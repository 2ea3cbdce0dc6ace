"""GPU: the fp8 two-stage search (e4m3 shortlist, exact bf16 re-rank) against float64 and against the restatement of
tests/fp8_two_stage.py (pinned on CPU by tests/test_fp8_two_stage_host.py), at the shortlist's edges, and a
multi-device fp8 Searcher bitwise the one-device one.

* Decoy corpora: e4m3 rounding puts 300 decoys ahead of a target that is exactly better.  At ``ndocs = 4 * 300`` the
  shortlist misses the target and the search returns the decoys, tied, in pid order; at ``4 * 301`` it returns the
  target.  Every form (unrestricted, ``filter_fn``, ``pids=`` on the listed and the bitmap scan, ``qid_to_pids``) and
  every device set gives exactly those rankings, also with the decoys in shard 0 and the target in a later shard, and
  with tied decoys on both sides of a shard boundary cut by the depth.
* A pairwise grid over form, k, ndocs, relu, deletions, Nq and the re-rank's gather size: e4m3 scores within the scan
  bound of float64, returned scores within the arg-max bound of float64 over the bf16 rows and in order, and returned
  ids and scores equal to the restatement run on the kernels' own scores (the scan's e4m3 scores of the same batch, the
  grouped arg-max over the gathered rows of the restatement's candidates).  Every non-deleted case also runs on
  ``devices=[0, 0]``, ``[0, 0, 0]`` (and ``[0, 1]``, ``"all"`` with two GPUs), bitwise the one-device result.

The largest error / bound ratios, the depths reached and whether the two arg-max kernels gave different bits are
printed at the end (run with -s)."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import fp8_two_stage as T
import scan_fp64 as S
from train_fp64 import C_BOUND, U, bf16_rows, pairwise_cases

pytestmark = pytest.mark.gpu

N_GPUS = torch.cuda.device_count() if torch.cuda.is_available() else 0
TWO_GPUS = pytest.mark.skipif(N_GPUS < 2, reason="needs at least two GPUs")
DEVICE_SETS = [[0, 0], [0, 0, 0]] + ([[0, 1], "all"] if N_GPUS >= 2 else [])
DEVICE_PARAMS = [pytest.param([0, 0], id="0-0"), pytest.param([0, 0, 0], id="0-0-0"),
                 pytest.param([0, 1], id="0-1", marks=TWO_GPUS), pytest.param("all", id="all", marks=TWO_GPUS)]
RATIOS = {}
NOTES = {"depth=k": 0, "depth<n": 0, "depth=n": 0, "argmax kernels differ": 0, "argmax kernels compared": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[fp8 two-stage] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[fp8 two-stage]   %-28s %.3e" % (k, RATIOS[k]))
    for k, v in NOTES.items():
        print("[fp8 two-stage]   %-28s %d" % (k, v))


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


@pytest.fixture(scope="module")
def SR(R):
    from ravqa_b200 import searcher
    return searcher


def _same(a, b, tag):
    assert torch.equal(a[1].cpu(), b[1].cpu()), "%s: ids differ" % tag
    assert torch.equal(a[0].cpu().view(torch.int32), b[0].cpu().view(torch.int32)), "%s: scores differ" % tag


def _path(monkeypatch, SR, form):
    """Force a restricted search onto the listed scan or the bitmap scan."""
    if form == "pids_listed":
        monkeypatch.setattr(SR, "LISTED_SCAN_MAX_ROW_FRACTION", float("inf"))
    elif form == "pids_bitmap":
        monkeypatch.setattr(SR, "LISTED_SCAN_MAX_ROW_FRACTION", -1.0)


def _search(searcher, Q, k, form, lists, keep):
    """One search of ``form``: (scores, pids) on the home device."""
    if form == "filter_fn":
        return searcher._search_tensors(Q, k, filter_fn=keep)
    if form in ("pids_listed", "pids_bitmap", "qid_to_pids"):
        return searcher._search_tensors(Q, k, pid_lists=lists)
    if form == "rescore":
        out = searcher.retrieve_and_rescore(Q.float(), k, generator=torch.Generator().manual_seed(k))
        return out["search_scores"], torch.as_tensor(out["retrieved_doc_ids"], device=out["search_scores"].device)
    return searcher._search_tensors(Q, k)


def _kept(pids):
    """bool: what ``_keep`` keeps (every planted passage of the decoy corpora among them)."""
    return (pids % 3 != 1) | (pids < 1100)


def _keep(pids):
    return pids[_kept(pids)]


# ---- decoy corpora ----------------------------------------------------------------------------------------------------
N_DECOY = 300


def _decoy_layout(better=False):
    """1200 passages: the decoys (pids 0..299) short (< 128 tokens), a run of long passages (128..180 tokens) from pid
    700 on, the target at 1000 (``better``: at 1151).  ``better``: decoys 0..199 plus 150 better decoys at 900..1049,
    tied with them in e4m3, in other shards than they are, and the target's exact twin after it at 1160."""
    rng = np.random.default_rng(17)
    dl = rng.integers(1, 100, 1200).astype(np.int32)
    dl[700:] = rng.integers(128, 181, 500)
    plant = {1151 if better else 1000: "target"}
    if better:
        plant.update({p: "decoy" for p in range(200)})
        plant.update({p: "better" for p in range(900, 1050)})
        plant[1160] = "twin"
    else:
        plant.update({p: "decoy" for p in range(N_DECOY)})
    return dl, plant


@pytest.fixture(scope="module")
def decoy_indexes(R, tmp_path_factory):
    out = {}
    for better in (False, True):
        dl, plant = _decoy_layout(better)
        D, dl = T.decoy_corpus(dl, plant, seed=5)
        path = str(tmp_path_factory.mktemp("decoys") / ("better" if better else "plain"))
        R.save_flat_index(path, torch.from_numpy(D).to(torch.bfloat16), dl)
        out[better] = (path, D, dl, plant)
    return out


def _decoy_lists(plant, n, B):
    """Per query: every planted passage plus fillers (query b: a different number of them), some listed twice."""
    rng = np.random.default_rng(B)
    planted = np.array(sorted(plant), np.int64)
    fill = np.setdiff1d(np.arange(n), planted)
    return [np.concatenate([planted, rng.choice(fill, 20 + 37 * b, replace=False), planted[:5]]) for b in range(B)]


def _decoy_admitted(form, plant, n, lists, b):
    if form in ("pids_listed", "pids_bitmap", "qid_to_pids"):
        adm = np.zeros(n, bool)
        adm[lists[b]] = True
        return adm
    if form == "filter_fn":
        return _kept(np.arange(n))
    return np.ones(n, bool)


DECOY_FORMS = ["all", "filter_fn", "pids_listed", "pids_bitmap", "qid_to_pids"]


def _check_decoys(searcher, Q, plant, n, ndocs, k, form, lists, tag):
    searcher.configure(ndocs=ndocs)
    s, p = _search(searcher, Q, k, form, lists, _keep)
    for b in range(Q.size(0)):
        adm = _decoy_admitted(form, plant, n, lists, b)
        n_cand = int(adm.sum()) if form not in ("pids_listed", "pids_bitmap", "qid_to_pids") else \
            int(T.allowed_counts(lists, np.ones(n, bool)).max())
        depth = T.shortlist_depth(min(k, n_cand), ndocs, n_cand)
        ws, wp = T.expected_decoy_ranking(plant, n, depth, k, adm)
        got_p = p[b].cpu().numpy()
        got_s = s[b].cpu().numpy()
        assert np.array_equal(got_p[got_p >= 0], wp[wp >= 0]), "%s b=%d depth=%d: ids" % (tag, b, depth)
        assert np.array_equal(got_s[got_p >= 0], ws[wp >= 0].astype(np.float32)), "%s b=%d: scores" % (tag, b)
    return s, p


@pytest.mark.parametrize("nq", [32, 320])
@pytest.mark.parametrize("form", DECOY_FORMS)
def test_decoys_decide_the_one_device_ranking(R, SR, monkeypatch, decoy_indexes, form, nq):
    path, D, dl, plant = decoy_indexes[False]
    n = len(dl)
    _path(monkeypatch, SR, form)
    one = R.Searcher(index=path, storage="fp8")
    Q = torch.from_numpy(T.decoy_queries(2, nq)).to(torch.bfloat16).cuda()
    lists = _decoy_lists(plant, n, 2)
    for k in (1, 10):
        s, p = _check_decoys(one, Q, plant, n, 4 * N_DECOY, k, form, lists, "%s k=%d miss" % (form, k))
        assert 1000 not in p.cpu().numpy()
        assert p[0, 0].item() == 0 and s[0, 0].item() == T.EXACT["decoy"]
        assert one._last_depth == N_DECOY
        s, p = _check_decoys(one, Q, plant, n, 4 * (N_DECOY + 1), k, form, lists, "%s k=%d find" % (form, k))
        assert (p[:, 0] == 1000).all() and (s[:, 0] == T.EXACT["target"]).all()
        assert one._last_depth == N_DECOY + 1
    one.configure(ndocs=4 * N_DECOY)
    qids = ["a", "b"]
    rk = one._search_all_Q(qids, Q, 10, qid_to_pids=dict(zip(qids, lists)) if form == "qid_to_pids" else None)
    assert rk.provenance()["shortlist_depth"] == N_DECOY
    # the bf16 Searcher has no shortlist: it finds the target whatever ndocs says
    bf = R.Searcher(index=path)
    bf.configure(ndocs=4 * N_DECOY)
    _, p = _search(bf, Q, 10, form, lists, _keep)
    assert (p[:, 0] == 1000).all()


@pytest.mark.parametrize("devices", DEVICE_PARAMS)
@pytest.mark.parametrize("better", [False, True], ids=["decoys-in-shard-0", "ties-across-shards"])
def test_decoys_multi_device_is_the_one_device_ranking(R, SR, monkeypatch, decoy_indexes, devices, better):
    path, D, dl, plant = decoy_indexes[better]
    n = len(dl)
    one = R.Searcher(index=path, storage="fp8")
    many = R.Searcher(index=path, storage="fp8", devices=devices)
    n_dev = N_GPUS if devices == "all" else len(devices)
    ranges = R.shard_ranges(dl, n_dev)
    assert [c.pid_base for c in many.shards] == [a for a, _ in ranges]
    owner = {p: next(i for i, (a, b) in enumerate(ranges) if a <= p < b) for p in plant}
    target = next(p for p, kind in plant.items() if kind == "target")
    assert owner[target] > 0
    if n_dev <= 3:                                       # shard 0 holds every plain decoy
        assert all(owner[p] == 0 for p, kind in plant.items() if kind == "decoy")
    if better:                                           # the e4m3 tie runs across shards
        assert len({owner[p] for p, kind in plant.items() if kind != "target"}) > 1
    lists = _decoy_lists(plant, n, 3)
    for nq in (32, 320):
        Q = torch.from_numpy(T.decoy_queries(3, nq)).to(torch.bfloat16).cuda()
        for form in DECOY_FORMS + ["rescore"]:
            with monkeypatch.context() as m:
                _path(m, SR, form)
                for ndocs, k in ((4 * N_DECOY, 10), (4 * (N_DECOY + 1), 10), (1000, 60), (4 * N_DECOY, 150),
                                 (1600, 10)):
                    tag = "%s %s nq=%d ndocs=%d k=%d" % (devices, form, nq, ndocs, k)
                    if form == "rescore":
                        one.configure(ndocs=ndocs)
                        many.configure(ndocs=ndocs)
                        a = _search(one, Q, k, form, lists, _keep)
                        b = _search(many, Q, k, form, lists, _keep)
                    else:
                        a = _check_decoys(one, Q, plant, n, ndocs, k, form, lists, tag)
                        b = _check_decoys(many, Q, plant, n, ndocs, k, form, lists, tag + " many")
                    _same(a, b, tag)
                    assert many._last_depth == one._last_depth, tag
    one.configure(ndocs=4 * N_DECOY)
    many.configure(ndocs=4 * N_DECOY)
    rk1 = one._search_all_Q(["a", "b", "c"], Q, 10)
    rk2 = many._search_all_Q(["a", "b", "c"], Q, 10)
    assert rk1.todict() == rk2.todict()
    assert rk2.provenance()["shortlist_depth"] == rk1.provenance()["shortlist_depth"] == N_DECOY


def test_k_above_the_select_capacity_is_refused(R, decoy_indexes):
    path = decoy_indexes[False][0]
    Q = torch.from_numpy(T.decoy_queries(1, 32)).to(torch.bfloat16).cuda()
    for s in (R.Searcher(index=path, storage="fp8"), R.Searcher(index=path, storage="fp8", devices=[0, 0])):
        with pytest.raises(ValueError):
            s._search_tensors(Q, 2049)


# ---- the certified grid -----------------------------------------------------------------------------------------------
N_GRID = 2600
GRID_FACTORS = {
    "form": ["all", "filter_fn", "pids_listed", "pids_bitmap", "qid_to_pids", "rescore"],
    "k": [1, 10, 128, 129, 2048],
    "ndocs": ["unset", "k", "lt_n", "n"],
    "relu": [False, True],
    "deleted": [False, True],
    "nq": [32, 320],
    "gather": ["default", "small"],
}


def _grid_allowed(case):
    return not (case.get("form") == "rescore" and case.get("deleted"))


@pytest.fixture(scope="module")
def grid(R, tmp_path_factory):
    """2600 passages of 1..180 tokens (the first 1300 under 100, so shard 0 of three holds no passage of 128 tokens),
    unit bf16 rows, with duplicated passages (exact ties in both scores) and decoy/target pairs planted; queries of 32
    (B = 3) and 320 (B = 2) rows."""
    g = torch.Generator().manual_seed(41)
    rng = np.random.default_rng(41)
    dl = rng.integers(1, 181, N_GRID).astype(np.int32)
    dl[:1300] = rng.integers(1, 100, 1300)
    D = bf16_rows((int(dl.sum()), 128), generator=g)
    off = np.concatenate([[0], np.cumsum(dl, dtype=np.int64)])
    for a, b in ((3, 1400), (40, 2500), (41, 2501), (1299, 1301)):
        dl_a = min(dl[a], dl[b])
        D[off[b]:off[b] + dl_a] = D[off[a]:off[a] + dl_a]
        D[off[b] + dl_a:off[b + 1]] = D[off[a]]
    path = str(tmp_path_factory.mktemp("grid") / "idx")
    R.save_flat_index(path, D.to(torch.bfloat16), dl)
    Qs = {32: bf16_rows((3, 32, 128), generator=g), 320: bf16_rows((2, 320, 128), generator=g)}
    Qs[32][1, 20:] = 0.0                                   # zero rows
    # the deleted variant: an fp8 corpus of the same rows with 700 passages deleted (fewer live passages than 2048)
    dead = np.sort(rng.choice(N_GRID, 700, replace=False))
    cd = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0, storage="fp8")
    cd.delete(dead)
    live = np.ones(N_GRID, bool)
    live[dead] = False
    searchers = {False: R.Searcher(index=path, storage="fp8"), True: R.Searcher(index=cd)}
    many = {str(d): R.Searcher(index=path, storage="fp8", devices=d) for d in DEVICE_SETS}
    refs = {}

    def ref(nq, relu, storage):
        if (nq, relu, storage) not in refs:
            refs[nq, relu, storage] = S.maxsim_packed(Qs[nq].cuda(), D.cuda(), dl, relu=relu, storage=storage)
        return refs[nq, relu, storage]
    return dict(D=D, dl=dl, path=path, Qs=Qs, live=live, searchers=searchers, many=many, ref=ref)


def _grid_lists(case, B, live, seed):
    """Per query, lists of very different sizes (a short list, one of ~1900 ids, one of ~400 with deleted ids and
    duplicates); ``qid_to_pids`` gives its last query none (the whole index)."""
    rng = np.random.default_rng(seed)
    sizes = [7, 1900, 400]
    lists = [np.concatenate([rng.choice(N_GRID, sizes[b % 3], replace=False), rng.choice(N_GRID, 5)])
             for b in range(B)]
    if case["form"] == "qid_to_pids":
        lists[-1] = None
    return lists


def _ndocs(opt, k, n_cand):
    if opt == "unset":
        return None
    if opt == "k":
        return 4 * k
    if opt == "lt_n":
        return 4 * max(k, (min(k, n_cand) + n_cand) // 2)
    return 4 * n_cand


def _rescore(R, SR, corpus, Q, cand, relu):
    """The kernels' own exact scores of the candidates ``cand`` (pid-sorted, -1: none): the gather and the grouped
    arg-max in the query steps the Searcher takes."""
    from ravqa_b200.maxsim import maxsim_argmax_grouped
    depth = cand.size(1)
    c = cand[cand >= 0].cpu().numpy()
    nd_max = int(corpus.doclens[c].max()) if c.size else 1
    step = max(1, SR.RERANK_GATHER_BYTES // (depth * nd_max * 128 * 2))
    out = []
    for q0 in range(0, Q.size(0), step):
        Dg, mask = corpus.gather_padded(cand[q0:q0 + step], nd_max)
        _, rowmax = maxsim_argmax_grouped(Q[q0:q0 + step], Dg.flatten(0, 1), mask.flatten(0, 1), depth,
                                            return_rowmax=True)
        if relu:
            rowmax = rowmax.clamp_min(0.0)
        out.append(rowmax.sum(dim=-1))
    return torch.cat(out).masked_fill(cand < 0, float("-inf"))


GRID = pairwise_cases(GRID_FACTORS, _grid_allowed)


@pytest.mark.parametrize("ci", range(len(GRID)), ids=["%d-%s-k%d-%s" % (i, c["form"], c["k"], c["ndocs"])
                                                      for i, c in enumerate(GRID)])
def test_grid_certified_and_multi_device_bitwise(R, SR, monkeypatch, grid, ci):
    case = GRID[ci]
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    form, k, relu, nq = case["form"], case["k"], case["relu"], case["nq"]
    one = grid["searchers"][case["deleted"]]
    corpus = one.corpus
    live = grid["live"] if case["deleted"] else np.ones(N_GRID, bool)
    Q = grid["Qs"][nq].to(torch.bfloat16).cuda()
    B = Q.size(0)
    _path(monkeypatch, SR, form)
    if case["gather"] == "small":
        monkeypatch.setattr(SR, "RERANK_GATHER_BYTES", 1)          # one query per gather step
    lists = _grid_lists(case, B, live, seed=ci)
    restricted = form in ("pids_listed", "pids_bitmap", "qid_to_pids")
    if restricted:
        adm = T.admitted_rows(lists, live)
        n_cand = int(T.allowed_counts(lists, live).max())
    else:
        adm = np.tile(live & (_kept(np.arange(N_GRID)) if form == "filter_fn" else True), (B, 1))
        n_cand = int(adm[0].sum())
    kk = max(5, k) if form == "rescore" else k
    kq = min(kk, n_cand)
    ndocs = _ndocs(case["ndocs"], kq, n_cand)
    depth = T.shortlist_depth(kq if restricted else kk, ndocs, n_cand)
    NOTES["depth=k" if depth == kq else ("depth=n" if depth == n_cand else "depth<n")] += 1
    one.configure(relu=relu, ndocs=ndocs)
    s, p = _search(one, Q, kk if form != "rescore" else k, form, lists, _keep)
    if form == "rescore":                                   # the search it made: compare that one below
        s_r, p_r = s, p
        s, p = one._search_tensors(Q, kk)
        if k >= 5:
            _same((s_r, p_r), (s, p), "rescore")
        else:
            for b in range(B):
                assert set(p_r[b].tolist()) <= set(p[b].tolist())
    assert one._last_depth == depth
    # the restatement on the kernels' own scores, in the same batch
    e8 = R.maxsim_scores(corpus, Q, relu=relu)
    cand = np.sort(T.shortlist(e8.cpu().numpy(), adm, depth), axis=1)
    cand_t = torch.from_numpy(cand).cuda()
    exact = _rescore(R, SR, corpus, Q, cand_t, relu)
    ws, wp = T.rerank(cand, exact.cpu().numpy(), kq)
    n_valid = p.size(1)
    assert np.array_equal(p.cpu().numpy(), wp[:, :n_valid]) and (wp[:, n_valid:] < 0).all(), "ids"
    assert np.array_equal(s.cpu().numpy(), ws[:, :n_valid].astype(np.float32)), "scores"
    # the two arg-max kernels on the same candidates
    try:
        got = {}
        for path in (1, 2):
            _cabi.check(L.flmr_debug_set_argmax_path(path))
            got[path] = _rescore(R, SR, corpus, Q, cand_t, relu)
    finally:
        L.flmr_debug_set_argmax_path(0)
    NOTES["argmax kernels compared"] += 1
    NOTES["argmax kernels differ"] += int(not torch.equal(got[1], got[2]))
    # float64: e4m3 scores within the scan bound, exact scores within the arg-max bound, in order
    s8_64, a8, r8 = grid["ref"](nq, relu, "fp8")
    s16_64, a16, r16 = grid["ref"](nq, relu, "bf16")
    lv = torch.from_numpy(live).cuda()
    S.check_ratio(RATIOS, "e4m3 scan", (e8.double() - s8_64)[:, lv].abs(), S.scan_bound(a8, r8, nq, "fp8")[:, lv])
    ebound = C_BOUND * U * a16 + nq * U * r16
    ok = cand_t >= 0
    cl = cand_t.clamp_min(0)
    S.check_ratio(RATIOS, "re-rank exact (candidates)", (exact.double() - s16_64.gather(1, cl))[ok].abs(),
                  ebound.gather(1, cl)[ok])
    hit = p >= 0
    pl = p.clamp_min(0)
    S.check_ratio(RATIOS, "returned scores", (s.double() - s16_64.gather(1, pl))[hit].abs(), ebound.gather(1, pl)[hit])
    assert (s[:, :-1] >= s[:, 1:]).all() or not hit.any(), "returned out of order"
    assert (torch.from_numpy(adm).cuda().gather(1, pl)[hit]).all(), "a returned id is not admitted"
    # multi-device: bitwise the one-device search
    if not case["deleted"]:
        if ci == 0:
            assert max(grid["dl"][a:b].max() for a, b in R.shard_ranges(grid["dl"], 3)[:1]) < 128
        one_s = _search(one, Q, kk if form != "rescore" else k, form, lists, _keep)
        for key, many in grid["many"].items():
            many.configure(relu=relu, ndocs=ndocs)
            _same(one_s, _search(many, Q, kk if form != "rescore" else k, form, lists, _keep),
                  "%s case %d" % (key, ci))
            assert many._last_depth == depth
