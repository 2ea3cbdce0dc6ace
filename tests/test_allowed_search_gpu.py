"""Restricted search on the GPU: per-query allow bitmaps tested in the scan's reducer.

(a) masking identity: restricted scores are bitwise the unrestricted ones where allowed, -inf elsewhere, for both
    storages, every scan variant, lane and warp mode, row-sliced passes, relu on and off, and bitmap densities 0-1;
(b) the fused top-k equals a stable sort of that masked matrix, filled with (-inf, -1);
(c) query indexing across passes, CTA pairs and the workspace's 64-query chunks;
(d) deletions and appends; (e) the C-level exchange; (f) the Searcher's pids= / qid_to_pids=, k > 128, fp8,
    launch counts; (g) a two-rank gloo Searcher.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN_DIR, golden_names, load_golden, placement_doclens
from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu

NEG = float("-inf")
SHAPES = [(12, 32), (4, 160), (16, 320), (3, 832)]   # lane mode, warp mode, warp mode (pair passes), row-sliced
DENSITIES = [0.0, 1e-3, 0.5, 1.0]


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    return ravqa_b200


def _unit_rows(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1).bfloat16()


def _queries(B, nq, seed):
    return _unit_rows(B * nq, seed).view(B, nq, 128).cuda()


def _set_variant(v):
    from ravqa_b200 import _cabi
    _cabi.check(_cabi.lib().flmr_debug_set_scan_variant(v))


@pytest.fixture(scope="module")
def corpora(R):
    """{(name, storage): corpus}: the placement fixture (many passage ends per tile, slots >= kFastSlots) and
    180-token passages."""
    dls = {"placement": placement_doclens(), "nd180": np.full(2000, 180, np.int32)}
    out = {}
    for name, dl in dls.items():
        D = _unit_rows(int(dl.sum()), 7)
        for storage in ("bf16", "fp8"):
            out[(name, storage)] = R.FlatCorpus(D, dl, storage=storage)
    yield out
    for c in out.values():
        c.close()


def _random_allow(c, B, density, seed):
    """(bitmaps [B, words] on the GPU, dense bool mask [B, n] on the GPU)."""
    n = c.n_passages
    mask = np.random.default_rng(seed).random((B, n)) < density
    allow = c.allow_bitmaps([np.nonzero(m)[0] + c.pid_base for m in mask])
    if density == 1.0:
        allow.fill_(-1)                                  # bits past n_passages set too: they are ignored
    return allow, torch.from_numpy(mask).cuda()


def _ranked(masked, k):
    """Stable descending sort of a masked score matrix: (scores, pids) [B, k] with (-inf, -1) fill."""
    vals, idx = torch.sort(masked, dim=1, descending=True, stable=True)
    vals, idx = vals[:, :k], idx[:, :k]
    if vals.size(1) < k:
        vals = torch.cat([vals, vals.new_full((vals.size(0), k - vals.size(1)), NEG)], 1)
        idx = torch.cat([idx, idx.new_full((idx.size(0), k - idx.size(1)), -1)], 1)
    return vals, idx.masked_fill(vals == NEG, -1)


# ---- (a) masking identity ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("variant", [0, 2, 3, 4])
@pytest.mark.parametrize("storage", ["bf16", "fp8"])
@pytest.mark.parametrize("name", ["placement", "nd180"])
def test_masking_identity(R, corpora, name, storage, variant, shape, relu):
    if storage == "fp8" and variant == 4:
        pytest.skip("the CTA-pair scan is bf16 only")
    c = corpora[(name, storage)]
    B, nq = shape
    Q = _queries(B, nq, seed=B * nq)
    _set_variant(variant)
    try:
        full = R.maxsim_scores(c, Q, relu=relu)
        for i, dens in enumerate(DENSITIES):
            allow, mask = _random_allow(c, B, dens, seed=i)
            got = R.maxsim_scores(c, Q, relu=relu, allow=allow)
            assert torch.equal(got, torch.where(mask, full, NEG)), dens
    finally:
        _set_variant(0)


# ---- (b) fused top-k -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 10, 128])
@pytest.mark.parametrize("shape", [(12, 32), (16, 320), (3, 832)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("storage,variant", [("bf16", 0), ("bf16", 4), ("fp8", 0)])
def test_fused_topk_is_stable_sort_of_masked_scores(R, corpora, storage, variant, shape, k):
    c = corpora[("placement", storage)]
    B, nq = shape
    Q = _queries(B, nq, seed=3 + nq)
    _set_variant(variant)
    try:
        full = R.maxsim_scores(c, Q)
        for i, dens in enumerate(DENSITIES):
            allow, mask = _random_allow(c, B, dens, seed=10 + i)
            s, p = R.maxsim_topk(c, Q, k, allow=allow)
            ws, wp = _ranked(torch.where(mask, full, NEG), k)
            assert torch.equal(p, wp), dens
            assert torch.equal(s, ws), dens
            if dens == 0.0:
                assert (p == -1).all() and torch.isneginf(s).all()
        # an all-ones bitmap is the unrestricted call
        s0, p0 = R.maxsim_topk(c, Q, k)
        ones = torch.full((B, (c.n_passages + 31) // 32), -1, dtype=torch.int32, device="cuda")
        s1, p1 = R.maxsim_topk(c, Q, k, allow=ones)
        assert torch.equal(p1, p0) and torch.equal(s1, s0)
        # one shared bitmap (stride 0) is that row repeated
        row, _ = _random_allow(c, 1, 0.5, seed=99)
        s2, p2 = R.maxsim_topk(c, Q, k, allow=row[0])
        s3, p3 = R.maxsim_topk(c, Q, k, allow=row.expand(B, -1))
        assert torch.equal(p2, p3) and torch.equal(s2, s3)
    finally:
        _set_variant(0)


# ---- (c) query indexing --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage,variant", [("bf16", 0), ("bf16", 4), ("fp8", 0)])
def test_each_query_reaches_its_own_passage(R, corpora, storage, variant):
    c = corpora[("placement", storage)]
    B = 100                                              # two chunks of the 64-query workspace
    targets = (np.arange(B) * 197 + 11) % c.n_passages
    allow = c.allow_bitmaps([[t] for t in targets])
    Q = _queries(B, 32, seed=5)
    _set_variant(variant)
    try:
        s, p = R.maxsim_topk(c, Q, 5, allow=allow)
        scores = R.maxsim_scores(c, Q, allow=allow)
    finally:
        _set_variant(0)
    assert p[:, 0].tolist() == targets.tolist()
    assert (p[:, 1:] == -1).all() and torch.isneginf(s[:, 1:]).all()
    assert torch.isfinite(scores).sum(1).tolist() == [1] * B
    assert torch.equal(scores[torch.arange(B), torch.from_numpy(targets).cuda()], s[:, 0])


# ---- (d) deletions and appends -------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_deleted_never_returned_and_appended_reachable(R, storage):
    dl = placement_doclens(3000, seed=4)
    c = R.FlatCorpus(_unit_rows(int(dl.sum()), 8), dl, storage=storage)
    try:
        Q = _queries(6, 32, seed=6)
        full = R.maxsim_scores(c, Q)
        allow, mask = _random_allow(c, 6, 0.3, seed=1)
        # delete the best allowed passages of every query
        best = _ranked(torch.where(mask, full, NEG), 3)[1]
        gone = torch.unique(best[best >= 0]).cpu().numpy()
        c.delete(gone)
        live = torch.ones(c.n_passages, dtype=torch.bool, device="cuda")
        live[torch.from_numpy(gone).cuda()] = False
        s, p = R.maxsim_topk(c, Q, 128, allow=allow)
        assert not np.isin(p.cpu().numpy(), gone).any()
        ws, wp = _ranked(torch.where(mask & live, full, NEG), 128)
        assert torch.equal(p, wp) and torch.equal(s, ws)
        assert torch.equal(R.maxsim_scores(c, Q, allow=allow), torch.where(mask & live, full, NEG))
        # after an append a bitmap built on the grown corpus reaches the new ids
        extra = placement_doclens(300, seed=5)
        new = c.append(_unit_rows(int(extra.sum()), 9), extra)
        with pytest.raises(ValueError):
            R.maxsim_topk(c, Q, 10, allow=allow)             # built for the old corpus: the wrong width
        pick = new[::3]
        s, p = R.maxsim_topk(c, Q, 128, allow=c.allow_bitmaps([pick] * 6))
        full2 = R.maxsim_scores(c, Q)
        m2 = torch.zeros_like(full2, dtype=torch.bool)
        m2[:, torch.from_numpy(pick).cuda()] = True
        ws, wp = _ranked(torch.where(m2, full2, NEG), 128)
        assert torch.equal(p, wp) and torch.equal(s, ws)
        assert (p[:, :len(pick)] >= new[0]).all()
    finally:
        c.close()


# ---- (e) the C-level exchange --------------------------------------------------------------------------------------
def test_sharded_allowed_world_one_equals_local(R, corpora):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    c = corpora[("placement", "bf16")]
    uid = (C.c_char * 128)()
    _cabi.check(L.flmr_comm_unique_id(C.cast(uid, C.c_void_p)))
    comm = C.c_void_p()
    _cabi.check(L.flmr_comm_create(C.cast(uid, C.c_void_p), 0, 1, int(c.device.index), C.byref(comm)))
    try:
        B, k = 12, 10
        Q = _queries(B, 32, seed=8)
        for allow in (_random_allow(c, B, 0.01, seed=3)[0], _random_allow(c, 1, 0.5, seed=4)[0][0]):
            stride = allow.size(1) if allow.dim() == 2 else 0
            s = torch.empty((B, k), dtype=torch.float32, device="cuda")
            p = torch.empty((B, k), dtype=torch.int64, device="cuda")
            _cabi.check(L.flmr_maxsim_topk_sharded_allowed(
                c.handle, c.workspace(), comm, C.c_void_p(Q.data_ptr()), B, 32, k, 0, C.c_void_p(allow.data_ptr()),
                stride, C.c_void_p(s.data_ptr()), C.c_void_p(p.data_ptr()),
                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            ws, wp = R.maxsim_topk(c, Q, k, allow=allow)
            assert torch.equal(p, wp) and torch.equal(s, ws)
        # a stride shorter than one bitmap is rejected
        bad = _cabi.lib().flmr_maxsim_topk_allowed(
            c.handle, c.workspace(), C.c_void_p(Q.data_ptr()), B, 32, k, 0, C.c_void_p(allow.data_ptr()), 1,
            C.c_void_p(s.data_ptr()), C.c_void_p(p.data_ptr()), None)
        assert bad == 1                                   # FLMR_ERR_INVALID_ARG
    finally:
        torch.cuda.synchronize()
        L.flmr_comm_destroy(comm)


# ---- (f) Searcher --------------------------------------------------------------------------------------------------
def _oracle_restricted(scores, lists, k):
    """{b: ids} of the exact ranking restricted to each list (None: everything), ties by lower id."""
    out = {}
    for b, ids in enumerate(lists):
        cand = np.arange(scores.shape[1]) if ids is None else np.unique(np.asarray(ids, dtype=np.int64))
        out[b] = cand[np.lexsort((cand, -scores[b, cand].astype(np.float64)))][:k].tolist()
    return out


def test_searcher_callsites_qid_to_pids_and_pids(R):
    z = np.load(os.path.join(GOLDEN_DIR, "callsites.npz"))
    Q = torch.from_numpy(z["queries"])
    n = z["exact_scores_bf16"].shape[1]
    rng = np.random.default_rng(0)
    lists = [rng.choice(n, size=s, replace=False).tolist() for s in (0, 1, 7, 40, 100)] + [None]
    lists[3] = lists[3] + lists[3][:5]                    # duplicates collapse
    qids = ["q%d" % i for i in range(Q.size(0))]
    with R.Run().context(R.RunConfig(root=os.path.join(GOLDEN_DIR, "callsites", "ckpt"), experiment="temp_index_0")):
        sr = R.Searcher(index="temp_index.nbits=8", config=R.ColBERTConfig())
    ranking = sr._search_all_Q(qids, Q, k=20, qid_to_pids=dict(zip(qids, lists)))
    want = _oracle_restricted(z["exact_scores_bf16"], lists, 20)
    got = ranking.todict()
    for b, qid in enumerate(qids):
        assert [pid for pid, _, _ in got[qid]] == want[b], b
        assert [r for _, r, _ in got[qid]] == list(range(1, len(want[b]) + 1))
        np.testing.assert_allclose([s for _, _, s in got[qid]], z["exact_scores_bf16"][b, want[b]], rtol=5e-4)
        pids, ranks, scores = sr.dense_search(Q[b:b + 1], k=20, pids=lists[b])
        assert pids == want[b]
    assert ranking.provenance()["restricted"] is True
    with pytest.raises(KeyError):
        sr._search_all_Q(qids, Q, k=5, qid_to_pids={})


@pytest.mark.parametrize("golden_name", golden_names())
def test_searcher_golden_filter_badid_k_beyond_corpus(R, golden_name):
    from ravqa_b200 import _cabi
    g = load_golden(golden_name)
    D, dl, Qn = g["D"], g["doclens"].astype(np.int32), g["Q"]
    c = R.FlatCorpus(torch.from_numpy(D).bfloat16(), dl)
    try:
        n = c.n_passages
        sr = R.Searcher(index=c)
        truth = R.maxsim_scores(c, torch.from_numpy(Qn)).cpu().numpy()
        ref = O.maxsim_scores(Qn, D, dl)
        rng = np.random.default_rng(1)
        B = Qn.shape[0]
        lists = [rng.choice(n, size=min(n, 5 + 13 * b), replace=False) for b in range(B)]
        rk = sr._search_all_Q(list(range(B)), torch.from_numpy(Qn), k=10,
                              qid_to_pids={b: lists[b] for b in range(B)}).todict()
        want = _oracle_restricted(truth, lists, 10)
        for b in range(B):
            assert [pid for pid, _, _ in rk[b]] == want[b]
            np.testing.assert_allclose([s for _, _, s in rk[b]], ref[b, want[b]], rtol=1e-3)
        # filter_fn applies within each list
        keep = lambda pids: pids[pids % 2 == 0]                                     # noqa: E731
        rk = sr._search_all_Q(list(range(B)), torch.from_numpy(Qn), k=10, filter_fn=keep,
                              qid_to_pids={b: lists[b] for b in range(B)}).todict()
        want = _oracle_restricted(truth, [l[l % 2 == 0] for l in lists], 10)
        assert all([pid for pid, _, _ in rk[b]] == want[b] for b in range(B))
        # a bad id anywhere in the batch: ValueError, nothing launched
        L = _cabi.lib()
        L.flmr_launch_count(1)
        with pytest.raises(ValueError):
            sr._search_all_Q(list(range(B)), torch.from_numpy(Qn), k=10,
                             qid_to_pids={b: (lists[b] if b else [0, n]) for b in range(B)})
        assert L.flmr_launch_count(0) == 0
        # k beyond the whole corpus: every allowed passage, rows trimmed per query
        big = [np.arange(0, n, 2), None] + [lists[b] for b in range(2, B)]
        rk = sr._search_all_Q(list(range(B)), torch.from_numpy(Qn), k=200,
                              qid_to_pids={b: big[b] for b in range(B)}).todict()
        want = _oracle_restricted(truth, big, 200)
        assert all([pid for pid, _, _ in rk[b]] == want[b] for b in range(B))
    finally:
        c.close()


@pytest.mark.parametrize("k,name", [(200, "nd180"), (3000, "placement")])
def test_searcher_k_beyond_fused_capacity(R, corpora, k, name):
    """k > 128 (all scores + topk_select) and k > 2048 (all scores + a stable sort), with queries that allow more and
    fewer than k live passages."""
    c = corpora[(name, "bf16")]
    n = c.n_passages
    rng = np.random.default_rng(k)
    sizes = (k + k // 2, k - 50, 7, 0, 2 * k, k // 3)
    lists = [rng.choice(n, size=s, replace=False) for s in sizes] + [None]
    Q = _queries(len(lists), 32, seed=k)
    truth = R.maxsim_scores(c, Q).cpu().numpy()
    rk = R.Searcher(index=c)._search_all_Q(list(range(len(lists))), Q, k=k,
                                          qid_to_pids=dict(enumerate(lists))).todict()
    want = _oracle_restricted(truth, lists, k)
    for b in range(len(lists)):
        got = rk[b]
        assert len(got) == min(k, n if lists[b] is None else len(lists[b])), b    # short rows trimmed per query
        assert [pid for pid, _, _ in got] == want[b], b
        assert [sc for _, _, sc in got] == truth[b, want[b]].tolist(), b
        assert [r for _, r, _ in got] == list(range(1, len(got) + 1))


def test_fp8_searcher_k_beyond_fused_capacity(R, corpora):
    c8, c16 = corpora[("nd180", "fp8")], corpora[("nd180", "bf16")]
    rng = np.random.default_rng(5)
    n = c8.n_passages
    lists = [rng.choice(n, size=s, replace=False) for s in (300, 150, 900, 0)] + [None]
    Q = _queries(len(lists), 32, seed=6)
    q2p = dict(enumerate(lists))
    sr8 = R.Searcher(index=c8)
    r8 = sr8._search_all_Q(list(range(len(lists))), Q, k=200, qid_to_pids=q2p).todict()
    r16 = R.Searcher(index=c16)._search_all_Q(list(range(len(lists))), Q, k=200, qid_to_pids=q2p).todict()
    exact = R.maxsim_scores(c16, Q).cpu().numpy()
    assert sr8._last_depth == 1024                                  # ndocs / 4, ndocs = 4096 for k > 100
    for b, ids in enumerate(lists):
        ids8 = [pid for pid, _, _ in r8[b]]
        assert len(ids8) == min(200, n if ids is None else len(ids))
        np.testing.assert_allclose([s for _, _, s in r8[b]], exact[b, ids8], rtol=1e-5, atol=1e-6)
        if ids is not None and len(ids) <= 1024:                    # the whole list is shortlisted
            assert ids8 == [pid for pid, _, _ in r16[b]], b


def test_restricted_launch_count_matches_unrestricted(R, corpora):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    c = corpora[("nd180", "bf16")]
    Q = _queries(16, 320, seed=2)
    allow, _ = _random_allow(c, 16, 0.5, seed=2)
    R.maxsim_topk(c, Q, 10, allow=allow)
    torch.cuda.synchronize()
    L.flmr_launch_count(1)
    R.maxsim_topk(c, Q, 10)
    n_plain = L.flmr_launch_count(1)
    R.maxsim_topk(c, Q, 10, allow=allow)
    n_allowed = L.flmr_launch_count(1)
    assert n_plain == n_allowed == 1 + 16 + 1


def test_fp8_searcher_exact_and_matches_bf16(R, corpora):
    c8, c16 = corpora[("nd180", "fp8")], corpora[("nd180", "bf16")]
    Q = _queries(8, 32, seed=4)
    rng = np.random.default_rng(3)
    n = c8.n_passages
    lists = [rng.choice(n, size=s, replace=False) for s in (1, 10, 50, 200, 255, 256, 600, 1500)]
    q2p = {b: lists[b] for b in range(8)}
    r8 = R.Searcher(index=c8)._search_all_Q(list(range(8)), Q, k=10, qid_to_pids=q2p).todict()
    r16 = R.Searcher(index=c16)._search_all_Q(list(range(8)), Q, k=10, qid_to_pids=q2p).todict()
    exact = R.maxsim_scores(c16, Q).cpu().numpy()
    depth = 256                                                     # ndocs / 4 for k = 10
    for b in range(8):
        ids8 = [pid for pid, _, _ in r8[b]]
        assert len(ids8) == min(10, len(lists[b]))
        np.testing.assert_allclose([s for _, _, s in r8[b]], exact[b, ids8], rtol=1e-5, atol=1e-6)
        if len(lists[b]) <= depth:                                  # the whole list is shortlisted
            assert ids8 == [pid for pid, _, _ in r16[b]], b


# ---- (g) two-rank gloo Searcher ------------------------------------------------------------------------------------
def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


TINY_LISTS = [[0], [], None, [0, 0]]                               # for the one-passage index


def _sharded_worker(rank, world, port, root, backend, storage, ret):
    """One rank of a restricted sharded Searcher on the 'flat' index and on the one-passage 'tiny' index (where a rank
    holds no shard); records {(rank, index, k): {row: [(pid, score), ...]}}."""
    import torch.distributed as dist
    import ravqa_b200 as R
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    kw = {"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    z = np.load(os.path.join(root, "case.npz"))
    lists = [z["l%d" % b] if b != 2 else None for b in range(int(z["B"]))]
    for index, qlists, ks in (("flat", lists, (10, 128)), ("tiny", TINY_LISTS, (5,))):
        with R.Run().context(R.RunConfig(root=root, experiment="e")):
            sr = R.Searcher(index=index, config=R.ColBERTConfig(total_visible_gpus=1), shard_across_ranks=True,
                            storage=storage)
        Q = torch.from_numpy(z["Q"][:len(qlists)])
        for k in ks:
            rk = sr._search_all_Q(list(range(len(qlists))), Q, k=k, qid_to_pids=dict(enumerate(qlists))).todict()
            ret[(rank, index, k)] = {b: [(pid, sc) for pid, _, sc in rk[b]] for b in rk}
    dist.barrier()
    dist.destroy_process_group()


def _sharded_case(R, tmp_path):
    """Writes the indexes and queries; returns (lists, unsharded bf16 results {(index, k): {row: [(pid, score)]}},
    exact bf16 scores of the 'flat' index [5, n])."""
    dl = placement_doclens(4000, seed=9)
    D = _unit_rows(int(dl.sum()), 10)
    Q = _unit_rows(5 * 32, 11).view(5, 32, 128)
    rng = np.random.default_rng(2)
    lists = {"l%d" % b: rng.choice(len(dl), size=s, replace=False) for b, s in enumerate((3, 40, 0, 500, 2000))}
    R.save_flat_index(str(tmp_path / "e" / "indexes" / "flat"), D, dl)
    R.save_flat_index(str(tmp_path / "e" / "indexes" / "tiny"), D[:int(dl[0])], dl[:1])
    np.savez(tmp_path / "case.npz", Q=Q.float().numpy().astype(np.float32), B=5, **lists)
    rows = [lists["l%d" % b] if b != 2 else None for b in range(5)]
    want = {}
    for index, corpus_args, qlists, ks in (("flat", (D, dl), rows, (10, 128)),
                                           ("tiny", (D[:int(dl[0])], dl[:1]), TINY_LISTS, (5,))):
        c = R.FlatCorpus(*corpus_args)
        try:
            if index == "flat":
                exact = R.maxsim_scores(c, Q).cpu().numpy()
            for k in ks:
                rk = R.Searcher(index=c)._search_all_Q(list(range(len(qlists))), Q[:len(qlists)], k=k,
                                                       qid_to_pids=dict(enumerate(qlists))).todict()
                want[(index, k)] = {b: [(pid, sc) for pid, _, sc in rk[b]] for b in rk}
        finally:
            c.close()
    return rows, want, exact


def _check_sharded(ret, world, rows, want, exact, storage):
    """bf16: the unsharded results exactly.  fp8: exact scores (passage 0 of 'tiny' is passage 0 of 'flat'), and the
    bf16 ranking wherever the whole list was shortlisted (depth 256 for k <= 100, else 1024)."""
    for rank in range(world):
        for (index, k), w in want.items():
            got = ret[(rank, index, k)]
            qlists = rows if index == "flat" else TINY_LISTS
            for b in w:
                if storage == "bf16":
                    assert got[b] == w[b], (rank, index, k, b)
                    continue
                assert len(got[b]) == len(w[b]), (rank, index, k, b)
                ids = [pid for pid, _ in got[b]]
                np.testing.assert_allclose([sc for _, sc in got[b]], exact[b, ids], rtol=1e-5, atol=1e-6)
                if qlists[b] is not None and len(qlists[b]) <= (256 if k <= 100 else 1024):
                    assert ids == [pid for pid, _ in w[b]], (rank, index, k, b)


@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_sharded_gloo_searcher_matches_unsharded(R, tmp_path, storage):
    """Two gloo ranks on one GPU: bf16 (scan, then exchange), fp8 (each rank re-ranks its shortlist, then exchange), and
    a one-passage index where one rank holds nothing."""
    import torch.multiprocessing as mp
    rows, want, exact = _sharded_case(R, tmp_path)
    ret = mp.Manager().dict()
    mp.spawn(_sharded_worker, args=(2, _free_port(), str(tmp_path), "gloo", storage, ret), nprocs=2, join=True)
    _check_sharded(ret, 2, rows, want, exact, storage)


def test_sharded_nccl_searcher_matches_unsharded(R, tmp_path):
    """The Searcher's C-level NCCL path (flmr_maxsim_topk_sharded_allowed) with one rank per GPU."""
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    rows, want, exact = _sharded_case(R, tmp_path)
    ret = mp.Manager().dict()
    mp.spawn(_sharded_worker, args=(world, _free_port(), str(tmp_path), "nccl", "bf16", ret), nprocs=world, join=True)
    _check_sharded(ret, world, rows, want, exact, "bf16")
