"""Restricted search over id lists on the GPU: the scan kernel over a per-call plan of the listed passages' rows
(flmr_maxsim_topk_listed / flmr_maxsim_scores_listed).

(a) bitwise the bitmap (_allowed) calls for the same sets: bf16, fp16 and e4m3 storage, scan variants 0, 2 and 6, relu
    on and off, lane / warp / row-sliced pass shapes, k = 1, 10, 128, lists that are empty, hold one passage, the
    shard's first and last, a long contiguous range (runs across CTA shares), random sets with duplicates and ids
    outside the shard, on the placement fixture (many passage ends per tile) and on 1000-5000-token passages (longer
    than a CTA's share);
(b) pid_base != 0, deleted, compacted-away and appended ids; (c) no stale candidates after a full search;
(d) the planner's invariants (flmr_debug_listed_plan); (e) the Searcher's pids= / qid_to_pids= on both paths, bf16,
    fp16 and fp8, k up to 3000, and two-rank Searchers (gloo; NCCL with two GPUs) with one rank on each path.
"""
import os

import numpy as np
import pytest
import torch

from helpers import placement_doclens

pytestmark = pytest.mark.gpu

NEG = float("-inf")
SHAPES = [(12, 32), (4, 160), (16, 320), (3, 832)]   # lane mode, warp mode, split kernel, row-sliced


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


def _long_doclens():
    rng = np.random.default_rng(5)
    return np.concatenate([rng.integers(1000, 5001, size=40), rng.integers(1, 200, size=300)]).astype(np.int32)


@pytest.fixture(scope="module")
def corpora(R):
    """{(name, storage): corpus}: the placement fixture and a corpus of 1000-5000-token passages among short ones."""
    dls = {"placement": placement_doclens(), "long": _long_doclens()}
    out = {}
    for name, dl in dls.items():
        D = _unit_rows(int(dl.sum()), 7)
        for storage in ("bf16", "fp16", "fp8"):
            out[(name, storage)] = R.FlatCorpus(D, dl, storage=storage)
    yield out
    for c in out.values():
        c.close()


def _lists(c, B, seed):
    """B lists of global ids of shard c, one of each kind, cycling."""
    rng = np.random.default_rng(seed)
    n, base = c.n_passages, c.pid_base
    kinds = [
        lambda: np.array([], np.int64),
        lambda: np.array([base + int(rng.integers(n))]),
        lambda: np.array([base + n - 1, base]),
        lambda: base + np.arange(n // 5, n // 5 + n // 3),                               # a run across CTA shares
        lambda: np.concatenate([base + rng.choice(n, 50), base + rng.choice(n, 20),     # duplicates
                                [base - 1, base + n, base + n + 7]]),                    # outside the shard
        lambda: base + rng.choice(n, n // 20, replace=False),
        lambda: base + rng.choice(n, 3),
    ]
    return [rng.permutation(kinds[(b + seed) % len(kinds)]()).astype(np.int64) for b in range(B)]


def _check_listed(R, c, Q, lists, relu, ks=(1, 10, 128)):
    allow = c.allow_bitmaps(lists)
    for k in ks:
        ws, wp = R.maxsim_topk(c, Q, k, relu=relu, allow=allow)
        gs, gp = R.maxsim_topk(c, Q, k, relu=relu, pids=lists)
        assert torch.equal(gp, wp), k
        assert torch.equal(gs.view(torch.int32), ws.view(torch.int32)), k
    full = R.maxsim_scores(c, Q, relu=relu, allow=allow)
    got = R.maxsim_scores_listed(c, Q, lists, relu=relu)
    want = []
    for b, ids in enumerate(lists):
        local = torch.as_tensor(ids, dtype=torch.int64) - c.pid_base
        inside = (local >= 0) & (local < c.n_passages)
        row = full[b].cpu()
        want.append(torch.where(inside, row[local.clamp(0, c.n_passages - 1)], torch.tensor(NEG)))
    want = torch.cat(want) if want else torch.empty(0)
    assert torch.equal(got.cpu().view(torch.int32), want.view(torch.int32))


# ---- (a) bitwise the bitmap calls ----------------------------------------------------------------------------------
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("variant", [0, 2, 6])
@pytest.mark.parametrize("storage", ["bf16", "fp16", "fp8"])
def test_listed_equals_allowed_placement(R, corpora, storage, variant, shape, relu):
    c = corpora[("placement", storage)]
    B, nq = shape
    Q = _queries(B, nq, seed=B * nq)
    _set_variant(variant)
    try:
        _check_listed(R, c, Q, _lists(c, B, seed=variant + B), relu)
    finally:
        _set_variant(0)


@pytest.mark.parametrize("shape", [(12, 32), (16, 320)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("storage", ["bf16", "fp16", "fp8"])
def test_listed_equals_allowed_long_passages(R, corpora, storage, shape):
    """Passages of 1000-5000 tokens: one passage is longer than a CTA's share of a large union."""
    c = corpora[("long", storage)]
    B, nq = shape
    Q = _queries(B, nq, seed=nq + 1)
    rng = np.random.default_rng(1)
    lists = _lists(c, B, seed=3)
    lists[0] = np.arange(c.n_passages)                                   # everything
    lists[1] = np.concatenate([np.arange(40), rng.choice(c.n_passages, 30)])
    _check_listed(R, c, Q, lists, relu=False)


def test_unsupported_variants_refused(R, corpora):
    from ravqa_b200 import _cabi
    c = corpora[("placement", "bf16")]
    Q = _queries(2, 32, seed=1)
    for v in (3, 4):
        _set_variant(v)
        try:
            with pytest.raises(_cabi.FlmrError, match="variant"):
                R.maxsim_topk(c, Q, 5, pids=[[0], [1]])
        finally:
            _set_variant(0)


# ---- (b) updates -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["bf16", "fp16", "fp8"])
def test_listed_after_delete_compact_append(R, storage):
    dl = placement_doclens(6000, seed=4)
    base = 100_000
    c = R.FlatCorpus(_unit_rows(int(dl.sum()), 3), dl, pid_base=base, storage=storage)
    try:
        rng = np.random.default_rng(0)
        Q = _queries(12, 32, seed=5)
        Q320 = _queries(3, 320, seed=6)

        def lists():
            n = c.n_passages
            out = _lists(c, 12, seed=int(rng.integers(100)))
            out[0] = np.concatenate([dead[:40], base + rng.choice(n, 60)])        # deleted ids
            out[1] = np.concatenate([np.arange(base + n - 30, base + n), [base + n + 1, 5]])
            return out

        dead = base + rng.choice(len(dl), 400, replace=False)
        c.delete(dead)
        _check_listed(R, c, Q, lists(), relu=False)
        c.compact()                                                  # compacted-away ids
        _check_listed(R, c, Q, lists(), relu=True)
        dl2 = np.array([5, 300, 17, 96, 97], np.int32)
        c.append(_unit_rows(int(dl2.sum()), 9), dl2)                 # appended since the compaction
        ls = lists()
        _check_listed(R, c, Q, ls, relu=False)
        _check_listed(R, c, Q320, ls[:3], relu=False, ks=(10,))
    finally:
        c.close()


# ---- (c) no stale candidates -------------------------------------------------------------------------------------
def test_full_search_then_short_list_fills(R, corpora):
    c = corpora[("placement", "bf16")]
    Q = _queries(12, 32, seed=8)
    R.maxsim_topk(c, Q, 128)
    s, p = R.maxsim_topk(c, Q, 128, pids=[[3, 9]] * 12)
    assert (p[:, 2:] == -1).all() and torch.isinf(s[:, 2:]).all()
    assert set(p[:, :2].flatten().tolist()) <= {3, 9}


# ---- (d) the planner -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["placement", "long"])
@pytest.mark.parametrize("shape", [(12, 32), (3, 832)], ids=lambda s: "%dx%d" % s)
def test_plan_invariants(R, corpora, name, shape):
    from ravqa_b200.maxsim import debug_listed_plan
    c = corpora[(name, "bf16")]
    B, nq = shape
    lists = _lists(c, B, seed=11)
    poff = np.concatenate([[0], np.cumsum((c.doclens.astype(np.int64) + 3) // 4 * 4)])
    plans = debug_listed_plan(c, B, nq, lists)
    covered = set()
    for pl in plans:
        qs = range(pl["q_first"], pl["q_first"] + pl["n_q"])
        want = sorted({int(i) for b in qs for i in lists[b] if 0 <= i < c.n_passages})
        assert pl["slots"].tolist() == want
        covered.update(qs)
        rows, mask, first, base = pl["tile_row"], pl["tile_mask"], pl["tile_first"], pl["cta_tile_base"]
        n_tiles = len(rows)
        assert n_tiles <= pl["tile_bound"]
        assert base[0] == 0 and base[-1] == n_tiles and (np.diff(base) >= 0).all()
        want_set = set(want)
        starts_at = {int(poff[s]): s for s in want}   # first stored row -> listed slot
        ends = {}       # slot -> tile index of its end
        share_rows = []
        for cta in range(pl["n_ctas"]):
            t0, t1 = int(base[cta]), int(base[cta + 1])
            for t in range(t0, t1):
                m = int(mask[t]) & 0xFFFFFFFF
                starts = (m >> 31) & 1
                # bit 31 exactly where a run or the CTA's share begins: the share's first tile, or a tile starting at a
                # listed slot whose predecessor is not listed; any other tile follows its predecessor by 96 rows
                run_start = t == t0 or (int(rows[t]) in starts_at and starts_at[int(rows[t])] - 1 not in want_set)
                assert starts == run_start, (cta, t)
                if not run_start:
                    assert rows[t] == rows[t - 1] + 96, (cta, t)
                k = 0
                for g in range(24):
                    if (m >> g) & 1:
                        slot = int(first[t]) + k
                        k += 1
                        assert slot in want_set, (t, g, slot)                    # every end is a listed slot
                        assert poff[slot + 1] - 1 == rows[t] + 4 * g + 3, slot   # at its padded end group
                        assert slot not in ends, slot
                        ends[slot] = t
            share_rows.append(sum(int(poff[s + 1] - poff[s]) for s, t in ends.items() if t0 <= t < t1))
        assert sorted(ends) == want                                  # every listed slot ends in exactly one tile
        if want:     # every share is within one passage plus one tile of the even share
            longest = max(int(poff[s + 1] - poff[s]) for s in want)
            even = sum(int(poff[s + 1] - poff[s]) for s in want) / pl["n_ctas"]
            assert max(abs(r - even) for r in share_rows) <= longest + 96
    assert covered == set(range(B))


# ---- (e) Searcher --------------------------------------------------------------------------------------------------
def _both_paths(R, sr, fn):
    import ravqa_b200.searcher as S
    keep = S.LISTED_SCAN_MAX_ROW_FRACTION
    try:
        S.LISTED_SCAN_MAX_ROW_FRACTION = float("inf")
        a = fn()
        S.LISTED_SCAN_MAX_ROW_FRACTION = -1.0
        b = fn()
    finally:
        S.LISTED_SCAN_MAX_ROW_FRACTION = keep
    return a, b


@pytest.mark.parametrize("k", [10, 128, 300, 3000])
@pytest.mark.parametrize("storage", ["bf16", "fp16", "fp8"])
def test_searcher_listed_and_bitmap_paths_agree(R, corpora, storage, k):
    if storage == "fp8" and k > 2048:
        pytest.skip("fp8 storage re-ranks at most 2048 candidates")
    c = corpora[("placement", storage)]
    sr = R.Searcher(index=c)
    Q = _queries(7, 32, seed=k)
    lists = [ids[(ids >= 0) & (ids < c.n_passages)] for ids in _lists(c, 7, seed=k)]   # the Searcher rejects others
    lists[3] = np.arange(5000)
    qid_to_pids = {"q%d" % b: lists[b] for b in range(7)}
    a, b = _both_paths(R, sr, lambda: sr._search_all_Q(list(qid_to_pids), Q, k, qid_to_pids=qid_to_pids).todict())
    assert a == b
    a, b = _both_paths(R, sr, lambda: sr.dense_search(Q[3:4], k, pids=lists[3]))
    assert a == b


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _sharded_worker(rank, world, port, root, backend, storage, ret):
    import torch.distributed as dist
    import ravqa_b200 as R
    import ravqa_b200.searcher as S
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    kw = {"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    z = np.load(os.path.join(root, "case.npz"))
    lists = {b: z["l%d" % b] for b in range(int(z["B"]))}
    with R.Run().context(R.RunConfig(root=root, experiment="e")):
        sr = R.Searcher(index="flat", config=R.ColBERTConfig(total_visible_gpus=1), shard_across_ranks=True,
                        storage=storage)
    Q = torch.from_numpy(z["Q"])
    # rank 0 takes the listed path, rank 1 the bitmap path, then the other way round: the same collectives either way
    for mode in (0, 1):
        S.LISTED_SCAN_MAX_ROW_FRACTION = float("inf") if (rank + mode) % 2 == 0 else -1.0
        for k in (10, 128):
            rk = sr._search_all_Q(list(lists), Q, k=k, qid_to_pids=lists).todict()
            ret[(rank, mode, k)] = {b: [(pid, sc) for pid, _, sc in rk[b]] for b in rk}
    dist.barrier()
    dist.destroy_process_group()


def _sharded_case(R, tmp_path, storage):
    """Writes the index and the queries; returns the unsharded Searcher's results {k: {row: [(pid, _, score)]}}."""
    dl = placement_doclens(4000, seed=9)
    D = _unit_rows(int(dl.sum()), 10)
    Q = _unit_rows(5 * 32, 11).view(5, 32, 128)
    rng = np.random.default_rng(2)
    lists = {"l%d" % b: rng.choice(len(dl), size=s, replace=False) for b, s in enumerate((3, 40, 0, 500, 2000))}
    R.save_flat_index(str(tmp_path / "e" / "indexes" / "flat"), D, dl)
    np.savez(tmp_path / "case.npz", Q=Q.float().numpy().astype(np.float32), B=5, **lists)
    c = R.FlatCorpus(D, dl, storage=storage)
    try:
        return {k: R.Searcher(index=c)._search_all_Q(list(range(5)), Q, k=k,
                                                     qid_to_pids={b: lists["l%d" % b] for b in range(5)}).todict()
                for k in (10, 128)}
    finally:
        c.close()


def _check_sharded(ret, want, storage):
    for rank in range(2):
        for mode in (0, 1):
            for k in (10, 128):
                got = ret[(rank, mode, k)]
                for b in range(5):
                    w = [(pid, sc) for pid, _, sc in want[k][b]]
                    if storage == "bf16":
                        assert got[b] == w, (rank, mode, k, b)
                    else:
                        assert len(got[b]) == len(w), (rank, mode, k, b)
                assert got == ret[(1 - rank, mode, k)]


@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_sharded_gloo_listed_matches_unsharded(R, tmp_path, storage):
    import torch.multiprocessing as mp
    want = _sharded_case(R, tmp_path, storage)
    ret = mp.Manager().dict()
    mp.spawn(_sharded_worker, args=(2, _free_port(), str(tmp_path), "gloo", storage, ret), nprocs=2, join=True)
    _check_sharded(ret, want, storage)


def test_sharded_nccl_listed_matches_unsharded(R, tmp_path):
    """The Searcher's C-level NCCL path, one rank per GPU: a rank on the listed scan (_listed_topk, then
    flmr_topk_exchange) next to a rank on the bitmap scan (flmr_maxsim_topk_sharded_allowed) makes the same
    collectives, and both answer bitwise as the unsharded bf16 Searcher."""
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    want = _sharded_case(R, tmp_path, "bf16")
    ret = mp.Manager().dict()
    mp.spawn(_sharded_worker, args=(2, _free_port(), str(tmp_path), "nccl", "bf16", ret), nprocs=2, join=True)
    _check_sharded(ret, want, "bf16")
