"""A passage's score is a function of the query and the passage's tokens only, and every ranking path orders exact
ties by its documented rule.

(a) relocation: the same passages scored after a prepended passage, a permutation, sharding (pid_base), an append
    and deletions, and under each forced scan variant, give bitwise the same scores — on a corpus of mostly 1-23
    token passages, where a 96-token tile holds more than the 4 passage ends the reducer sums from row maxima;
(b) batching: a query scored alone, inside a batch of 13 and through a workspace of 2 queries gives the same bits;
(c) duplicate passages rank in ascending id with one score through the fused top-k, topk_select, deletions, the
    shard merge and the fp8 two-stage Searcher;
(d) flmr_topk_merge orders ties by pid across many lists and canonicalises -0.0;
(e) the arg-max kernels pick the lowest unmasked index among exactly tied tokens, and the backward puts the
    gradient on that token only.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from fp8_oracle import maxsim_scores_fp8
from helpers import placement_doclens, placement_tracked, scan_slots
from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu

NQS = [32, 128, 129, 320, 832]   # lane-mode reducer (rbq <= 4), warp mode, row-sliced


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    return ravqa_b200


def _unit_rows(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1).bfloat16()


def _queries(B, nq, seed):
    return _unit_rows(B * nq, seed).view(B, nq, 128)


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def _set_variant(L, v):
    from ravqa_b200 import _cabi
    _cabi.check(L.flmr_debug_set_scan_variant(v))


# ---- (a) relocation invariance ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def placed(R):
    from ravqa_b200.sharded import shard_ranges
    dl = placement_doclens()
    n = len(dl)
    D = _unit_rows(int(dl.sum()), 1)
    off = np.concatenate([[0], np.cumsum(dl)])
    perm = np.random.default_rng(2).permutation(n)
    D_perm = D[torch.from_numpy(np.concatenate([np.arange(off[p], off[p + 1]) for p in perm]))]
    extra_dl = placement_doclens(500, seed=1)
    extra = _unit_rows(int(extra_dl.sum()), 3)
    tracked = placement_tracked(n)
    gone = np.setdiff1d(np.arange(5, n, 101), tracked)               # deleted originals (none tracked)
    built = {}
    for storage in ("bf16", "fp8"):
        mk = lambda T, d, **kw: R.FlatCorpus(T, d, storage=storage, **kw)
        cs = {"base": mk(D, dl), "perm": mk(D_perm, dl[perm])}
        for g in range(1, 6):
            cs["shim%d" % g] = mk(torch.cat([_unit_rows(4 * g, 10 + g), D]), np.concatenate([[4 * g], dl]))
        for w in (2, 4):
            cs["shards%d" % w] = [(p0, mk(D[off[p0]:off[p1]], dl[p0:p1], pid_base=p0))
                                  for p0, p1 in shard_ranges(dl, w)]
        grown = mk(D, dl)
        new_ids = grown.append(extra, extra_dl)
        grown.delete(np.concatenate([new_ids[::2], gone]))
        cs["grown"] = grown
        built[storage] = cs
    yield dict(dl=dl, D=D, n=n, perm=perm, tracked=tracked, gone=gone, corpora=built)
    for cs in built.values():
        for v in cs.values():
            for c in (v if isinstance(v, list) else [v]):
                (c[1] if isinstance(c, tuple) else c).close()


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("nq", NQS)
@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_score_does_not_depend_on_placement(R, placed, storage, nq, relu):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    cs, n, dl = placed["corpora"][storage], placed["n"], placed["dl"]
    Q = _queries(3, nq, 100 + nq)
    score = lambda c: R.maxsim_scores(c, Q, relu=relu)
    base = score(cs["base"])

    for g in range(1, 6):
        assert torch.equal(score(cs["shim%d" % g])[:, 1:], base), "prepended passage of %d groups" % g
    assert torch.equal(score(cs["perm"]), base[:, torch.from_numpy(placed["perm"]).cuda()]), "permutation"
    for w in (2, 4):
        parts = [score(c) for _, c in cs["shards%d" % w]]
        assert torch.equal(torch.cat(parts, dim=1), base), "%d shards" % w
    grown = score(cs["grown"])[:, :n]
    gone = torch.from_numpy(placed["gone"]).cuda()
    assert torch.isneginf(grown[:, gone]).all()
    live = torch.ones(n, dtype=torch.bool, device="cuda")
    live[gone] = False
    assert torch.equal(grown[:, live], base[:, live]), "append + delete"
    try:
        for variant in ((2, 3) if storage == "fp8" else (2, 3, 4)):
            _set_variant(L, variant)
            assert torch.equal(score(cs["base"]), base), "scan variant %d" % variant
    finally:
        L.flmr_debug_set_scan_variant(0)

    tr = placed["tracked"]
    off = np.concatenate([[0], np.cumsum(dl)])
    rows = np.concatenate([np.arange(off[p], off[p + 1]) for p in tr])
    Qf, Df = Q.float().numpy(), placed["D"][torch.from_numpy(rows)].float().numpy()
    got = base[:, torch.from_numpy(tr).cuda()].cpu().numpy()
    if storage == "fp8":   # the e4m3 wgmma does not accumulate to fp32 accuracy (tests/test_fp8_gpu.py: 1e-4)
        np.testing.assert_allclose(got, maxsim_scores_fp8(Qf, Df, dl[tr], relu=relu), rtol=1e-4, atol=1e-5 * nq)
    else:
        np.testing.assert_allclose(got, O.maxsim_scores(Qf, Df, dl[tr], relu=relu), rtol=2e-5, atol=2e-5)


# ---- (b) batch invariance ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("nq", NQS)
@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_score_does_not_depend_on_the_batch(R, placed, storage, nq, relu):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    corpus = placed["corpora"][storage]["base"]
    Q = _queries(13, nq, 200 + nq).cuda()
    batch = R.maxsim_scores(corpus, Q, relu=relu)
    for b in range(13):
        assert torch.equal(R.maxsim_scores(corpus, Q[b:b + 1], relu=relu)[0], batch[b]), b
    ws = C.c_void_p()
    _cabi.check(L.flmr_workspace_create(corpus.handle, 2, nq, C.byref(ws)))
    try:
        out = torch.empty_like(batch)
        _cabi.check(L.flmr_maxsim_scores(corpus.handle, ws, C.c_void_p(Q.data_ptr()), 13, nq,
                                         _cabi.FLAG_RELU if relu else 0, C.c_void_p(out.data_ptr()),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
    finally:
        L.flmr_workspace_destroy(ws)
    assert torch.equal(out, batch)


# ---- (c) duplicate passages ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dup_corpus():
    dl = placement_doclens(20_000, seed=4)
    n = len(dl)
    copies = np.sort(np.random.default_rng(5).choice(np.arange(n), 40, replace=False))
    dl[copies] = 12
    D = _unit_rows(int(dl.sum()), 6)
    P = _unit_rows(12, 7)
    off = np.concatenate([[0], np.cumsum(dl)])
    for p in copies:
        D[off[p]:off[p] + 12] = P
    return dl, D, P, copies


@pytest.mark.parametrize("nq", [32, 320, 832])
def test_duplicate_passages_rank_by_id(R, dup_corpus, nq):
    from ravqa_b200.sharded import shard_ranges
    dl, D, P, copies = dup_corpus
    Q = _queries(2, nq, 300 + nq)
    Q[0, ::2] = P[torch.arange(0, nq, 2) % 12]                          # the copies fill the top of the ranking
    Q[1, 1::2] = P[torch.arange(1, nq, 2) % 12]
    off = np.concatenate([[0], np.cumsum(dl)])
    corpus = R.FlatCorpus(D, dl)
    try:
        slots = scan_slots(dl, corpus.info.n_ctas)[copies]
        assert (slots < 4).any() and (slots >= 4).any(), "copies in both reducer forms"
        want = torch.from_numpy(copies).cuda()
        s128, p128 = R.maxsim_topk(corpus, Q, 128)
        for k in (1, 17, 128):
            s, p = R.maxsim_topk(corpus, Q, k)
            m = min(k, len(copies))
            assert torch.equal(p[:, :m], want[:m].expand(2, m)), k
            assert (s[:, :m] == s[:, :1]).all(), "one score for the class (k=%d)" % k
            assert torch.equal(p, p128[:, :k]) and torch.equal(s, s128[:, :k])
        assert (s128[:, len(copies):] < s128[:, :1]).all()

        sel_s, sel_p = R.Searcher(index=corpus)._search_tensors(Q, 300)  # all scores + topk_select
        assert torch.equal(sel_p[:, :128], p128) and torch.equal(sel_s[:, :128], s128)

        parts = []
        for p0, p1 in shard_ranges(dl, 4):
            c =R.FlatCorpus(D[off[p0]:off[p1]], dl[p0:p1], pid_base=p0)
            parts.append(R.maxsim_topk(c, Q, 128))
            c.close()
        ms, mp_ = R.topk_merge(torch.stack([x[0] for x in parts]), torch.stack([x[1] for x in parts]), 128)
        assert torch.equal(mp_, p128) and torch.equal(ms, s128)

        c8 = R.FlatCorpus(D, dl, storage="fp8")
        try:
            s8, p8 = R.Searcher(index=c8)._search_tensors(Q, len(copies))
            assert torch.equal(p8, want.expand(2, len(copies)))
            assert (s8 == s8[:, :1]).all()
        finally:
            c8.close()

        corpus.delete(copies[:5])                                       # the next ids are promoted
        s, p = R.maxsim_topk(corpus, Q, 17)
        assert torch.equal(p, want[5:22].expand(2, 17)) and torch.equal(s, s128[:, :17])
    finally:
        corpus.close()


# ---- (d) merge ties --------------------------------------------------------------------------------------------------
def _merge_ref(s, p, k_out):
    out_s, out_p = [], []
    for b in range(s.shape[1]):
        fs, fp = s[:, b].reshape(-1) + np.float32(0.0), p[:, b].reshape(-1)   # -0.0 + 0.0 = +0.0
        keep = fp >= 0
        fs, fp = fs[keep], fp[keep]
        order = np.lexsort((fp, -fs.astype(np.float64)))[:k_out]
        out_s.append(fs[order])
        out_p.append(fp[order])
    return np.stack(out_s), np.stack(out_p)


@pytest.mark.parametrize("n_lists,k_in,k_out", [(160, 128, 128), (132, 128, 100), (40, 512, 77), (2, 3, 5)])
def test_topk_merge_ties_and_signed_zero(R, n_lists, k_in, k_out):
    rng = np.random.default_rng(n_lists + k_in)
    B = 3
    levels = np.array([2.0, 1.0, 0.5, 0.0, -0.0, -1.0], np.float32)
    s = levels[rng.integers(0, len(levels), size=(n_lists, B, k_in))]
    s[:, 1] = np.where(rng.random((n_lists, k_in)) < 0.5, np.float32(-0.0), np.float32(0.0))   # zeros only
    p = rng.permutation(n_lists * B * k_in).reshape(n_lists, B, k_in).astype(np.int64)
    p[-1, :, -1] = -1
    ms, mp_ = R.topk_merge(torch.from_numpy(s).cuda(), torch.from_numpy(p).cuda(), k_out)
    rs, rp = _merge_ref(s, p, k_out)
    m = min(k_out, rp.shape[1])
    assert np.array_equal(mp_.cpu().numpy()[:, :m], rp[:, :m])
    assert np.array_equal(_bits(ms.cpu().numpy()[:, :m]), _bits(rs[:, :m])), "-0.0 comes back as +0.0"


def test_topk_merge_minus_zero_ranks_by_pid(R):
    s = torch.tensor([[[-0.0]], [[0.0]]], device="cuda")
    p = torch.tensor([[[1]], [[7]]], device="cuda")
    ms, mp_ = R.topk_merge(s, p, 2)
    assert mp_.tolist() == [[1, 7]]
    assert _bits(ms.cpu().numpy()).tolist() == [[0, 0]]


# ---- (e) arg-max ties --------------------------------------------------------------------------------------------------
def _tied_docs(n, nd, seed):
    """Documents with duplicated token rows: copies adjacent, 64 and 128 positions apart with masked holes between,
    a masked copy before the winner, and a copy pair on both sides of the wgmma path's 128-token chunk boundary in
    the compacted layout.  Returns D [n, nd, 128] bf16, mask [n, nd] and plants [(p, j, copies)]."""
    rng = np.random.default_rng(seed)
    D = _unit_rows(n * nd, seed).view(n, nd, 128).clone()
    mask = torch.from_numpy(rng.random((n, nd)) > 0.1)
    plants = []
    for p in range(n):
        length = int(rng.integers(nd * 3 // 4, nd + 1))
        mask[p, length:] = False
        a = int(rng.integers(1, max(2, length - 130)))
        mask[p, a] = True
        mask[p, a - 1] = False                                          # masked copy before the winner
        cps = [j for j in (a + 1, a + 64, a + 128) if j < length]
        for j in [a - 1] + cps:
            D[p, j] = D[p, a]
        for j in cps:
            mask[p, j] = True
        plants.append((p, a, cps))
        unmasked = torch.nonzero(mask[p]).flatten().tolist()
        j0, j1 = (unmasked[127], unmasked[128]) if len(unmasked) > 129 else (a, a)   # compacted positions 127, 128
        if not {j0, j1} & {a - 1, a, *cps}:
            D[p, j1] = D[p, j0]
            plants.append((p, j0, [j1]))
    return D, mask, plants


def _check_argmax(Q, D, mask, arg, rowmax, docs):
    """One query Q [1, nq, 128] against documents D[p], p in docs: arg / rowmax [1, len(docs), nq] against fp64."""
    Q64, D64 = Q[0].double().numpy(), D.double().numpy()
    m = mask.numpy()
    n_tied = 0
    for p in docs:
        S = Q64 @ D64[p].T                                              # [nq, nd]; copies of a row tie exactly
        S[:, ~m[p]] = -np.inf
        best = S.max(axis=1)
        at_best = S == best[:, None]
        first = at_best.argmax(axis=1)                                  # lowest index among the exact maxima
        a, r = arg[0, p].numpy(), rowmax[0, p].numpy()
        np.testing.assert_allclose(r, best, rtol=0, atol=1e-6)
        tied = at_best.sum(axis=1) > 1
        n_tied += int(tied.sum())
        assert np.array_equal(a[tied], first[tied]), (p, np.nonzero(a[tied] != first[tied]))
        assert m[p][a].all(), "arg on a masked token"
        assert (S[np.arange(len(a)), a] >= best - 1e-5).all()
    return n_tied


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("nq,nd", [(70, 512), (832, 512), (70, 200)])
def test_argmax_ties_pick_lowest_index_and_backward_follows(R, path, nq, nd):
    from ravqa_b200 import _cabi
    from ravqa_b200.maxsim import (maxsim_argmax, maxsim_argmax_grouped, maxsim_backward,
                                   maxsim_backward_grouped)
    L = _cabi.lib()
    B, n = 2, 6
    D, mask, plants = _tied_docs(n, nd, seed=nq + nd)
    Q = _queries(B, nq, 400 + nq)
    for i, (p, j, _) in enumerate(plants):                              # query row i of query (i % B) hits token j
        Q[i % B, i // B] = D[p, j]
    grad = torch.from_numpy(np.random.default_rng(8).standard_normal((B, n)).astype(np.float32))
    try:
        _cabi.check(L.flmr_debug_set_argmax_path(path))
        arg, rowmax = maxsim_argmax(Q.cuda(), D.cuda(), mask.cuda(), return_rowmax=True)
        _, dD = maxsim_backward(Q.cuda(), D.cuda(), arg, grad.cuda(), need_dq=False)
        r = n // B
        garg, growmax = maxsim_argmax_grouped(Q.cuda(), D.cuda(), mask.cuda(), r, return_rowmax=True)
        _, gdD = maxsim_backward_grouped(Q.cuda(), D.cuda(), garg, grad[:, :r].cuda(), need_dq=False)
    finally:
        L.flmr_debug_set_argmax_path(0)
    arg, rowmax, dD = arg.cpu(), rowmax.cpu(), dD.cpu().double().numpy()
    garg, growmax, gdD = garg.cpu(), growmax.cpu(), gdD.cpu().double().numpy()
    # all-pairs
    Qb = Q.double().numpy()
    ref = np.zeros((n, nd, 128))
    n_tied = 0
    for b in range(B):
        n_tied += _check_argmax(Q[b:b + 1], D, mask, arg[b:b + 1], rowmax[b:b + 1], range(n))
        for p in range(n):
            np.add.at(ref[p], arg[b, p].numpy(), grad[b, p].item() * Qb[b])
    assert n_tied >= len(plants), "every planted row meets its copies"
    np.testing.assert_allclose(dD, ref, rtol=1e-5, atol=1e-5)
    # grouped: query b meets documents [b r, (b + 1) r)
    gref = np.zeros((n, nd, 128))
    for b in range(B):
        _check_argmax(Q[b:b + 1], D[b * r:(b + 1) * r], mask[b * r:(b + 1) * r], garg[b:b + 1], growmax[b:b + 1],
                      range(r))
        for p in range(r):
            np.add.at(gref[b * r + p], garg[b, p].numpy(), grad[b, p].item() * Qb[b])
    np.testing.assert_allclose(gdD, gref, rtol=1e-5, atol=1e-5)
    # the copies of a planted token (after the winner) receive nothing
    for p, j, cps in plants:
        for c in cps:
            assert not dD[p, c].any() and not gdD[p, c].any(), (p, j, c)
