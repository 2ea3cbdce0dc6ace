"""GPU parity tests proper: the CUDA path (through the C ABI) against
  (a) golden vectors produced by the reference's own code (tests/golden/*.npz),
  (b) the CPU oracle on seeded inputs at sizes it finishes in seconds,
  (c) size-independent properties at large sizes (fused top-k == top-k of all scores, agreement with
      the independent SIMT kernel, permutation / concatenation invariance, idempotence).
Tolerance: bf16 inputs are exact in both paths, accumulation is fp32 in both; the north star allows
1e-3 relative, the tests hold 2e-5 relative.  Top-k ids must be identical.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import golden_names, load_golden
from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu

RTOL = 2e-5


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    return ravqa_b200


def _corpus(R, D, doclens, **kw):
    return R.FlatCorpus(torch.from_numpy(np.ascontiguousarray(D)).to(torch.bfloat16), doclens, **kw)


def _check(R, Q, D, doclens, k, relu=False, ref=None):
    corpus = _corpus(R, D, doclens)
    if ref is None:
        ref = O.maxsim_scores(Q, D, doclens, relu=relu)
    Qt = torch.from_numpy(Q)
    got = R.maxsim_scores(corpus, Qt, relu=relu).cpu().numpy()
    np.testing.assert_allclose(got, ref, rtol=RTOL, atol=1e-5)
    ts, tp = R.maxsim_topk(corpus, Qt, k, relu=relu)
    rs, rp = O.topk(ref, k)
    assert np.array_equal(tp.cpu().numpy(), rp), "top-k ids differ from the oracle"
    valid = rp >= 0
    np.testing.assert_allclose(ts.cpu().numpy()[valid], rs[valid], rtol=RTOL, atol=1e-5)
    assert np.isneginf(ts.cpu().numpy()[~valid]).all()
    corpus.close()


# ---- (a) golden vectors from the reference ------------------------------------------------------
@pytest.mark.parametrize("name", golden_names())
def test_golden_true_max(R, name):
    g = load_golden(name)
    corpus = _corpus(R, g["D"], g["doclens"])
    got = R.maxsim_scores(corpus, torch.from_numpy(g["Q"])).cpu().numpy()
    np.testing.assert_allclose(got, g["scores_true_max"], rtol=RTOL, atol=1e-5)
    k = g["topk_pids"].shape[1]
    ts, tp = R.maxsim_topk(corpus, torch.from_numpy(g["Q"]), k)
    assert np.array_equal(tp.cpu().numpy(), g["topk_pids"])
    np.testing.assert_allclose(ts.cpu().numpy(), g["topk_scores"], rtol=RTOL, atol=1e-5)


@pytest.mark.parametrize("name", golden_names())
def test_golden_relu_variant(R, name):
    """FLMR_FLAG_RELU reproduces the reference CPU packed path (segmented_maxsim.cpp zero init)."""
    g = load_golden(name)
    corpus = _corpus(R, g["D"], g["doclens"])
    got = R.maxsim_scores(corpus, torch.from_numpy(g["Q"]), relu=True).cpu().numpy()
    np.testing.assert_allclose(got, g["scores_relu"], rtol=RTOL, atol=1e-5)


# ---- (b) oracle on seeded inputs ------------------------------------------------------------------
def test_config_c1_16q_1k_passages(R):
    """BASELINE.json configs[0]: 16 queries x 1k passages, Nq=32, Nd=64, d=128."""
    Q, D, dl = O.synth(1000, 64, 16, 32, seed=0)
    _check(R, Q, D, dl, k=5)


@pytest.mark.parametrize("n,nd,B,nq,k,ragged,relu,seed", [
    (1000, 64, 16, 32, 10, True, False, 1),      # ragged lengths (group padding + repack path)
    (700, 12, 5, 32, 7, True, True, 2),          # short docs, ReLU path differs from true max
    (3000, 180, 2, 320, 5, False, False, 3),     # north-star shape: 3 resident query tiles
    (900, 200, 3, 96, 100, True, False, 4),      # several queries per pass, k = 100
    (600, 150, 2, 832, 20, True, False, 5),      # FLMR full query (512 text + 320 vision): row slices
    (400, 90, 1, 400, 128, True, True, 6),       # 2 slices, k = FLMR_MAX_K, relu
    (500, 120, 7, 832, 5, True, False, 15),      # 7 long queries: tail slices share passes in groups of 6 (6+1)
    (300, 60, 3, 1500, 9, True, True, 16),       # 4 slices (384+384+384+348): tail groups of 1, relu
    (200, 50, 2, 1280, 4, True, False, 17),      # 4 slices, 128-row tails in groups of 3 (one pass)
    (257, 33, 13, 45, 3, True, False, 7),        # nq not a multiple of 32, 13 queries (3 passes)
    (50, 700, 2, 64, 5, True, False, 8),         # passages longer than several 128-token tiles
    (5000, 3, 2, 32, 10, True, False, 9),        # tiny passages: up to 32 passage ends per tile
])
def test_seeded_vs_oracle(R, n, nd, B, nq, k, ragged, relu, seed):
    Q, D, dl = O.synth(n, nd, B, nq, seed=seed, ragged=ragged)
    _check(R, Q, D, dl, k=k, relu=relu)


def test_empty_ragged_and_tiny_corpora(R):
    for n, k in [(1, 1), (1, 5), (2, 5), (3, 128), (149, 5)]:
        Q, D, dl = O.synth(n, 9, 2, 32, seed=n, ragged=True)
        _check(R, Q, D, dl, k=k)
    # zero queries is a no-op
    Q, D, dl = O.synth(10, 8, 1, 32, seed=0)
    corpus = _corpus(R, D, dl)
    s = R.maxsim_scores(corpus, torch.zeros(0, 32, 128))
    assert tuple(s.shape) == (0, 10)


def test_zero_query_rows_and_zero_passage_rejected(R):
    Q, D, dl = O.synth(300, 40, 2, 40, seed=11, ragged=True)
    Q[:, 30:, :] = 0.0                              # masked query tokens are exact zero rows
    _check(R, Q, D, dl, k=5)
    with pytest.raises(Exception, match="zero-length"):
        R.FlatCorpus(torch.zeros(4, 128, dtype=torch.bfloat16), [4, 0])


def test_corpus_creation_paths_agree(R):
    """host pointer (chunked staging) / device copy+repack / zero-copy adoption give identical scores."""
    Q, D, dl = O.synth(500, 64, 2, 32, seed=12)               # doclens multiple of 4 -> adoptable
    Dt = torch.from_numpy(D).to(torch.bfloat16)
    c_host = R.FlatCorpus(Dt, dl)
    c_copy = R.FlatCorpus(Dt.cuda(), dl, adopt=False)
    c_adopt = R.FlatCorpus(Dt.cuda(), dl, adopt=True)
    assert c_adopt.info.adopted == 1 and c_copy.info.adopted == 0 and c_host.info.adopted == 0
    Qt = torch.from_numpy(Q)
    a = R.maxsim_scores(c_host, Qt)
    assert torch.equal(a, R.maxsim_scores(c_copy, Qt)) and torch.equal(a, R.maxsim_scores(c_adopt, Qt))
    Q2, D2, dl2 = O.synth(500, 61, 2, 32, seed=13, ragged=True)   # not adoptable: falls back to repack
    c2 = R.FlatCorpus(torch.from_numpy(D2).to(torch.bfloat16).cuda(), dl2, adopt=True)
    assert c2.info.adopted == 0 and c2.info.n_rows >= c2.info.n_tokens
    np.testing.assert_allclose(R.maxsim_scores(c2, torch.from_numpy(Q2)).cpu().numpy(),
                               O.maxsim_scores(Q2, D2, dl2), rtol=RTOL)


def test_pid_base_and_error_codes(R):
    Q, D, dl = O.synth(200, 20, 2, 32, seed=14, ragged=True)
    corpus = _corpus(R, D, dl, pid_base=1_000_000)
    ts, tp = R.maxsim_topk(corpus, torch.from_numpy(Q), 5)
    rs, rp = O.topk(O.maxsim_scores(Q, D, dl), 5, pid_base=1_000_000)
    assert np.array_equal(tp.cpu().numpy(), rp)
    with pytest.raises(ValueError):
        R.maxsim_topk(corpus, torch.from_numpy(Q), 129)
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    out_s = torch.empty(2, 200, device="cuda")
    rc = L.flmr_maxsim_topk(corpus.handle, corpus.workspace(), C.c_void_p(out_s.data_ptr()), 2, 32, 500, 0,
                            C.c_void_p(out_s.data_ptr()), C.c_void_p(out_s.data_ptr()), None)
    assert rc == 3 and b"k=500" in L.flmr_last_error()


def test_topk_merge_kernel(R):
    rng = np.random.default_rng(0)
    n_lists, B, k_in, k_out = 8, 5, 20, 20
    s = rng.standard_normal((n_lists, B, k_in)).astype(np.float32)
    s[0, :, :3] = s[1, :, :3]                                   # force score ties across lists
    p = rng.permutation(n_lists * B * k_in).reshape(n_lists, B, k_in).astype(np.int64)
    p[2, :, -2:] = -1                                           # padding entries are ignored
    ms, mp_ = R.topk_merge(torch.from_numpy(s).cuda(), torch.from_numpy(p).cuda(), k_out)
    for b in range(B):
        fs, fp = s[:, b].reshape(-1), p[:, b].reshape(-1)
        keep = fp >= 0
        fs, fp = fs[keep], fp[keep]
        order = np.lexsort((fp, -fs.astype(np.float64)))[:k_out]
        assert np.array_equal(mp_[b].cpu().numpy(), fp[order])
        assert np.array_equal(ms[b].cpu().numpy(), fs[order])


# ---- (c) properties at sizes the oracle cannot reach ----------------------------------------------
@pytest.fixture(scope="module")
def big(R):
    n_p, nd, nq = 120_000, 180, 320                            # 21.6M tokens = 5.5 GB of bf16
    g = torch.Generator(device="cuda").manual_seed(0)
    D = torch.nn.functional.normalize(torch.randn((n_p * nd, 128), device="cuda", generator=g), dim=-1)
    D = D.to(torch.bfloat16)
    Q = torch.nn.functional.normalize(torch.randn((3, nq, 128), device="cuda", generator=g), dim=-1)
    Q = Q.to(torch.bfloat16)
    corpus = R.FlatCorpus(D, np.full(n_p, nd, dtype=np.int32))
    yield corpus, D, Q, n_p, nd
    corpus.close()


def test_big_fused_topk_equals_topk_of_all_scores(R, big):
    corpus, D, Q, n_p, nd = big
    s_all = R.maxsim_scores(corpus, Q)
    for k in (1, 5, 100):
        ts, tp = R.maxsim_topk(corpus, Q, k)
        rs, rp = torch.sort(s_all, dim=1, descending=True, stable=True)
        assert torch.equal(tp, rp[:, :k]) and torch.equal(ts, rs[:, :k])
    # idempotence: the scan is deterministic (fixed-order reductions, no atomics)
    assert torch.equal(s_all, R.maxsim_scores(corpus, Q))


def test_big_agrees_with_independent_simt_kernel_and_torch(R, big):
    corpus, D, Q, n_p, nd = big
    s_all = R.maxsim_scores(corpus, Q[:1])
    s_simt = R.debug_scores_simt(corpus, Q[:1])
    rel = ((s_all - s_simt).abs() / s_simt.abs().clamp_min(1e-6)).max().item()
    assert rel < RTOL, rel
    # torch fp32 reference (colbert_score semantics) on the top-5 and 2000 random passages
    _, tp = R.maxsim_topk(corpus, Q[:1], 5)
    pick = torch.cat([tp[0], torch.randint(0, n_p, (2000,), device="cuda")])
    Dp = D.view(n_p, nd, 128)[pick].float()
    ref = (Dp @ Q[0].float().T).max(dim=1).values.sum(dim=-1)
    np.testing.assert_allclose(s_all[0, pick].cpu().numpy(), ref.cpu().numpy(), rtol=RTOL)


def test_big_planted_positive_recall(R, big):
    """Recall@5 with a known positive: copy 24 token rows of a passage into the query."""
    corpus, D, Q, n_p, nd = big
    g = torch.Generator(device="cuda").manual_seed(1)
    targets = torch.randint(0, n_p, (3,), device="cuda", generator=g)
    Qp = Q.clone()
    for b, t in enumerate(targets.tolist()):
        Qp[b, :24] = D[t * nd: t * nd + 24]
    _, tp = R.maxsim_topk(corpus, Qp, 5)
    assert all(int(targets[b]) == int(tp[b, 0]) for b in range(3))


def test_shard_concatenation_invariance(R):
    """Sharding property (SURVEY 8e): top-k over the whole corpus == merge of per-shard top-k, bitwise.
    30-60-token passages: at most 4 passage ends per 96-token tile."""
    _check_shard_concatenation(R, 4000, 60, 21)


def test_shard_concatenation_invariance_short_passages(R):
    """The same property on 12-23-token passages: a tile holds more than 4 passage ends, so sharding moves passages
    between the reducer's two forms of partial sums (parked row maxima and the consumer warps' 16-row sums)."""
    _check_shard_concatenation(R, 8000, 23, 22)


def _check_shard_concatenation(R, n, nd, seed):
    from ravqa_b200.sharded import shard_ranges
    Q, D, dl = O.synth(n, nd, 4, 64, seed=seed, ragged=True)
    whole = _corpus(R, D, dl)
    ws, wp = R.maxsim_topk(whole, torch.from_numpy(Q), 10)
    off = np.concatenate([[0], np.cumsum(dl)])
    parts_s, parts_p = [], []
    for p0, p1 in shard_ranges(dl, 4):
        c = _corpus(R, D[off[p0]:off[p1]], dl[p0:p1], pid_base=p0)
        s, p = R.maxsim_topk(c, torch.from_numpy(Q), 10)
        parts_s.append(s)
        parts_p.append(p)
    ms, mp_ = R.topk_merge(torch.stack(parts_s), torch.stack(parts_p), 10)
    assert torch.equal(mp_, wp) and torch.equal(ms, ws)


def test_searcher_facade(R, tmp_path):
    """colbert.Searcher call surface: _search_all_Q / dense_search / Ranking.todict (searcher.py:73-132)."""
    Q, D, dl = O.synth(800, 50, 6, 32, seed=31, ragged=True)
    path = R.save_flat_index(str(tmp_path / "temp_index.nbits=8"), torch.from_numpy(D), dl)
    searcher = R.Searcher(index=path)
    queries = {"q%d" % i: "text %d" % i for i in range(6)}
    ranking = searcher._search_all_Q(queries, torch.from_numpy(Q), k=10, progress=False)
    ref_s, ref_p = O.topk(O.maxsim_scores(Q, D, dl), 10)
    d = ranking.todict()
    assert list(d.keys()) == list(queries.keys())
    for i, qid in enumerate(queries):
        pids, ranks, scores = zip(*d[qid])
        assert list(pids) == ref_p[i].tolist() and list(ranks) == list(range(1, 11))
        np.testing.assert_allclose(scores, ref_s[i], rtol=RTOL)
    pids, ranks, scores = searcher.dense_search(torch.from_numpy(Q[2:3]), k=5)
    assert pids == ref_p[2, :5].tolist() and ranks == [1, 2, 3, 4, 5]
    # filter_fn (IndexScorer.rank filter hook): keep even pids only
    pids, _, _ = searcher.dense_search(torch.from_numpy(Q[0:1]), k=5, filter_fn=lambda p: p[p % 2 == 0])
    s0 = O.maxsim_scores(Q[0:1], D, dl)[0]
    even = np.arange(0, 800, 2)
    assert pids == even[np.argsort(-s0[even], kind="stable")[:5]].tolist()
    # k beyond the fused top-k capacity (FLMR_MAX_K = 128): all scores from the scan + selection
    pids, ranks, scores = searcher.dense_search(torch.from_numpy(Q[1:2]), k=300)
    s1 = O.maxsim_scores(Q[1:2], D, dl)[0]
    assert pids == np.argsort(-s1, kind="stable")[:300].tolist() and len(ranks) == 300
    # the reference's (dead) default flag is accepted; the search still runs on the GPU
    assert R.Searcher(index=path, disable_gpu=True).corpus.device.type == "cuda"


def test_topk_select_kernel(R):
    """flmr_topk_select (k beyond the fused capacity): radix select + ordered compaction + bitonic sort."""
    rng = np.random.default_rng(5)
    for n, k in [(50_000, 1000), (4097, 2048), (300, 500), (1, 1), (70_000, 129)]:
        s = rng.standard_normal((3, n)).astype(np.float32)
        s[1] = np.round(s[1], 1)                                   # massive ties -> lower pid first
        if n > 10:
            s[2, :7] = np.inf
            s[2, 7:9] = -np.inf
        vs, ps = R.topk_select(torch.from_numpy(s).cuda(), k, pid_base=10)
        rs, rp = O.topk(s, k, pid_base=10)
        assert np.array_equal(ps.cpu().numpy(), rp), (n, k)
        assert np.array_equal(vs.cpu().numpy(), rs), (n, k)
    with pytest.raises(ValueError):
        R.topk_select(torch.zeros(2, 10, device="cuda"), 4096)


@pytest.mark.parametrize("case", [
    (3000, 60, 1, 32, True, False, 5), (3000, 60, 2, 64, True, True, 7), (2000, 180, 1, 320, False, False, 5),
    (2000, 180, 2, 320, True, False, 100), (1500, 90, 3, 129, True, False, 5), (1200, 100, 5, 97, True, False, 3),
    (900, 64, 20, 32, True, False, 5), (700, 50, 3, 832, True, False, 10), (5, 7, 2, 320, True, False, 5),
    (2500, 13, 2, 320, True, False, 5), (800, 200, 16, 320, True, False, 5),
    # row-sliced queries under CTA pairs: 6 queries of Nq = 832 per pair group (+1 left over), 4 of Nq = 1500 (+1),
    # and Nq = 641 whose one-row tails fill a pair group only from 40 queries up
    (700, 50, 7, 832, True, False, 10), (600, 40, 5, 1500, True, True, 5), (400, 30, 43, 641, True, False, 4)])
def test_three_warpgroup_scan_kernel_is_bit_identical(case):
    """flmr_scan_kernel<3> (three consumer warpgroups; the product uses it for passes with three resident query
    tiles) forced onto every pass shape: scores and fused top-k bit-identical to flmr_scan_kernel<2>'s and within
    2e-5 of the oracle."""
    import ravqa_b200 as R
    from ravqa_b200 import _cabi
    n, nd, B, nq, ragged, relu, k = case
    L = _cabi.lib()
    Q, D, dl = O.synth(n, nd, B, nq, seed=n + nq, ragged=ragged)
    corpus = R.FlatCorpus(torch.from_numpy(D).to(torch.bfloat16), dl, device=0)
    Qt = torch.from_numpy(Q)
    try:
        outs = {}
        for variant in (2, 3, 0, 4):
            _cabi.check(L.flmr_debug_set_scan_variant(variant))
            outs[variant] = (R.maxsim_scores(corpus, Qt, relu=relu), *R.maxsim_topk(corpus, Qt, min(k, n), relu=relu))
    finally:
        L.flmr_debug_set_scan_variant(0)
    for x, y in zip(outs[2], outs[3]):
        assert torch.equal(x, y)
    # CTA-pair passes (variant 4) partition the passages differently; every passage end is summed in the same order,
    # so the scores are bitwise those of the single-CTA kernel too
    for variant in (4, 0):
        for x, y in zip(outs[variant], outs[2]):
            assert torch.equal(x, y), variant
    ref = O.maxsim_scores(Q, D, dl, relu=relu)
    np.testing.assert_allclose(outs[3][0].cpu().numpy(), ref, rtol=2e-5)


def test_c2_shape_against_the_c_oracle():
    """BASELINE.json configs[1] (PreFLMR ViT-B on OK-VQA's GoogleSearch corpus) at its exact query shape — the full
    832-row FLMR query (512 text + 320 vision rows), row-sliced over passes, k = max(Ks) = 100
    (FLMR_base_preload_vision_features.jsonnet:141) — over a 2,000-passage ragged slice (90..180 tokens), against the
    plain-C oracle: scores within 2e-5, the 100 ids identical."""
    import ravqa_b200 as R
    from helpers import c_oracle_scores
    rng = np.random.default_rng(77)
    n, nq, B, k = 2000, 832, 3, 100
    dl = rng.integers(90, 181, size=n).astype(np.int32)
    g = torch.Generator().manual_seed(77)
    D = torch.nn.functional.normalize(torch.randn(int(dl.sum()), 128, generator=g), dim=-1).bfloat16().float().numpy()
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).bfloat16().float().numpy()
    corpus = R.FlatCorpus(torch.from_numpy(D).to(torch.bfloat16), dl, device=0)
    ref = c_oracle_scores(Q, D, dl, nthreads=8)
    got = R.maxsim_scores(corpus, torch.from_numpy(Q)).cpu().numpy()
    np.testing.assert_allclose(got, ref, rtol=2e-5)
    s, p = R.Searcher(index=corpus)._search_tensors(torch.from_numpy(Q), k)
    rs, rp = O.topk(ref, k)
    assert np.array_equal(p.cpu().numpy(), rp)
    np.testing.assert_allclose(s.cpu().numpy(), rs, rtol=2e-5)


def test_big_cta_pair_passes_properties(R, big):
    """120k passages, SIX Nq = 320 queries through three CTA-pair passes (variant 4: clusters of two CTAs, TMA
    multicast, one query resident in each CTA).  Fused top-k == stable sort of all scores (same call pattern),
    deterministic, and bitwise equal to the single-CTA kernel forced onto all six (another tile partition, the same
    summation order)."""
    from ravqa_b200 import _cabi
    corpus, D, Q3, n_p, nd = big
    L = _cabi.lib()
    g = torch.Generator(device="cuda").manual_seed(9)
    Q = torch.nn.functional.normalize(torch.randn((6, 320, 128), device="cuda", generator=g), dim=-1).to(torch.bfloat16)
    for b, t in enumerate([0, 1, n_p // 2, n_p - 1, 77, n_p - 2]):        # planted positives incl. both corpus ends
        Q[b, :32] = D[t * nd: t * nd + 32]
    try:
        _cabi.check(L.flmr_debug_set_scan_variant(4))
        L.flmr_launch_count(1)
        s_all = R.maxsim_scores(corpus, Q)
        assert L.flmr_launch_count(1) == 4                                # one staging launch + three pair passes of 2
        for k in (5, 100):
            ts, tp = R.maxsim_topk(corpus, Q, k)
            rs, rp = torch.sort(s_all, dim=1, descending=True, stable=True)
            assert torch.equal(tp, rp[:, :k]) and torch.equal(ts, rs[:, :k])
        assert [int(tp[b, 0]) for b in range(6)] == [0, 1, n_p // 2, n_p - 1, 77, n_p - 2]
        assert torch.equal(s_all, R.maxsim_scores(corpus, Q))
        _cabi.check(L.flmr_debug_set_scan_variant(2))
        s_single = R.maxsim_scores(corpus, Q)
        _, tp_single = R.maxsim_topk(corpus, Q, 100)
    finally:
        L.flmr_debug_set_scan_variant(0)
    assert torch.equal(s_all, s_single)
    assert torch.equal(tp, tp_single)


def test_search_call_is_cuda_graph_capturable(R):
    """flmr_maxsim_topk / flmr_maxsim_scores enqueue their launches (query staging, single-CTA and cluster scan
    passes, merges) on the caller's stream and synchronise nothing: a call captured into a CUDA graph and replayed
    on NEW query contents gives exactly what the eager call gives — whole queries, CTA-pair passes forced, the product's
    split kernel and row-sliced queries (variant 0), fp16 and e4m3 corpora, allow bitmaps (replayed with new contents
    too), and a compacted corpus with deletions, whose score rows and bitmaps go through stream-ordered scratch."""
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    cases = [  # n, nd, B, nq, k, variant, storage, allow, compact
        (3000, 60, 5, 97, 7, 0, "bf16", False, False), (2000, 120, 6, 320, 10, 4, "bf16", False, False),
        (900, 50, 7, 832, 5, 4, "bf16", False, False), (2000, 120, 6, 320, 10, 0, "bf16", False, False),
        (900, 50, 3, 832, 128, 0, "bf16", False, False), (1500, 80, 12, 32, 128, 0, "fp16", False, False),
        (1500, 80, 4, 320, 16, 0, "fp8", False, False), (2500, 60, 5, 97, 128, 0, "bf16", True, False),
        (2500, 60, 3, 320, 20, 0, "fp8", True, True), (2500, 60, 6, 32, 50, 0, "fp16", False, True),
        (1200, 40, 2, 832, 9, 0, "bf16", True, True)]
    for (n, nd, B, nq, k, variant, storage, with_allow, compact) in cases:
        Q0, D, dl = O.synth(n, nd, B, nq, seed=17 + nq, ragged=True)
        dt = torch.float16 if storage == "fp16" else torch.bfloat16
        corpus = R.FlatCorpus(torch.from_numpy(D).to(dt), dl, device=0, storage=storage)
        try:
            if compact:
                corpus.delete(np.arange(0, n, 3))
                corpus.compact()
            _cabi.check(L.flmr_debug_set_scan_variant(variant))
            Qs = torch.from_numpy(Q0).cuda().to(dt)
            rng = np.random.default_rng(nq)
            allow = (corpus.allow_bitmaps([rng.choice(n, 60, replace=False) for _ in range(B)])
                     if with_allow else None)
            R.maxsim_topk(corpus, Qs, k, allow=allow)         # first call outside capture (sizes the workspace)
            R.maxsim_scores(corpus, Qs, allow=allow)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                gs, gp = R.maxsim_topk(corpus, Qs, k, allow=allow)
                ga = R.maxsim_scores(corpus, Qs, allow=allow)
            for seed in (1, 2):
                Q1, _, _ = O.synth(4, 4, B, nq, seed=seed)
                Qs.copy_(torch.from_numpy(Q1).cuda().to(dt))
                if with_allow:
                    allow.copy_(corpus.allow_bitmaps([rng.choice(n, 60, replace=False) for _ in range(B)]))
                graph.replay()
                torch.cuda.synchronize()
                es, ep = R.maxsim_topk(corpus, Qs, k, allow=allow)
                ea = R.maxsim_scores(corpus, Qs, allow=allow)
                assert torch.equal(gs, es) and torch.equal(gp, ep) and torch.equal(ga, ea), (nq, variant, storage)
                if storage == "bf16" and not with_allow and not compact:
                    ref = O.maxsim_scores(Q1, D, dl)
                    np.testing.assert_allclose(ga.cpu().numpy(), ref, rtol=2e-5)
        finally:
            L.flmr_debug_set_scan_variant(0)
            corpus.close()
