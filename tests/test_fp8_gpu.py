"""e4m3 corpus storage on the GPU: the fp8 scan against the fp8 oracle and the SIMT kernel, its top-k and warpgroup
variants, the two load paths, and the two-stage Searcher (fp8 shortlist + exact bf16 re-rank) against the bf16
Searcher.  Observed errors are printed (run with -s to see them)."""
import ctypes as C

import numpy as np
import pytest
import torch

import fp8_oracle as F8
from helpers import golden_names, load_golden
from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


def _corpus(R, D, dl, storage="fp8", **kw):
    return R.FlatCorpus(torch.from_numpy(np.ascontiguousarray(D)).to(torch.bfloat16), dl, device=0, storage=storage,
                        **kw)


def _rel(got, ref):
    return float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-3)))


def _check_scores(R, Q, D, dl, relu=False, tag=""):
    """wgmma within 1e-4 relative of the fp8 oracle and of SIMT; SIMT within 1e-6 of the oracle.  These are smoke
    tolerances, not the accuracy contract: the fp8 MMA keeps 13 bits below a k-step's leading bit, and the bound a
    score is held to, derived from measured accumulator probes, is scan_fp64.ROW_COEF["fp8"] (checked in
    tests/test_scan_kernels_fp64_gpu.py)."""
    corpus = _corpus(R, D, dl)
    try:
        assert corpus.storage == "fp8"
        Qt = torch.from_numpy(Q)
        got = R.maxsim_scores(corpus, Qt, relu=relu).cpu().numpy()
        simt = R.debug_scores_simt(corpus, Qt, relu=relu).cpu().numpy()
    finally:
        corpus.close()
    ref = F8.maxsim_scores_fp8(Q, D, dl, relu=relu)
    print("[fp8] %s wgmma-vs-oracle %.2e  wgmma-vs-simt %.2e  simt-vs-oracle %.2e"
          % (tag, _rel(got, ref), _rel(got, simt), _rel(simt, ref)))
    np.testing.assert_allclose(simt, ref, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(got, simt, rtol=1e-4, atol=1e-5)
    return got


@pytest.mark.parametrize("name", golden_names())
@pytest.mark.parametrize("relu", [False, True])
def test_golden_fp8_scores(R, name, relu):
    g = load_golden(name)
    _check_scores(R, g["Q"], g["D"], g["doclens"], relu=relu, tag=name + (" relu" if relu else ""))


@pytest.mark.parametrize("n,nd,B,nq,ragged,relu", [
    (1, 9, 2, 32, True, False), (2, 9, 2, 32, True, True), (3, 7, 3, 32, True, False),   # tiny corpora
    (1500, 180, 2, 320, True, False),     # the flagship pass shape
    (900, 64, 12, 32, True, True),        # twelve queries in one pass
    (300, 64, 2, 832, True, False),       # row-sliced queries (three passes of partial scores)
])
def test_seeded_fp8_scores(R, n, nd, B, nq, ragged, relu):
    Q, D, dl = O.synth(n, nd, B, nq, seed=n + nq, ragged=ragged)
    _check_scores(R, Q, D, dl, relu=relu, tag="n=%d nd=%d B=%d nq=%d" % (n, nd, B, nq))


def test_zero_query_rows_stay_zero(R):
    Q, D, dl = O.synth(700, 40, 3, 64, seed=5, ragged=True)
    Q[0, 20:] = 0.0
    Q[2, :] = 0.0                    # an all-zero query scores exactly 0 everywhere
    got = _check_scores(R, Q, D, dl, tag="zero rows")
    assert np.all(got[2] == 0.0)


def test_120k_passages_against_simt(R):
    g = torch.Generator(device="cuda").manual_seed(120)
    dl = torch.randint(24, 65, (120_000,), generator=g, device="cuda").cpu().numpy().astype(np.int32)
    D = torch.randn((int(dl.sum()), 128), generator=g, device="cuda")
    D = torch.nn.functional.normalize(D, dim=1).to(torch.bfloat16)
    Q = torch.nn.functional.normalize(torch.randn((3, 64, 128), generator=g, device="cuda"), dim=2)
    corpus = R.FlatCorpus(D, dl, device=0, storage="fp8")
    del D
    try:
        got = R.maxsim_scores(corpus, Q).cpu().numpy()
        simt = R.debug_scores_simt(corpus, Q).cpu().numpy()
    finally:
        corpus.close()
    print("[fp8] 120k passages wgmma-vs-simt %.2e" % _rel(got, simt))
    np.testing.assert_allclose(got, simt, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("k", [1, 5, 128])
def test_fused_topk_is_a_stable_sort_of_own_scores(R, k):
    Q, D, dl = O.synth(2000, 90, 6, 64, seed=k, ragged=True)
    corpus = _corpus(R, D, dl, pid_base=1000)
    try:
        s = R.maxsim_scores(corpus, torch.from_numpy(Q)).cpu().numpy()
        ts, tp = R.maxsim_topk(corpus, torch.from_numpy(Q), k)
    finally:
        corpus.close()
    rs, rp = O.topk(s, k, pid_base=1000)
    assert np.array_equal(tp.cpu().numpy(), rp)
    assert np.array_equal(ts.cpu().numpy(), rs)


def test_warpgroup_variants_bit_identical_and_no_pair_variant(R):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    Q, D, dl = O.synth(1500, 180, 2, 320, seed=9, ragged=True)
    corpus = _corpus(R, D, dl)
    out = {}
    try:
        for variant in (2, 3):
            assert L.flmr_debug_set_scan_variant(variant) == 0
            s = R.maxsim_scores(corpus, torch.from_numpy(Q))
            ts, tp = R.maxsim_topk(corpus, torch.from_numpy(Q), 17)
            out[variant] = (s.cpu(), ts.cpu(), tp.cpu())
        assert L.flmr_debug_set_scan_variant(4) == 0
        with pytest.raises(_cabi.FlmrError) as e:
            R.maxsim_topk(corpus, torch.from_numpy(Q), 5)
        assert e.value.code == 3   # FLMR_ERR_UNSUPPORTED
    finally:
        L.flmr_debug_set_scan_variant(0)
        corpus.close()
    for a, b in zip(out[2], out[3]):
        assert torch.equal(a, b), "two- and three-warpgroup fp8 kernels differ"


def test_fp8_adopt_is_rejected(R):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    D = torch.randn((16, 128), device="cuda").to(torch.bfloat16)
    dl = np.full(4, 4, dtype=np.int32)
    h = C.c_void_p()
    rc = L.flmr_corpus_create(C.c_void_p(D.data_ptr()), dl.ctypes.data_as(C.c_void_p), 4, 128, 0, 0,
                              _cabi.CORPUS_FP8 | _cabi.CORPUS_ADOPT, C.byref(h))
    assert rc == 1 and not h.value


@pytest.mark.parametrize("ragged", [False, True])
def test_load_paths_bit_identical(R, tmp_path, ragged):
    Q, D, dl = O.synth(3000, 64, 4, 32, seed=int(ragged), ragged=ragged)
    path = R.save_flat_index(str(tmp_path / "idx"), torch.from_numpy(D), dl)
    a = _corpus(R, D, dl)
    b = R.FlatCorpus.from_index(path, device=0, storage="fp8")
    bf = _corpus(R, D, dl, storage="bf16")
    try:
        assert a.storage == b.storage == "fp8" and bf.storage == "bf16"
        sa = R.maxsim_scores(a, torch.from_numpy(Q))
        sb = R.maxsim_scores(b, torch.from_numpy(Q))
        assert torch.equal(sa, sb)
        pids = torch.arange(0, 3000, 7, device="cuda")
        ga, gb, gf = a.gather_padded(pids), b.gather_padded(pids), bf.gather_padded(pids)
        assert torch.equal(ga[0], gb[0]) and torch.equal(ga[0], gf[0]) and torch.equal(ga[1], gf[1])
        print("[fp8] hbm_bytes fp8 %d / bf16 %d" % (a.info.hbm_bytes, bf.info.hbm_bytes))
        assert a.info.hbm_bytes == b.info.hbm_bytes
        assert 0.45 < a.info.hbm_bytes / bf.info.hbm_bytes < 0.55
        from ravqa_b200 import _cabi
        st, host = C.c_int(-1), C.c_int64(-1)
        _cabi.check(_cabi.lib().flmr_corpus_storage(a.handle, C.byref(st), C.byref(host)))
        assert st.value == 1 and host.value == a.info.n_rows * 256
    finally:
        a.close()
        b.close()
        bf.close()


# ---- the two-stage Searcher ---------------------------------------------------------------------------------------
def _compare_searchers(R, Q, D, dl, ks, filters, tag):
    """Searcher(storage="fp8") against Searcher(): scores within 2e-5 relative rank by rank; ids identical wherever
    the exact gap at rank k exceeds 1e-4 relative (and, inside the top k, where neighbours are that far apart)."""
    c8, c16 = _corpus(R, D, dl), _corpus(R, D, dl, storage="bf16")
    try:
        s8, s16 = R.Searcher(index=c8, storage="fp8"), R.Searcher(index=c16)
        exact = R.maxsim_scores(c16, torch.from_numpy(Q)).cpu().numpy()
        for filter_fn in filters:
            ex = exact
            if filter_fn is not None:
                keep = filter_fn(torch.arange(len(dl))).numpy()
                ex = np.full_like(exact, -np.inf)
                ex[:, keep] = exact[:, keep]
            order = np.sort(ex, axis=1)[:, ::-1]
            for k in ks:
                a_s, a_p = s8._search_tensors(torch.from_numpy(Q), k, filter_fn)
                b_s, b_p = s16._search_tensors(torch.from_numpy(Q), k, filter_fn)
                a_s, a_p, b_s, b_p = (t.cpu().numpy() for t in (a_s, a_p, b_s, b_p))
                assert a_s.shape == b_s.shape
                np.testing.assert_allclose(a_s, b_s, rtol=2e-5, atol=1e-6)
                n_mism = 0
                for q in range(Q.shape[0]):
                    kk = a_p.shape[1]
                    top = order[q, :kk + 1]
                    gaps = np.abs(np.diff(top)) / np.maximum(np.abs(top[:-1]), 1e-6)
                    if kk < order.shape[1] and np.isfinite(top[kk]) and gaps[kk - 1] <= 1e-4:
                        n_mism += int(set(a_p[q]) != set(b_p[q]))
                        continue
                    assert set(a_p[q]) == set(b_p[q]), (tag, k, q)
                    sure = np.ones(kk, bool)          # positions whose neighbours are clearly apart
                    sure[1:] &= gaps[:kk - 1] > 1e-4
                    sure[:-1] &= gaps[:kk - 1] > 1e-4
                    assert np.array_equal(a_p[q][sure], b_p[q][sure]), (tag, k, q)
                print("[fp8] searcher %s k=%d filter=%s depth=%s near-tie boundaries differing=%d"
                      % (tag, k, filter_fn is not None, s8._last_depth, n_mism))
        # the RAG block re-scores the retrieved passages from the bf16 master: same doc_scores
        ra = s8.retrieve_and_rescore(torch.from_numpy(Q).cuda(), 5)
        rb = s16.retrieve_and_rescore(torch.from_numpy(Q).cuda(), 5)
        assert np.array_equal(ra["retrieved_doc_ids"], rb["retrieved_doc_ids"])
        assert torch.equal(ra["doc_scores"], rb["doc_scores"])
        rk = s8._search_all_Q(None, torch.from_numpy(Q[:1]), 5)
        assert rk.provenance()["storage"] == "fp8" and rk.provenance()["shortlist_depth"] == min(256, len(dl))
    finally:
        c8.close()
        c16.close()


def _even(pids):
    return pids[pids % 2 == 0]


@pytest.mark.parametrize("name", golden_names())
def test_searcher_fp8_golden(R, name):
    g = load_golden(name)
    _compare_searchers(R, g["Q"], g["D"], g["doclens"], [1, 5, 10, 100], [None, _even], name)


def test_searcher_fp8_20k_isotropic(R):
    Q, D, dl = O.synth(20_000, 180, 8, 32, seed=20)
    _compare_searchers(R, Q, D, dl, [1, 5, 10, 100], [None, _even], "20k x 180")


def test_searcher_storage_mismatch_and_from_index(R, tmp_path):
    Q, D, dl = O.synth(500, 32, 2, 32, seed=3)
    c16 = _corpus(R, D, dl, storage="bf16")
    with pytest.raises(ValueError):
        R.Searcher(index=c16, storage="fp8")
    c16.close()
    path = R.save_flat_index(str(tmp_path / "temp_index.nbits=8"), torch.from_numpy(D), dl)
    s = R.Searcher(index=path, storage="fp8")
    assert s.corpus.storage == "fp8" and s.storage == "fp8"
    pids, _, scores = s.dense_search(torch.from_numpy(Q[:1]), k=5)
    ref_s, ref_p = O.topk(O.maxsim_scores(Q[:1], D, dl), 5)
    assert pids == ref_p[0].tolist()
    np.testing.assert_allclose(scores, ref_s[0], rtol=2e-5)
