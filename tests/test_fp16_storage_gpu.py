"""GPU: fp16 corpus storage (``FlatCorpus(..., storage="fp16")``, FLMR_CORPUS_FP16): the fp16 wgmma scan and the SIMT
cross-check against float64, and every search path on an fp16 shard.

* Exact read-backs: every finite fp16 value (+-0 and the subnormals included) in one-token passages against one-hot
  queries, and transposed in one-row queries against one-hot passages: every score is bitwise the value.  Whether the
  fp16 MMA keeps fp16 subnormals is recorded.
* Accumulator probes (DESIGN.md §2): ``1 + 2^-j`` and one dominant product plus 31 / 127 small ones give the bits an
  fp16 k-step keeps below its leading term; the grid's row bound is derived from that measurement.
* The float64 grid: operands with full fp16 mantissas, Nq around 32 / 384 / 832, lane and warp reducer modes, both
  warpgroup kernels (variants 2 and 6, and 0), ragged lengths, relu, zero query rows.
* Cross-storage identity on inputs exact in bf16 and in fp16's normal range.
* Every path: deletions, allow bitmaps, append, pid_base shards, adoption, the streaming builder, Searcher (k <= 128 and
  k > 128), an fp16 index written by Indexer.
* The call-site PLAID fixture decoded to fp16.

Largest error / bound ratios and the measured model are printed at the end (run with -s)."""
import os

import numpy as np
import pytest
import torch

import scan_fp64 as S
from helpers import GOLDEN_DIR
from oracle import maxsim_oracle as O
from train_fp64 import pairwise_cases

pytestmark = pytest.mark.gpu

RATIOS = {}
REPORT = []
U = 2.0 ** -24


def _check(name, err, bound):
    err, bound = err.double().reshape(-1), bound.double().reshape(-1)
    assert not torch.isnan(err).any(), name
    if err.numel() == 0:
        return
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    worst = int(ratio.argmax())
    r = float(ratio[worst])
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)
    assert r <= 1.0, "%s: error %.3e > bound %.3e (ratio %.3g)" % (name, err[worst], bound[worst], r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[fp16] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[fp16]   %-28s %.3e" % (k, RATIOS[k]))
    for line in REPORT:
        print("[fp16] " + line)


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


@pytest.fixture()
def scan_variant(R):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    yield lambda v: _cabi.check(L.flmr_debug_set_scan_variant(v))
    L.flmr_debug_set_scan_variant(0)


def _f16(R, D, dl, **kw):
    return R.FlatCorpus(D.to(torch.float16), dl, device=0, storage="fp16", **kw)


def _bits(x):
    return x.float().contiguous().view(torch.int32)


# ---- read-backs ---------------------------------------------------------------------------------------------------
def finite_f16_values() -> torch.Tensor:
    """Every finite fp16 value (63,488 bit patterns = 496 rows of 128), as float32, in bit-pattern order."""
    x = torch.arange(1 << 16, dtype=torch.int32).to(torch.int16).view(torch.float16).float()
    return x[torch.isfinite(x)].view(496, 128)


def _readback(tag, got, src):
    got = got.cpu()
    want = src.clone()
    want[want == 0] = 0.0                      # -0 reads back as +0: the reducer adds the query's zero rows
    sub = (src != 0) & (src.abs() < 2.0 ** -14)
    same = _bits(got) == _bits(want)
    bad = ~same & ~sub
    assert not bad.any(), "%s: %d values differ, e.g. %s -> %s" % (tag, int(bad.sum()), src[bad][:4].tolist(),
                                                                     got[bad][:4].tolist())
    kept, flushed = int((sub & same).sum()), int((sub & (_bits(got) == 0)).sum())
    assert kept + flushed == int(sub.sum()), "%s: an fp16 subnormal came back as neither itself nor +0" % tag
    REPORT.append("%s: fp16 subnormals kept %d, flushed to +0 %d" % (tag, kept, flushed))
    return kept, flushed


@pytest.mark.parametrize("variant", [0, 2, 6])
def test_corpus_readback_every_f16_value(R, scan_variant, variant):
    V = finite_f16_values()
    D = torch.cat([torch.roll(V, shifts=r, dims=1) for r in range(16)])   # 7,936 one-token passages
    dl = np.ones(D.size(0), np.int32)
    c = _f16(R, D, dl)
    try:
        scan_variant(variant)
        got = R.maxsim_scores(c, torch.eye(128).view(128, 1, 128))
        scan_variant(0)
        simt = R.debug_scores_simt(c, torch.eye(128).view(128, 1, 128)) if variant == 0 else None
    finally:
        c.close()
    _readback("corpus v%d" % variant, got, D.T.contiguous())
    if simt is not None:
        k_simt, _ = _readback("corpus simt", simt, D.T.contiguous())
        assert k_simt == int(((D != 0) & (D.abs() < 2.0 ** -14)).sum())   # fp32 FMA keeps every fp16 subnormal


@pytest.mark.parametrize("variant", [0, 2, 6])
def test_query_staging_readback_every_f16_value(R, scan_variant, variant):
    V = finite_f16_values()
    c = _f16(R, torch.eye(128), np.ones(128, np.int32))
    try:
        scan_variant(variant)
        got = R.maxsim_scores(c, V.view(496, 1, 128))
        scan_variant(0)
        simt = R.debug_scores_simt(c, V.view(496, 1, 128)) if variant == 0 else None
    finally:
        c.close()
    _readback("staging v%d" % variant, got, V)
    if simt is not None:
        _readback("staging simt", simt, V)


def test_unsupported_variants_are_refused(R, scan_variant):
    from ravqa_b200._cabi import FlmrError
    c = _f16(R, torch.eye(128), np.ones(128, np.int32))
    try:
        for v in (3, 4):
            scan_variant(v)
            with pytest.raises(FlmrError) as e:
                R.maxsim_scores(c, torch.eye(128).view(128, 1, 128))
            assert e.value.code == 3      # FLMR_ERR_UNSUPPORTED
    finally:
        scan_variant(0)
        c.close()


# ---- accumulator probes -------------------------------------------------------------------------------------------
def _probes():
    """name -> (q, D, exponents j): products 1 and 2^-j (q = 2^-14 times d = 2^(14 - j): both normal fp16)."""
    fam = {}
    one_j, small_j = list(range(1, 29)), list(range(16, 29))
    qs, dsc = 2.0 ** -14, lambda j: 2.0 ** (14 - j)
    for name, k in (("1+2^-j same step", 1), ("1+2^-j other step", 64)):
        q = torch.zeros(128)
        q[0], q[k] = 1.0, qs
        D = torch.zeros((len(one_j), 128))
        D[:, 0] = 1.0
        D[:, k] = torch.tensor([dsc(j) for j in one_j])
        fam[name] = (q, D, one_j)
    for n in (31, 127):
        q = torch.zeros(128)
        q[0], q[1:n + 1] = 1.0, qs
        D = torch.zeros((len(small_j), 128))
        D[:, 0] = 1.0
        D[:, 1:n + 1] = torch.tensor([dsc(j) for j in small_j])[:, None]
        fam["1+%d x 2^-j" % n] = (q, D, small_j)
    return fam


@pytest.fixture(scope="module")
def f16_model(R):
    """Runs the probes once: the bits m an fp16 k-step keeps below its leading term, and the row coefficient derived
    from them as for bf16 (scan_fp64 docstring): c = 8 (16 2^-m + 2^-23)."""
    fam = _probes()
    names = list(fam)
    Q = torch.stack([fam[n][0] for n in names]).view(len(names), 1, 128)
    D = torch.cat([fam[n][1] for n in names])
    c = _f16(R, D, np.ones(D.size(0), np.int32))
    try:
        got = R.maxsim_scores(c, Q).cpu().double()
        simt = R.debug_scores_simt(c, Q).cpu().double()
    finally:
        c.close()
    out, p0, bits = {}, 0, None
    for f, name in enumerate(names):
        q, Df, js = fam[name]
        m = Df.size(0)
        s64, amax, rabs = S.maxsim_packed(q.view(1, 1, 128), Df, np.ones(m, np.int32))
        out[name] = (got[f, p0:p0 + m], simt[f, p0:p0 + m], s64[0], amax[0], rabs[0], js)
        if name.startswith("1+127"):
            err = (got[f, p0:p0 + m] - s64[0]).abs()
            lost = [j for i, j in enumerate(js) if float(err[i]) == 127 * 2.0 ** -j]
            assert lost, "no probe lost its small products: widen the exponents"
            bits = lost[0] - 1
            assert all(j in lost for j in js if j > bits), lost
        p0 += m
    coef = 8 * (16 * 2.0 ** -bits + 2.0 ** -23)
    REPORT.append("fp16 k-step keeps %d bits below its leading term: row coefficient %.1f u" % (bits, coef / U))
    return {"bits": bits, "coef": coef, "probes": out}


def test_accumulator_probes(f16_model):
    bits, coef = f16_model["bits"], f16_model["coef"]
    for name, (g, sm, s64, amax, rabs, js) in f16_model["probes"].items():
        err = (g - s64).abs()
        _check("probe scan", err, coef * amax + U * rabs)
        _check("probe simt", (sm - s64).abs(), S.simt_bound(amax, rabs, 1))
        if name.startswith("1+2^-j"):
            kept = 0
            while kept < len(js) and float(g[kept]) == 1.0 + 2.0 ** -js[kept]:
                kept += 1
            REPORT.append("%-18s keeps 1 + 2^-j for j <= %d (an fp32 result holds 23)" % (name, kept))
            assert kept == min(bits, 23), (name, kept)
        else:
            n = int(name.split("+")[1].split(" ")[0])
            REPORT.append("%-18s error / 2^-23 at j = %d..%d: %s" % (name, js[0], js[-1],
                                                                   [round(float(e) / 2.0 ** -23, 2) for e in err]))
            assert float(err[js.index(bits)]) < 2.0 ** -22, name
            assert float(err[js.index(bits + 1)]) == n * 2.0 ** -(bits + 1), name


# ---- the float64 grid ---------------------------------------------------------------------------------------------
FACTORS = {
    "variant": [0, 2, 6],
    "relu": [False, True],
    "nq": [1, 31, 32, 33, 320, 383, 384, 385, 832],
    "B": [1, 12, 13, 65],
    "lengths": ["1", "le4", "mix", "96", "192", "ragged", "long"],
    "n": [1, 3, 133, 2000],
    "rows": ["unit", "norms", "negative", "cancel", "ties"],
    "zeros": ["none", "trailing", "query"],
}
GRID = pairwise_cases(FACTORS, lambda c: True)


def f16_case_data(case, seed):
    """scan_fp64.case_data's structure with every operand given a full fp16 mantissa (a relative perturbation of
    2^-9, then rounded to fp16); ties re-planted after the perturbation."""
    Q, D, dl = S.case_data(dict(case, storage="bf16"), seed)
    g = torch.Generator().manual_seed(seed + 1)
    Q = (Q * (1 + 2.0 ** -9 * torch.randn(Q.shape, generator=g))).half().float()
    D = (D * (1 + 2.0 ** -9 * torch.randn(D.shape, generator=g))).half().float()
    if case["rows"] == "ties":
        off = np.concatenate([[0], np.cumsum(dl)])
        D[off[1:] - 1] = D[off[:-1]]
        for b in range(Q.size(0)):
            Q[b, 0] = D[off[b % len(dl)]]
    if case["zeros"] == "trailing":
        Q[:, Q.size(1) - max(1, Q.size(1) // 3):] = 0.0
    elif case["zeros"] == "query":
        Q[0] = 0.0
    return Q.contiguous(), D.contiguous(), dl


def _check_topk(scores, ts, tp, s64, bound, k, tag):
    rs, rp = O.topk(scores.cpu().numpy(), k)
    assert np.array_equal(tp.cpu().numpy(), rp) and np.array_equal(ts.cpu().numpy(), rs), tag
    lo, hi = s64 - bound, s64 + bound
    n = s64.size(1)
    for b in range(s64.size(0)):
        ids = tp[b][tp[b] >= 0]
        assert ids.numel() == min(k, n), tag
        out = torch.ones(n, dtype=torch.bool, device=s64.device)
        out[ids] = False
        if out.any():
            assert lo[b][out].max() <= hi[b][ids].min(), tag
        assert (hi[b][ids[:-1]] >= lo[b][ids[1:]]).all(), tag


@pytest.mark.parametrize("ci", range(len(GRID)), ids=lambda i: "c%03d" % i)
def test_scan_grid_f16(R, scan_variant, f16_model, ci):
    c = GRID[ci]
    relu, nq = c["relu"], c["nq"]
    tag = "case %d %s" % (ci, c)
    Q, D, dl = f16_case_data(c, 7000 + ci)
    Qd = Q.cuda()
    corpus = _f16(R, D, dl)
    try:
        scan_variant(c["variant"])
        got = R.maxsim_scores(corpus, Qd, relu=relu)
        tops = {k: R.maxsim_topk(corpus, Qd, k, relu=relu) for k in (1, 10, 128)}
        scan_variant(0)
        simt = R.debug_scores_simt(corpus, Qd, relu=relu)
    finally:
        corpus.close()
    s64, amax, rabs = S.maxsim_packed(Qd, D.cuda(), dl, relu=relu)
    bound = f16_model["coef"] * amax + nq * U * rabs
    _check("scan fp16", (got.double() - s64).abs(), bound)
    _check("simt fp16", (simt.double() - s64).abs(), S.simt_bound(amax, rabs, nq))
    if c["zeros"] == "query":
        assert (got[0] == 0).all() and (simt[0] == 0).all(), tag
    for k, (ts, tp) in tops.items():
        _check_topk(got, ts, tp, s64, bound, k, "%s k=%d" % (tag, k))


@pytest.mark.parametrize("nq,B,lengths", [(32, 16, "ragged"), (320, 16, "ragged"), (832, 3, "96")])
def test_cross_storage_identity(R, f16_model, nq, B, lengths):
    """bf16 values inside fp16's normal range are exact in both storages: the two MMAs give equal scores when they
    accumulate alike, and the largest difference is recorded and held to the bound either way."""
    case = dict(nq=nq, B=B, lengths=lengths, n=2000, rows="unit", zeros="none")
    Q, D, dl = S.case_data(dict(case, storage="bf16"), 9000 + nq)
    Q[Q.abs() < 2.0 ** -14] = 0.0
    D[D.abs() < 2.0 ** -14] = 0.0
    out = {}
    for storage in ("bf16", "fp16"):
        c = R.FlatCorpus(D, dl, device=0, storage=storage)
        try:
            out[storage] = (R.maxsim_scores(c, Q), *R.maxsim_topk(c, Q, 100))
        finally:
            c.close()
    diff = (out["fp16"][0] - out["bf16"][0]).abs()
    REPORT.append("cross-storage nq=%d: largest |fp16 - bf16| score difference %.3e, bitwise equal: %s" % (
        nq, float(diff.max()), bool(torch.equal(out["fp16"][0], out["bf16"][0]))))
    s64, amax, rabs = S.maxsim_packed(Q.cuda(), D.cuda(), dl)
    _check("cross-storage", diff.double(), 2 * (f16_model["coef"] * amax + nq * U * rabs))
    if torch.equal(out["fp16"][0], out["bf16"][0]):
        assert torch.equal(out["fp16"][1], out["bf16"][1]) and torch.equal(out["fp16"][2], out["bf16"][2])


# ---- every path ---------------------------------------------------------------------------------------------------
def _data(n=700, seed=3, aligned=False):
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    dl = (rng.integers(1, 12, n) * (4 if aligned else 1) + (0 if aligned else rng.integers(0, 4, n))).astype(np.int32)
    dl = np.maximum(dl, 1)
    D = torch.nn.functional.normalize(torch.randn(int(dl.sum()), 128, generator=g), dim=1).half()
    Q = torch.nn.functional.normalize(torch.randn(6, 40, 128, generator=g), dim=2).half()
    return Q, D, dl


def _ref_scores(R, Q, D, dl):
    c = R.FlatCorpus(D, dl, device=0, storage="fp16", adopt=False)
    try:
        assert c.storage == "fp16" and c.dtype == torch.float16
        return R.maxsim_scores(c, Q).cpu()
    finally:
        c.close()


def test_deletions_and_allow_bitmaps(R):
    Q, D, dl = _data()
    ref = _ref_scores(R, Q, D, dl)
    c = R.FlatCorpus(D, dl, device=0, storage="fp16")
    try:
        dead = np.array([0, 5, 17, 699])
        c.delete(dead)
        s = R.maxsim_scores(c, Q).cpu()
        live = np.setdiff1d(np.arange(len(dl)), dead)
        assert torch.isinf(s[:, dead]).all() and torch.equal(s[:, live], ref[:, live])
        ts, tp = R.maxsim_topk(c, Q, 20)
        want = ref.clone()
        want[:, dead] = -torch.inf
        rs, rp = O.topk(want.numpy(), 20)
        assert np.array_equal(tp.cpu().numpy(), rp)
        lists = [list(range(b, 700, 3)) for b in range(Q.size(0))]
        for allow in (c.allow_bitmaps(lists), c.allow_bitmaps([lists[0]])[0]):
            s = R.maxsim_scores(c, Q, allow=allow).cpu()
            ts, tp = R.maxsim_topk(c, Q, 10, allow=allow)
            for b in range(Q.size(0)):
                ok = np.setdiff1d(lists[b] if allow.dim() == 2 else lists[0], dead)
                assert torch.equal(s[b, ok], ref[b, ok])
                assert set(tp[b].cpu().tolist()) <= set(ok.tolist())
    finally:
        c.close()


def test_append_across_sm_count_and_shards(R):
    Q, D, dl = _data()
    ref = _ref_scores(R, Q, D, dl)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    off = np.concatenate([[0], np.cumsum(dl)])
    n0 = sms // 2                                     # fewer passages than SMs, then past the SM count
    c = R.FlatCorpus(D[:off[n0]], dl[:n0], device=0, storage="fp16")
    try:
        ids = c.append(D[off[n0]:].float(), dl[n0:])  # converted to fp16 on the way in
        assert ids[0] == n0 and c.n_passages == len(dl) and c.info.n_ctas == sms
        assert torch.equal(R.maxsim_scores(c, Q).cpu(), ref)
    finally:
        c.close()
    # two pid_base shards: concatenated scores and merged top-k of the whole corpus
    h = len(dl) // 2
    a = R.FlatCorpus(D[:off[h]], dl[:h], device=0, storage="fp16")
    b = R.FlatCorpus(D[off[h]:], dl[h:], device=0, storage="fp16", pid_base=h)
    try:
        assert torch.equal(torch.cat([R.maxsim_scores(a, Q), R.maxsim_scores(b, Q)], 1).cpu(), ref)
        sa, pa = R.maxsim_topk(a, Q, 50)
        sb, pb = R.maxsim_topk(b, Q, 50)
        ms, mp = R.topk_merge(torch.stack([sa, sb]), torch.stack([pa, pb]), 50)
        rs, rp = O.topk(ref.numpy(), 50)
        assert np.array_equal(mp.cpu().numpy(), rp)
    finally:
        a.close()
        b.close()


def test_adoption_gather_and_conversion(R):
    Q, D, dl = _data(aligned=True)
    ref = _ref_scores(R, Q, D, dl)
    Dg = D.cuda()
    c = R.FlatCorpus(Dg, dl, device=0, storage="fp16")
    try:
        assert c.info.adopted == 1
        assert torch.equal(R.maxsim_scores(c, Q).cpu(), ref)
        assert torch.equal(R.maxsim_scores(c, Q.float()).cpu(), ref)      # fp32 queries: converted with .half()
        E, M = c.gather_padded(torch.tensor([3, 4]))
        assert E.dtype == torch.float16
        off = np.concatenate([[0], np.cumsum(dl)])
        assert torch.equal(E[0][M[0].squeeze(-1)].cpu(), D[off[3]:off[4]])
    finally:
        c.close()
    # fp32 beyond fp16's range becomes +-inf, as torch's .half() (and the reference) make it
    big = torch.zeros(4, 128)
    big[0, 0] = 1e6
    c = R.FlatCorpus(big, np.array([4], np.int32), device=0, storage="fp16")
    try:
        E, _ = c.gather_padded(torch.tensor([0]))
        assert torch.isinf(E[0, 0, 0]) and E[0, 0, 0] > 0
    finally:
        c.close()
    import ctypes as C
    from ravqa_b200._cabi import CORPUS_FP8, CORPUS_FP16, lib
    h = C.c_void_p()
    rc = lib().flmr_corpus_create(C.c_void_p(Dg.data_ptr()), dl.ctypes.data_as(C.c_void_p), len(dl), 128, 0, 0,
                                  CORPUS_FP8 | CORPUS_FP16, C.byref(h))
    assert rc == 1 and not h.value                                       # FLMR_ERR_INVALID_ARG


def test_index_files_builder_searcher_and_indexer(R, tmp_path):
    from ravqa_b200 import Indexer, Searcher, save_flat_index
    Q, D, dl = _data(n=400)
    ref = _ref_scores(R, Q, D, dl)
    path = str(tmp_path / "flat16")
    save_flat_index(path, D.float(), dl, dtype="float16")
    c = R.FlatCorpus.from_index(path, device=0)                  # streamed by the builder, fp16 by default
    try:
        assert c.storage == "fp16" and c.load_stats is not None
        assert torch.equal(R.maxsim_scores(c, Q).cpu(), ref)
    finally:
        c.close()
    c = R.FlatCorpus.from_index(path, device=0, storage="bf16")  # converted once on the way in
    try:
        assert c.storage == "bf16"
        want = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0)
        assert torch.equal(R.maxsim_scores(c, Q).cpu(), R.maxsim_scores(want, Q).cpu())
        want.close()
    finally:
        c.close()
    s = Searcher(path)
    assert s.storage == "fp16"
    for k in (10, 200):
        sc, ids = s._search_tensors(Q.cuda(), k)
        rs, rp = O.topk(ref.numpy(), k)
        assert np.array_equal(ids.cpu().numpy(), rp), k
    # an fp16 index written by Indexer, read back by Searcher
    off = np.concatenate([[0], np.cumsum(dl)])
    passages = list(range(len(dl)))
    enc = lambda ps: (torch.cat([D[off[p]:off[p + 1]].float() for p in ps]), [int(dl[p]) for p in ps])  # noqa: E731
    ipath = Indexer(encode_fn=enc, chunksize=150, storage="fp16").index(str(tmp_path / "idx16"), passages)
    s = Searcher(ipath)
    assert s.storage == "fp16"
    sc, ids = s._search_tensors(Q.cuda(), 10)
    assert np.array_equal(ids.cpu().numpy(), O.topk(ref.numpy(), 10)[1])


# ---- the call-site PLAID fixture, decoded to fp16 -----------------------------------------------------------------
def _fp32_decode(path):
    """The fixture's nbits = 8 PLAID decode in fp32 (torch): centroid + bucket weight of the bit-reversed byte,
    L2-normalised."""
    cen = torch.load(os.path.join(path, "centroids.pt"), map_location="cpu").float()
    _, w = torch.load(os.path.join(path, "buckets.pt"), map_location="cpu")
    codes = torch.load(os.path.join(path, "0.codes.pt"), map_location="cpu").long()
    res = torch.load(os.path.join(path, "0.residuals.pt"), map_location="cpu").long()
    rev = torch.tensor([int("{:08b}".format(i)[::-1], 2) for i in range(256)])
    emb = cen[codes] + w.float()[rev[res]]
    return torch.nn.functional.normalize(emb, dim=-1)


def test_callsite_fixture_from_plaid_fp16(R):
    path = os.path.join(GOLDEN_DIR, "callsites", "ckpt", "temp_index_0", "indexes", "temp_index.nbits=8")
    z = np.load(os.path.join(GOLDEN_DIR, "callsites.npz"))
    corpus = R.FlatCorpus.from_plaid(path, storage="fp16")
    try:
        assert corpus.storage == "fp16"
        n = corpus.n_passages
        E, M = corpus.gather_padded(torch.arange(n))
        got = torch.cat([E[p][M[p].squeeze(-1)] for p in range(n)]).float().cpu()
        ref32 = _fp32_decode(path)[:got.size(0)]
        # within half an fp16 ulp of the fp32 decode (+ fp32 slack: the two normalise in different orders)
        ulp = torch.where(ref32.abs() < 2.0 ** -14, torch.full_like(ref32, 2.0 ** -24),
                          2.0 ** (torch.floor(torch.log2(ref32.abs().clamp_min(2.0 ** -14))) - 10))
        _check("plaid fp16 decode", (got - ref32).abs(), 0.5 * ulp + 2.0 ** -20 * ref32.abs())
        Q = torch.from_numpy(z["queries"])
        s = R.maxsim_scores(corpus, Q).cpu().numpy()
        exact = z["exact_scores"]
        rel = np.abs(s - exact) / np.abs(exact)
        REPORT.append("call-site fixture, fp16 storage: largest relative score error vs the fp32 decode %.3e "
                      "(bf16 storage is held to 3e-3)" % rel.max())
        # the bf16 test's 3e-3 is a bf16 rounding budget (2^-8 relative per operand); fp16 rounds at 2^-11: 3e-3 / 8
        assert rel.max() <= 3e-3 / 8
        k = int(z["k"])
        ts, tp = R.maxsim_topk(corpus, Q, k)
        want = np.argsort(-exact, axis=1, kind="stable")[:, :k]
        assert np.array_equal(tp.cpu().numpy(), want)
    finally:
        corpus.close()
