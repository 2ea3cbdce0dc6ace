"""GPU: the corpus scan (``maxsim_scores`` / ``maxsim_topk`` over a FlatCorpus, bf16 and e4m3 storage, every scan
variant) and its SIMT cross-check against the float64 restatement of tests/scan_fp64.py (pinned on CPU by
tests/test_scan_fp64_host.py).

* Exact read-backs: every finite bf16 value goes through the corpus conversion (repack / scatter) and through the
  query staging, against one-hot operands, and must come back bitwise (e4m3: as its round-to-nearest-even,
  saturated e4m3 value) — ties to even, the +-448 saturation and the 2^-9 subnormal steps included.
* Accumulator probes: the bits each MMA keeps of ``1 + 2^-j`` and of one dominant product plus 31 / 127 small
  ones, printed; every probe within the bound the grid uses.
* A pairwise grid over storage, variant, relu, Nq, B, passage lengths, corpus size, row kinds and zero query rows:
  every score within its bound, the fused top-k certified against float64 and equal to a stable sort of the
  kernel's own scores.

Each check records its largest error / bound ratio; the module prints them, and the accumulator bits, at the end
(run with -s)."""
import numpy as np
import pytest
import torch

import scan_fp64 as S
from helpers import scan_partition

pytestmark = pytest.mark.gpu

RATIOS = {}
REPORT = []


def _check(name, err, bound):
    S.check_ratio(RATIOS, name, err, bound)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[scan fp64] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[scan fp64]   %-24s %.3e" % (k, RATIOS[k]))
    for line in REPORT:
        print("[scan fp64] " + line)


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


def _corpus(R, D, dl, storage):
    return R.FlatCorpus(D.to(torch.bfloat16), dl, device=0, storage=storage)


def _bits(x):
    return x.float().contiguous().view(torch.int32)


VARIANTS = [("bf16", 0), ("bf16", 2), ("bf16", 3), ("bf16", 4), ("fp8", 0), ("fp8", 2), ("fp8", 3)]


def _readback(tag, storage, got, src):
    """got == src (e4m3: e4m3_round(src)) bitwise, with -0 read as +0 (the reducer adds the query's zero rows).  bf16
    subnormals of a bf16 operand are reported, kept or flushed to +0, each entry one or the other."""
    got = got.cpu()
    want = S.e4m3_round(src) if storage == "fp8" else src.clone()
    want[want == 0] = 0.0
    sub = S.bf16_is_subnormal(src) if storage == "bf16" else torch.zeros_like(src, dtype=torch.bool)
    same = _bits(got) == _bits(want)
    bad = ~same & ~sub
    assert not bad.any(), "%s: %d values differ, e.g. %s -> %s (want %s)" % (
        tag, int(bad.sum()), src[bad][:4].tolist(), got[bad][:4].tolist(), want[bad][:4].tolist())
    if storage == "fp8":   # the edges, by name: saturation, ties to even, subnormal steps
        for x, y in ((1e30, 448.0), (-464.0, -448.0), (1.0625, 1.0), (1.1875, 1.25), (3 * 2.0 ** -10, 2.0 ** -8),
                     (2.0 ** -10, 0.0), (2.0 ** -9, 2.0 ** -9)):
            hit = src == torch.tensor(x, dtype=torch.bfloat16).float()
            assert hit.any() and (got[hit] == y).all(), (tag, x, y)
    if sub.any():
        kept = int((sub & same).sum())
        flushed = int((sub & (_bits(got) == 0)).sum())
        assert kept + flushed == int(sub.sum()), "%s: a bf16 subnormal came back as neither itself nor +0" % tag
        REPORT.append("%s: bf16 subnormals kept %d, flushed to +0 %d" % (tag, kept, flushed))


@pytest.mark.parametrize("storage,variant", VARIANTS)
def test_corpus_readback_every_bf16_value(R, scan_variant, storage, variant):
    """8,192 one-token passages carrying every finite bf16 value (16 rotated copies: every reducer slot 0..23 in
    use) against 128 one-hot queries (Nq = 1, two 64-query chunks): score[b, p] == D[p, b]."""
    D, dl = S.readback_corpus()
    part = scan_partition(dl, torch.cuda.get_device_properties(0).multi_processor_count)
    assert set(part["slot"].tolist()) == set(range(S.SLOTS))
    Q = torch.eye(128).view(128, 1, 128)
    c = _corpus(R, D, dl, storage)
    try:
        scan_variant(variant)
        got = R.maxsim_scores(c, Q)
        scan_variant(0)
        simt = R.debug_scores_simt(c, Q) if variant == 0 else None
    finally:
        c.close()
    _readback("corpus %s v%d" % (storage, variant), storage, got, D.T.contiguous())
    if simt is not None:
        _readback("corpus %s simt" % storage, storage, simt, D.T.contiguous())


@pytest.mark.parametrize("storage,variant", VARIANTS)
def test_query_staging_readback_every_bf16_value(R, scan_variant, storage, variant):
    """The transpose: 512 one-row queries carrying every finite bf16 value against 128 one-hot passages, so the
    values go through the query staging kernel (e4m3: its conversion): score[b, k] == Q[b, 0, k]."""
    V = S.readback_values()
    D, dl = torch.eye(128), np.ones(128, np.int32)
    c = _corpus(R, D, dl, storage)
    try:
        scan_variant(variant)
        got = R.maxsim_scores(c, V.view(512, 1, 128))
        scan_variant(0)
        simt = R.debug_scores_simt(c, V.view(512, 1, 128)) if variant == 0 else None
    finally:
        c.close()
    _readback("staging %s v%d" % (storage, variant), storage, got, V)
    if simt is not None:
        _readback("staging %s simt" % storage, storage, simt, V)


# ---- accumulator probes ----------------------------------------------------------------------------------------------
def _probes(storage):
    """Families of one-token passages against one query row each: name -> (q [128], D [m, 128], exponents j).
    'step j, same' / 'other': 1 + 2^-j with the two products in one k-step of the MMA (dims 0 and 1) or in different
    ones (dims 0 and 64); 'n small': the product 1 on dim 0 plus n products 2^-j on dims 1..n."""
    fam = {}
    if storage == "bf16":
        one_j, small_j = range(1, 31), range(16, 31)
        qs, dsc = 1.0, lambda j: 2.0 ** -j
    else:   # e4m3: q = 2^-9 (the smallest subnormal), d = 2^(9 - j): products 2^-j down to 2^-18
        one_j, small_j = range(1, 19), range(6, 19)
        qs, dsc = 2.0 ** -9, lambda j: 2.0 ** (9 - j)
    for name, k in (("1+2^-j same step", 1), ("1+2^-j other step", 64)):
        q = torch.zeros(128)
        q[0], q[k] = 1.0, qs
        D = torch.zeros((len(one_j), 128))
        D[:, 0] = 1.0
        D[:, k] = torch.tensor([dsc(j) for j in one_j])
        fam[name] = (q, D, list(one_j))
    for n in (31, 127):
        q = torch.zeros(128)
        q[0], q[1:n + 1] = 1.0, qs
        D = torch.zeros((len(small_j), 128))
        D[:, 0] = 1.0
        D[:, 1:n + 1] = torch.tensor([dsc(j) for j in small_j])[:, None]
        fam["1+%d x 2^-j" % n] = (q, D, list(small_j))
    return fam


@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_accumulator_probes(R, storage):
    """The accumulator model behind scan_fp64.ROW_COEF, measured: the leading-bit alignment keeps ALIGN_BITS bits of
    a k-step (1 + 2^-j, both products in one step or in different steps), and a dominant product plus 31 / 127 small
    ones loses every small one just below that cut.  Every probe stays within the grid's bound; the SIMT kernel
    within its rigorous one."""
    fam = _probes(storage)
    names = list(fam)
    Q = torch.stack([fam[n][0] for n in names]).view(len(names), 1, 128)
    D = torch.cat([fam[n][1] for n in names])
    dl = np.ones(D.size(0), np.int32)
    c = _corpus(R, D, dl, storage)
    try:
        got = R.maxsim_scores(c, Q).cpu().double()
        simt = R.debug_scores_simt(c, Q).cpu().double()
    finally:
        c.close()
    p0 = 0
    for f, name in enumerate(names):
        q, Df, js = fam[name]
        m = Df.size(0)
        s64, amax, rabs = S.maxsim_packed(q.view(1, 1, 128), Df, np.ones(m, np.int32), storage=storage)
        g, sm = got[f, p0:p0 + m], simt[f, p0:p0 + m]
        err = (g - s64[0]).abs()
        _check("probe scan " + storage, err, S.scan_bound(amax, rabs, 1, storage)[0])
        _check("probe simt " + storage, (sm - s64[0]).abs(), S.simt_bound(amax, rabs, 1)[0])
        bits = S.ALIGN_BITS[storage]
        if name.startswith("1+2^-j"):
            exact = [float(g[i]) == 1.0 + 2.0 ** -j for i, j in enumerate(js)]
            kept = 0
            while kept < len(js) and exact[kept]:
                kept += 1
            REPORT.append("%s %-18s keeps 1 + 2^-j for j <= %d (an fp32 result holds 23)" % (storage, name, kept))
            assert kept == min(bits, 23), (storage, name, kept)
        else:
            n = int(name.split("+")[1].split(" ")[0])
            REPORT.append("%s %-18s error / 2^-23 at j = %d..%d: %s" % (storage, name, js[0], js[-1], [
                round(float(e) / 2.0 ** -23, 2) for e in err]))
            # products 2^-m below the leading one are kept (up to the final fp32 truncation), 2^-(m+1) all lost
            assert float(err[js.index(bits)]) < 2.0 ** -22, (storage, name)
            assert float(err[js.index(bits + 1)]) == n * 2.0 ** -(bits + 1), (storage, name)
        p0 += m


# ---- the float64 grid ------------------------------------------------------------------------------------------------
GRID = S.scan_grid()


@pytest.mark.parametrize("ci", range(len(GRID)), ids=lambda i: "c%03d" % i)
def test_scan_grid(R, scan_variant, ci):
    c = GRID[ci]
    storage, relu, nq = c["storage"], c["relu"], c["nq"]
    tag = "case %d %s" % (ci, c)
    Q, D, dl = S.case_data(c, S.case_seed(ci))
    Qd = Q.cuda()
    corpus = _corpus(R, D, dl, storage)
    try:
        scan_variant(c["variant"])
        got = R.maxsim_scores(corpus, Qd, relu=relu)
        tops = {k: R.maxsim_topk(corpus, Qd, k, relu=relu) for k in (1, 10, 128)}
        scan_variant(0)
        simt = R.debug_scores_simt(corpus, Qd, relu=relu)
    finally:
        corpus.close()
    s64, amax, rabs = S.maxsim_packed(Qd, D.cuda(), dl, relu=relu, storage=storage)
    bound = S.scan_bound(amax, rabs, nq, storage)
    _check("scan " + storage, (got.double() - s64).abs(), bound)
    _check("simt " + storage, (simt.double() - s64).abs(), S.simt_bound(amax, rabs, nq))
    if c["zeros"] == "query":
        assert (got[0] == 0).all() and (simt[0] == 0).all(), tag
    for k, (ts, tp) in tops.items():
        S.check_topk(got, ts, tp, s64, bound, k, "%s k=%d" % (tag, k))
