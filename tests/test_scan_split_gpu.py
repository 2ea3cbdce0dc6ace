"""GPU: flmr_scan_split_kernel (scan variant 6, three consumer warpgroups folding one half of each tile while the other
half's MMAs run) against flmr_scan_kernel<3> (variant 3; fp16 corpora, which have no such kernel, against the
two-warpgroup fp16 kernel of variant 2): bitwise the same scores and fused top-k, and the default selection (variant 0)
with them.

The cases cover every storage, relu on and off, passes of five and six occupied 64-row blocks (2/2/1 and 2/2/2 over
the warpgroups: Nq 288 / 320 / 321 / 384, the row slices of Nq 832, 10-12 queries of 32 rows per pass in the reducer's
lane mode), passages of 1 token (24 ends per tile: slots past kFastSlots in both halves) to thousands (open across
many tiles), ends on either side of the half boundary (4-token groups 11 and 12), corpora below, at and above 132
passages, k = 1, 10 and 128, and each case again with tombstones and per-query allow bitmaps."""
import numpy as np
import pytest
import torch

import scan_fp64 as S
from helpers import scan_partition

pytestmark = pytest.mark.gpu

# (storage, relu, nq, B, lengths, n)
CASES = [
    ("bf16", False, 320, 3, "1", 2000),
    ("fp8", True, 320, 2, "long", 133),
    ("bf16", True, 288, 2, "mix", 132),
    ("fp8", False, 288, 2, "halves", 2000),
    ("bf16", False, 321, 2, "halves", 100),
    ("fp8", False, 384, 2, "1", 133),
    ("bf16", False, 832, 3, "ragged", 2000),
    ("fp8", True, 832, 2, "mix", 132),
    ("bf16", False, 32, 12, "le4", 2000),
    ("fp8", False, 32, 10, "1", 2000),
    ("bf16", True, 32, 11, "long", 133),
    ("bf16", False, 384, 1, "long", 2000),
    ("fp8", False, 321, 1, "ragged", 100),
    ("bf16", True, 320, 2, "halves", 2000),
    ("fp16", False, 320, 3, "1", 2000),
    ("fp16", True, 384, 2, "halves", 133),
    ("fp16", False, 832, 2, "ragged", 2000),
    ("fp16", False, 32, 12, "le4", 2000),
]


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


def _doclens(kind, n, seed):
    if kind == "halves":   # ends every 44-52 tokens: many in the 4-token groups 11 and 12 of a tile
        return np.random.default_rng(seed).choice([44, 45, 48, 49, 52], n).astype(np.int32)
    return S.case_doclens(dict(n=n, lengths=kind), seed)


def _data(B, nq, dl, relu, seed):
    g = torch.Generator().manual_seed(seed)
    unit = lambda *shape: torch.nn.functional.normalize(torch.randn(shape, generator=g), dim=-1).bfloat16().float()
    Q, D = unit(B, nq, 128), unit(int(dl.sum()), 128)
    if relu:   # every other token scores below zero against every query row: relu decides its rows' maxima
        Q = Q.abs()
        D[::2] = -D[::2].abs()
    return Q, D


def _run(R, L, corpus, Q, relu, variant, allow=None):
    from ravqa_b200 import _cabi
    _cabi.check(L.flmr_debug_set_scan_variant(variant))
    try:
        scores = R.maxsim_scores(corpus, Q, relu=relu, allow=allow)
        tops = [R.maxsim_topk(corpus, Q, k, relu=relu, allow=allow) for k in (1, 10, 128)]
        torch.cuda.synchronize()
    finally:
        L.flmr_debug_set_scan_variant(0)
    return scores, tops


def _same(a, b, tag):
    (sa, ta), (sb, tb) = a, b
    assert torch.equal(sa, sb), "%s: scores differ at %d entries" % (tag, int((sa != sb).sum()))
    for k, (x, y) in zip((1, 10, 128), zip(ta, tb)):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]), "%s: top-%d differs" % (tag, k)


@pytest.mark.parametrize("ci", range(len(CASES)), ids=lambda i: "%s-relu%d-nq%d-B%d-%s-n%d" % CASES[i])
def test_split_kernel_is_bitwise_the_serial_kernel(R, ci):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    storage, relu, nq, B, kind, n = CASES[ci]
    ref_variant = 2 if storage == "fp16" else 3
    seed = 7000 + ci
    dl = _doclens(kind, n, seed)
    if kind == "halves":
        part = scan_partition(dl, torch.cuda.get_device_properties(0).multi_processor_count)
        masks = part["end_mask"].astype(np.int64)
        assert ((masks >> 11) & 1).any() and ((masks >> 12) & 1).any(), "no end in group 11 or 12"
    # the case reaches a pass of five or six occupied blocks (row-sliced queries add a short tail pass)
    blocks = {S.occupied_blocks(int(r[1]), int(r[4])) for plan in S.call_plans(B, nq) for r in plan}
    assert blocks & {5, 6}, (CASES[ci], blocks)
    Q, D = _data(B, nq, dl, relu, seed)
    Qd = Q.cuda()
    corpus = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0, storage=storage)
    try:
        ref = _run(R, L, corpus, Qd, relu, ref_variant)
        _same(ref, _run(R, L, corpus, Qd, relu, 6), "variant 6")
        _same(ref, _run(R, L, corpus, Qd, relu, 0), "variant 0")
        # tombstones and per-query allow bitmaps
        rng = np.random.default_rng(seed)
        corpus.delete(rng.choice(n, size=max(1, n // 10), replace=False))
        allow = corpus.allow_bitmaps([rng.choice(n, size=max(1, (7 * n) // 10), replace=False) for _ in range(B)])
        ref = _run(R, L, corpus, Qd, relu, ref_variant, allow)
        _same(ref, _run(R, L, corpus, Qd, relu, 6, allow), "variant 6, filtered")
        _same(ref, _run(R, L, corpus, Qd, relu, 0, allow), "variant 0, filtered")
    finally:
        corpus.close()
