"""GPU: flmr_scan_udesc_kernel (scan variant 7: the split-tile loop with its MMA descriptors built from warp-uniform
bases) against flmr_scan_kernel<3> (variant 3; fp16 corpora, which have no such kernel, against the two-warpgroup
fp16 kernel of variant 2): bitwise the same scores and fused top-k, and the default selection (variant 0) with them.

The cases are those of the split kernel's test (both storages, relu on and off, five- and six-block passes, ends on
either side of the half boundary, lane and warp mode, k = 1, 10 and 128, tombstones and allow bitmaps) plus fp16
corpora of the same kinds."""
import numpy as np
import pytest
import torch

import scan_fp64 as S
from helpers import scan_partition
from test_scan_split_gpu import CASES as SPLIT_CASES, _data, _doclens, _run, _same

pytestmark = pytest.mark.gpu

# (storage, relu, nq, B, lengths, n)
CASES = SPLIT_CASES + [
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


@pytest.mark.parametrize("ci", range(len(CASES)), ids=lambda i: "%s-relu%d-nq%d-B%d-%s-n%d" % CASES[i])
def test_udesc_kernel_is_bitwise_the_serial_kernel(R, ci):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    storage, relu, nq, B, kind, n = CASES[ci]
    ref_variant = 2 if storage == "fp16" else 3
    seed = 7100 + ci
    dl = _doclens(kind, n, seed)
    if kind == "halves":
        part = scan_partition(dl, torch.cuda.get_device_properties(0).multi_processor_count)
        masks = part["end_mask"].astype(np.int64)
        assert ((masks >> 11) & 1).any() and ((masks >> 12) & 1).any(), "no end in group 11 or 12"
    blocks = {S.occupied_blocks(int(r[1]), int(r[4])) for plan in S.call_plans(B, nq) for r in plan}
    assert blocks & {5, 6}, (CASES[ci], blocks)
    Q, D = _data(B, nq, dl, relu, seed)
    Qd = Q.cuda()
    corpus = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0, storage=storage)
    try:
        ref = _run(R, L, corpus, Qd, relu, ref_variant)
        _same(ref, _run(R, L, corpus, Qd, relu, 7), "variant 7")
        _same(ref, _run(R, L, corpus, Qd, relu, 0), "variant 0")
        rng = np.random.default_rng(seed)
        corpus.delete(rng.choice(n, size=max(1, n // 10), replace=False))
        allow = corpus.allow_bitmaps([rng.choice(n, size=max(1, (7 * n) // 10), replace=False) for _ in range(B)])
        ref = _run(R, L, corpus, Qd, relu, ref_variant, allow)
        _same(ref, _run(R, L, corpus, Qd, relu, 7, allow), "variant 7, filtered")
        _same(ref, _run(R, L, corpus, Qd, relu, 0, allow), "variant 0, filtered")
    finally:
        corpus.close()


def test_variant_7_has_no_listed_kernel(R):
    """Plan-mode (listed) searches have no uniform-descriptor kernel: forcing variant 7 refuses them."""
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    dl = np.full(64, 8, np.int32)
    Q, D = _data(2, 32, dl, False, 5)
    corpus = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0)
    try:
        _cabi.check(L.flmr_debug_set_scan_variant(7))
        with pytest.raises(_cabi.FlmrError, match="variant"):
            R.maxsim_topk(corpus, Q.cuda(), 5, pids=[[0], [1]])
    finally:
        L.flmr_debug_set_scan_variant(0)
        corpus.close()
