"""The scan kernel's consumer loop: MMAs of the next (tile, query block) overlap the fold of the current one, and only
the 64-row query blocks that hold resident rows are issued.

CPU: what ptxas made of it (no serialised wgmma, no spills, the overlapped wait in the SASS).
GPU: pass shapes whose last 64-row block is half used (Nq = 288, 352, 3 x Nq = 32) or whose last 128-row tile ends on
a block boundary (12 x Nq = 32), against the oracle, with the two- and three-warpgroup kernels bit-identical.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import maxsim_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200")
SRC = os.path.join(PKG, "csrc", "flmr_maxsim.cu")
SCAN = re.compile(r"flmr_scan_kernelILi(\d)ELNS_4ElemE(\d)ELb(\d)E")
# (kWgs, Elem value, kPair) of every flmr_scan_kernel instantiation
KERNELS = {(2, 0, False), (3, 0, False), (2, 0, True), (2, 1, False), (2, 2, False), (3, 2, False)}


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    return nvcc


@pytest.fixture(scope="module")
def ptxas_build(tmp_path_factory):
    """Compiles the library with -Xptxas -v into a temporary directory: (ptxas log, SASS)."""
    nvcc = _nvcc()
    out = str(tmp_path_factory.mktemp("scan_pipeline") / "lib.so")
    proc = subprocess.run([nvcc, "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-shared", "-Xcompiler", "-fPIC", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out],
                          capture_output=True, text=True, check=True).stdout
    return proc.stderr, sass


def _per_scan_kernel(text, header):
    """{(kWgs, Elem value, kPair): lines} for the sections of `text` that start with a line matching `header`."""
    sections, cur = {}, None
    for line in text.splitlines():
        if re.search(header, line):
            m = SCAN.search(line)
            cur = (int(m.group(1)), int(m.group(2)), bool(int(m.group(3)))) if m else None
            if cur:
                sections[cur] = []
            continue
        if cur:
            sections[cur].append(line)
    return sections


def test_ptxas_no_serialised_wgmma_and_no_spills(ptxas_build):
    log, _ = ptxas_build
    assert "C7518" not in log and "C7517" not in log and "C7511" not in log and "C7512" not in log, \
        [l for l in log.splitlines() if "C75" in l]
    kernels = _per_scan_kernel(log, r"Compiling entry function")
    assert set(kernels) == KERNELS
    for key, lines in kernels.items():
        spill = next(l for l in lines if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (key, spill)


def test_sass_overlaps_mma_with_fold(ptxas_build):
    _, sass = ptxas_build
    kernels = _per_scan_kernel(sass, r"Function : ")
    assert set(kernels) == KERNELS
    for key, lines in kernels.items():
        waits = [l for l in lines if "WARPGROUP.DEPBAR.LE gsb0" in l]
        overlapped = [l for l in waits if "gsb0, 0x1" in l]
        if key[0] == 2:   # two accumulators: wait for all but the group just issued
            assert overlapped, key
        else:             # three warpgroups have the registers for one accumulator: serial loop
            assert waits and not overlapped, key


# ---- GPU ------------------------------------------------------------------------------------------------------
SHAPES = [   # (n, nd, B, nq): rows per pass and its last 64-row block
    (1500, 180, 2, 288),   # 288 rows: block 4 half used
    (1500, 180, 2, 352),   # 352 rows: block 5 half used
    (900, 64, 12, 32),     # 12 queries x 32 rows = 384 rows in one pass
    (900, 64, 3, 32),      # 96 rows: block 1 half used
]


@pytest.mark.gpu
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("n,nd,B,nq", SHAPES)
def test_partial_last_block(n, nd, B, nq, relu):
    import ravqa_b200 as R
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    Q, D, dl = O.synth(n, nd, B, nq, seed=n + nq + B, ragged=True)
    corpus = R.FlatCorpus(torch.from_numpy(D).to(torch.bfloat16), dl, device=0)
    Qt = torch.from_numpy(Q)
    k = 7
    out = {}
    try:
        for variant in (2, 3):
            assert L.flmr_debug_set_scan_variant(variant) == 0
            s = R.maxsim_scores(corpus, Qt, relu=relu)
            ts, tp = R.maxsim_topk(corpus, Qt, k, relu=relu)
            torch.cuda.synchronize()
            out[variant] = (s.cpu(), ts.cpu(), tp.cpu())
    finally:
        L.flmr_debug_set_scan_variant(0)
        corpus.close()
    for a, b in zip(out[2], out[3]):
        assert torch.equal(a, b), "two- and three-warpgroup kernels differ"
    ref = O.maxsim_scores(Q, D, dl, relu=relu)
    np.testing.assert_allclose(out[2][0].numpy(), ref, rtol=2e-5, atol=1e-5)
    rs, rp = O.topk(ref, k)
    assert np.array_equal(out[2][2].numpy(), rp)
