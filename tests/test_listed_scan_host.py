"""CPU: the plan-mode scan kernels (the listed search): registers and no spills, the MMAs of their storage, the
two-warpgroup loop's overlapped wait, the new exports, and the Searcher's path choice."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from helpers import ROOT
from ravqa_b200 import _cabi

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
# plan-mode kernel (mangled-name pattern) -> registers ptxas gives it, and the MMA its SASS must hold
LISTED_KERNELS = {r"23flmr_scan_listed_kernelILNS_4ElemE0E": (167, "HGMMA.64x96x16.F32.BF16"),
                  r"23flmr_scan_listed_kernelILNS_4ElemE2E": (159, "QGMMA.64x96x32.F32.E4M3.E4M3"),
                  r"23flmr_scan_listed_kernelILNS_4ElemE1E": (167, "HGMMA.64x96x16.F32 "),
                  r"29flmr_scan_listed_split_kernelILNS_4ElemE0E": (109, "HGMMA.64x48x16.F32.BF16"),
                  r"29flmr_scan_listed_split_kernelILNS_4ElemE2E": (102, "QGMMA.64x48x32.F32.E4M3.E4M3"),
                  r"29flmr_scan_listed_split_kernelILNS_4ElemE1E": (109, "HGMMA.64x48x16.F32 ")}


@pytest.fixture(scope="module")
def ptxas_build(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("listed_scan") / "lib.so")
    proc = subprocess.run([nvcc, "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-shared", "-Xcompiler", "-fPIC", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out],
                          capture_output=True, text=True, check=True).stdout
    nm = subprocess.run(["nm", "-D", out], capture_output=True, text=True, check=True).stdout
    return proc.stderr, sass, nm


def _sections(text, header):
    out, cur = {}, None
    for line in text.splitlines():
        if re.search(header, line):
            m = re.search(r"(_ZN4flmr\d+flmr_scan\w*)", line)
            cur = m.group(1) if m else None
            if cur:
                out[cur] = []
            continue
        if cur:
            out[cur].append(line)
    return out


def _find(sections, pattern):
    hits = [k for k in sections if re.search(pattern, k)]
    assert len(hits) == 1, (pattern, hits)
    return sections[hits[0]]


def test_listed_kernels_registers_and_no_spills(ptxas_build):
    log, _, _ = ptxas_build
    kernels = _sections(log, r"Compiling entry function")
    for pattern, (regs, _) in LISTED_KERNELS.items():
        lines = _find(kernels, pattern)
        spill = next(l for l in lines if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (pattern, spill)
        used = int(re.search(r"Used (\d+) registers", next(l for l in lines if "Used" in l)).group(1))
        assert used == regs, (pattern, used)


def test_listed_kernels_issue_their_mmas_and_overlap_the_fold(ptxas_build):
    _, sass, _ = ptxas_build
    kernels = _sections(sass, r"Function : ")
    for pattern, (_, mma) in LISTED_KERNELS.items():
        text = "\n".join(_find(kernels, pattern))
        assert mma in text, pattern
        if pattern.endswith("ElemE1E"):   # fp16
            assert ".BF16" not in text and "QGMMA" not in text, pattern
        assert "WARPGROUP.DEPBAR.LE gsb0, 0x1" in text, pattern


def test_listed_symbols_declared_and_exported(ptxas_build):
    _, _, nm = ptxas_build
    with open(os.path.join(ROOT, "include", "flmr_maxsim.h")) as f:
        hdr = f.read()
    assert "#define FLMR_ABI_VERSION 2" in hdr
    for name in _cabi.LISTED_SYMBOLS:
        assert name in _cabi.SYMBOLS and re.search(r"int %s\(" % name, hdr), name
        assert re.search(r" T %s$" % name, nm, re.M), name
        assert hasattr(_cabi.lib(), name), name


class _FakeInfo:
    n_rows = 0


class _FakeCorpus:
    def __init__(self, doclens, pid_base=0):
        self.doclens = np.asarray(doclens, np.int32)
        self.n_passages = len(doclens)
        self.pid_base = pid_base
        self.info = _FakeInfo()
        self.info.n_rows = int(((self.doclens + 3) // 4 * 4).sum())


@pytest.mark.parametrize("fraction,want", [(0.5, True), (0.01, False)])
def test_searcher_chooses_by_listed_rows(monkeypatch, fraction, want):
    """The listed scan is taken while the batch's listed rows are small against the rows its bitmap scan streams."""
    import torch
    import ravqa_b200.searcher as S
    monkeypatch.setattr(S, "LISTED_SCAN_MAX_ROW_FRACTION", fraction)
    sr = S.Searcher.__new__(S.Searcher)
    sr.corpus = _FakeCorpus(np.full(1000, 180), pid_base=50)
    Q = torch.zeros(2, 32, 128)
    lists = [torch.arange(50, 100), torch.tensor([0, 10_000, 60])]          # ids outside the shard do not count
    assert sr._listed_is_cheaper(Q, lists) is want                          # 51 of 1000 passages in one pass
    assert sr._listed_is_cheaper(Q, [torch.arange(50, 60), None]) is False  # a query without a list: bitmaps
