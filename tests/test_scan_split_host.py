"""CPU: what ptxas made of flmr_scan_split_kernel (the three-warpgroup scan whose consumers fold one half of each tile
while the other half's MMAs run).  Three consumer warpgroups leave 128 registers per thread; the split loop must fit
them without spilling, issue m64n48 MMAs and keep one commit group in flight across each fold (wait_group 1)."""
import os
import re
import shutil
import subprocess

import pytest

from helpers import ROOT

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
SPLIT = re.compile(r"flmr_scan_split_kernelILb(\d)E")


@pytest.fixture(scope="module")
def ptxas_build(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("split_scan") / "lib.so")
    proc = subprocess.run([nvcc, "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-shared", "-Xcompiler", "-fPIC", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out],
                          capture_output=True, text=True, check=True).stdout
    return proc.stderr, sass


def _sections(text, header):
    """fp8 flag -> lines of that split-kernel instantiation, for the lines of `text` that follow a `header` line."""
    out, cur = {}, None
    for line in text.splitlines():
        if re.search(header, line):
            m = SPLIT.search(line)
            cur = int(m.group(1)) if m else None
            if cur is not None:
                out[cur] = []
            continue
        if cur is not None:
            out[cur].append(line)
    return out


def test_split_kernels_fit_128_registers_without_spills(ptxas_build):
    log, _ = ptxas_build
    kernels = _sections(log, r"Compiling entry function")
    assert set(kernels) == {0, 1}
    for fp8, lines in kernels.items():
        spill = next(l for l in lines if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (fp8, spill)
        regs = int(re.search(r"Used (\d+) registers", next(l for l in lines if "Used" in l)).group(1))
        assert regs <= 128, (fp8, regs)


def test_split_kernels_issue_n48_mmas_and_overlap_the_fold(ptxas_build):
    _, sass = ptxas_build
    kernels = _sections(sass, r"Function : ")
    assert set(kernels) == {0, 1}
    for fp8, lines in kernels.items():
        text = "\n".join(lines)
        if fp8:
            assert "QGMMA.64x48x32.F32.E4M3.E4M3" in text and "HGMMA" not in text
        else:
            assert "HGMMA.64x48x16.F32.BF16" in text and "64x96" not in text
        assert "WARPGROUP.DEPBAR.LE gsb0, 0x1" in text, fp8
