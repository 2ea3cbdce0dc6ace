"""e4m3 corpus storage, CPU side: what ptxas made of the fp8 scan kernels, the fp8 oracle against torch's e4m3 cast,
and the shortlist depth of the exact re-rank."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import fp8_oracle as F8
from helpers import ROOT, golden_names, load_golden

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
FP8_SCAN = re.compile(r"flmr_scan_kernelILi(\d)ELNS_4ElemE2ELb0E")


@pytest.fixture(scope="module")
def ptxas_build(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("fp8_scan") / "lib.so")
    proc = subprocess.run([nvcc, "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-shared", "-Xcompiler", "-fPIC", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out],
                          capture_output=True, text=True, check=True).stdout
    return proc.stderr, sass


def _sections(text, header):
    """{kWgs: lines} of the fp8 scan kernels in `text`, sections starting at lines matching `header`."""
    out, cur = {}, None
    for line in text.splitlines():
        if re.search(header, line):
            m = FP8_SCAN.search(line)
            cur = int(m.group(1)) if m else None
            if cur:
                out[cur] = []
            continue
        if cur:
            out[cur].append(line)
    return out


def test_fp8_scan_kernels_build_without_spills(ptxas_build):
    log, _ = ptxas_build
    kernels = _sections(log, r"Compiling entry function")
    assert set(kernels) == {2, 3}
    for wgs, lines in kernels.items():
        spill = next(l for l in lines if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (wgs, spill)


def test_fp8_scan_kernels_issue_e4m3_wgmma(ptxas_build):
    _, sass = ptxas_build
    kernels = _sections(sass, r"Function : ")
    assert set(kernels) == {2, 3}
    for wgs, lines in kernels.items():
        text = "\n".join(lines)
        assert "QGMMA.64x96x32.F32.E4M3.E4M3" in text, wgs
        assert "HGMMA" not in text, wgs            # no bf16 MMA left in the fp8 kernels
        overlapped = "WARPGROUP.DEPBAR.LE gsb0, 0x1" in text
        assert overlapped == (wgs == 2), wgs       # two warpgroups overlap MMA and fold, three run serially


@pytest.mark.parametrize("name", golden_names())
def test_e4m3_round_matches_torch_cast(name):
    g = load_golden(name)
    for x in (g["Q"], g["D"]):
        want = torch.from_numpy(np.ascontiguousarray(x)).to(torch.float8_e4m3fn).float().numpy()
        assert np.array_equal(F8.e4m3_round(x), want)


def test_e4m3_round_edges():
    x = np.array([0.0, -0.0, 2.0 ** -10, 1.5 * 2.0 ** -9, 2.0 ** -6 * 1.0625, 1.0625, 1.1875, 447.0, 500.0, -1e4],
                 dtype=np.float32)
    want = torch.from_numpy(np.clip(x, -448, 448)).to(torch.float8_e4m3fn).float().numpy()
    got = F8.e4m3_round(x)
    assert np.array_equal(got, want)
    assert got[-2] == 448.0 and got[-1] == -448.0   # saturated
    assert F8.e4m3_round(np.float32(1.0625)) == 1.0 and F8.e4m3_round(np.float32(1.1875)) == 1.25   # ties to even


def test_fp8_oracle_scores_round_both_operands():
    g = load_golden(golden_names()[0])
    q8, d8 = F8.e4m3_round(g["Q"]), F8.e4m3_round(g["D"])
    from oracle import maxsim_oracle as O
    np.testing.assert_array_equal(F8.maxsim_scores_fp8(g["Q"], g["D"], g["doclens"]),
                                  O.maxsim_scores(q8, d8, g["doclens"]))
    rel = np.abs(F8.maxsim_scores_fp8(g["Q"], g["D"], g["doclens"]) - g["scores_true_max"])
    assert rel.max() > 0   # e4m3 is not bf16: the first stage is approximate


def test_shortlist_depth_rule():
    from ravqa_b200.searcher import shortlist_depth
    # ndocs unset: the reference's own default from k (1024 for k <= 100, max(4k, 4096) above), divided by four
    assert shortlist_depth(5, None, 10 ** 6) == 256
    assert shortlist_depth(100, None, 10 ** 6) == 256
    assert shortlist_depth(101, None, 10 ** 6) == 1024
    assert shortlist_depth(1500, None, 10 ** 6) == 1500
    # a configured ndocs, never below k
    assert shortlist_depth(10, 2000, 10 ** 6) == 500
    assert shortlist_depth(300, 1024, 10 ** 6) == 300
    # clamps: the select kernel's capacity and the candidates there are
    assert shortlist_depth(10, 10 ** 5, 10 ** 6) == 2048
    assert shortlist_depth(5, None, 40) == 40
    assert shortlist_depth(5, None, 3) == 3
    with pytest.raises(ValueError):
        shortlist_depth(2049, None, 10 ** 6)


def test_storage_argument_is_validated():
    from ravqa_b200 import corpus
    with pytest.raises(ValueError):
        corpus._storage_flag("int8")
    assert corpus._storage_flag("bf16") == 0 and corpus._storage_flag("fp8") == 2
