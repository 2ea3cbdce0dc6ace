"""CPU: what ptxas made of flmr_scan_udesc_kernel (the split-tile scan loop whose MMAs take their descriptors from
warp-uniform bases).  Like the split kernel it must fit the 128 registers of three consumer warpgroups without
spilling, issue m64n48 MMAs of its storage's type and keep one commit group in flight across each fold; unlike it, the
MMAs of a commit group follow each other with no more than a few instructions between them instead of a descriptor
rebuilt from regular registers before each one."""
import os
import re
import shutil
import statistics
import subprocess

import pytest

from helpers import ROOT

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
# Elem value in the mangled name -> the storage's MMA
UDESC = {0: "HGMMA.64x48x16.F32.BF16", 1: "HGMMA.64x48x16.F32 ", 2: "QGMMA.64x48x32.F32.E4M3.E4M3"}
MMA = re.compile(r"\b[HQ]GMMA\.")


@pytest.fixture(scope="module")
def ptxas_build(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("udesc_scan") / "lib.so")
    proc = subprocess.run([nvcc, "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-shared", "-Xcompiler", "-fPIC", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out],
                          capture_output=True, text=True, check=True).stdout
    return proc.stderr, sass


def _sections(text, header, name):
    """{group 1 of `name`: lines} for the kernels whose `header` line matches `name`."""
    out, cur = {}, None
    for line in text.splitlines():
        if re.search(header, line):
            m = re.search(name, line)
            cur = m.group(1) if m else None
            if cur is not None:
                out[cur] = []
            continue
        if cur is not None:
            out[cur].append(line)
    return out


def _udesc(text, header):
    return {int(k): v for k, v in _sections(text, header, r"22flmr_scan_udesc_kernelILNS_4ElemE(\d)E").items()}


def _commit_groups(lines):
    """Per commit group (MMAs up to one that sets gsb0): the instruction counts between its consecutive MMAs."""
    instr = [l for l in lines if re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+\S", l)]
    groups, gaps, prev = [], [], None
    for i, l in enumerate(instr):
        if MMA.search(l):
            if prev is not None:
                gaps.append(i - prev - 1)
            prev = i
            if "gsb0" in l:
                groups.append(gaps)
                gaps, prev = [], None
    return groups


def test_udesc_kernels_fit_128_registers_without_spills(ptxas_build):
    log, _ = ptxas_build
    kernels = _udesc(log, r"Compiling entry function")
    assert set(kernels) == set(UDESC)
    for elem, lines in kernels.items():
        spill = next(l for l in lines if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (elem, spill)
        regs = int(re.search(r"Used (\d+) registers", next(l for l in lines if "Used" in l)).group(1))
        assert regs <= 128, (elem, regs)


def test_udesc_kernels_issue_n48_mmas_and_overlap_the_fold(ptxas_build):
    _, sass = ptxas_build
    kernels = _udesc(sass, r"Function : ")
    assert set(kernels) == set(UDESC)
    for elem, lines in kernels.items():
        text = "\n".join(lines)
        assert UDESC[elem] in text, elem
        assert "64x96" not in text, elem
        assert len({m.group(0) for m in re.finditer(r"[HQ]GMMA\.64x48x\d+\.F32(\.\w+)*", text)}) == 1, elem
        assert "WARPGROUP.DEPBAR.LE gsb0, 0x1" in text, elem


def test_udesc_mma_groups_issue_back_to_back(ptxas_build):
    """Inside a commit group the MMAs are separated by a few instructions only.  ptxas schedules the group's remaining
    descriptor set-up behind its first MMA and fills some later slots with the loop's own bookkeeping (the next tile's
    end-mask load), so the bound is on the mean gap after the first MMA of each group; and over the whole kernel the
    gaps add up to well under half of the split kernel's, whose MMAs each wait for a descriptor rebuilt in regular
    registers."""
    _, sass = ptxas_build
    udesc = _udesc(sass, r"Function : ")
    split = {int(k): v for k, v in _sections(sass, r"Function : ", r"22flmr_scan_split_kernelILb(\d)E").items()}
    for elem, lines in udesc.items():
        groups = _commit_groups(lines)
        k_steps = 4 if elem == 2 else 8
        assert len(groups) == 12 and all(len(g) == k_steps - 1 for g in groups), (elem, groups)
        for g in groups:
            assert statistics.mean(g[1:]) <= 4, (elem, groups)
        twin = _commit_groups(split[1 if elem == 2 else 0])
        if elem != 1:   # the split kernel's fp16 form has its own name (flmr_scan_split_f16_kernel)
            assert 2 * sum(map(sum, groups)) < sum(map(sum, twin)), (elem, groups, twin)


def test_variant_7_is_accepted():
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    try:
        assert L.flmr_debug_set_scan_variant(7) == 0
        assert L.flmr_debug_set_scan_variant(5) != 0
    finally:
        L.flmr_debug_set_scan_variant(0)
