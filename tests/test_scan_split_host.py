"""CPU: what ptxas made of the split-tile scan loop (flmr_scan_split_kernel and flmr_scan_listed_split_kernel: three
consumer warpgroups that fold one half of each tile while the other half's MMAs run, issued from warp-uniform
descriptors), for every storage.  Three consumer warpgroups leave 128 registers per thread; the loop must fit them
without spilling, issue only its storage's m64n48 MMAs, keep one commit group in flight across each fold
(wait_group 1), and issue the MMAs of a commit group with no more than a few instructions between them instead of a
descriptor rebuilt from regular registers before each one."""
import os
import re
import shutil
import statistics
import subprocess

import pytest

from helpers import ROOT

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
SPLIT = re.compile(r"(22flmr_scan_split_kernel|29flmr_scan_listed_split_kernel)ILNS_4ElemE(\d)E")
# Elem value in the mangled name -> the storage's MMA
MMA_OF = {0: "HGMMA.64x48x16.F32.BF16", 1: "HGMMA.64x48x16.F32 ", 2: "QGMMA.64x48x32.F32.E4M3.E4M3"}
KERNELS = {(listed, elem) for listed in (False, True) for elem in MMA_OF}
MMA = re.compile(r"\b[HQ]GMMA\.")
# Whole-kernel instruction gaps inside the commit groups of the partition split kernel when it rebuilt both
# descriptors of every MMA in regular registers (the listed split kernels had 997 bf16 / fp16 and 415 e4m3).  Every
# split kernel must keep its gaps under half of these.
GAPS_REBUILT = {0: 973, 1: 973, 2: 401}


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
    """(listed, Elem value) -> lines of that split-kernel instantiation, for the lines of `text` that follow a `header`
    line."""
    out, cur = {}, None
    for line in text.splitlines():
        if re.search(header, line):
            m = SPLIT.search(line)
            cur = ("listed" in m.group(1), int(m.group(2))) if m else None
            if cur is not None:
                out[cur] = []
            continue
        if cur is not None:
            out[cur].append(line)
    return out


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


def test_split_kernels_fit_128_registers_without_spills(ptxas_build):
    log, _ = ptxas_build
    kernels = _sections(log, r"Compiling entry function")
    assert set(kernels) == KERNELS
    for key, lines in kernels.items():
        spill = next(l for l in lines if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (key, spill)
        regs = int(re.search(r"Used (\d+) registers", next(l for l in lines if "Used" in l)).group(1))
        assert regs <= 128, (key, regs)


def test_split_kernels_issue_n48_mmas_and_overlap_the_fold(ptxas_build):
    _, sass = ptxas_build
    kernels = _sections(sass, r"Function : ")
    assert set(kernels) == KERNELS
    for (listed, elem), lines in kernels.items():
        text = "\n".join(lines)
        assert MMA_OF[elem] in text, (listed, elem)
        assert "64x96" not in text, (listed, elem)
        assert len({m.group(0) for m in re.finditer(r"[HQ]GMMA\.64x48x\d+\.F32(\.\w+)*", text)}) == 1, (listed, elem)
        assert "WARPGROUP.DEPBAR.LE gsb0, 0x1" in text, (listed, elem)


def test_split_mma_groups_issue_back_to_back(ptxas_build):
    """Inside a commit group the MMAs are separated by a few instructions only.  ptxas schedules the group's remaining
    descriptor set-up behind its first MMA and fills some later slots with the loop's own bookkeeping (the next tile's
    end-mask load), so the bound is on the mean gap after the first MMA of each group; and over the whole kernel the
    gaps add up to under half of the loop's with descriptors rebuilt for each MMA (GAPS_REBUILT)."""
    _, sass = ptxas_build
    kernels = _sections(sass, r"Function : ")
    assert set(kernels) == KERNELS
    for (listed, elem), lines in kernels.items():
        groups = _commit_groups(lines)
        k_steps = 4 if elem == 2 else 8
        assert len(groups) == 12 and all(len(g) == k_steps - 1 for g in groups), (listed, elem, groups)
        for g in groups:
            assert statistics.mean(g[1:]) <= 4, (listed, elem, groups)
        assert 2 * sum(map(sum, groups)) < GAPS_REBUILT[elem], (listed, elem, groups)


def test_variant_6_is_accepted_and_5_and_7_refused():
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    try:
        assert L.flmr_debug_set_scan_variant(6) == 0
        assert L.flmr_debug_set_scan_variant(5) != 0
        assert L.flmr_debug_set_scan_variant(7) != 0
    finally:
        L.flmr_debug_set_scan_variant(0)
