"""fp16 training / re-scoring kernels, CPU side: the four _fp16 entry points (exported, declared alike in the header and
the binding, refusing what their bf16 forms refuse), and what ptxas made of the fp16 kernels: f16 MMAs, no spills,
the registers of their bf16 twins, the wgmma kernel's pipeline intact; and the bf16 kernels' registers as they were
before the fp16 forms existed."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from ravqa_b200 import _cabi
from helpers import ROOT

CSRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc")
# fp16 kernel -> its bf16 twin
TWINS = {"flmr_argmax_tc_f16_kernel": "flmr_argmax_tc_kernel",
         "flmr_argmax_mma_f16_kernel": "flmr_argmax_mma_kernel",
         "flmr_argmax_f16_kernel": "flmr_argmax_kernel",
         "flmr_bwd_dq_f16_kernel": "flmr_bwd_dq_kernel",
         "flmr_bwd_dd_f16_kernel": "flmr_bwd_dd_kernel"}
# registers of the training kernels in the revision before the fp16 forms (ptxas of CUDA 12.9, sm_90a, -O3)
REGISTERS_BEFORE = {"flmr_argmax_tc_kernel": 106, "flmr_argmax_mma_kernel": 77, "flmr_argmax_kernel": 64,
                    "flmr_bwd_dq_kernel": 32, "flmr_bwd_dd_kernel": 28, "flmr_compact_docs_kernel": 30}
INVALID_ARG, UNSUPPORTED = 1, 3


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """(ptxas log, SASS) of the training kernels, compiled from the library's own headers."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("fp16_train")
    tu = d / "train.cu"
    tu.write_text('#include "flmr_train_kernels.cuh"\n#include "flmr_train_tc_kernel.cuh"\n')
    out = str(d / "train.cubin")
    proc = subprocess.run([nvcc, "-cubin", "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                           "-std=c++17", "-I", CSRC, "-o", out, str(tu)], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out],
                          capture_output=True, text=True, check=True).stdout
    return proc.stderr, sass


def _sections(text, header):
    """{kernel name: lines} of the flmr kernels in `text`, sections starting at lines matching `header`."""
    out, cur = {}, None
    for line in text.splitlines():
        if re.search(header, line):
            m = re.search(r"_ZN4flmr\d+(flmr_\w+?)E", line)
            cur = m.group(1) if m else None
            if cur:
                out[cur] = []
            continue
        if cur:
            out[cur].append(line)
    return out


def _registers(lines):
    spill = next(l for l in lines if "spill stores" in l)
    assert "0 bytes spill stores, 0 bytes spill loads" in spill, spill
    return int(re.search(r"Used (\d+) registers", next(l for l in lines if "Used" in l)).group(1))


def test_fp16_kernels_no_spills_and_the_registers_of_their_twins(compiled):
    kernels = _sections(compiled[0], r"Compiling entry function")
    for f16, twin in TWINS.items():
        regs, twin_regs = _registers(kernels[f16]), _registers(kernels[twin])
        if f16 == "flmr_argmax_f16_kernel":
            # the debug-only SIMT cross-check: widening fp16 takes one HADD2.F32 per element where bf16 takes a
            # shift, and ptxas needs two registers fewer for it
            assert regs <= twin_regs, (f16, regs, twin_regs)
        else:
            assert regs == twin_regs, (f16, regs, twin_regs)


def test_bf16_kernels_keep_their_registers(compiled):
    kernels = _sections(compiled[0], r"Compiling entry function")
    for name, regs in REGISTERS_BEFORE.items():
        assert _registers(kernels[name]) == regs, name


def _opcodes(lines, pattern):
    ops = []
    for l in lines:
        m = re.search(r"\*/\s+(@!?U?P\w+\s+)?([A-Z][\w.]*)", l)
        if m and re.match(pattern, m.group(2)):
            ops.append(m.group(2))
    return ops


def test_fp16_kernels_issue_f16_mmas(compiled):
    kernels = _sections(compiled[1], r"Function : ")
    tc = "\n".join(kernels["flmr_argmax_tc_f16_kernel"])
    assert "HGMMA.64x128x16.F32 " in tc and ".BF16" not in tc
    mma = "\n".join(kernels["flmr_argmax_mma_f16_kernel"])
    assert "HMMA.16816.F32 " in mma and ".BF16" not in mma
    assert "HGMMA.64x128x16.F32.BF16" in "\n".join(kernels["flmr_argmax_tc_kernel"])
    assert "HMMA.16816.F32.BF16" in "\n".join(kernels["flmr_argmax_mma_kernel"])
    for name in ("flmr_argmax_f16_kernel", "flmr_bwd_dq_f16_kernel", "flmr_bwd_dd_f16_kernel"):
        text = "\n".join(kernels[name])
        assert "HADD2.F32" in text and ".BF16" not in text, name     # fp16 widened to fp32 on load


def test_fp16_wgmma_kernel_keeps_the_pipeline_of_its_twin(compiled):
    """Same MMA count, same warpgroup waits and the same mbarrier / TMA operations, in the same order."""
    kernels = _sections(compiled[1], r"Function : ")
    f16, bf16 = kernels["flmr_argmax_tc_f16_kernel"], kernels["flmr_argmax_tc_kernel"]
    pat = r"(WARPGROUP|SYNCS|UTMALDG|HGMMA|WARPSYNC)"
    strip = lambda ops: [re.sub(r"\.BF16$", "", o) for o in ops]
    assert strip(_opcodes(f16, pat)) == strip(_opcodes(bf16, pat))
    assert _opcodes(f16, r"HGMMA").count("HGMMA.64x128x16.F32") == 8
    depbar = [l.split("*/")[1].split(";")[0].strip() for l in f16 if "WARPGROUP.DEPBAR" in l]
    assert depbar and depbar == [l.split("*/")[1].split(";")[0].strip() for l in bf16 if "WARPGROUP.DEPBAR" in l]


def test_new_symbols_are_declared_and_exported():
    with open(os.path.join(ROOT, "include", "flmr_maxsim.h")) as f:
        hdr = f.read()
    L = _cabi.lib()
    for name in _cabi.FP16_TRAIN_SYMBOLS:
        assert name in _cabi.SYMBOLS and hasattr(L, name), name
        twin = name[:-len("_fp16")]
        decl = re.search(r"int %s\(([^)]*)\);" % name, hdr)
        twin_decl = re.search(r"int %s\(([^)]*)\);" % twin, hdr)
        assert decl and twin_decl, name
        # the same parameters as the bf16 call, and as many as the binding declares
        norm = lambda s: [p.split()[-1].lstrip("*") for p in s.replace("\n", " ").split(",")]
        assert norm(decl.group(1)) == norm(twin_decl.group(1)), name
        assert len(getattr(L, name).argtypes) == len(norm(decl.group(1))), name
        assert getattr(L, name).argtypes == getattr(L, twin).argtypes, name
        assert getattr(L, name).restype == C.c_int, name
    assert "INPUT ELEMENT TYPE" in hdr and "_fp16 names" in hdr


def _argmax_calls(L, suffix, q, d, m, nq, n, nd, arg):
    """(rc, message) of flmr_maxsim_argmax{suffix} and its grouped form on the given pointers and shapes."""
    out = []
    for grouped in (False, True):
        f = getattr(L, ("flmr_maxsim_argmax_grouped" if grouped else "flmr_maxsim_argmax") + suffix)
        rc = f(q, 2, nq, d, m, n, nd, arg, None, 0, None)
        out.append((rc, L.flmr_last_error() if rc else b""))
    return out


def _backward_calls(L, suffix, q, d, nq, n, nd, arg, g, dq):
    out = []
    for grouped in (False, True):
        f = getattr(L, ("flmr_maxsim_backward_grouped" if grouped else "flmr_maxsim_backward") + suffix)
        rc = f(q, 2, nq, d, n, nd, arg, g, dq, None, 0, None)
        out.append((rc, L.flmr_last_error() if rc else b""))
    return out


# (q, d, mask, argmax, nq, n_docs, nd) -> every case is refused before any device is touched
BAD_ARGMAX = [(None, 1, 1, 1, 8, 2, 8), (1, None, 1, 1, 8, 2, 8), (1, 1, None, 1, 8, 2, 8), (1, 1, 1, None, 8, 2, 8),
              (1, 1, 1, 1, 0, 2, 8), (1, 1, 1, 1, 8, 2, 0), (1, 1, 1, 1, 8, -1, 8), (1, 1, 1, 1, 8, 65536, 8)]


@pytest.mark.parametrize("case", range(len(BAD_ARGMAX)))
def test_fp16_argmax_refuses_what_bf16_refuses(case):
    L = _cabi.lib()
    q, d, m, a, nq, n, nd = BAD_ARGMAX[case]
    ptr = lambda x: None if x is None else C.c_void_p(0x1000 * x)
    args = (ptr(q), ptr(d), ptr(m), nq, n, nd, ptr(a))
    bf16, f16 = _argmax_calls(L, "", *args), _argmax_calls(L, "_fp16", *args)
    assert f16 == bf16, (BAD_ARGMAX[case], bf16, f16)
    assert all(rc in (INVALID_ARG, UNSUPPORTED) for rc, _ in f16), f16


BAD_BACKWARD = [(None, 1, 1, 1, 8, 2, 8), (1, None, 1, 1, 8, 2, 8), (1, 1, None, 1, 8, 2, 8), (1, 1, 1, None, 8, 2, 8),
                (1, 1, 1, 1, 0, 2, 8), (1, 1, 1, 1, 8, 2, 0), (1, 1, 1, 1, 8, -1, 8)]


@pytest.mark.parametrize("case", range(len(BAD_BACKWARD)))
def test_fp16_backward_refuses_what_bf16_refuses(case):
    L = _cabi.lib()
    q, d, a, g, nq, n, nd = BAD_BACKWARD[case]
    ptr = lambda x: None if x is None else C.c_void_p(0x1000 * x)
    args = (ptr(q), ptr(d), nq, n, nd, ptr(a), ptr(g), None)
    bf16, f16 = _backward_calls(L, "", *args), _backward_calls(L, "_fp16", *args)
    assert f16 == bf16, (BAD_BACKWARD[case], bf16, f16)
    assert all(rc == INVALID_ARG for rc, _ in f16), f16
