"""fp16 corpus storage, CPU side: what ptxas made of the fp16 scan kernels (f16 HGMMA, no spills, registers no higher
than their bf16 twins, the overlapped wait), that the bf16 and e4m3 scan kernels keep their registers, the new
exports, and the fp16 flat index on disk."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ravqa_b200 import _cabi
from ravqa_b200 import index_io as I
from helpers import ROOT

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
# fp16 kernel -> its bf16 twin (the kernel the same launch runs on a bf16 corpus)
F16_KERNELS = {r"flmr_scan_kernelILi2ELNS_4ElemE1ELb0E": r"flmr_scan_kernelILi2ELNS_4ElemE0ELb0E",
               r"flmr_scan_split_kernelILNS_4ElemE1E": r"flmr_scan_split_kernelILNS_4ElemE0E"}
# registers of every bf16 and e4m3 scan instantiation (kernel name pattern -> registers)
REGISTERS_BEFORE = {r"flmr_scan_kernelILi2ELNS_4ElemE0ELb0E": 167, r"flmr_scan_kernelILi3ELNS_4ElemE0ELb0E": 119,
                    r"flmr_scan_kernelILi2ELNS_4ElemE2ELb0E": 167, r"flmr_scan_kernelILi3ELNS_4ElemE2ELb0E": 109,
                    r"flmr_scan_kernelILi2ELNS_4ElemE0ELb1E": 168, r"flmr_scan_split_kernelILNS_4ElemE0E": 109,
                    r"flmr_scan_split_kernelILNS_4ElemE2E": 102}


@pytest.fixture(scope="module")
def ptxas_build(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("fp16_scan") / "lib.so")
    proc = subprocess.run([nvcc, "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-shared", "-Xcompiler", "-fPIC", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out],
                          capture_output=True, text=True, check=True).stdout
    return proc.stderr, sass


def _sections(text, header):
    """{mangled kernel name: lines} of the scan kernels in `text`, sections starting at lines matching `header`."""
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
    hits = [k for k in sections if re.search(r"\d%s" % pattern if pattern.startswith("flmr") else pattern, k)]
    assert len(hits) == 1, (pattern, hits)
    return sections[hits[0]]


def _registers(lines):
    spill = next(l for l in lines if "spill stores" in l)
    assert "0 bytes spill stores, 0 bytes spill loads" in spill, spill
    return int(re.search(r"Used (\d+) registers", next(l for l in lines if "Used" in l)).group(1))


def test_f16_kernels_no_spills_and_no_more_registers_than_bf16(ptxas_build):
    log, _ = ptxas_build
    kernels = _sections(log, r"Compiling entry function")
    for f16, twin in F16_KERNELS.items():
        regs = _registers(_find(kernels, f16))
        assert regs <= _registers(_find(kernels, twin)), (f16, regs)


def test_existing_scan_kernels_keep_their_registers(ptxas_build):
    log, _ = ptxas_build
    kernels = _sections(log, r"Compiling entry function")
    for pattern, regs in REGISTERS_BEFORE.items():
        assert _registers(_find(kernels, pattern)) == regs, pattern


def test_f16_kernels_issue_f16_hgmma_and_overlap_the_fold(ptxas_build):
    _, sass = ptxas_build
    kernels = _sections(sass, r"Function : ")
    for f16, shape in zip(F16_KERNELS, ("64x96x16", "64x48x16")):
        text = "\n".join(_find(kernels, f16))
        assert "HGMMA.%s.F32 " % shape in text, f16
        assert ".BF16" not in text and "QGMMA" not in text, f16      # no bf16 or e4m3 MMA in the fp16 kernels
        assert "WARPGROUP.DEPBAR.LE gsb0, 0x1" in text, f16
    for twin in F16_KERNELS.values():                                # and their bf16 twins stay bf16
        assert "HGMMA" in "\n".join(_find(kernels, twin)) and ".BF16" in "\n".join(_find(kernels, twin))


def test_new_symbols_are_declared_and_exported():
    with open(os.path.join(ROOT, "include", "flmr_maxsim.h")) as f:
        hdr = f.read()
    assert re.search(r"#define FLMR_CORPUS_FP16 4u", hdr)
    assert "#define FLMR_ABI_VERSION 2" in hdr
    for name in _cabi.FP16_SYMBOLS:
        assert name in _cabi.SYMBOLS and re.search(r"int %s\(" % name, hdr), name
        assert hasattr(_cabi.lib(), name), name
    assert _cabi.STORAGES[2] == "fp16" and _cabi.CORPUS_FP16 == 4


def test_storage_flags_and_element_types():
    from ravqa_b200 import corpus
    assert corpus._storage_flag("fp16") == _cabi.CORPUS_FP16
    assert corpus.element_dtype("fp16") == torch.float16
    assert corpus.element_dtype("bf16") == corpus.element_dtype("fp8") == torch.bfloat16


def _tokens(n_rows, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_rows, 128, generator=g)


@pytest.mark.parametrize("chunked", [False, True])
def test_fp16_index_round_trips_and_bf16_readers_refuse_it(tmp_path, chunked):
    rng = np.random.default_rng(0)
    dl = rng.integers(1, 9, size=10).astype(np.int32)
    toks = _tokens(int(dl.sum()), 0)
    toks[0, 0] = 1e6                      # beyond fp16: +inf, as torch's .half() makes it
    path = str(tmp_path / "idx")
    if chunked:
        off = np.concatenate([[0], np.cumsum(dl)])
        I.save_flat_chunk(path, 0, 0, toks[:off[6]], dl[:6], dtype="float16")
        I.save_flat_chunk(path, 1, 6, toks[off[6]:], dl[6:], dtype="float16")
        assert I.chunk_exists(path, 1, "float16") and not I.chunk_exists(path, 1)
        I.finalize_chunked_index(path, 2, I.FORMAT_F16)
    else:
        I.save_flat_index(path, toks, dl, dtype="float16")
    t, d, meta = I.load_flat_index(path)
    assert meta["format"] == I.FORMAT_F16 and meta["dtype"] == "float16" and I.index_dtype(meta) == "float16"
    assert t.dtype == torch.float16 and torch.equal(t.view(torch.int16), toks.half().view(torch.int16))
    assert torch.isinf(t[0, 0]) and np.array_equal(d, dl)
    # a reader of bf16 indexes only: its format set and its token files are not there
    assert meta["format"] not in ("flmr-flat-v1", "flmr-flat-v2")
    assert not [f for f in os.listdir(path) if f.endswith(".bf16")]
    all_dl, files = I.index_token_files(path)
    assert all(f.endswith(".f16") for f, *_ in files) and np.array_equal(all_dl, dl)
    # appends and deletions keep the dtype: f16-v2 with deletions, f16 chunks for the new passages
    meta = I.persist_updates(path, _tokens(5, 1), np.array([2, 3], dtype=np.int32), [3])
    assert meta["format"] == I.FORMAT_F16_V2 and meta["dtype"] == "float16"
    assert np.array_equal(I.read_deleted(path), [3])
    t2, d2, _ = I.load_flat_index(path)
    assert t2.dtype == torch.float16 and torch.equal(t2[:t.size(0)].view(torch.int16), t.view(torch.int16))
    meta = I.persist_updates(path, None, [], [])
    assert meta["format"] == I.FORMAT_F16
    from ravqa_b200.searcher import detect_index_kind
    assert detect_index_kind(path) == "flat"
    with open(os.path.join(path, "metadata.json")) as f:
        assert json.load(f)["format"] == "flmr-flat-f16-v1"


def test_bf16_index_is_unchanged(tmp_path):
    dl = np.array([3, 5], np.int32)
    path = I.save_flat_index(str(tmp_path / "b"), _tokens(8, 2), dl)
    meta = I.read_metadata(path)
    assert meta["format"] == I.FORMAT and meta["dtype"] == "bfloat16" and I.index_dtype(meta) == "bfloat16"
    assert os.path.exists(os.path.join(path, "tokens.bf16"))
    assert I.load_flat_index(path)[0].dtype == torch.bfloat16


def test_indexer_storage_argument():
    from ravqa_b200 import Indexer
    assert Indexer(encode_fn=lambda p: None, storage="fp16").dtype == "float16"
    assert Indexer(encode_fn=lambda p: None).dtype == "bfloat16"
    with pytest.raises(ValueError):
        Indexer(encode_fn=lambda p: None, storage="fp8")
