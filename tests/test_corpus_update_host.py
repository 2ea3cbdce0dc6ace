"""Corpus updates, CPU side: the flat index's persistence of appended passages and deletions (format v1 / v2, chunk
conversion, per-shard deletion ranges), what ptxas made of the scan kernels with the reducer's tombstone test, and the
new exports."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ravqa_b200 import index_io as I
from ravqa_b200 import _cabi
from helpers import ROOT

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
SCAN = re.compile(r"flmr_scan_kernelILi(\d)ELNS_4ElemE([02])ELb(\d)E")   # bf16 and e4m3
# registers of each scan instantiation (kWgs, kPair, kFp8) before the tombstone test was added: it must not raise them
REGISTERS_BEFORE = {(2, 0, 0): 167, (3, 0, 0): 119, (2, 0, 1): 167, (3, 0, 1): 111, (2, 1, 0): 168}


def _tokens(n_rows, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_rows, 128, generator=g).to(torch.bfloat16)


def _index(tmp_path, chunked, n=10, seed=0):
    rng = np.random.default_rng(seed)
    dl = rng.integers(1, 9, size=n).astype(np.int32)
    toks = _tokens(int(dl.sum()), seed)
    path = str(tmp_path / ("chunked" if chunked else "single"))
    if chunked:
        off = np.concatenate([[0], np.cumsum(dl)])
        I.save_flat_chunk(path, 0, 0, toks[:off[6]], dl[:6])
        I.save_flat_chunk(path, 1, 6, toks[off[6]:], dl[6:])
        I.finalize_chunked_index(path, 2)
    else:
        I.save_flat_index(path, toks, dl)
    return path, toks, dl


@pytest.mark.parametrize("chunked", [False, True])
def test_v1_index_loads_as_before(tmp_path, chunked):
    path, toks, dl = _index(tmp_path, chunked)
    t, d, meta = I.load_flat_index(path)
    assert meta["format"] == I.FORMAT == "flmr-flat-v1"
    assert torch.equal(t.view(torch.int16), toks.view(torch.int16)) and np.array_equal(d, dl)
    assert I.read_deleted(path).size == 0
    all_dl, files = I.index_token_files(path)
    assert np.array_equal(all_dl, dl) and len(files) == (2 if chunked else 1)


def test_single_file_index_becomes_chunked_on_append(tmp_path):
    path, toks, dl = _index(tmp_path, chunked=False)
    new_dl = np.array([3, 1, 7], dtype=np.int32)
    new = _tokens(int(new_dl.sum()), 1)
    meta = I.persist_updates(path, new, new_dl, [])
    assert meta["format"] == I.FORMAT and meta["num_chunks"] == 2 and meta["n_passages"] == 13
    names = set(os.listdir(path))
    assert "tokens.bf16" not in names and "doclens.npy" not in names
    assert {"tokens.0.bf16", "doclens.0.npy", "0.metadata.json", "tokens.1.bf16", "1.metadata.json"} <= names
    assert "deleted.npy" not in names
    t, d, _ = I.load_flat_index(path)
    assert torch.equal(t.view(torch.int16), torch.cat([toks, new]).view(torch.int16))
    assert np.array_equal(d, np.concatenate([dl, new_dl]))
    # a second append adds a chunk behind the others; small chunks split the appended passages
    meta = I.persist_updates(path, _tokens(5, 2), np.array([2, 3], dtype=np.int32), [], chunksize=1)
    assert meta["num_chunks"] == 4 and meta["n_passages"] == 15
    assert np.array_equal(I.index_token_files(path)[0], np.concatenate([dl, new_dl, [2, 3]]))


@pytest.mark.parametrize("chunked", [False, True])
def test_deleted_ids_round_trip_and_v2_only_with_deletions(tmp_path, chunked):
    path, toks, dl = _index(tmp_path, chunked)
    meta = I.persist_updates(path, None, [], [])
    assert meta["format"] == I.FORMAT                        # nothing deleted: still v1
    meta = I.persist_updates(path, None, [], [7, 2, 7])
    assert meta["format"] == I.FORMAT_V2 == "flmr-flat-v2"
    assert meta["num_chunks"] == (2 if chunked else 0)       # deletions alone keep the layout
    assert np.array_equal(I.read_deleted(path), [2, 7])
    assert I.read_deleted(path).dtype == np.int64
    t, d, _ = I.load_flat_index(path)                         # deleted passages keep their rows and ids
    assert np.array_equal(d, dl) and t.shape[0] == int(dl.sum())
    with open(os.path.join(path, "metadata.json")) as f:      # a reader of v1 only refuses the index
        assert json.load(f)["format"] != "flmr-flat-v1"
    with pytest.raises(ValueError):
        I.persist_updates(path, None, [], [10])               # outside the index


def test_v2_index_is_detected_as_flat(tmp_path):
    from ravqa_b200.searcher import detect_index_kind
    path, _, _ = _index(tmp_path, chunked=True)
    I.persist_updates(path, _tokens(4, 3), np.array([4], dtype=np.int32), [10, 0])
    assert detect_index_kind(path) == "flat"
    assert np.array_equal(I.read_deleted(path), [0, 10])


def test_deletions_split_by_shard_ranges():
    from ravqa_b200.sharded import shard_ranges
    dl = np.full(100, 8, dtype=np.int32)
    dead = np.array([0, 3, 49, 50, 51, 99], dtype=np.int64)
    ranges = shard_ranges(dl, 2)
    parts = [I.deleted_in_range(dead, p0, p1) for p0, p1 in ranges]
    assert ranges[0][1] == ranges[1][0]
    assert np.array_equal(np.concatenate(parts), dead)
    for (p0, p1), part in zip(ranges, parts):
        assert ((part >= p0) & (part < p1)).all()


def test_updater_rejects_sharded_and_plaid_persist():
    from ravqa_b200 import IndexUpdater

    class _S:
        _sharded = object()
        corpus = None
    with pytest.raises(NotImplementedError):
        IndexUpdater(searcher=_S())
    with pytest.raises(ValueError):
        IndexUpdater()


def test_new_symbols_are_declared_and_exported():
    for name in ("flmr_corpus_append", "flmr_corpus_delete", "flmr_corpus_deleted"):
        assert name in _cabi.SYMBOLS
        assert hasattr(_cabi.lib(), name), name
    with open(os.path.join(ROOT, "include", "flmr_maxsim.h")) as f:
        hdr = f.read()
    assert "#define FLMR_ABI_VERSION 2" in hdr
    for name in ("flmr_corpus_append", "flmr_corpus_delete", "flmr_corpus_deleted"):
        assert re.search(r"int %s\(" % name, hdr), name


@pytest.fixture(scope="module")
def ptxas_build(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("update_scan") / "lib.so")
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
            m = SCAN.search(line)
            cur = (int(m.group(1)), int(m.group(3)), int(m.group(2) == "2")) if m else None
            if cur:
                out[cur] = []
            continue
        if cur:
            out[cur].append(line)
    return out


def test_scan_kernels_keep_registers_and_no_spills(ptxas_build):
    log, _, _ = ptxas_build
    kernels = _sections(log, r"Compiling entry function")
    assert set(kernels) == set(REGISTERS_BEFORE)
    for key, lines in kernels.items():
        spill = next(l for l in lines if "spill stores" in l)
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (key, spill)
        regs = int(re.search(r"Used (\d+) registers", next(l for l in lines if "Used" in l)).group(1))
        assert regs <= REGISTERS_BEFORE[key], (key, regs)


def test_scan_kernels_keep_their_sass(ptxas_build):
    _, sass, _ = ptxas_build
    kernels = _sections(sass, r"Function : ")
    assert set(kernels) == set(REGISTERS_BEFORE)
    for (wgs, pair, fp8), lines in kernels.items():
        text = "\n".join(lines)
        assert ("QGMMA.64x96x32.F32.E4M3.E4M3" if fp8 else "HGMMA") in text
        assert ("WARPGROUP.DEPBAR.LE gsb0, 0x1" in text) == (wgs == 2), (wgs, pair, fp8)


def test_library_resolves_the_driver_at_run_time(ptxas_build):
    _, _, nm = ptxas_build
    undefined = [l.split()[-1] for l in nm.splitlines() if l.split()[0] == "U"]
    assert not [s for s in undefined if re.match(r"cu[A-Z]", s)], "libcuda symbols linked directly"
    for name in ("flmr_corpus_append", "flmr_corpus_delete", "flmr_corpus_deleted"):
        assert re.search(r" T %s$" % name, nm, re.M), name
