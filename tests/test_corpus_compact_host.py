"""Corpus compaction, CPU side: the row-move schedule flmr_corpus_compact executes (flmr_debug_compact_plan), replayed
on a numpy matrix for adversarial deletion patterns; argument checks that need no device; the new exports; and what
ptxas made of the new kernels."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from helpers import ROOT
from ravqa_b200 import _cabi

SRC = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
NEW_SYMBOLS = ("flmr_corpus_compact", "flmr_corpus_stored", "flmr_debug_compact_plan")
NEW_KERNELS = ("flmr_move_rows_kernel", "flmr_slot_allow_kernel", "flmr_slot_ids_kernel",
               "flmr_expand_slot_scores_kernel")
GROUP = _cabi.TOKEN_GROUP


def _plan(doclens, deleted, chunk_rows):
    L = _cabi.lib()
    dl = np.ascontiguousarray(doclens, dtype=np.int32)
    dead = np.ascontiguousarray(deleted, dtype=np.int64)
    n = C.c_int64(0)
    _cabi.check(L.flmr_debug_compact_plan(dl.ctypes.data, len(dl), dead.ctypes.data, len(dead), chunk_rows, None, 0,
                                          C.byref(n)))
    out = np.zeros((n.value, 5), dtype=np.int64)
    _cabi.check(L.flmr_debug_compact_plan(dl.ctypes.data, len(dl), dead.ctypes.data, len(dead), chunk_rows,
                                          out.ctypes.data, n.value, C.byref(n)))
    return out


def _replay(doclens, deleted, chunk_rows):
    """Run the schedule on a matrix whose row r holds r: the result must be the compacted layout, no row may be
    written before every move that reads it has read it, and a staged chunk never holds more than chunk_rows rows."""
    padded = (np.asarray(doclens, dtype=np.int64) + GROUP - 1) // GROUP * GROUP
    poff = np.concatenate([[0], np.cumsum(padded)])
    rows = int(poff[-1])
    keep = np.ones(len(doclens), dtype=bool)
    keep[np.asarray(deleted, dtype=np.int64)] = False
    want = np.concatenate([np.arange(poff[p], poff[p + 1]) for p in np.flatnonzero(keep)])
    plan = _plan(doclens, deleted, chunk_rows)
    mat = np.arange(rows, dtype=np.int64)
    # rows some move has yet to read: a write to one of them would clobber it
    pending = np.zeros(rows, dtype=np.int64)
    for src, _, n, _, _ in plan:
        pending[src:src + n] += 1
    assert np.all(plan[:, 2] > 0)
    assert np.all(plan[:, 1] <= plan[:, 0]), "a destination above its source"
    assert np.all(np.diff(plan[:, 1]) > 0), "moves not in destination order"
    assert np.all(np.diff(plan[:, 4]) >= 0)
    for chunk in np.unique(plan[:, 4]):
        moves = plan[plan[:, 4] == chunk]
        staged = set(moves[:, 3].tolist())
        assert len(staged) == 1, "a chunk is either staged or not"
        assert moves[:, 2].sum() <= chunk_rows, "a chunk beyond the staging bound"
        assert np.all(moves[1:, 1] == moves[:-1, 1] + moves[:-1, 2]), "a chunk's destinations are contiguous"
        reads = [mat[s:s + n].copy() for s, _, n, _, _ in moves]   # a staged chunk reads everything first
        read_rows = np.concatenate([np.arange(s, s + n) for s, _, n, _, _ in moves])
        write_rows = np.concatenate([np.arange(d, d + n) for _, d, n, _, _ in moves])
        if not moves[0, 3]:
            # copied directly, all moves of the chunk at once: none of its writes may land on one of its reads
            assert not np.intersect1d(read_rows, write_rows).size, "an unstaged chunk overlaps its own sources"
        for (s, _, n, _, _) in moves:
            pending[s:s + n] -= 1
        assert not pending[write_rows].any(), "a row is overwritten before it is read"
        for (_, d, n, _, _), v in zip(moves, reads):
            mat[d:d + n] = v
    assert np.array_equal(mat[:len(want)], want)
    return plan


def _ragged(n, seed, aligned=False):
    rng = np.random.default_rng(seed)
    dl = rng.integers(1, 40, size=n).astype(np.int32)
    if aligned:
        dl = (dl + 3) // 4 * 4
    return dl


PATTERNS = {
    "first": lambda n: [0],
    "last": lambda n: [n - 1],
    "alternating": lambda n: list(range(0, n, 2)),
    "alternating_odd": lambda n: list(range(1, n, 2)),
    "long_runs": lambda n: list(range(5, 40)) + list(range(60, 61)) + list(range(120, n - 3)),
    "all_but_one": lambda n: [p for p in range(n) if p != n // 2],
    "all_but_first": lambda n: list(range(1, n)),
    "all_but_last": lambda n: list(range(n - 1)),
    "random_30": lambda n: sorted(np.random.default_rng(7).choice(n, n * 3 // 10, replace=False).tolist()),
}


@pytest.mark.parametrize("aligned", [False, True])
@pytest.mark.parametrize("chunk_rows", [4, 37, 256, 100_000])
@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_schedule_compacts_without_clobbering(pattern, chunk_rows, aligned):
    dl = _ragged(200, 3, aligned)
    _replay(dl, PATTERNS[pattern](len(dl)), chunk_rows)


def test_first_passage_deleted_shifts_every_row_through_staging():
    # every kept row moves down by one 4-row group: each chunk overlaps its own source, so each is staged
    dl = np.full(100, 8, dtype=np.int32)
    plan = _replay(dl, [0], 64)
    assert plan[:, 3].all()
    assert np.all(plan[:, 0] - plan[:, 1] == 8)
    assert plan[:, 2].sum() == 99 * 8 and plan[:, 2].max() <= 64


def test_rows_in_front_of_the_first_deletion_stay_put():
    dl = np.full(50, 5, dtype=np.int32)
    assert _plan(dl, [49], 0).shape[0] == 0      # deleting the last passage moves nothing
    plan = _replay(dl, [10], 1 << 20)
    assert plan[0, 1] == 10 * 8 and plan[:, 2].sum() == 39 * 8
    # a removal wider than a chunk: the source of each chunk lies wholly above its destination, so no staging
    plan = _replay(np.full(40, 4, dtype=np.int32), list(range(0, 20)), 16)
    assert not plan[:, 3].any()


def test_default_bound_is_256_mib_of_bf16_rows():
    dl = np.full(10, 4, dtype=np.int32)
    plan = _plan(dl, [0], 0)
    assert plan.shape[0] == 1 and plan[0, 2] == 36 and plan[0, 3] == 1
    # a corpus larger than the bound is cut into chunks of exactly 2^20 rows (256 MiB of 256-byte rows)
    big = np.full(300_000, 8, dtype=np.int32)
    plan = _plan(big, [0], 0)
    sizes = [plan[plan[:, 4] == c, 2].sum() for c in np.unique(plan[:, 4])]
    assert max(sizes) == (256 << 20) // (128 * 2) and sum(sizes) == (300_000 - 1) * 8


def test_plan_argument_checks():
    L = _cabi.lib()
    dl = np.full(4, 4, dtype=np.int32)
    bad = np.array([4], dtype=np.int64)
    n = C.c_int64(0)
    assert L.flmr_debug_compact_plan(dl.ctypes.data, 4, bad.ctypes.data, 1, 0, None, 0, C.byref(n)) == 1
    assert L.flmr_debug_compact_plan(None, 4, None, 0, 0, None, 0, C.byref(n)) == 1
    assert L.flmr_debug_compact_plan(dl.ctypes.data, 4, None, 1, 0, None, 0, C.byref(n)) == 1
    ok = np.array([1], dtype=np.int64)
    out = np.zeros(5, dtype=np.int64)
    assert L.flmr_debug_compact_plan(dl.ctypes.data, 4, ok.ctypes.data, 1, 0, out.ctypes.data, 0, C.byref(n)) == 1
    assert b"capacity" in L.flmr_last_error()


def test_compact_and_stored_reject_a_null_corpus_and_take_null_outputs():
    L = _cabi.lib()
    removed, released = C.c_int64(7), C.c_int64(7)
    assert L.flmr_corpus_compact(None, C.byref(removed), C.byref(released)) == _cabi.FLMR_OK + 1
    assert removed.value == 0 and released.value == 0          # outputs are cleared before the check
    assert L.flmr_corpus_compact(None, None, None) == 1
    assert L.flmr_corpus_stored(None, None, None) == 1
    assert b"null" in L.flmr_last_error()


def test_new_symbols_are_declared_and_exported():
    L = _cabi.lib()
    with open(os.path.join(ROOT, "include", "flmr_maxsim.h")) as f:
        hdr = f.read()
    assert "#define FLMR_ABI_VERSION 2" in hdr
    for name in NEW_SYMBOLS:
        assert name in _cabi.SYMBOLS
        assert hasattr(L, name), name
        assert re.search(r"int %s\(" % name, hdr), name
        assert getattr(L, name).argtypes is not None, name


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("compact") / "lib.so")
    proc = subprocess.run([nvcc, "-Xptxas=-v", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-shared", "-Xcompiler", "-fPIC", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    nm = subprocess.run(["nm", "-D", out], capture_output=True, text=True, check=True).stdout
    return proc.stderr, nm


def test_new_kernels_compile_for_sm90a_without_spills(ptxas_log):
    log, nm = ptxas_log
    seen = {}
    cur = None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)' for 'sm_90a'", line)
        if m:
            cur = next((k for k in NEW_KERNELS if k in m.group(1)), None)
            continue
        if cur and "spill stores" in line:
            seen[cur] = line
    assert set(seen) == set(NEW_KERNELS)
    for name, line in seen.items():
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
    for name in NEW_SYMBOLS:
        assert re.search(r" T %s$" % name, nm, re.M), name
