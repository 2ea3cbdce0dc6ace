"""CPU: a streamed corpus (rows in pinned host memory, scanned window by window) — its C declarations and bindings,
the window plan against a numpy restatement, and the Python argument checks."""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np
import pytest

from ravqa_b200 import _cabi
from ravqa_b200.corpus import FlatCorpus, _check_residency

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "flmr_maxsim.h")
NEW = ("flmr_corpus_create_streamed", "flmr_corpus_builder_create_streamed", "flmr_corpus_residency",
       "flmr_debug_window_plan")
ROW = _cabi.DIM * 2
TILE = _cabi.TILE_TOKENS


def test_header_declares_and_cabi_binds_the_streamed_calls():
    src = open(HEADER).read()
    L = _cabi.lib()
    for name in NEW:
        assert re.search(r"\bint\s+%s\s*\(" % name, src), name
        assert name in _cabi.SYMBOLS
        assert getattr(L, name).argtypes, name


# ---- numpy restatement of the plan ----------------------------------------------------------------------------------
def _poff(doclens):
    rows = (np.asarray(doclens, np.int64) + 3) // 4 * 4
    return np.concatenate([[0], np.cumsum(rows)])


def np_windows(doclens, window_bytes):
    """Contiguous slot ranges, each taking every slot whose rows still fit window_bytes // 256 rows; None when a
    passage alone is longer than that."""
    poff = _poff(doclens)
    cap = window_bytes // ROW
    out, s0, n = [], 0, len(doclens)
    while s0 < n:
        s1 = s0
        while s1 < n and poff[s1 + 1] - poff[s0] <= cap:
            s1 += 1
        if s1 == s0:
            return None
        out.append((s0, s1))
        s0 = s1
    return out


def np_partition(doclens, n_ctas):
    """build_partition: token-balanced CTA ranges of whole passages, tiles of TILE rows per CTA, per tile the mask of
    4-row groups a passage ends with and the first passage ending in it."""
    poff = _poff(doclens)
    n, rows = len(doclens), int(poff[-1])
    pbeg = [0]
    for c in range(1, n_ctas):
        p = int(np.searchsorted(poff, rows * c // n_ctas, side="left"))
        pbeg.append(min(max(p, pbeg[-1]), n))
    pbeg.append(n)
    rb = np.array([poff[p] for p in pbeg], np.int64)
    tiles = [(rb[c + 1] - rb[c] + TILE - 1) // TILE for c in range(n_ctas)]
    tb = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int64)
    em = np.zeros(int(tb[-1]), np.uint32)
    fp = np.zeros(int(tb[-1]), np.int64)
    for c in range(n_ctas):
        seen = set()
        for p in range(pbeg[c], pbeg[c + 1]):
            last = poff[p + 1] - 1 - rb[c]
            t = int(tb[c] + last // TILE)
            em[t] |= np.uint32(1 << int((last % TILE) // 4))
            if t not in seen:
                seen.add(t)
                fp[t] = p
    return rb, tb, em, fp


def np_window_plan(doclens, window_bytes, n_ctas):
    wins = np_windows(doclens, window_bytes)
    if wins is None:
        return None
    poff = _poff(doclens)
    table, rb, tb, em, fp = [], [], [], [], []
    for s0, s1 in wins:
        nc = min(n_ctas, s1 - s0)
        r, t, e, f = np_partition(doclens[s0:s1], nc)
        table.append((s0, s1, poff[s0], poff[s1] - poff[s0], nc, len(e)))
        rb.append(r), tb.append(t), em.append(e), fp.append(f + s0)
    return (np.array(table, np.int64), np.concatenate(rb), np.concatenate(tb), np.concatenate(em),
            np.concatenate(fp))


def lib_window_plan(doclens, window_bytes, n_ctas):
    L = _cabi.lib()
    dl = np.ascontiguousarray(doclens, np.int32)
    nw, nt = C.c_int64(), C.c_int64()
    rc = L.flmr_debug_window_plan(dl.ctypes.data, len(dl), int(window_bytes), n_ctas, None, 0, C.byref(nw), None,
                                  None, None, None, 0, C.byref(nt))
    if rc != 0:
        return rc
    table = np.zeros((nw.value, 6), np.int64)
    cap = int(_poff(dl)[-1]) // TILE + nw.value * (n_ctas + 2) + 1
    rb, tb = np.zeros(cap, np.int32), np.zeros(cap, np.int64)
    em, fp = np.zeros(cap, np.uint32), np.zeros(cap, np.int32)
    _cabi.check(L.flmr_debug_window_plan(dl.ctypes.data, len(dl), int(window_bytes), n_ctas, table.ctypes.data,
                                         nw.value, C.byref(nw), rb.ctypes.data, tb.ctypes.data, em.ctypes.data,
                                         fp.ctypes.data, cap, C.byref(nt)))
    n_entries = int((table[:, 4] + 1).sum())
    return table, rb[:n_entries], tb[:n_entries], em[:nt.value], fp[:nt.value]


def _cases():
    rng = np.random.default_rng(7)
    yield "ragged", rng.integers(1, 200, 3000).astype(np.int32), 256 * 1024, 132
    yield "short", rng.integers(1, 9, 5000).astype(np.int32), 64 * 1024, 132
    yield "one-cta", rng.integers(1, 40, 400).astype(np.int32), 40 * 1024, 1
    yield "whole", rng.integers(1, 180, 500).astype(np.int32), 1 << 30, 132
    # a window of exactly one 64-row passage; a passage exactly as long as the window; a last window of one passage
    dl = np.array([10, 20, 64, 3, 5, 64, 7, 8, 9, 64], np.int32)
    yield "edges", dl, 64 * ROW, 132
    yield "odd-bytes", rng.integers(1, 100, 700).astype(np.int32), 100 * ROW + 255, 7
    # one window of exactly every row, as a resident corpus plans it
    dl = rng.integers(1, 300, 900).astype(np.int32)
    yield "exact", dl, int(_poff(dl)[-1]) * ROW, 7


@pytest.mark.parametrize("name,doclens,window_bytes,n_ctas", list(_cases()), ids=[c[0] for c in _cases()])
def test_window_plan_matches_numpy(name, doclens, window_bytes, n_ctas):
    want = np_window_plan(doclens, window_bytes, n_ctas)
    got = lib_window_plan(doclens, window_bytes, n_ctas)
    for a, b, what in zip(got, want, ("windows", "cta_row_begin", "cta_tile_base", "tile_end_mask", "tile_first_pid")):
        assert np.array_equal(a.astype(np.int64), b.astype(np.int64)), "%s: %s differs" % (name, what)
    table = got[0]
    poff = _poff(doclens)
    # contiguous, covering every slot, in order; rows are the slots' stored rows; none exceeds the window
    assert table[0, 0] == 0 and table[-1, 1] == len(doclens)
    assert np.array_equal(table[1:, 0], table[:-1, 1])
    assert (table[:, 1] > table[:, 0]).all()
    assert np.array_equal(table[:, 2], poff[table[:, 0]])
    assert np.array_equal(table[:, 3], poff[table[:, 1]] - poff[table[:, 0]])
    assert (table[:, 3] <= window_bytes // ROW).all()
    # a window is closed only by a passage that does not fit it
    nxt = table[:-1, 1]
    assert (table[:-1, 3] + (poff[nxt + 1] - poff[nxt]) > window_bytes // ROW).all()
    # every passage ends in exactly one tile of its window
    ends = sum(bin(int(m)).count("1") for m in got[3])
    assert ends == len(doclens)
    if name == "edges":
        sizes = table[:, 1] - table[:, 0]
        assert 1 in sizes[:-1] and sizes[-1] == 1
        assert (table[:, 3] == 64).any()
    if window_bytes >= poff[-1] * ROW:
        # one window of every slot, whose partition is exactly flmr_debug_build_partition's: the resident corpus's
        assert len(table) == 1
        L, dl, nt = _cabi.lib(), np.ascontiguousarray(doclens, np.int32), C.c_int64()
        nc = min(n_ctas, len(dl))
        want = (np.zeros(nc + 1, np.int32), np.zeros(nc + 1, np.int64), np.zeros(len(got[3]), np.uint32),
                np.zeros(len(got[3]), np.int32))
        _cabi.check(L.flmr_debug_build_partition(dl.ctypes.data, len(dl), n_ctas, *(a.ctypes.data for a in want),
                                                 len(got[3]), C.byref(nt)))
        assert table[0, 4] == nc and nt.value == len(got[3])
        for a, b in zip(got[1:], want):
            assert np.array_equal(a, b)


def test_window_plan_refuses_a_passage_longer_than_the_window():
    dl = np.array([4, 8, 65, 4], np.int32)                # 68 stored rows
    assert np_windows(dl, 64 * ROW) is None
    assert lib_window_plan(dl, 64 * ROW, 132) == 3        # FLMR_ERR_UNSUPPORTED
    assert lib_window_plan(dl, 68 * ROW, 132)[0].shape[0] >= 1
    assert lib_window_plan(dl, ROW - 1, 132) == 1         # not one row: FLMR_ERR_INVALID_ARG


@pytest.mark.parametrize("bad", [0, -1, ROW - 1, 1.5e9, "1GB", True, None])
def test_bad_window_bytes_raise(bad):
    with pytest.raises(ValueError):
        _check_residency("host", "bf16", bad)
    import torch
    with pytest.raises(ValueError):
        FlatCorpus(torch.zeros(4, _cabi.DIM), [4], residency="host", window_bytes=bad)


def test_fp8_and_unknown_residency_raise():
    import torch
    with pytest.raises(ValueError, match="fp8"):
        _check_residency("host", "fp8", 1 << 30)
    with pytest.raises(ValueError, match="fp8"):
        FlatCorpus(torch.zeros(4, _cabi.DIM), [4], storage="fp8", residency="host")
    with pytest.raises(ValueError, match="residency"):
        FlatCorpus(torch.zeros(4, _cabi.DIM), [4], residency="pinned")
    _check_residency("host", "bf16", ROW)
    _check_residency("host", "fp16", np.int64(1 << 26))
    _check_residency("device", "fp8", None)       # window_bytes is read only for residency="host"
