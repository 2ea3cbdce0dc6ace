"""Shared helpers for the test-suite (golden fixtures, C oracle loader)."""
from __future__ import annotations

import ctypes as C
import glob
import json
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def bf16_bits_to_f32(bits: np.ndarray) -> np.ndarray:
    return (bits.astype(np.uint32) << 16).view(np.float32)


def load_golden(name: str) -> dict:
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    g = {k: z[k] for k in z.files}
    g["Q"] = bf16_bits_to_f32(g.pop("Q_bf16"))
    g["D"] = bf16_bits_to_f32(g.pop("D_bf16"))
    g["meta"] = json.loads(str(g["meta"]))
    return g


def golden_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "g[0-9]*.npz")))


def placement_doclens(n: int = 20_000, seed: int = 0) -> np.ndarray:
    """Passage lengths of the placement fixture: most passages 1-23 tokens, so that a 96-token scan tile holds more
    than the 4 passage ends whose row maxima the reducer sums itself; one in 16 is 24-200 tokens long."""
    rng = np.random.default_rng(seed)
    dl = rng.integers(1, 24, size=n)
    long = rng.random(n) < 1 / 16
    dl[long] = rng.integers(24, 201, size=int(long.sum()))
    return dl.astype(np.int32)


def placement_tracked(n: int) -> np.ndarray:
    """Tracked passages of the placement fixture: the front of the corpus (the first two of 132 CTAs, where a
    prepended passage shifts every passage) and every 97th passage after it."""
    return np.concatenate([np.arange(300), np.arange(300, n, 97)])


def scan_partition(doclens, n_ctas: int = 132) -> dict:
    """The scan's partition for ``min(n_ctas, n)`` CTAs (host-only ``flmr_debug_build_partition``; passages padded to
    multiples of 4 rows, 96-row tiles) and what the tests read off it: per-CTA rows and tile ranges, per-tile end masks,
    and per passage its first / last tile (global tile index) and its slot (the how-manyth passage to end in its
    tile)."""
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    dl = np.ascontiguousarray(doclens, dtype=np.int32)
    n = len(dl)
    nc = min(n_ctas, n)
    rows = (dl.astype(np.int64) + 3) // 4 * 4
    poff = np.concatenate([[0], np.cumsum(rows)])
    rb = np.zeros(nc + 1, np.int32)
    tb = np.zeros(nc + 1, np.int64)
    cap = int(poff[-1] // 96 + nc + 1)
    em = np.zeros(cap, np.uint32)
    fp = np.zeros(cap, np.int32)
    nt = C.c_int64()
    _cabi.check(L.flmr_debug_build_partition(dl.ctypes.data, n, nc, rb.ctypes.data, tb.ctypes.data, em.ctypes.data,
                                             fp.ctypes.data, cap, C.byref(nt)))
    em, fp = em[:nt.value], fp[:nt.value]
    cta_of_row = np.searchsorted(rb[1:], poff[:-1], side="right")          # CTA of each passage's first row
    first_tile = tb[cta_of_row] + (poff[:-1] - rb[cta_of_row]) // 96
    last_tile = tb[cta_of_row] + (poff[1:] - 1 - rb[cta_of_row]) // 96
    slot = np.full(n, -1, np.int64)
    for mask, first in zip(em.tolist(), fp.tolist()):
        k = bin(mask).count("1")
        slot[first:first + k] = np.arange(k)
    return {"n_ctas": nc, "row_begin": rb, "tile_base": tb, "end_mask": em, "first_pid": fp, "rows": rows,
            "n_rows": int(poff[-1]), "first_tile": first_tile, "last_tile": last_tile, "slot": slot,
            "cta_rows": np.diff(rb.astype(np.int64)), "cta_tiles": np.diff(tb)}


def scan_slots(doclens, n_ctas: int = 132) -> np.ndarray:
    """Slot of every passage in the scan's partition for `n_ctas` CTAs: the passage is the slot-th passage to end in
    its 96-token tile.  The reducer sums slots 0-3 from parked row maxima and later slots from the consumer warps'
    16-row sums."""
    slot = scan_partition(doclens, n_ctas)["slot"]
    assert (slot >= 0).all()
    return slot


def c_oracle():
    """Build (if needed) and load oracle/_ref/libmaxsim_oracle.so."""
    path = os.path.join(ROOT, "oracle", "_ref", "libmaxsim_oracle.so")
    src = os.path.join(ROOT, "oracle", "maxsim_oracle.c")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, capture_output=True)
    L = C.CDLL(path)
    L.flmr_oracle_maxsim_scores.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                            C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.flmr_oracle_topk.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]
    return L


def c_oracle_scores(Q, D, doclens, relu=False, nthreads=4):
    L = c_oracle()
    Q = np.ascontiguousarray(Q, dtype=np.float32)
    D = np.ascontiguousarray(D, dtype=np.float32)
    dl = np.ascontiguousarray(doclens, dtype=np.int32)
    out = np.empty((Q.shape[0], len(dl)), dtype=np.float32)
    rc = L.flmr_oracle_maxsim_scores(Q.ctypes.data, Q.shape[0], Q.shape[1], D.ctypes.data, dl.ctypes.data,
                                     len(dl), Q.shape[2], int(relu), nthreads, out.ctypes.data)
    assert rc == 0
    return out
