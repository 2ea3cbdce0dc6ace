"""CPU: a PLAID-coded streamed corpus (codes and residuals in pinned host memory, decoded per window on the GPU) — its C
declarations, bindings and prototypes, the Python argument refusals, the builder refusals that happen before any CUDA
call, and a numpy restatement of the padded compressed layout."""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np
import pytest

from ravqa_b200 import _cabi
from ravqa_b200.corpus import FlatCorpus

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "flmr_maxsim.h")
NEW = {"flmr_corpus_builder_create_plaid": 12, "flmr_corpus_builder_append_plaid": 4, "flmr_corpus_codec": 2}
ROW = _cabi.DIM * 2
INVALID, UNSUPPORTED = 1, 3


def test_header_declares_and_cabi_binds_the_plaid_streamed_calls():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    L = _cabi.lib()
    for name, n_params in NEW.items():
        m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, src)
        assert m, name
        assert m.group(1).count(",") + 1 == n_params, name
        assert name in _cabi.SYMBOLS and name in _cabi.PLAID_STREAMED_SYMBOLS
        assert hasattr(L, name) and len(getattr(L, name).argtypes) == n_params, name
    assert L.flmr_abi_version() == 2


# ---- the builder's refusals before any CUDA call ----------------------------------------------------------------------
def _create(doclens=(3, 5), dim=128, flags=0, window_bytes=1 << 20, nbits=2, n_centroids=8, tables=True):
    L = _cabi.lib()
    d = np.ascontiguousarray(doclens, np.int32)
    cen = np.zeros((max(n_centroids, 1), 128), np.float32)
    w = np.zeros(256, np.float32)
    b = C.c_void_p(123)
    rc = L.flmr_corpus_builder_create_plaid(d.ctypes.data if len(d) else None, len(d), dim, 0, 0, flags,
                                            window_bytes, nbits, cen.ctypes.data if tables else None, n_centroids,
                                            w.ctypes.data if tables else None, C.byref(b))
    assert not b.value, "a refused builder hands back no handle"
    return rc


@pytest.mark.parametrize("kwargs,code", [
    ({"window_bytes": ROW - 1}, INVALID),
    ({"window_bytes": 0, "flags": _cabi.CORPUS_FP8}, INVALID),          # window first, as the streamed builder
    ({"flags": _cabi.CORPUS_FP8}, UNSUPPORTED),
    ({"flags": _cabi.CORPUS_ADOPT}, UNSUPPORTED),
    ({"flags": _cabi.CORPUS_FP8, "dim": 64}, UNSUPPORTED),
    ({"dim": 64}, UNSUPPORTED),
    ({"dim": 64, "nbits": 3}, UNSUPPORTED),                            # dim before nbits
    ({"doclens": ()}, INVALID),
    ({"nbits": 3}, INVALID),
    ({"nbits": 0}, INVALID),
    ({"nbits": 16}, INVALID),
    ({"tables": False}, INVALID),
    ({"n_centroids": 0}, INVALID),
    ({"doclens": (3, 0)}, INVALID),
    ({"nbits": 3, "doclens": (3, 0)}, INVALID),
    ({"doclens": (3, 300), "window_bytes": 100 * ROW}, UNSUPPORTED),   # a passage longer than a window
])
def test_builder_refusals(kwargs, code):
    assert _create(**kwargs) == code


def test_append_refusals_without_a_builder():
    L = _cabi.lib()
    codes = np.zeros(4, np.int32)
    resid = np.zeros((4, 32), np.uint8)
    assert L.flmr_corpus_builder_append_plaid(None, codes.ctypes.data, resid.ctypes.data, 4) == INVALID
    nb = C.c_int(5)
    assert L.flmr_corpus_codec(None, C.byref(nb)) == INVALID


# ---- Python refusals ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kwargs", [
    {"compressed": True},                                        # residency="device"
    {"compressed": True, "residency": "device"},
    {"compressed": True, "residency": "host", "storage": "fp8"},
    {"compressed": True, "storage": "fp8"},
    {"compressed": 1, "residency": "host"},
])
def test_from_plaid_refuses_compressed_without_a_host_residency(tmp_path, kwargs):
    with pytest.raises(ValueError):
        FlatCorpus.from_plaid(str(tmp_path), **kwargs)


def test_searcher_refuses_compressed_on_a_flat_index(tmp_path):
    import json
    from ravqa_b200 import Searcher
    from ravqa_b200.index_io import FORMATS as FLAT_FORMATS
    path = tmp_path / "flat"
    path.mkdir()
    with open(path / "metadata.json", "w") as f:
        json.dump({"format": sorted(FLAT_FORMATS)[0]}, f)
    with pytest.raises(ValueError, match="compressed"):
        Searcher(index=str(path), residency="host", compressed=True)


# ---- the padded compressed layout ---------------------------------------------------------------------------------------
def padded_source_rows(doclens) -> np.ndarray:
    """For every stored row of the padded layout, the packed token row whose code and residual it holds: a passage's
    own rows in order, then its last row repeated up to a multiple of 4 rows."""
    out, s = [], 0
    for n in np.asarray(doclens, np.int64):
        rows = (n + 3) // 4 * 4
        out.append(s + np.minimum(np.arange(rows), n - 1))
        s += n
    return np.concatenate(out) if out else np.empty(0, np.int64)


def scatter(codes, residuals, doclens, pieces):
    """The builder's fill, restated: packed rows fed in `pieces` (row counts, cutting passages anywhere) land in the
    padded arrays as host_scatter_rows puts them."""
    doclens = np.asarray(doclens, np.int64)
    soff = np.concatenate([[0], np.cumsum(doclens)])
    poff = np.concatenate([[0], np.cumsum((doclens + 3) // 4 * 4)])
    out_c = np.full(poff[-1], -1, np.int32)
    out_r = np.zeros((poff[-1], residuals.shape[1]), np.uint8)
    r = 0
    for n in pieces:
        for row in range(r, r + n):
            p = int(np.searchsorted(soff, row, side="right")) - 1
            dst = poff[p] + row - soff[p]
            out_c[dst], out_r[dst] = codes[row], residuals[row]
            if row == soff[p + 1] - 1:
                for j in range(poff[p] + doclens[p], poff[p + 1]):
                    out_c[j], out_r[j] = codes[row], residuals[row]
        r += n
    return out_c, out_r


@pytest.mark.parametrize("seed", range(4))
def test_padded_layout_repeats_each_passage_last_row(seed):
    rng = np.random.default_rng(seed)
    dl = rng.integers(1, 30, size=40)
    n = int(dl.sum())
    codes = rng.integers(0, 1000, size=n).astype(np.int32)
    residuals = rng.integers(0, 256, size=(n, 16 * [1, 2, 4, 8][seed])).astype(np.uint8)
    cuts = np.sort(rng.choice(np.arange(1, n), size=7, replace=False))
    pieces = np.diff(np.concatenate([[0], cuts, [n]]))
    c, r = scatter(codes, residuals, dl, pieces)
    src = padded_source_rows(dl)
    assert len(src) == int(((dl + 3) // 4 * 4).sum()) and len(src) % 4 == 0
    assert np.array_equal(c, codes[src]) and np.array_equal(r, residuals[src])
    # a window is a contiguous range of stored rows in both arrays: the bytes a window copies, from its row range
    poff = np.concatenate([[0], np.cumsum((dl + 3) // 4 * 4)])
    a, b = int(poff[10]), int(poff[25])
    assert (b - a) * (4 + residuals.shape[1]) == c[a:b].nbytes + r[a:b].nbytes
