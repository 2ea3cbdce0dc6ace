"""Float64 restatement of the paths that put a corpus into HBM, and the corpora that reach their loops' edges.

* ``decode_fp64``: PLAID residual decode (``flmr_plaid_decode`` / ``_fp16``, csrc/flmr_maxsim.cu).  The embedding is
  ``v = fl32(centroid[code] + w[idx])``, one fp32 addition as in the reference's ``decompress_residuals_cpp``; the
  normalised row ``y = v / max(||v||, eps)`` is then computed in float64.
* ``check_rounding``: a kernel's bf16 / fp16 output against ``y``: round to nearest even of ``y``, except within the
  kernel's fp32 error band of a rounding midpoint, where either neighbour is accepted.
* ``write_plaid``: the reference's PLAID directory layout (as tests/golden/plaid_nbits*/).
* ``design_doclens`` / ``design_rows``: corpora whose passage ends and straddling passages sit at the multiples of a
  staging size, and whose rows make a wrong padding row change a score.
* ``load_constants``: the staging sizes, read from the CUDA source, so that a change of one of them fails the host
  tests instead of silently moving the boundaries out of the GPU tests' reach.

Pinned on CPU by tests/test_corpus_load_host.py; used by tests/test_corpus_load_gpu.py.  Torch float64 ops run on
either device.
"""
from __future__ import annotations

import json
import os
import re

import numpy as np
import torch

from helpers import ROOT

CU_PATH = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "csrc", "flmr_maxsim.cu")
DIM = 128
EPS = float(np.float32(1e-12))   # F.normalize's eps as the fp32 kernel holds it (1e-12 itself differs by 2^-28)

# The kernel's error band, relative to |y|.  v is exact (the model makes the same fp32 addition).  The sum of squares
# is 4 in-lane terms (3 additions, the products rounded or fused) and 5 butterfly levels: all terms are >= 0, so its
# relative error is below (4 + 5) u.  sqrt halves that (4.5 u) and adds its own rounding (5.5 u), the reciprocal and
# the final multiply add one u each: 7.5 u, u = 2^-24.  The band takes 16 u = 2^-20, about twice that.  A kernel
# value v' = y (1 + d) rounds differently from y only if a rounding midpoint lies between them, i.e. within |d| |y|.
BAND = 2.0 ** -20

_FMT = {  # mantissa bits (with the implicit one), smallest normal exponent, largest finite value
    torch.bfloat16: (8, -126, (2.0 - 2.0 ** -7) * 2.0 ** 127),
    torch.float16: (11, -14, 65504.0),
}


# ---- PLAID decode ----------------------------------------------------------------------------------------------------
def bucket_index(residuals, nbits: int) -> torch.Tensor:
    """int64 ``[n, 128]``: the bucket of every dim.  Dim i is field ``i % (8 / nbits)`` (from the most significant bits)
    of byte ``i / (8 / nbits)``; the reference packs each index least significant bit first, so the field is read
    bit-reversed."""
    r = torch.as_tensor(np.asarray(residuals)).to(torch.int64)
    keys = 8 // nbits
    i = torch.arange(DIM)
    byte = r[:, i // keys]
    field = (byte >> (8 - nbits * (i % keys + 1))) & ((1 << nbits) - 1)
    idx = torch.zeros_like(field)
    for b in range(nbits):
        idx |= ((field >> b) & 1) << (nbits - 1 - b)
    return idx


def decode_fp32(codes, residuals, centroids, weights, nbits: int) -> torch.Tensor:
    """``v = fl32(centroids[code] + weights[idx])`` float32 ``[n, 128]`` (CPU)."""
    c = torch.as_tensor(np.asarray(centroids)).float()
    w = torch.as_tensor(np.asarray(weights)).float()
    code = torch.as_tensor(np.asarray(codes)).to(torch.int64)
    return c[code] + w[bucket_index(residuals, nbits)]


def decode_fp64(codes, residuals, centroids, weights, nbits: int, normalize: bool = True) -> torch.Tensor:
    """Float64 ``y``: ``v`` itself, or ``v / max(||v||, eps)`` computed in float64."""
    v = decode_fp32(codes, residuals, centroids, weights, nbits).double()
    if not normalize:
        return v
    return v / v.norm(dim=1, keepdim=True).clamp_min(EPS)


# ---- the rounding classifier -----------------------------------------------------------------------------------------
def _pow2(n: torch.Tensor) -> torch.Tensor:
    """2^n exactly, built from its bits (``torch.pow`` on a GPU may miss a power of two by an ulp)."""
    return ((n.to(torch.int64) + 1023) << 52).view(torch.float64)


def rounding_neighbours(y: torch.Tensor, dtype: torch.dtype):
    """(lo, hi, rn, mid): float64 values of ``dtype`` with ``lo <= y < hi`` (overflow beyond the largest finite value
    as +-inf), the round-to-nearest-even of ``y`` and the midpoint of lo and hi.  Every value here is exact."""
    p, emin, fmax = _FMT[dtype]
    y = y.double()
    _, e = torch.frexp(y)                                     # |y| in [2^(e-1), 2^e)
    ulp = _pow2(torch.clamp(e - 1, min=emin) - (p - 1))
    k = torch.floor(y / ulp)
    lo, hi = k * ulp, (k + 1) * ulp
    dlo, dhi = y - lo, hi - y
    even_lo = torch.remainder(k, 2) == 0
    rn = torch.where((dlo < dhi) | ((dlo == dhi) & even_lo), lo, hi)

    def inf(x):
        return torch.where(x.abs() > fmax, torch.copysign(torch.full_like(x, torch.inf), x), x)
    return inf(lo), inf(hi), inf(rn), lo + ulp / 2


def check_rounding(got: torch.Tensor, y: torch.Tensor, tag: str = "") -> int:
    """``got`` (bf16 or fp16) must be RN(y) in its type; within ``BAND |y|`` of a rounding midpoint either neighbour is
    accepted.  A flush of a subnormal to zero fails like any other wrong value.  Returns how many elements fell
    inside the band."""
    lo, hi, rn, mid = rounding_neighbours(y, got.dtype)
    g = got.double()
    y = y.double()
    band = (y - mid).abs() <= BAND * y.abs()
    ok = (g == rn) | (band & ((g == lo) | (g == hi)))
    if not bool(ok.all()):
        bad = (~ok).nonzero()[0].tolist()
        at = tuple(bad)
        raise AssertionError("%s: %d of %d elements misrounded; first at %s: got %r, float64 %r, rn %r" % (
            tag, int((~ok).sum()), ok.numel(), at, float(g[at]), float(y[at]), float(rn[at])))
    return int(band.sum())


# ---- the reference's PLAID directory -----------------------------------------------------------------------------
def write_plaid(path: str, nbits: int, centroids: torch.Tensor, cutoffs: torch.Tensor, weights: torch.Tensor,
                chunks) -> None:
    """A PLAID index directory as the reference's indexer writes it: ``chunks`` is a list of (codes int32 [n],
    residuals uint8 [n, 128 * nbits / 8], doclens [passages]).  Centroids are stored fp16, ``buckets.pt`` holds
    ``(cutoffs, weights)``."""
    os.makedirs(path, exist_ok=True)
    torch.save(torch.as_tensor(centroids).half(), os.path.join(path, "centroids.pt"))
    torch.save((torch.as_tensor(cutoffs).float(), torch.as_tensor(weights).float()), os.path.join(path, "buckets.pt"))
    n_emb = n_pass = 0
    for c, (codes, residuals, doclens) in enumerate(chunks):
        codes = torch.as_tensor(codes).to(torch.int32)
        residuals = torch.as_tensor(residuals).to(torch.uint8)
        doclens = [int(x) for x in doclens]
        assert codes.numel() == sum(doclens) == residuals.size(0) and residuals.size(1) == DIM * nbits // 8
        torch.save(codes, os.path.join(path, "%d.codes.pt" % c))
        torch.save(residuals, os.path.join(path, "%d.residuals.pt" % c))
        with open(os.path.join(path, "doclens.%d.json" % c), "w") as f:
            json.dump(doclens, f)
        with open(os.path.join(path, "%d.metadata.json" % c), "w") as f:
            json.dump({"passage_offset": n_pass, "num_passages": len(doclens), "num_embeddings": len(codes),
                       "embedding_offset": n_emb}, f)
        n_emb += len(codes)
        n_pass += len(doclens)
    with open(os.path.join(path, "metadata.json"), "w") as f:
        json.dump({"config": {"nbits": nbits, "dim": DIM}, "num_chunks": len(chunks),
                   "num_partitions": int(centroids.shape[0]), "num_embeddings": n_emb,
                   "avg_doclen": n_emb / n_pass}, f)


def fixture_weights(nbits: int, g: torch.Generator) -> torch.Tensor:
    """Bucket weights shaped like the reference's (sorted quantiles of residuals, about +-0.3)."""
    return torch.sort(0.1 * torch.randn(1 << nbits, generator=g)).values


def random_codes(n: int, n_centroids: int, nbits: int, g: torch.Generator):
    codes = torch.randint(0, n_centroids, (n,), generator=g, dtype=torch.int32)
    residuals = torch.randint(0, 256, (n, DIM * nbits // 8), generator=g, dtype=torch.uint8)
    return codes, residuals


# ---- corpus designers ------------------------------------------------------------------------------------------------
def _fill(n: int, rng, aligned: bool) -> list:
    """Random passage lengths summing to exactly n (1..180, every residue mod 4; aligned: multiples of 4)."""
    out = []
    while n > 0:
        x = 4 * int(rng.integers(1, 46)) if aligned else int(rng.integers(1, 181))
        x = n if n - x < (4 if aligned else 1) else x
        out.append(x)
        n -= x
    return out


def design_doclens(n_rows: int, period: int, kind: str, seed: int, aligned: bool = False) -> np.ndarray:
    """Passage lengths summing to ``n_rows`` with, at every multiple ``m * period < n_rows``:

    * kind "ends": passage ends at ``m P - 1``, ``m P`` and ``m P + 1`` (two 1-row passages; aligned: at ``m P - 4``,
      ``m P``, ``m P + 4``);
    * kind "straddle": one passage that starts at least 2 rows before ``m P`` and ends at least 2 rows after it.

    The first passage is 1 row long (aligned: 4) and the corpus ends in passages of 1, 2 and 3 rows (aligned: 4 and
    8), so the first and the last rows of a load are passage edges too."""
    rng = np.random.default_rng(seed)
    step = 4 if aligned else 1
    assert n_rows % step == 0 and period % step == 0
    tail = [4, 8] if aligned else [1, 2, 3]
    fixed = []                                    # (start, lengths) of the designed pieces, in row order
    fixed.append((0, [step]))
    for m in range(1, (n_rows - 1) // period + 1):
        b = m * period
        if kind == "ends":
            fixed.append((b - step, [step, step]))
        elif kind == "straddle":
            a, c = step * rng.integers(-(-2 // step), 40 // step + 1, 2)    # >= 2 rows on either side
            fixed.append((b - int(a), [int(a + c)]))
        else:
            raise ValueError(kind)
    fixed.append((n_rows - sum(tail), tail))
    out, pos = [], 0
    for start, lens in fixed:
        assert start >= pos, "period too short for the designed pieces"
        out += _fill(start - pos, rng, aligned) + lens
        pos = start + sum(lens)
    assert pos == n_rows
    return np.asarray(out, dtype=np.int32)


def offsets(doclens) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(np.asarray(doclens, dtype=np.int64))])


def design_rows(n: int, seed: int, negative: bool = True) -> torch.Tensor:
    """bf16 ``[n, 128]`` unit rows; ``negative``: every row has ``x0 >= 0.5``, so the query row ``-e0`` has a negative
    product with every stored row and a padding row of zeros (or of another passage's token) changes its MaxSim."""
    g = torch.Generator().manual_seed(seed)
    out = torch.empty((n, DIM), dtype=torch.bfloat16)
    for r0 in range(0, n, 1 << 18):          # in blocks: a few million rows stay within a few GB of host memory
        m = min(n, r0 + (1 << 18)) - r0
        x = torch.randn((m, DIM), generator=g)
        x = x / x.norm(dim=1, keepdim=True)
        if negative:
            x0 = 0.5 + 0.5 * torch.rand(m, generator=g)
            rest = x[:, 1:]
            rest = rest / rest.norm(dim=1, keepdim=True) * (1 - x0 * x0).sqrt()[:, None]
            x = torch.cat([x0[:, None], rest], dim=1)
        out[r0:r0 + m] = x
    return out


def probe_queries() -> torch.Tensor:
    """``[2, 4, 128]``: query 0 is four rows ``-e0`` (every product with a ``design_rows`` row is below -0.5), query
    1 four random unit rows."""
    g = torch.Generator().manual_seed(7)
    q = torch.zeros((2, 4, DIM))
    q[0, :, 0] = -1.0
    r = torch.randn((4, DIM), generator=g)
    q[1] = r / r.norm(dim=1, keepdim=True)
    return q.to(torch.bfloat16).float()


# ---- the staging sizes, from the CUDA source -------------------------------------------------------------------------
def load_constants() -> dict:
    """``buf_rows``: the streamed builder's staging buffer (``kBufRows``); ``host_chunk_rows``: the host-source pack
    chunk; ``decode_blocks_per_sm`` / ``decode_threads``: the decode grid cap, as they are written in
    csrc/flmr_maxsim.cu."""
    src = open(CU_PATH).read()
    kdim = int(re.search(r"constexpr int kDim = (\d+);",
                         open(os.path.join(os.path.dirname(CU_PATH), "flmr_scan_kernel.cuh")).read()).group(1))
    m = re.search(r"kBufRows = \((\d+)ll << (\d+)\) / \(kDim \* 2\);", src)
    buf_rows = (int(m.group(1)) << int(m.group(2))) // (kdim * 2)
    m = re.search(r"const int64_t chunk_rows = std::min<int64_t>\(soff\[n_passages\], \((\d+)ll << (\d+)\) / "
                  r"\(kDim \* 2\)\);", src)
    host_chunk = (int(m.group(1)) << int(m.group(2))) // (kdim * 2)
    dec = src[src.index("int plaid_decode("):]
    dec = dec[:dec.index("\n}\n")]
    threads = int(re.search(r"const int threads = (\d+);", dec).group(1))
    per_sm = int(re.search(r"static_cast<int64_t>\(sms\) \* (\d+)\)", dec).group(1))
    assert "(n_tokens * 32 + threads - 1) / threads" in dec     # one warp per token
    return {"dim": kdim, "buf_rows": buf_rows, "host_chunk_rows": host_chunk, "decode_threads": threads,
            "decode_blocks_per_sm": per_sm}


def decode_stride(sms: int) -> int:
    """Tokens one pass of the decode grid covers: one warp per token, ``sms * blocks_per_sm`` blocks."""
    k = load_constants()
    return sms * k["decode_blocks_per_sm"] * k["decode_threads"] // 32
