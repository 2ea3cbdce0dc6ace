"""TEST INFRASTRUCTURE: a numpy restatement of ``flmr_plaid_encode`` (include/flmr_maxsim.h), the inverse of
``oracle.maxsim_oracle.plaid_decode`` with ``normalize=False``:

    code[t]   = argmax_c <x_t, C_c>                    (float64 scores of the fp16 values, the lowest c on ties)
    r_t       = fp16(float32(x_t) - float32(C_code))   per dim
    bucket    = #{j : cutoffs[j] < float32(r_t)}       (torch.bucketize, right=False)
    residuals = bit j of dim d's bucket at position d * nbits + j of the row's bit string, np.packbits (MSB first)

``encode_torch`` has the signature of ``plaid.encode`` so that a test can substitute it for the kernel and drive the
Indexer's PLAID build on a machine without a GPU (the tests/oracle_backend.py pattern).
"""
from __future__ import annotations

import numpy as np
import torch


def assign(x, centroids) -> np.ndarray:
    """Nearest-centroid codes of fp16-valued rows, float64 scores, the lowest index on exact ties."""
    x = np.asarray(x, dtype=np.float64)
    c = np.asarray(centroids, dtype=np.float64)
    codes = np.empty(x.shape[0], dtype=np.int32)
    for a in range(0, x.shape[0], 4096):
        codes[a:a + 4096] = np.argmax(x[a:a + 4096] @ c.T, axis=1)
    return codes


def residual_bytes(x, centroids, codes, cutoffs, nbits: int) -> np.ndarray:
    """The packed residual rows ``[n, 16 nbits]`` of fp16-valued rows given their codes."""
    x32 = np.asarray(x, dtype=np.float16).astype(np.float32)
    c32 = np.asarray(centroids, dtype=np.float16).astype(np.float32)
    r = (x32 - c32[np.asarray(codes, dtype=np.int64)]).astype(np.float16).astype(np.float32)
    return pack_buckets(np.searchsorted(np.asarray(cutoffs, dtype=np.float32), r, side="left"), nbits)


def pack_buckets(buckets, nbits: int) -> np.ndarray:
    """ResidualCodec.binarize's packing of bucket indices ``[n, 128]``."""
    buckets = np.asarray(buckets, dtype=np.uint8)
    bits = (buckets[..., None] >> np.arange(nbits, dtype=np.uint8)) & 1          # [n, 128, nbits], bit j last
    return np.packbits(bits.reshape(buckets.shape[0], -1), axis=1)


def encode(x, centroids, cutoffs=None, nbits: int = 2):
    codes = assign(x, centroids)
    res = None if cutoffs is None else residual_bytes(x, centroids, codes, cutoffs, nbits)
    return codes, res


def encode_torch(x, centroids, cutoffs=None, nbits: int = 2, return_best: bool = False):
    """``plaid.encode`` computed by the restatement, on CPU tensors."""
    assert x.dtype == torch.float16 and centroids.dtype == torch.float16
    xn, cn = x.cpu().numpy(), centroids.cpu().numpy()
    codes, res = encode(xn, cn, None if cutoffs is None else cutoffs.cpu().float().numpy(), nbits)
    out = (torch.from_numpy(codes), None if res is None else torch.from_numpy(res))
    if return_best:
        best = (xn.astype(np.float64) * cn.astype(np.float64)[codes]).sum(1).astype(np.float32)
        out = out + (torch.from_numpy(best),)
    return out


def straddle_rows(x, centroids, codes, cutoffs) -> np.ndarray:
    """Rows where the reference's CPU compress (an fp32 residual, not rounded to fp16) and the fp16-rounded residual
    fall on different sides of a cutoff: the only rows whose residual bytes may differ between the two."""
    x32 = np.asarray(x, dtype=np.float32)
    c32 = np.asarray(centroids, dtype=np.float32)[np.asarray(codes, dtype=np.int64)]
    r32 = x32 - c32
    r16 = r32.astype(np.float16).astype(np.float32)
    cut = np.asarray(cutoffs, dtype=np.float32)
    return (np.searchsorted(cut, r32, side="left") != np.searchsorted(cut, r16, side="left")).any(axis=1)


def lloyd_float64(points, init, niters: int, eps: float = 1.0 / 1024):
    """Float64 Lloyd iterations from the centroids ``init``: assignment with the centroids rounded to fp16 (as the
    kernel sees them), means in float64 rounded once to float32, and an empty cluster split off the largest one
    (the lowest index among equals), scaled by (1 +- eps) on alternating dims."""
    x = np.asarray(points, dtype=np.float64)
    C = np.asarray(init, dtype=np.float32).copy()
    K = C.shape[0]
    sign = np.where(np.arange(C.shape[1]) % 2 == 0, 1.0, -1.0).astype(np.float32)
    for _ in range(niters):
        codes = assign(x, C.astype(np.float16))
        counts = np.bincount(codes, minlength=K)
        sums = np.zeros((K, C.shape[1]), dtype=np.float64)
        np.add.at(sums, codes, x)
        live = counts > 0
        C[live] = (sums[live] / counts[live][:, None]).astype(np.float32)
        counts = counts.tolist()
        for ci in [i for i in range(K) if counts[i] == 0]:
            cj = max(range(K), key=lambda c: (counts[c], -c))
            C[ci] = C[cj] * (1 + eps * sign)
            C[cj] = C[cj] * (1 - eps * sign)
            counts[ci] = counts[cj] // 2
            counts[cj] -= counts[ci]
    return C
