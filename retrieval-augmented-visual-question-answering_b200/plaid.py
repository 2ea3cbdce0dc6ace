"""Reader for the reference's PLAID index directories (SURVEY.md Appendix C; written by
third_party/ColBERT/colbert/indexing/collection_indexer.py + index_saver.py + codecs/residual.py)
and GPU decode into the flat bf16 store the scan kernel streams (SURVEY.md 8f-3), so a user of the
reference can switch without re-encoding the collection.

Only what the exhaustive scan needs is read: ``metadata.json`` (nbits, dim, num_chunks),
``centroids.pt``, ``buckets.pt``, ``<c>.codes.pt``, ``<c>.residuals.pt``, ``doclens.<c>.json``.
The IVF (``ivf.pid.pt``) and ``avg_residual.pt`` only serve PLAID's candidate generation / pruning.

The writing side (``indexer.Indexer(index_format="plaid")``) uses ``encode``, ``kmeans``, ``residual_buckets`` and
``build_ivf`` below: k-means assignment, codes and packed residuals come from one wgmma kernel
(``flmr_plaid_encode``); the rest is small torch plumbing on the same device.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from typing import Optional, Tuple

import numpy as np
import torch

from . import _cabi


def read_plaid_metadata(path: str) -> dict:
    with open(os.path.join(path, "metadata.json")) as f:
        meta = json.load(f)
    cfg = meta["config"]
    return {"nbits": int(cfg["nbits"]), "dim": int(cfg["dim"]), "num_chunks": int(meta["num_chunks"]),
            "num_embeddings": int(meta.get("num_embeddings", -1))}


def decode_chunk(codes: torch.Tensor, residuals: torch.Tensor, centroids: torch.Tensor,
                 bucket_weights: torch.Tensor, nbits: int, out: torch.Tensor, normalize: bool = True) -> None:
    """GPU decode of one chunk into ``out`` (bf16 or fp16 ``[n, 128]`` CUDA, may be a slice of the corpus matrix):
    computed in fp32, normalised, rounded once to ``out``'s type."""
    dev = out.device
    codes = codes.to(dev, torch.int32).contiguous()
    residuals = residuals.to(dev, torch.uint8).contiguous()
    n = codes.numel()
    if residuals.shape != (n, _cabi.DIM * nbits // 8) or out.shape != (n, _cabi.DIM) or \
            out.dtype not in (torch.bfloat16, torch.float16):
        raise ValueError("shape mismatch: codes %s residuals %s out %s" % (tuple(codes.shape),
                         tuple(residuals.shape), tuple(out.shape)))
    if not out.is_contiguous():
        raise ValueError("out must be contiguous")
    with torch.cuda.device(dev):
        decode = _cabi.lib().flmr_plaid_decode_fp16 if out.dtype == torch.float16 else _cabi.lib().flmr_plaid_decode
        _cabi.check(decode(
            C.c_void_p(codes.data_ptr()), C.c_void_p(residuals.data_ptr()), n,
            C.c_void_p(centroids.data_ptr()), centroids.size(0), C.c_void_p(bucket_weights.data_ptr()),
            nbits, _cabi.DIM, int(normalize), C.c_void_p(out.data_ptr()), int(dev.index),
            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))


def read_plaid_doclens(path: str, num_chunks: int):
    """Per-chunk passage lengths (``doclens.<c>.json``, index_saver.py:83-85)."""
    out = []
    for c in range(num_chunks):
        with open(os.path.join(path, "doclens.%d.json" % c)) as f:
            out.append(np.asarray(json.load(f), dtype=np.int64))
    return out


def _plaid_pieces(path: str, device, passage_range: Optional[Tuple[int, int]]):
    """What a decode of the passages ``[p0, p1)`` of a PLAID index reads: (device, metadata, centroids and bucket
    weights on the device, pieces ``(chunk, first token row, one-past-last row, doclens slice, chunk rows)``)."""
    if not torch.cuda.is_available():
        raise RuntimeError("PLAID decode runs on the GPU; there is no CPU fallback")
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    meta, centroids, weights, pieces = _plaid_plan(path, passage_range)
    return device, meta, centroids.to(device), weights.to(device), pieces


def _plaid_plan(path: str, passage_range: Optional[Tuple[int, int]]):
    """(metadata, centroids and bucket weights as fp32 CPU tensors, the pieces of ``_plaid_pieces``) of the passages
    ``[p0, p1)`` of a PLAID index."""
    meta = read_plaid_metadata(path)
    if meta["dim"] != _cabi.DIM:
        raise ValueError("dim=%d (only %d is supported)" % (meta["dim"], _cabi.DIM))
    centroids = torch.load(os.path.join(path, "centroids.pt"), map_location="cpu").float().contiguous()
    _cutoffs, weights = torch.load(os.path.join(path, "buckets.pt"), map_location="cpu")
    weights = weights.float().contiguous()
    chunk_doclens = read_plaid_doclens(path, meta["num_chunks"])
    n_total = int(sum(len(d) for d in chunk_doclens))
    p0, p1 = (0, n_total) if passage_range is None else passage_range
    p1 = n_total if p1 is None else p1
    if not 0 <= p0 <= p1 <= n_total:
        raise ValueError("passage_range %s outside [0, %d]" % (passage_range, n_total))
    pieces, c0 = [], 0                       # (chunk, first token row, one-past-last row, doclens slice)
    for c, dl in enumerate(chunk_doclens):
        a, b = max(p0, c0) - c0, min(p1, c0 + len(dl)) - c0
        if a < b:
            off = np.concatenate([[0], np.cumsum(dl)])
            pieces.append((c, int(off[a]), int(off[b]), dl[a:b], int(off[-1])))
        c0 += len(dl)
    return meta, centroids, weights, pieces


def _load_piece(path: str, c: int, n_chunk: int):
    codes = torch.load(os.path.join(path, "%d.codes.pt" % c), map_location="cpu")
    residuals = torch.load(os.path.join(path, "%d.residuals.pt" % c), map_location="cpu")
    if codes.numel() != n_chunk:
        raise ValueError("chunk %d holds %d codes but its doclens sum to %d" % (c, codes.numel(), n_chunk))
    return codes, residuals


def _piece_doclens(pieces) -> np.ndarray:
    doclens = np.concatenate([p[3] for p in pieces]) if pieces else np.empty(0, dtype=np.int64)
    return doclens.astype(np.int32)


def plaid_to_flat(path: str, device=None, passage_range: Optional[Tuple[int, int]] = None,
                  dtype: torch.dtype = torch.bfloat16) -> Tuple[torch.Tensor, np.ndarray]:
    """Decode a PLAID index — all of it, or the passages ``[p0, p1)`` only (one GPU's shard: only the chunks
    that overlap are read) — into (tokens ``[n_tokens, 128]`` of ``dtype``, bf16 or fp16, on the GPU, doclens
    int32)."""
    device, meta, centroids, weights, pieces = _plaid_pieces(path, device, passage_range)
    tokens = torch.empty((sum(p[2] - p[1] for p in pieces), _cabi.DIM), dtype=dtype, device=device)
    row = 0
    for c, r0, r1, _, n_chunk in pieces:
        codes, residuals = _load_piece(path, c, n_chunk)
        decode_chunk(codes[r0:r1], residuals[r0:r1], centroids, weights, meta["nbits"], tokens[row:row + r1 - r0])
        row += r1 - r0
    return tokens, _piece_doclens(pieces)


# token rows one decode step of plaid_to_host_chunks holds on the GPU (32 MiB of bf16 rows)
HOST_DECODE_ROWS = 1 << 17


def plaid_to_host_chunks(path: str, device=None, passage_range: Optional[Tuple[int, int]] = None,
                         dtype: torch.dtype = torch.bfloat16, rows_per_step: int = HOST_DECODE_ROWS):
    """The decode of ``plaid_to_flat`` for a corpus kept in host memory: (device, doclens int32, an iterator of host
    token tensors ``[rows, 128]`` of ``dtype`` that concatenate to ``plaid_to_flat``'s tokens).  Each step decodes at
    most ``rows_per_step`` rows on the GPU, with the same kernels, and copies them down; the GPU never holds more."""
    device, meta, centroids, weights, pieces = _plaid_pieces(path, device, passage_range)

    def steps():
        buf = torch.empty((min(rows_per_step, max((p[2] - p[1] for p in pieces), default=1)), _cabi.DIM),
                          dtype=dtype, device=device)
        for c, r0, r1, _, n_chunk in pieces:
            codes, residuals = _load_piece(path, c, n_chunk)
            for a in range(r0, r1, rows_per_step):
                b = min(r1, a + rows_per_step)
                out = buf[:b - a]
                decode_chunk(codes[a:b], residuals[a:b], centroids, weights, meta["nbits"], out)
                yield out.cpu()
    return device, _piece_doclens(pieces), steps()


def plaid_compressed_chunks(path: str, passage_range: Optional[Tuple[int, int]] = None):
    """The compressed form of the passages ``[p0, p1)`` of a PLAID index, read on the host with nothing decoded:
    (nbits, centroids fp32 ``[K, 128]``, bucket weights fp32 ``[2^nbits]``, doclens int32, an iterator of
    (codes int32 ``[n]``, residuals uint8 ``[n, 16 nbits]``) CPU tensors, one per chunk the range overlaps, that
    concatenate to the range's packed token rows)."""
    meta, centroids, weights, pieces = _plaid_plan(path, passage_range)
    nbits = meta["nbits"]

    def steps():
        for c, r0, r1, _, n_chunk in pieces:
            codes, residuals = _load_piece(path, c, n_chunk)
            codes = codes[r0:r1].to(torch.int32).contiguous()
            residuals = residuals[r0:r1].to(torch.uint8).contiguous()
            if residuals.shape != (r1 - r0, _cabi.DIM * nbits // 8):
                raise ValueError("chunk %d: residuals of shape %s for nbits=%d" % (c, tuple(residuals.shape), nbits))
            yield codes, residuals
    return nbits, centroids, weights, _piece_doclens(pieces), steps()


# ---------------------------------------------------------------------------------------------------------------------
# writing a PLAID index
# ---------------------------------------------------------------------------------------------------------------------
def encode(x: torch.Tensor, centroids: torch.Tensor, cutoffs: Optional[torch.Tensor] = None, nbits: int = 2,
           return_best: bool = False):
    """``flmr_plaid_encode``: (codes int32 ``[n]``, packed residuals uint8 ``[n, 16 nbits]`` or None when ``cutoffs``
    is None, [the winning scores fp32 ``[n]`` with ``return_best``]) of fp16 token rows ``x [n, 128]`` against fp16
    ``centroids [K, 128]``, both on the same GPU.  ``codes[t]`` is the centroid of the largest fp32-accumulated dot
    product, the lowest index on exact ties; the residual bytes are what ``ResidualCodec.binarize`` writes for
    ``fp16(x - C[code])`` bucketed against ``cutoffs`` (non-decreasing fp32 ``[2^nbits - 1]``).  Asynchronous on the
    current stream."""
    if not (x.is_cuda and centroids.is_cuda):
        raise ValueError("plaid.encode runs on the GPU: x and centroids must be CUDA tensors")
    if x.dtype != torch.float16 or centroids.dtype != torch.float16:
        raise ValueError("plaid.encode takes fp16 rows and centroids, got %s and %s" % (x.dtype, centroids.dtype))
    if x.dim() != 2 or x.size(1) != _cabi.DIM or centroids.dim() != 2 or centroids.size(1) != _cabi.DIM:
        raise ValueError("shape mismatch: x %s centroids %s" % (tuple(x.shape), tuple(centroids.shape)))
    dev = x.device
    x, centroids = x.contiguous(), centroids.to(dev).contiguous()
    n = x.size(0)
    codes = torch.empty(n, dtype=torch.int32, device=dev)
    residuals = None
    if cutoffs is not None:
        cutoffs = cutoffs.to(dev, torch.float32).contiguous()
        if cutoffs.numel() != (1 << nbits) - 1:
            raise ValueError("%d cutoffs for nbits=%d" % (cutoffs.numel(), nbits))
        residuals = torch.empty((n, _cabi.DIM * nbits // 8), dtype=torch.uint8, device=dev)
    best = torch.empty(n, dtype=torch.float32, device=dev) if return_best else None
    ptr = (lambda t: C.c_void_p(t.data_ptr() if t is not None else None))
    with torch.cuda.device(dev):
        _cabi.check(_cabi.lib().flmr_plaid_encode(
            ptr(x), n, ptr(centroids), centroids.size(0), ptr(cutoffs), nbits, ptr(codes), ptr(residuals), ptr(best),
            int(dev.index), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return (codes, residuals, best) if return_best else (codes, residuals)


def _assign(x: torch.Tensor, centroids: torch.Tensor) -> torch.Tensor:
    """Nearest-centroid codes (int64) through ``encode``'s assignment-only mode, looked up at call time so that a
    test can substitute ``encode``."""
    return encode(x, centroids)[0].long()


# points per centroid k-means trains on at most (faiss's max_points_per_centroid)
KMEANS_MAX_POINTS_PER_CENTROID = 256


def _centroid_means(points: torch.Tensor, codes: torch.Tensor, K: int, rows_per_step: int = 1 << 20):
    """(per-centroid means fp32 ``[K, 128]``, counts int64 ``[K]``), the same bits on every run: the fp16 points are
    summed as fixed-point int64 (``round(v * 2^shift)``, exact for unit-norm fp16 rows, whose values are multiples of
    2^-24), so the order of the additions cannot change the sums; each mean is rounded once from float64."""
    dev = points.device
    counts = torch.bincount(codes, minlength=K)
    amax = float(points.abs().max()) if points.numel() else 0.0
    # keep |sum| < 2^62 for any assignment of all points to one centroid
    shift = 24 if amax == 0.0 else min(24, int(np.floor(62 - np.log2(max(1.0, points.size(0) * amax)))))
    sums = torch.zeros((K, points.size(1)), dtype=torch.int64, device=dev)
    for a in range(0, points.size(0), rows_per_step):
        q = torch.round(points[a:a + rows_per_step].double() * (2.0 ** shift)).to(torch.int64)
        sums.index_add_(0, codes[a:a + rows_per_step], q)
    means = (sums.double() / (2.0 ** shift)) / counts.clamp(min=1).double()[:, None]
    return means.float(), counts


def _split_empty(C_: torch.Tensor, counts: torch.Tensor, eps: float = 1.0 / 1024) -> None:
    """faiss's split of empty clusters (Clustering.cpp split_clusters), made deterministic: each empty centroid, in
    index order, takes a copy of the currently largest cluster's centroid (the lowest index among equals), the copy
    scaled by (1 + eps) on even dims and (1 - eps) on odd ones and the original the other way, and half its points."""
    empty = (counts == 0).nonzero().flatten().tolist()
    if not empty:
        return
    sign = torch.ones(C_.size(1), dtype=C_.dtype, device=C_.device)
    sign[1::2] = -1.0
    counts_h = counts.tolist()
    for ci in empty:
        cj = max(range(len(counts_h)), key=lambda c: (counts_h[c], -c))
        C_[ci] = C_[cj] * (1 + eps * sign)
        C_[cj] = C_[cj] * (1 - eps * sign)
        counts_h[ci] = counts_h[cj] // 2
        counts_h[cj] -= counts_h[ci]


def kmeans(sample: torch.Tensor, K: int, niters: int = 4, seed: int = 123, return_raw: bool = False):
    """Seeded Lloyd k-means of fp16 rows ``sample [N, 128]`` (the reference trains faiss.Kmeans here,
    collection_indexer.py:258-288; this is NOT faiss, so its centroids differ from the reference's):

    * at most ``256 K`` points (faiss's ``max_points_per_centroid``), a seeded random subset;
    * initial centroids: K distinct sample rows chosen by a ``torch.Generator`` seeded with ``seed``;
    * each iteration assigns every point to its nearest centroid with fp16 operands and fp32 accumulation (the
      assignment-only mode of ``encode``), then sets each centroid to the fp32 mean of its points
      (``_centroid_means``: bitwise the same on every run), and an empty cluster takes a split of the largest one;
    * the result is L2-normalised and cast to fp16, as ``_train_kmeans`` does.

    Returns the fp16 centroids ``[K, 128]`` (with ``return_raw``: also the fp32 centroids before normalisation)."""
    N = sample.size(0)
    if not 1 <= K <= N:
        raise ValueError("k-means of %d points into K=%d clusters" % (N, K))
    g = torch.Generator().manual_seed(int(seed))
    points = sample
    if N > KMEANS_MAX_POINTS_PER_CENTROID * K:
        keep = torch.randperm(N, generator=g)[:KMEANS_MAX_POINTS_PER_CENTROID * K]
        points = sample[keep.to(sample.device)]
    init = torch.randperm(points.size(0), generator=g)[:K]
    C_ = points[init.to(points.device)].float()
    for _ in range(int(niters)):
        codes = _assign(points, C_.half())
        means, counts = _centroid_means(points, codes, K)
        C_ = torch.where((counts > 0)[:, None], means, C_)
        _split_empty(C_, counts)
    out = torch.nn.functional.normalize(C_, dim=-1).half()
    return (out, C_) if return_raw else out


def residual_buckets(centroids: torch.Tensor, heldout: torch.Tensor, nbits: int):
    """(bucket cutoffs fp32 ``[2^nbits - 1]``, bucket weights fp32 ``[2^nbits]``, average residual, a 0-d fp16 tensor)
    from the held-out rows, as CollectionIndexer._compute_avg_residual computes them on the GPU
    (collection_indexer.py:290-314): fp16 residuals to each row's nearest centroid, their quantiles."""
    codes = _assign(heldout, centroids)
    res = heldout - centroids[codes]
    avg_residual = torch.abs(res).mean(dim=0).cpu().mean()
    num_options = 2 ** nbits
    quantiles = torch.arange(0, num_options, device=res.device) * (1 / num_options)
    cutoffs = res.float().quantile(quantiles[1:])
    weights = res.float().quantile(quantiles + (0.5 / num_options))
    return cutoffs.cpu(), weights.cpu(), avg_residual


def build_ivf(codes: torch.Tensor, doclens, K: int):
    """``ivf.pid.pt``'s (ivf int32, ivf_lengths int64) as optimize_ivf builds it (indexing/utils.py:8-48): for each
    centroid in order, the sorted distinct pids of the tokens coded to it.  ``codes`` are every token's codes in
    index order; the sort runs on their device."""
    dev = codes.device
    doclens = torch.as_tensor(np.asarray(doclens, dtype=np.int64), device=dev)
    n_passages = int(doclens.numel())
    pids = torch.repeat_interleave(torch.arange(n_passages, device=dev), doclens)
    keys = torch.unique(codes.long() * n_passages + pids)                       # sorted: by code, then pid
    ivf = (keys % n_passages).to(torch.int32)
    lengths = torch.bincount(keys // n_passages, minlength=K)
    return ivf.cpu(), lengths.cpu()
