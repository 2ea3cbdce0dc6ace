"""Reader for the reference's PLAID index directories (SURVEY.md Appendix C; written by
third_party/ColBERT/colbert/indexing/collection_indexer.py + index_saver.py + codecs/residual.py)
and GPU decode into the flat bf16 store the scan kernel streams (SURVEY.md 8f-3), so a user of the
reference can switch without re-encoding the collection.

Only what the exhaustive scan needs is read: ``metadata.json`` (nbits, dim, num_chunks),
``centroids.pt``, ``buckets.pt``, ``<c>.codes.pt``, ``<c>.residuals.pt``, ``doclens.<c>.json``.
The IVF (``ivf.pid.pt``) and ``avg_residual.pt`` only serve PLAID's candidate generation / pruning.
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
