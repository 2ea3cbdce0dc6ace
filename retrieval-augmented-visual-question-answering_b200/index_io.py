"""Flat index on disk: the format that replaces the reference's PLAID index directory
(``centroids.pt`` / ``*.codes.pt`` / ``*.residuals.pt`` / ``ivf.pid.pt`` ..., SURVEY.md Appendix C;
written by third_party/ColBERT/colbert/indexing/collection_indexer.py + index_saver.py).

A flat index is simply what the scan kernel streams, in one piece or in chunks of passages
(the reference also writes per-chunk files, index_saver.py:75-90):

    metadata.json          {"format": "flmr-flat-v1", "n_passages", "n_tokens", "dim",
                            "dtype": "bfloat16", "num_chunks": C}            (C = 0: single file)
    single file layout     doclens.npy (int32 [n_passages]) + tokens.bf16 (raw bf16 [n_tokens, dim])
    chunked layout         doclens.<c>.npy + tokens.<c>.bf16 + <c>.metadata.json
                           {"passage_offset", "num_passages", "num_embeddings"}   for c < C

An index whose corpus lost passages after it was built (``IndexUpdater.remove``) is written as "flmr-flat-v2": the
same files plus ``deleted.npy`` (int64, the sorted ids of the deleted passages, which keep their rows and ids).
Readers of v1 refuse a v2 index instead of bringing the deleted passages back; v2 is written only when there are
deletions.

An index of fp16 tokens (``save_flat_index(..., dtype="float16")``, ``Indexer(..., storage="fp16")``: the precision the
reference's encoder and codec produce) is "flmr-flat-f16-v1" (with deletions "flmr-flat-f16-v2"), "dtype": "float16",
and its token files are ``tokens.f16`` / ``tokens.<c>.f16``.  A reader of bf16 indexes only refuses it (unknown format,
no ``.bf16`` files) instead of reading fp16 bits as bf16.
"""
from __future__ import annotations

import json
import os
import shutil
from typing import Optional, Tuple

import numpy as np
import torch

FORMAT = "flmr-flat-v1"
FORMAT_V2 = "flmr-flat-v2"        # FORMAT + deleted.npy
FORMAT_F16 = "flmr-flat-f16-v1"   # FORMAT with fp16 tokens
FORMAT_F16_V2 = "flmr-flat-f16-v2"
FORMATS = (FORMAT, FORMAT_V2, FORMAT_F16, FORMAT_F16_V2)
# token dtype of an index -> (torch dtype, token file suffix, format without / with deletions)
DTYPES = {"bfloat16": (torch.bfloat16, "bf16", FORMAT, FORMAT_V2),
          "float16": (torch.float16, "f16", FORMAT_F16, FORMAT_F16_V2)}


def _dtype_info(dtype: str):
    if dtype not in DTYPES:
        raise ValueError("dtype must be one of %s, got %r" % (tuple(DTYPES), dtype))
    return DTYPES[dtype]


def index_dtype(meta: dict) -> str:
    """Token dtype of a flat index ("bfloat16" or "float16") from its metadata."""
    return "float16" if meta["format"] in (FORMAT_F16, FORMAT_F16_V2) else "bfloat16"


def read_metadata(path: str) -> dict:
    """metadata.json of a flat index of either format version."""
    with open(os.path.join(path, "metadata.json")) as f:
        meta = json.load(f)
    if meta.get("format") not in FORMATS:
        raise ValueError("%s is not a %s index" % (path, " / ".join(FORMATS)))
    return meta


def read_deleted(path: str) -> np.ndarray:
    """Sorted global ids of the passages deleted from the index at ``path`` (empty for a v1 index)."""
    if read_metadata(path)["format"] not in (FORMAT_V2, FORMAT_F16_V2):
        return np.empty(0, dtype=np.int64)
    return np.load(os.path.join(path, "deleted.npy")).astype(np.int64)


def deleted_in_range(deleted: np.ndarray, p0: int, p1: int) -> np.ndarray:
    """The deleted ids that fall in the passage shard ``[p0, p1)``."""
    deleted = np.asarray(deleted, dtype=np.int64)
    return deleted[(deleted >= p0) & (deleted < p1)]


def _write_tokens(path: str, tokens: torch.Tensor, dtype: str = "bfloat16") -> None:
    tokens = tokens.detach().to("cpu", _dtype_info(dtype)[0]).contiguous()
    tmp = path + ".tmp"
    tokens.view(torch.int16).numpy().tofile(tmp)
    os.replace(tmp, path)          # a chunk either exists completely or not at all (resume safety)


def save_flat_index(path: str, tokens: torch.Tensor, doclens, dtype: str = "bfloat16") -> str:
    """A single-file flat index of ``tokens`` stored as ``dtype`` ("bfloat16", or "float16": converted with torch's
    ``.half()``, values beyond +-65504 becoming +-inf as in the reference)."""
    _, sfx, fmt, _ = _dtype_info(dtype)
    os.makedirs(path, exist_ok=True)
    doclens = np.ascontiguousarray(np.asarray(doclens), dtype=np.int32)
    if tokens.dim() != 2 or int(doclens.sum()) != tokens.size(0):
        raise ValueError("tokens must be [sum(doclens), dim]")
    _write_tokens(os.path.join(path, "tokens." + sfx), tokens, dtype)
    np.save(os.path.join(path, "doclens.npy"), doclens)
    with open(os.path.join(path, "metadata.json"), "w") as f:
        json.dump({"format": fmt, "n_passages": int(doclens.shape[0]), "n_tokens": int(tokens.size(0)),
                   "dim": int(tokens.size(1)), "dtype": dtype, "num_chunks": 0}, f)
    return path


def save_flat_chunk(path: str, chunk_idx: int, passage_offset: int, tokens: torch.Tensor, doclens,
                    dtype: str = "bfloat16") -> None:
    """One chunk of a chunked flat index (cf. IndexSaver._write_chunk_to_disk, index_saver.py:75-90), its tokens
    stored as ``dtype``.  The chunk's metadata file is written LAST: its presence marks the chunk complete."""
    sfx = _dtype_info(dtype)[1]
    os.makedirs(path, exist_ok=True)
    doclens = np.ascontiguousarray(np.asarray(doclens), dtype=np.int32)
    if tokens.dim() != 2 or int(doclens.sum()) != tokens.size(0):
        raise ValueError("tokens must be [sum(doclens), dim]")
    _write_tokens(os.path.join(path, "tokens.%d.%s" % (chunk_idx, sfx)), tokens, dtype)
    np.save(os.path.join(path, "doclens.%d.npy" % chunk_idx), doclens)
    meta = {"passage_offset": int(passage_offset), "num_passages": int(doclens.shape[0]),
            "num_embeddings": int(tokens.size(0)), "dim": int(tokens.size(1))}
    tmp = os.path.join(path, "%d.metadata.json.tmp" % chunk_idx)
    with open(tmp, "w") as f:
        json.dump(meta, f)
    os.replace(tmp, os.path.join(path, "%d.metadata.json" % chunk_idx))


def chunk_exists(path: str, chunk_idx: int, dtype: str = "bfloat16") -> bool:
    """cf. IndexSaver.check_chunk_exists (index_saver.py:30-50)."""
    return all(os.path.exists(os.path.join(path, n % chunk_idx))
               for n in ("%d.metadata.json", "doclens.%d.npy", "tokens.%d." + _dtype_info(dtype)[1]))


def finalize_chunked_index(path: str, num_chunks: int, fmt: str = FORMAT) -> dict:
    """Check the chunks tile the passage range and write the index-level metadata.json
    (cf. CollectionIndexer.finalize, collection_indexer.py:341-444, minus codec/IVF)."""
    offset = n_tokens = 0
    dim = None
    for c in range(num_chunks):
        with open(os.path.join(path, "%d.metadata.json" % c)) as f:
            m = json.load(f)
        if m["passage_offset"] != offset:
            raise ValueError("chunk %d starts at passage %d, expected %d" % (c, m["passage_offset"], offset))
        offset += m["num_passages"]
        n_tokens += m["num_embeddings"]
        dim = m["dim"] if dim is None else dim
    meta = {"format": fmt, "n_passages": offset, "n_tokens": n_tokens, "dim": dim,
            "dtype": index_dtype({"format": fmt}), "num_chunks": num_chunks}
    tmp = os.path.join(path, "metadata.json.tmp")
    with open(tmp, "w") as f:
        json.dump(meta, f)
    os.replace(tmp, os.path.join(path, "metadata.json"))
    return meta


def persist_updates(path: str, new_tokens: Optional[torch.Tensor], new_doclens, deleted,
                    chunksize: int = 25_000) -> dict:
    """Bring the flat index at ``path`` up to date with a corpus that was appended to and / or lost passages:
    ``new_tokens [sum(new_doclens), dim]`` are the passages behind the ``n_passages`` the index holds (may be empty),
    ``deleted`` every deleted id.  Appended passages become new chunks of at most ``chunksize`` passages; a
    single-file index is first turned into chunk 0 (its files are linked under the chunk names and the old names
    removed only after the new metadata.json is in place).  ``deleted.npy`` is written when there are deletions,
    and metadata.json last, as "flmr-flat-v2" when there are deletions and "flmr-flat-v1" otherwise."""
    meta = read_metadata(path)
    dtype = index_dtype(meta)
    _, sfx, fmt_plain, fmt_deleted = DTYPES[dtype]
    n_old = int(meta["n_passages"])
    num_chunks = int(meta.get("num_chunks", 0))
    new_doclens = np.ascontiguousarray(np.asarray(new_doclens if new_doclens is not None else [], dtype=np.int32))
    n_new = int(new_doclens.shape[0])
    deleted = np.unique(np.asarray(deleted if deleted is not None else [], dtype=np.int64))
    if deleted.size and (deleted[0] < 0 or deleted[-1] >= n_old + n_new):
        raise ValueError("deleted ids must lie in [0, %d)" % (n_old + n_new))
    stale = []
    if n_new:
        if new_tokens is None or new_tokens.dim() != 2 or int(new_doclens.sum()) != new_tokens.size(0):
            raise ValueError("new_tokens must be [sum(new_doclens), dim]")
        if num_chunks == 0:                                  # single file -> chunk 0
            for old, new in (("tokens." + sfx, "tokens.0." + sfx), ("doclens.npy", "doclens.0.npy")):
                src, dst = os.path.join(path, old), os.path.join(path, new)
                if os.path.exists(dst):
                    os.remove(dst)
                try:
                    os.link(src, dst)
                except OSError:
                    shutil.copyfile(src, dst)
                stale.append(src)
            m0 = {"passage_offset": 0, "num_passages": n_old, "num_embeddings": int(meta["n_tokens"]),
                  "dim": int(meta["dim"])}
            with open(os.path.join(path, "0.metadata.json"), "w") as f:
                json.dump(m0, f)
            num_chunks = 1
        off = np.concatenate([[0], np.cumsum(new_doclens, dtype=np.int64)])
        for a in range(0, n_new, chunksize):
            b = min(n_new, a + chunksize)
            save_flat_chunk(path, num_chunks, n_old + a, new_tokens[int(off[a]):int(off[b])], new_doclens[a:b], dtype)
            num_chunks += 1
    fmt = fmt_deleted if deleted.size else fmt_plain
    dpath = os.path.join(path, "deleted.npy")
    if deleted.size:
        with open(dpath + ".tmp", "wb") as f:
            np.save(f, deleted)
        os.replace(dpath + ".tmp", dpath)
    if num_chunks:
        meta = finalize_chunked_index(path, num_chunks, fmt)
    else:
        meta = dict(meta, format=fmt)
        tmp = os.path.join(path, "metadata.json.tmp")
        with open(tmp, "w") as f:
            json.dump(meta, f)
        os.replace(tmp, os.path.join(path, "metadata.json"))
    for f in stale:
        os.remove(f)
    if not deleted.size and os.path.exists(dpath):
        os.remove(dpath)
    return meta


def index_token_files(path: str):
    """(doclens of the whole index int32 [n_passages], [(token file, first passage, passages, rows), ...]) —
    what a streaming loader needs to pick the byte ranges of a passage shard without reading any token."""
    meta = read_metadata(path)
    sfx = DTYPES[index_dtype(meta)][1]
    if meta.get("num_chunks", 0) == 0:
        doclens = np.load(os.path.join(path, "doclens.npy")).astype(np.int32)
        return doclens, [(os.path.join(path, "tokens." + sfx), 0, len(doclens), int(doclens.sum()))]
    dls, files, offset = [], [], 0
    for c in range(meta["num_chunks"]):
        dl = np.load(os.path.join(path, "doclens.%d.npy" % c)).astype(np.int32)
        files.append((os.path.join(path, "tokens.%d.%s" % (c, sfx)), offset, len(dl), int(dl.sum())))
        dls.append(dl)
        offset += len(dl)
    return np.concatenate(dls), files


def _read_tokens(fname: str, n_rows: int, dim: int, row0: int = 0, row1: Optional[int] = None,
                 dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    row1 = n_rows if row1 is None else row1
    mm = np.memmap(fname, dtype=np.int16, mode="r", shape=(n_rows, dim))
    return torch.from_numpy(np.array(mm[row0:row1], copy=True)).view(dtype)


def load_flat_index(path: str, passage_range: Optional[Tuple[int, int]] = None
                    ) -> Tuple[torch.Tensor, np.ndarray, dict]:
    """Returns (tokens [n_tok, dim] on CPU in the index's dtype — bf16, or fp16 for an "flmr-flat-f16" index —,
    doclens int32, metadata) of the whole index or of the passages ``[p0, p1)`` only (a GPU's shard, SURVEY.md 8e) —
    only the chunks that overlap are read.  Deleted passages of a v2 index are included (their ids stay valid);
    ``read_deleted`` lists them."""
    meta = read_metadata(path)
    dim = meta["dim"]
    tdtype, sfx = DTYPES[index_dtype(meta)][:2]
    p0, p1 = passage_range if passage_range is not None else (0, meta["n_passages"])
    if not 0 <= p0 <= p1 <= meta["n_passages"]:
        raise ValueError("passage_range %s outside [0, %d]" % (passage_range, meta["n_passages"]))
    if meta.get("num_chunks", 0) == 0:
        doclens = np.load(os.path.join(path, "doclens.npy"))
        off = np.concatenate([[0], np.cumsum(doclens, dtype=np.int64)])
        tokens = _read_tokens(os.path.join(path, "tokens." + sfx), meta["n_tokens"], dim, int(off[p0]), int(off[p1]),
                              tdtype)
        return tokens, doclens[p0:p1], meta
    toks, dls = [], []
    for c in range(meta["num_chunks"]):
        with open(os.path.join(path, "%d.metadata.json" % c)) as f:
            m = json.load(f)
        c0, c1 = m["passage_offset"], m["passage_offset"] + m["num_passages"]
        if c1 <= p0 or c0 >= p1:
            continue
        doclens = np.load(os.path.join(path, "doclens.%d.npy" % c))
        off = np.concatenate([[0], np.cumsum(doclens, dtype=np.int64)])
        a, b = max(p0, c0) - c0, min(p1, c1) - c0
        toks.append(_read_tokens(os.path.join(path, "tokens.%d.%s" % (c, sfx)), m["num_embeddings"], dim,
                                 int(off[a]), int(off[b]), tdtype))
        dls.append(doclens[a:b])
    tokens = torch.cat(toks) if toks else torch.empty((0, dim), dtype=tdtype)
    doclens = np.concatenate(dls) if dls else np.empty(0, dtype=np.int32)
    return tokens, doclens.astype(np.int32), meta
