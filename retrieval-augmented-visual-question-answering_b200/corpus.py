"""Resident passage-token corpus shard (replaces the PLAID index residency of the reference:
``IndexScorer.__init__`` / ``IndexLoader``, third_party/ColBERT/colbert/search/index_storage.py:21-66,
index_loader.py:13-86).

The reference keeps centroids + residual codes + an IVF and decompresses ~256 survivors per query;
here the whole shard is a flat bf16 ``[sum(doclens), 128]`` matrix in HBM plus ``doclens`` — exactly
the ``(D_packed, D_lengths)`` operand pair of ``colbert_score_packed`` (colbert/modeling/colbert.py:289)
— scanned exhaustively by the fused kernel.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Union

import numpy as np
import torch

from . import _cabi


def _as_doclens(doclens) -> np.ndarray:
    if isinstance(doclens, torch.Tensor):
        doclens = doclens.detach().cpu().numpy()
    arr = np.ascontiguousarray(np.asarray(doclens), dtype=np.int32)
    if arr.ndim != 1:
        raise ValueError("doclens must be 1-D")
    return arr


def _storage_flag(storage: str) -> int:
    if storage not in _cabi.STORAGES:
        raise ValueError("storage must be one of %s, got %r" % (_cabi.STORAGES, storage))
    return {"bf16": 0, "fp8": _cabi.CORPUS_FP8, "fp16": _cabi.CORPUS_FP16}[storage]


def element_dtype(storage: str) -> torch.dtype:
    """The element type of the rows a corpus of ``storage`` takes and gathers, and of the queries it is searched
    with: fp16 for "fp16", bf16 for "bf16" and "fp8" (whose exact rows are bf16)."""
    _storage_flag(storage)
    return torch.float16 if storage == "fp16" else torch.bfloat16


RESIDENCIES = ("device", "host")
DEFAULT_WINDOW_BYTES = 1 << 30


def _check_residency(residency: str, storage: str, window_bytes) -> None:
    """The arguments of a corpus's residency: "device" (its rows in HBM) or "host" (a streamed corpus: its rows in
    pinned host memory, copied through two HBM windows of at most ``window_bytes`` per search)."""
    if residency not in RESIDENCIES:
        raise ValueError("residency must be one of %s, got %r" % (RESIDENCIES, residency))
    if residency == "host":
        if storage == "fp8":
            raise ValueError("residency='host' streams bf16 or fp16 rows; storage='fp8' is held in HBM only")
        if isinstance(window_bytes, bool) or not isinstance(window_bytes, (int, np.integer)) \
                or window_bytes < _cabi.DIM * 2:
            raise ValueError("window_bytes must be an int of at least one row (%d bytes), got %r"
                             % (_cabi.DIM * 2, window_bytes))


def _read_storage(handle) -> str:
    code = C.c_int(0)
    _cabi.check(_cabi.lib().flmr_corpus_storage(handle, C.byref(code), None))
    return _cabi.STORAGES[code.value]


def allow_bitmaps(pid_lists: Sequence, n_passages: int, pid_base: int = 0,
                  device: Optional[Union[str, torch.device]] = None) -> torch.Tensor:
    """Per-query allow bitmaps of a shard for ``maxsim_scores`` / ``maxsim_topk`` / ``NcclExchange.search``: int32
    ``[len(pid_lists), ceil(n_passages / 32)]``, bit ``p & 31`` of word ``p >> 5`` of row b set <=> query b may return
    the shard's local passage ``p`` (global id ``pid_base + p``).

    ``pid_lists[b]`` is a sequence or tensor of GLOBAL ids, or None (the whole shard: an all-ones row).  Ids outside
    ``[pid_base, pid_base + n_passages)`` are dropped, so every rank of a sharded search can pass the same global lists;
    duplicates collapse.  Plain torch, on ``device`` (CPU by default), with one byte of scratch per (query, passage)
    and no host synchronisation on a GPU."""
    dev = torch.device(device) if device is not None else torch.device("cpu")
    n, words, B = int(n_passages), (int(n_passages) + 31) // 32, len(pid_lists)
    lists = [torch.as_tensor(ids if ids is not None else [], dtype=torch.int64).reshape(-1) for ids in pid_lists]
    lens = torch.tensor([x.numel() for x in lists], dtype=torch.int64)
    total = int(lens.sum())
    flat = torch.cat([x.to(dev) for x in lists]) if total else torch.empty(0, dtype=torch.int64, device=dev)
    rows = torch.repeat_interleave(torch.arange(B, device=dev), lens.to(dev), output_size=total)
    local = flat - int(pid_base)
    inside = (local >= 0) & (local < n)
    # one bool per (query, passage); ids outside the shard land in a spare row B, so nothing waits for the device
    dense = torch.zeros((B + 1, words * 32), dtype=torch.bool, device=dev)
    dense[torch.where(inside, rows, B), torch.where(inside, local, 0)] = True
    none_rows = [b for b, ids in enumerate(pid_lists) if ids is None]
    if none_rows:
        dense[torch.tensor(none_rows, device=dev)] = True
    # 8 bools -> one byte (bit q = passage 8 j + q), four little-endian bytes -> one int32 word
    shifts = torch.arange(8, dtype=torch.uint8, device=dev)
    packed = (dense[:B].view(B, words * 4, 8).to(torch.uint8) << shifts).sum(-1, dtype=torch.uint8)
    return packed.view(torch.int32)


class FlatCorpus:
    """One GPU's shard of the passage-token matrix, resident in HBM.

    tokens   : ``[sum(doclens), 128]`` tensor in the storage's element type (``element_dtype``: bf16, or fp16 for
               ``storage="fp16"``; other dtypes are converted once), on CPU or on the target GPU.  A CUDA tensor
               of that type whose doclens are all multiples of 4 is adopted zero-copy (and kept alive by this
               object).
    doclens  : per-passage token counts (>= 1 each).
    pid_base : global id of this shard's first passage (sharded search, SURVEY.md §8e).
    storage  : "bf16" (default) or "fp8": HBM holds the tokens as e4m3 (half the bytes; the scan's scores become
               approximate, ``Searcher`` re-ranks a shortlist exactly) and the library keeps the exact bf16 rows
               in pinned host memory, where ``gather_padded`` reads them.  An fp8 corpus never adopts ``tokens``.
               Or "fp16": HBM holds fp16 tokens (the reference's own precision: ``ColBERT.doc`` returns ``D.half()``)
               and the scan runs fp16 MMAs, at the bytes and layout of bf16.  fp32 / bf16 sources are converted
               with torch's ``.half()`` as the reference does (beyond +-65504 they become +-inf); queries are
               converted to fp16 for the search, and ``gather_padded`` returns fp16 rows.
    residency: "device" (default): the rows live in HBM.  "host": a STREAMED corpus — the rows live in pinned host
               memory and every search copies them through two HBM windows of at most ``window_bytes`` (default
               1 GiB) while it scans them, so the corpus takes no HBM for its rows; its results are bitwise those of
               the same rows held in HBM.  For a shard that does not fit beside what the GPU already holds (a
               validation corpus searched inside a training process), or one larger than the card.  bf16 or fp16
               only; it cannot be appended to or compacted (``FlmrError``), and restricted searches test bitmaps.
    """

    def __init__(self, tokens: torch.Tensor, doclens, device: Optional[Union[int, torch.device]] = None,
                 pid_base: int = 0, adopt: bool = True, storage: str = "bf16", residency: str = "device",
                 window_bytes: int = DEFAULT_WINDOW_BYTES):
        _check_residency(residency, storage, window_bytes)
        if not torch.cuda.is_available():
            raise RuntimeError("FlatCorpus needs a CUDA device: there is no CPU fallback for this path")
        sflag = _storage_flag(storage)
        dtype = element_dtype(storage)
        L = _cabi.lib()
        self.doclens = _as_doclens(doclens)
        if tokens.dim() != 2 or tokens.size(1) != _cabi.DIM:
            raise ValueError("tokens must be [sum(doclens), %d], got %s" % (_cabi.DIM, tuple(tokens.shape)))
        if int(self.doclens.sum()) != tokens.size(0):
            raise ValueError("sum(doclens)=%d != tokens rows=%d" % (int(self.doclens.sum()), tokens.size(0)))
        if device is None:
            device = tokens.device if tokens.is_cuda else torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device) if not isinstance(device, torch.device) else device
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        tokens = tokens.detach()
        if tokens.dtype != dtype:
            tokens = tokens.to(dtype)
        tokens = tokens.contiguous()
        if tokens.is_cuda and tokens.device != device:
            tokens = tokens.to(device)
        # an fp8 corpus keeps its own copies; bf16 and fp16 adopt a CUDA tensor of their element type
        flags = sflag | (_cabi.CORPUS_ADOPT if (adopt and tokens.is_cuda and storage != "fp8") else _cabi.CORPUS_COPY)
        if tokens.is_cuda:
            torch.cuda.current_stream(device).synchronize()  # producer kernels of `tokens` are done
        handle = C.c_void_p()
        if residency == "host":
            _cabi.check(L.flmr_corpus_create_streamed(C.c_void_p(tokens.data_ptr()),
                                                      self.doclens.ctypes.data_as(C.c_void_p),
                                                      int(self.doclens.shape[0]), _cabi.DIM, int(device.index),
                                                      int(pid_base), sflag, int(window_bytes), C.byref(handle)))
        else:
            _cabi.check(L.flmr_corpus_create(C.c_void_p(tokens.data_ptr()),
                                             self.doclens.ctypes.data_as(C.c_void_p),
                                             int(self.doclens.shape[0]), _cabi.DIM, int(device.index),
                                             int(pid_base), flags, C.byref(handle)))
        self._h = handle
        info = _cabi.CorpusInfo()
        _cabi.check(L.flmr_corpus_info(self._h, C.byref(info)))
        self.info = info
        self.storage = _read_storage(self._h)
        self._keepalive = tokens if info.adopted else None
        self._ws = None
        self.pid_base = int(pid_base)
        self.load_stats = None

    @classmethod
    def _from_handle(cls, handle, doclens: np.ndarray, device: torch.device, pid_base: int) -> "FlatCorpus":
        self = cls.__new__(cls)
        self.doclens = doclens
        self.device = device
        self._h = handle
        info = _cabi.CorpusInfo()
        _cabi.check(_cabi.lib().flmr_corpus_info(self._h, C.byref(info)))
        self.info = info
        self.storage = _read_storage(self._h)
        self._keepalive = None
        self._ws = None
        self.pid_base = int(pid_base)
        self.load_stats = None
        return self

    @property
    def residency(self) -> str:
        """"host" for a streamed corpus (rows in pinned host memory), "device" for one whose rows are in HBM."""
        return "host" if self.residency_info()["streamed"] else "device"

    def residency_info(self) -> dict:
        """``{"streamed", "window_bytes", "host_bytes"}`` of ``flmr_corpus_residency``."""
        streamed, window, host = C.c_int(0), C.c_int64(0), C.c_int64(0)
        _cabi.check(_cabi.lib().flmr_corpus_residency(self.handle, C.byref(streamed), C.byref(window), C.byref(host)))
        return {"streamed": bool(streamed.value), "window_bytes": int(window.value), "host_bytes": int(host.value)}

    @property
    def codec_nbits(self) -> int:
        """The PLAID codec's bits per dimension of a PLAID-coded streamed corpus (``from_plaid(..., compressed=True)``),
        0 for any other corpus."""
        nbits = C.c_int(0)
        _cabi.check(_cabi.lib().flmr_corpus_codec(self.handle, C.byref(nbits)))
        return int(nbits.value)

    @property
    def dtype(self) -> torch.dtype:
        """Element type of the rows this corpus takes (``append``) and gathers, and of its queries."""
        return element_dtype(self.storage)

    @classmethod
    def from_index(cls, path: str, device=None, rank: int = 0, world_size: int = 1,
                   storage: Optional[str] = None, residency: str = "device",
                   window_bytes: int = DEFAULT_WINDOW_BYTES) -> "FlatCorpus":
        """Load a flat index (index_io.py) — or, with world_size > 1, only this rank's contiguous,
        token-balanced passage shard of it (SURVEY.md 8e) — into HBM.

        The token files are streamed by the C-level corpus builder: ``pread`` straight into two pinned staging
        buffers (8 reader threads, the fill of one buffer overlaps the DMA of the other) and from there into the
        padded layout — no numpy copy of the shard, no pageable ``cudaMemcpy``.  ``load_stats`` records seconds
        and GB/s (replaces IndexLoader / ResidualEmbeddings.load_chunks, colbert/search/index_loader.py:24-62).
        ``storage="fp8"``: the staged rows fill the bf16 master in pinned host memory, HBM receives e4m3.
        ``storage=None`` (default) keeps the index's own dtype: "fp16" for an fp16 index ("flmr-flat-f16"), "bf16"
        otherwise.  A storage of another element type converts the shard once on its way in (read on the host,
        ``.to()`` the storage's type) instead of streaming the files.
        The deletions an index records (``deleted.npy``, format v2) are applied to the passages of this shard.
        ``residency="host"``: a streamed corpus (see the class); the files are read straight into its pinned host
        matrix, with no device copy."""
        import time
        from .index_io import deleted_in_range, index_dtype, index_token_files, load_flat_index, read_deleted, \
            read_metadata
        from .sharded import shard_ranges
        if storage is not None:
            _check_residency(residency, storage, window_bytes)
        if not torch.cuda.is_available():
            raise RuntimeError("FlatCorpus needs a CUDA device: there is no CPU fallback for this path")
        disk_storage = "fp16" if index_dtype(read_metadata(path)) == "float16" else "bf16"
        storage = disk_storage if storage is None else storage
        flags = _storage_flag(storage)
        _check_residency(residency, storage, window_bytes)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device) if not isinstance(device, torch.device) else device
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        all_doclens, files = index_token_files(path)        # files: [(path, first passage, n passages, n rows)]
        p0, p1 = shard_ranges(all_doclens, world_size)[rank] if world_size > 1 else (0, len(all_doclens))
        if p0 == p1:
            return None          # more ranks than passages: this rank holds nothing (Searcher copes)
        doclens = np.ascontiguousarray(all_doclens[p0:p1], dtype=np.int32)
        if element_dtype(storage) != element_dtype(disk_storage):
            tokens, _, _ = load_flat_index(path, (p0, p1))
            self = cls(tokens, doclens, device=device, pid_base=p0, storage=storage, residency=residency,
                       window_bytes=window_bytes)
            dead = deleted_in_range(read_deleted(path), p0, p1)
            if dead.size:
                self.delete(dead)
            return self
        t0 = time.perf_counter()

        def feed(L, b):
            for fname, f0, fn, _rows in files:
                a, e = max(p0, f0), min(p1, f0 + fn)
                if a >= e:
                    continue
                row_a = int(all_doclens[f0:a].sum())
                rows = int(all_doclens[a:e].sum())
                _cabi.check(L.flmr_corpus_builder_append_file(b, fname.encode(), row_a * _cabi.DIM * 2, rows))

        self, fill_s = cls._build(doclens, device, p0, flags, residency, window_bytes, feed)
        dead = deleted_in_range(read_deleted(path), p0, p1)    # this shard's share of the index's deletions
        if dead.size:
            self.delete(dead)
        dt = time.perf_counter() - t0
        gb = float(doclens.sum()) * _cabi.DIM * 2 / 1e9
        self.load_stats = {"seconds": dt, "gigabytes": gb, "gb_per_s": gb / dt, "host_fill_seconds": fill_s,
                           "rank": rank, "world_size": world_size}
        return self

    @classmethod
    def from_plaid(cls, path: str, device=None, rank: int = 0, world_size: int = 1,
                   storage: str = "bf16", residency: str = "device",
                   window_bytes: int = DEFAULT_WINDOW_BYTES, compressed: bool = False) -> "FlatCorpus":
        """Decode a reference PLAID index directory on the GPU (plaid.py) and keep it resident — with
        world_size > 1 only this rank's contiguous, token-balanced passage shard (SURVEY.md 8e).  ``storage="fp16"``
        decodes straight to fp16 (``flmr_plaid_decode_fp16``), the type the reference's codec decodes to.
        ``residency="host"``: a streamed corpus (see the class), decoded on the GPU in bounded chunks
        (``plaid_to_host_chunks``), each copied down into its pinned host matrix.
        ``residency="host", compressed=True``: a PLAID-coded streamed corpus.  Nothing is decoded at load time: the
        pinned host memory holds each token's centroid code and packed residual (4 + 16 nbits bytes instead of 256),
        and every search copies a window's compressed rows and decodes them on the GPU before scanning them.  Its
        results are bitwise those of the resident ``from_plaid`` corpus of the same storage.  bf16 or fp16 only."""
        from .plaid import plaid_compressed_chunks, plaid_to_flat, plaid_to_host_chunks, read_plaid_doclens, \
            read_plaid_metadata
        from .sharded import shard_ranges
        _storage_flag(storage)
        _check_residency(residency, storage, window_bytes)
        if not isinstance(compressed, bool):
            raise ValueError("compressed must be a bool, got %r" % (compressed,))
        if compressed and residency != "host":
            raise ValueError("compressed=True streams a PLAID index's compressed form and needs residency='host'")
        if residency == "host":
            if world_size == 1:
                p0, p1 = 0, None
            else:
                all_doclens = np.concatenate(read_plaid_doclens(path, read_plaid_metadata(path)["num_chunks"]))
                p0, p1 = shard_ranges(all_doclens, world_size)[rank]
                if p0 == p1:
                    return None
            if compressed:
                if not torch.cuda.is_available():
                    raise RuntimeError("FlatCorpus needs a CUDA device: there is no CPU fallback for this path")
                device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
                if device.index is None:
                    device = torch.device("cuda", torch.cuda.current_device())
                nbits, centroids, weights, doclens, chunks = plaid_compressed_chunks(path, passage_range=(p0, p1))

                def feed_codes(L, b):
                    for codes, residuals in chunks:
                        _cabi.check(L.flmr_corpus_builder_append_plaid(b, C.c_void_p(codes.data_ptr()),
                                                                       C.c_void_p(residuals.data_ptr()),
                                                                       codes.numel()))

                return cls._build(np.ascontiguousarray(doclens, dtype=np.int32), device, p0, _storage_flag(storage),
                                  residency, window_bytes, feed_codes, codec=(nbits, centroids, weights))[0]
            device, doclens, pieces = plaid_to_host_chunks(path, device, passage_range=(p0, p1),
                                                           dtype=element_dtype(storage))

            def feed(L, b):
                for t in pieces:
                    _cabi.check(L.flmr_corpus_builder_append(b, C.c_void_p(t.data_ptr()), t.size(0)))

            return cls._build(np.ascontiguousarray(doclens, dtype=np.int32), device, p0, _storage_flag(storage),
                              residency, window_bytes, feed)[0]
        if world_size == 1:
            tokens, doclens = plaid_to_flat(path, device, dtype=element_dtype(storage))
            return cls(tokens, doclens, device=tokens.device, storage=storage)
        all_doclens = np.concatenate(read_plaid_doclens(path, read_plaid_metadata(path)["num_chunks"]))
        p0, p1 = shard_ranges(all_doclens, world_size)[rank]
        if p0 == p1:
            return None
        tokens, doclens = plaid_to_flat(path, device, passage_range=(p0, p1), dtype=element_dtype(storage))
        return cls(tokens, doclens, device=tokens.device, pid_base=p0, storage=storage)

    @classmethod
    def _build(cls, doclens: np.ndarray, device: torch.device, pid_base: int, flags: int, residency: str,
               window_bytes: int, feed, codec=None) -> tuple:
        """A corpus of ``doclens`` (int32) built through the C-level builder of ``residency``: ``feed(L, builder)``
        appends every packed row in order (``L``: the library).  ``codec = (nbits, centroids, bucket weights)`` (fp32
        CPU tensors) builds a PLAID-coded streamed corpus.  Returns the corpus and the host fill seconds."""
        L = _cabi.lib()
        b = C.c_void_p()
        if codec is not None:
            nbits, centroids, weights = codec
            centroids = centroids.float().contiguous()
            weights = weights.float().contiguous()
            _cabi.check(L.flmr_corpus_builder_create_plaid(doclens.ctypes.data_as(C.c_void_p), len(doclens),
                                                           _cabi.DIM, int(device.index), int(pid_base), flags,
                                                           int(window_bytes), int(nbits),
                                                           C.c_void_p(centroids.data_ptr()), centroids.size(0),
                                                           C.c_void_p(weights.data_ptr()), C.byref(b)))
        elif residency == "host":
            _cabi.check(L.flmr_corpus_builder_create_streamed(doclens.ctypes.data_as(C.c_void_p), len(doclens),
                                                              _cabi.DIM, int(device.index), int(pid_base), flags,
                                                              int(window_bytes), C.byref(b)))
        else:
            _cabi.check(L.flmr_corpus_builder_create_ex(doclens.ctypes.data_as(C.c_void_p), len(doclens), _cabi.DIM,
                                                        int(device.index), int(pid_base), flags, C.byref(b)))
        try:
            feed(L, b)
            handle, fill_s = C.c_void_p(), C.c_double(0)
            _cabi.check(L.flmr_corpus_builder_finish(b, C.byref(handle), C.byref(fill_s)))
            b = None
        finally:
            if b is not None:
                L.flmr_corpus_builder_destroy(b)
        return cls._from_handle(handle, doclens, device, pid_base), fill_s.value

    # -- properties ---------------------------------------------------------------------------
    @property
    def n_passages(self) -> int:
        return int(self.info.n_passages)

    @property
    def n_tokens(self) -> int:
        return int(self.info.n_tokens)

    @property
    def handle(self) -> C.c_void_p:
        if self._h is None:
            raise RuntimeError("corpus was closed")
        return self._h

    @property
    def n_deleted(self) -> int:
        n = C.c_int64(0)
        _cabi.check(_cabi.lib().flmr_corpus_deleted(self.handle, C.byref(n), None, 0))
        return int(n.value)

    @property
    def n_live(self) -> int:
        """Passages a search can return: every passage but the deleted ones."""
        return self.n_passages - self.n_deleted

    @property
    def n_stored(self) -> int:
        """Passages whose rows are held in HBM and scanned: all ``n_passages`` until ``compact`` removes the deleted
        ones.  ``n_passages`` is the id extent and never shrinks."""
        n = C.c_int64(0)
        _cabi.check(_cabi.lib().flmr_corpus_stored(self.handle, C.byref(n), None))
        return int(n.value)

    def deleted_pids(self) -> np.ndarray:
        """Global ids of the deleted passages, ascending (int64)."""
        n = C.c_int64(0)
        L = _cabi.lib()
        _cabi.check(L.flmr_corpus_deleted(self.handle, C.byref(n), None, 0))
        out = np.empty(n.value, dtype=np.int64)
        _cabi.check(L.flmr_corpus_deleted(self.handle, C.byref(n), out.ctypes.data_as(C.c_void_p), out.size))
        return out

    def allow_bitmaps(self, pid_lists: Sequence) -> torch.Tensor:
        """``allow_bitmaps`` of this shard (its ``n_passages`` and ``pid_base``), on the corpus' device.  A bitmap
        describes the shard as it is now: after ``append`` build a new one to reach the new passages."""
        return allow_bitmaps(pid_lists, self.n_passages, self.pid_base, self.device)

    def live_pids(self) -> torch.Tensor:
        """Global ids of the passages that are not deleted, ascending, on the corpus' device."""
        pids = torch.arange(self.n_passages, dtype=torch.int64) + self.pid_base
        dead = self.deleted_pids()
        if dead.size:
            keep = torch.ones(self.n_passages, dtype=torch.bool)
            keep[torch.from_numpy(dead - self.pid_base)] = False
            pids = pids[keep]
        return pids.to(self.device)

    def append(self, tokens: torch.Tensor, doclens) -> np.ndarray:
        """Append passages (``tokens [sum(doclens), 128]``, on the CPU or on the corpus' GPU, converted to ``dtype``;
        ``doclens`` >= 1 each) behind the stored ones, in place; returns their global ids (int64), which continue the
        shard's ids.  An adopted token tensor is copied into library memory by the first append and released."""
        doclens = _as_doclens(doclens)
        if tokens.dim() != 2 or tokens.size(1) != _cabi.DIM:
            raise ValueError("tokens must be [sum(doclens), %d], got %s" % (_cabi.DIM, tuple(tokens.shape)))
        if int(doclens.sum()) != tokens.size(0):
            raise ValueError("sum(doclens)=%d != tokens rows=%d" % (int(doclens.sum()), tokens.size(0)))
        tokens = tokens.detach()
        if tokens.dtype != self.dtype:
            tokens = tokens.to(self.dtype)
        tokens = tokens.contiguous()
        if tokens.is_cuda and tokens.device != self.device:
            tokens = tokens.to(self.device)
        if tokens.is_cuda:
            torch.cuda.current_stream(self.device).synchronize()   # producer kernels of `tokens` are done
        first = C.c_int64(0)
        _cabi.check(_cabi.lib().flmr_corpus_append(self.handle, C.c_void_p(tokens.data_ptr()),
                                                   doclens.ctypes.data_as(C.c_void_p), int(doclens.shape[0]),
                                                   C.byref(first)))
        self.doclens = np.concatenate([self.doclens, doclens])
        self._refresh()
        return np.arange(first.value, first.value + doclens.shape[0], dtype=np.int64)

    def delete(self, pids) -> None:
        """Delete passages by global id: they are never returned by a search again and gather as all-masked rows.
        Every id must belong to this shard (else nothing is deleted and ``FlmrError`` is raised); deleting a deleted
        id does nothing."""
        if isinstance(pids, torch.Tensor):
            pids = pids.detach().cpu().numpy()
        arr = np.ascontiguousarray(np.asarray(pids, dtype=np.int64).reshape(-1))
        _cabi.check(_cabi.lib().flmr_corpus_delete(self.handle, arr.ctypes.data_as(C.c_void_p), int(arr.size)))
        self._refresh()

    def compact(self) -> dict:
        """Remove the rows of the deleted passages from HBM and from every later search, keeping every id: every call
        on the corpus returns bitwise what it returned before, in less memory and time.  Physical memory behind the
        new end of the token matrix is returned to the device; an adopted token tensor is copied once and released.
        Waits for the device first, so searches already enqueued see the corpus as it was.  Returns ``{"removed",
        "rows_before", "rows_after", "bytes_released", "seconds"}``; nothing happens when no stored passage is deleted,
        and ``FlmrError`` is raised (nothing changes) when every one is."""
        import time
        rows_before = int(self.info.n_rows)
        removed, released = C.c_int64(0), C.c_int64(0)
        t0 = time.perf_counter()
        _cabi.check(_cabi.lib().flmr_corpus_compact(self.handle, C.byref(removed), C.byref(released)))
        seconds = time.perf_counter() - t0
        self._refresh()
        return {"removed": int(removed.value), "rows_before": rows_before, "rows_after": int(self.info.n_rows),
                "bytes_released": int(released.value), "seconds": seconds}

    def _refresh(self) -> None:
        info = _cabi.CorpusInfo()
        _cabi.check(_cabi.lib().flmr_corpus_info(self.handle, C.byref(info)))
        self.info = info
        if not info.adopted:
            self._keepalive = None

    def workspace(self) -> C.c_void_p:
        """Default per-corpus scratch (single-threaded use, like the reference Searcher)."""
        if self._ws is None:
            ws = C.c_void_p()
            _cabi.check(_cabi.lib().flmr_workspace_create(self.handle, 64, 1024, C.byref(ws)))
            self._ws = ws
        return self._ws

    def gather_padded(self, pids: torch.Tensor, nd_max: Optional[int] = None):
        """Retrieved passages as a padded batch, straight out of HBM (an fp8 corpus: the exact bf16 rows of its
        pinned host master): ``pids`` (any shape, global ids) ->
        (tokens ``[*pids.shape, nd_max, 128]`` of ``dtype`` — bf16, fp16 on an fp16 corpus —, mask bool
        ``[*pids.shape, nd_max, 1]``).  ``nd_max``
        defaults to the longest requested passage.  Ids outside this shard and deleted ids give an all-masked zero
        row.
        Replaces the host-dictionary lookup + stack + H2D of rag_model_blip.py:414-425."""
        shape = tuple(pids.shape)
        flat = pids.detach().reshape(-1).to(device=self.device, dtype=torch.int64).contiguous()
        if nd_max is None:
            local = (flat - self.pid_base).clamp(0, self.n_passages - 1).cpu().numpy()
            nd_max = int(self.doclens[local].max()) if flat.numel() else 1
        out = torch.empty((flat.numel(), nd_max, _cabi.DIM), dtype=self.dtype, device=self.device)
        mask = torch.empty((flat.numel(), nd_max), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _cabi.check(_cabi.lib().flmr_corpus_gather(
                self.handle, C.c_void_p(flat.data_ptr()), flat.numel(), int(nd_max), C.c_void_p(out.data_ptr()),
                C.c_void_p(mask.data_ptr()), C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
        return out.view(*shape, nd_max, _cabi.DIM), mask.bool().view(*shape, nd_max, 1)

    def close(self) -> None:
        L = _cabi.lib()
        if self._ws is not None:
            L.flmr_workspace_destroy(self._ws)
            self._ws = None
        if self._h is not None:
            torch.cuda.synchronize(self.device)
            L.flmr_corpus_destroy(self._h)
            self._h = None
        self._keepalive = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __repr__(self) -> str:
        i = self.info
        return ("FlatCorpus(n_passages=%d, n_tokens=%d, device=%s, pid_base=%d, n_ctas=%d, adopted=%d, storage=%s)"
                % (i.n_passages, i.n_tokens, self.device, i.pid_base, i.n_ctas, i.adopted, self.storage))
