"""``Indexer`` with the call surface of the reference's ``colbert.Indexer``
(third_party/ColBERT/colbert/indexer.py:15-84) that writes the FLAT store the scan kernel streams,
instead of a PLAID index (k-means centroids + residual codes + IVF,
colbert/indexing/collection_indexer.py:56-73).  This is the step *before* the hot path
(SURVEY.md 8f-1): the document encoder stays PyTorch and is passed in as ``encode_fn``.

    indexer = Indexer(checkpoint=..., config=..., encode_fn=lambda passages: (embs [T, d], doclens))
    path = indexer.index(name="temp_index.nbits=8", collection=passages, overwrite=True)

``encode_fn`` has the contract of ``CollectionEncoder.encode_passages``
(colbert/indexing/collection_encoder.py:13-45): a list of passages -> (packed embeddings, doclens).
Chunks of 25,000 passages (colbert/data/collection.py:77-78) are owned round-robin by ranks
(collection.py:58-75), written by a background saver thread through a bounded queue
(index_saver.py:52-73), and skipped when already complete under ``overwrite='resume'``
(index_saver.py:30-50, collection_indexer.py:325-327).
"""
from __future__ import annotations

import os
import queue
import threading
from typing import Callable, Optional, Sequence

import torch

from .index_io import DTYPES, chunk_exists, finalize_chunked_index, save_flat_chunk
from .infra import resolve_index_path, run_context_open


class Indexer:
    def __init__(self, checkpoint=None, config=None, encode_fn: Optional[Callable] = None,
                 index_root: Optional[str] = None, chunksize: int = 25_000, rank: int = 0, nranks: int = 1,
                 storage: str = "bf16"):
        self.checkpoint = checkpoint
        self.config = config
        self.encode_fn = encode_fn
        self.index_root = index_root      # None: addressed through config + the Run() context, like the reference
        self._checkpoint_model = None
        self.chunksize = int(chunksize)
        self.rank, self.nranks = int(rank), int(nranks)
        self.index_path = None
        # token dtype of the index written: "bf16", or "fp16" (the encoder's own output type, ColBERT.doc's D.half(),
        # written as an "flmr-flat-f16" index that Searcher loads as an fp16 corpus)
        if storage not in ("bf16", "fp16"):
            raise ValueError("Indexer storage must be 'bf16' or 'fp16', got %r" % (storage,))
        self.dtype = "float16" if storage == "fp16" else "bfloat16"

    def get_index(self):
        return self.index_path

    def erase(self):
        """colbert.Indexer.erase (indexer.py:33-56): delete the index files already at index_path."""
        assert self.index_path is not None
        deleted = []
        for fn in sorted(os.listdir(self.index_path)):
            if fn.endswith((".bf16", ".f16", ".npy", ".json", ".tmp")):
                os.remove(os.path.join(self.index_path, fn))
                deleted.append(fn)
        return deleted

    def _path(self, name: str) -> str:
        """colbert/indexer.py:66-68 (``config.index_path_`` after ``from_existing(checkpoint_config, config,
        Run().config)``): ``<root>/<experiment>/indexes/<name>`` of the open Run context unless an explicit
        ``index_root=`` (an extension) or an absolute name says otherwise."""
        if os.path.isabs(name):
            return name
        if self.index_root is None and self.config is None and not run_context_open():
            return name                                  # no config, no context: relative to the working directory
        return resolve_index_path(name, self.config, self.index_root)

    def _reference_encode_fn(self) -> Callable:
        """Document encoder of the reference, built on first use: ``Checkpoint(checkpoint, colbert_config=config)``
        and the batching of ``CollectionEncoder.encode_passages`` (collection_encoder.py:13-45) around its
        ``docFromText(..., keep_dims='flatten')``.  It stays PyTorch; nothing of it is reimplemented here."""
        if self._checkpoint_model is None:
            if self.checkpoint is None:
                raise RuntimeError("Indexer needs encode_fn=... or checkpoint=...: the document encoder (ColBERT.doc "
                                   "/ Checkpoint.docFromText) stays in PyTorch and is out of scope here")
            try:
                from colbert.modeling.checkpoint import Checkpoint
            except ImportError as e:
                raise RuntimeError("Indexer(checkpoint=%r) needs the reference's colbert package on sys.path "
                                   "(third_party/ColBERT), or pass encode_fn=..." % (self.checkpoint,)) from e
            model = Checkpoint(self.checkpoint, colbert_config=self.config)
            self._checkpoint_model = model.cuda() if torch.cuda.is_available() else model
        model, bsize = self._checkpoint_model, int(getattr(self.config, "bsize", 32) or 32)

        def encode(passages):
            embs, doclens = [], []
            with torch.inference_mode():
                for b0 in range(0, len(passages), bsize * 50):
                    e, d = model.docFromText(passages[b0:b0 + bsize * 50], bsize=bsize, keep_dims="flatten",
                                             showprogress=False)
                    embs.append(e)
                    doclens.extend(d)
            return torch.cat(embs), doclens
        return encode

    def _barrier(self) -> None:
        """All ranks of a multi-rank build meet here.  The reference erases and plans in the parent process before
        it launches the workers (colbert/indexer.py:58-84); ranks that call ``index`` independently need the same
        ordering, so a multi-rank build requires an initialised ``torch.distributed`` process group."""
        if self.nranks > 1:
            if not (torch.distributed.is_available() and torch.distributed.is_initialized()):
                raise RuntimeError("Indexer(nranks=%d) needs an initialised torch.distributed process group: rank 0 "
                                   "erases / finalizes, the others must wait for it" % self.nranks)
            torch.distributed.barrier()

    @staticmethod
    def _cast_collection(collection) -> Sequence:
        """colbert.data.Collection.cast (collection.py:86-96): a list of passages, an object with ``data``, or the
        path of a ``pid \\t passage [\\t title]`` TSV (evaluation/loaders.py:155-176: title is prepended with ' | ')."""
        if isinstance(collection, str):
            out = []
            with open(collection) as f:
                for line_idx, line in enumerate(f):
                    pid, passage, *rest = line.strip("\n\r ").split("\t")
                    assert pid == "id" or int(pid) == line_idx, (pid, line_idx)
                    out.append(rest[0] + " | " + passage if rest else passage)
            return out
        data = getattr(collection, "data", None)
        return collection if data is None else data

    def index(self, name: str, collection: Sequence, overwrite=False) -> str:
        assert overwrite in [True, False, "reuse", "resume"]
        collection = self._cast_collection(collection)
        if self.encode_fn is None:
            self.encode_fn = self._reference_encode_fn()
        self.index_path = self._path(name)
        # rank 0 decides about the directory (exists? erase?) BEFORE any rank writes a chunk into it; the others
        # wait at the barrier, so a fast rank can neither have its chunks erased nor trip the exists-check
        reuse = False
        if self.rank == 0:
            exists = os.path.exists(os.path.join(self.index_path, "metadata.json")) or (
                os.path.isdir(self.index_path) and len(os.listdir(self.index_path)) > 0)
            assert overwrite in [True, "reuse", "resume"] or not exists, self.index_path
            os.makedirs(self.index_path, exist_ok=True)
            if overwrite is True:
                self.erase()
            reuse = bool(exists and overwrite == "reuse"
                         and os.path.exists(os.path.join(self.index_path, "metadata.json")))
        if self.nranks > 1:
            self._barrier()
            flag = [reuse]
            torch.distributed.broadcast_object_list(flag, src=0)
            reuse = flag[0]
        if reuse:
            return self.index_path
        self._encode(collection, resume=(overwrite == "resume"))
        return self.index_path

    # -- encode -> compress(no-op: bf16) -> save, chunk by chunk ---------------------------------------
    def _encode(self, collection: Sequence, resume: bool) -> None:
        n = len(collection)
        chunksize = min(self.chunksize, 1 + n // self.nranks)       # Collection.get_chunksize
        num_chunks = (n + chunksize - 1) // chunksize
        q: "queue.Queue" = queue.Queue(maxsize=3)                     # IndexSaver.thread (index_saver.py:52-66)
        errors = []

        def saver():
            for item in iter(q.get, None):
                try:
                    save_flat_chunk(self.index_path, *item, dtype=self.dtype)
                except Exception as e:   # surfaced after join
                    errors.append(e)

        th = threading.Thread(target=saver)
        th.start()
        try:
            for c in range(num_chunks):
                if c % self.nranks != self.rank:                       # round-robin chunk ownership
                    continue
                if resume and chunk_exists(self.index_path, c, self.dtype):
                    continue
                p0, p1 = c * chunksize, min(n, (c + 1) * chunksize)
                embs, doclens = self.encode_fn(list(collection[p0:p1]))
                embs = torch.as_tensor(embs)
                if len(doclens) != p1 - p0 or int(sum(doclens)) != embs.size(0):
                    raise ValueError("encode_fn returned %d doclens / %d embeddings for %d passages"
                                     % (len(doclens), embs.size(0), p1 - p0))
                q.put((c, p0, embs.detach().to("cpu", DTYPES[self.dtype][0]), list(doclens)))
        finally:
            q.put(None)
            th.join()
        if errors:
            raise errors[0]
        self._barrier()                                   # every rank's chunks are on disk
        if self.rank == 0:
            finalize_chunked_index(self.index_path, num_chunks, DTYPES[self.dtype][2])
        self._barrier()                                   # nobody returns before metadata.json exists
