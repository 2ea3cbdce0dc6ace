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

``Indexer(..., index_format="plaid")`` writes a PLAID directory in the reference's on-disk format instead
(CollectionIndexer, collection_indexer.py:75-444), entirely on the GPU: seeded k-means (``plaid.kmeans``, not faiss)
on a sample of the collection, bucket cutoffs and weights from a held-out part of it, then every chunk's codes and
packed residuals from one kernel (``plaid.encode``) and the IVF.  Searcher, ``FlatCorpus.from_plaid`` and the
reference's own IndexScorer / Searcher open it.
"""
from __future__ import annotations

import json
import os
import queue
import random
import threading
from typing import Callable, Optional, Sequence

import numpy as np
import torch

from . import plaid
from .index_io import DTYPES, chunk_exists, finalize_chunked_index, save_flat_chunk
from .infra import resolve_index_path, run_context_open


class Indexer:
    def __init__(self, checkpoint=None, config=None, encode_fn: Optional[Callable] = None,
                 index_root: Optional[str] = None, chunksize: int = 25_000, rank: int = 0, nranks: int = 1,
                 storage: str = "bf16", index_format: str = "flat", nbits: Optional[int] = None, seed: int = 123):
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
        # "flat": the token store above; "plaid": a PLAID directory with nbits bits per dim (default config.nbits)
        if index_format not in ("flat", "plaid"):
            raise ValueError("Indexer index_format must be 'flat' or 'plaid', got %r" % (index_format,))
        self.index_format = index_format
        self.nbits = int(nbits if nbits is not None else getattr(config, "nbits", None) or 2)
        if index_format == "plaid" and self.nbits not in (1, 2, 4, 8):
            raise ValueError("PLAID nbits must be 1, 2, 4 or 8, got %d" % self.nbits)
        self.seed = int(seed)

    def get_index(self):
        return self.index_path

    def erase(self):
        """colbert.Indexer.erase (indexer.py:33-56): delete the index files already at index_path (a PLAID build also
        its .pt files, as the reference's erase does)."""
        assert self.index_path is not None
        deleted = []
        ends = (".bf16", ".f16", ".npy", ".json", ".tmp") + ((".pt",) if self.index_format == "plaid" else ())
        for fn in sorted(os.listdir(self.index_path)):
            if fn.endswith(ends):
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
        if self.index_format == "plaid":
            self._encode_plaid(collection, resume=(overwrite == "resume"))
        else:
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

    # -- PLAID: sample -> k-means -> buckets -> encode each chunk -> IVF (CollectionIndexer.run) -------------------
    def _device(self) -> torch.device:
        if torch.cuda.is_available():
            return torch.device("cuda", torch.cuda.current_device())
        return torch.device("cpu")        # only with plaid.encode substituted: the real encode refuses CPU tensors

    def _encode_chunk_embs(self, passages) -> tuple:
        embs, doclens = self.encode_fn(list(passages))
        embs = torch.as_tensor(embs)
        if len(doclens) != len(passages) or int(sum(doclens)) != embs.size(0):
            raise ValueError("encode_fn returned %d doclens / %d embeddings for %d passages"
                             % (len(doclens), embs.size(0), len(passages)))
        return embs.detach().to(self._device(), torch.float16), [int(d) for d in doclens]

    def _plaid_files_exist(self) -> bool:
        return all(os.path.exists(os.path.join(self.index_path, f))
                   for f in ("plan.json", "centroids.pt", "buckets.pt", "avg_residual.pt"))

    def _plaid_chunk_exists(self, c: int) -> bool:
        """IndexSaver.check_chunk_exists (index_saver.py:30-50)."""
        return all(os.path.exists(os.path.join(self.index_path, n % c))
                   for n in ("doclens.%d.json", "%d.metadata.json", "%d.codes.pt", "%d.residuals.pt"))

    def _encode_plaid(self, collection: Sequence, resume: bool) -> None:
        n = len(collection)
        chunksize = min(self.chunksize, 1 + n // self.nranks)        # Collection.get_chunksize
        num_chunks = (n + chunksize - 1) // chunksize
        owned = [c for c in range(num_chunks) if c % self.nranks == self.rank]
        reuse_plan = resume and self._plaid_files_exist()
        if self.nranks > 1:
            flag = [reuse_plan]
            torch.distributed.broadcast_object_list(flag, src=0)
            reuse_plan = flag[0]
        if not reuse_plan:
            self._train_plaid(collection, n, chunksize, num_chunks, owned)
        self._barrier()                                              # the codec is on disk
        with open(os.path.join(self.index_path, "plan.json")) as f:
            plan = json.load(f)
        dev = self._device()
        centroids = torch.load(os.path.join(self.index_path, "centroids.pt"), map_location="cpu").to(dev)
        cutoffs, _weights = torch.load(os.path.join(self.index_path, "buckets.pt"), map_location="cpu")
        cutoffs = cutoffs.to(dev)
        q: "queue.Queue" = queue.Queue(maxsize=3)                     # IndexSaver.thread (index_saver.py:52-73)
        errors = []

        def saver():
            for c, p0, codes, residuals, doclens in iter(q.get, None):
                try:
                    prefix = os.path.join(self.index_path, str(c))
                    torch.save(codes.cpu(), prefix + ".codes.pt")
                    torch.save(residuals.cpu(), prefix + ".residuals.pt")
                    with open(os.path.join(self.index_path, "doclens.%d.json" % c), "w") as f:
                        json.dump(doclens, f)
                    with open(prefix + ".metadata.json", "w") as f:      # written last: it marks the chunk complete
                        json.dump({"passage_offset": p0, "num_passages": len(doclens),
                                   "num_embeddings": int(codes.numel())}, f)
                except Exception as e:   # surfaced after join
                    errors.append(e)

        th = threading.Thread(target=saver)
        th.start()
        try:
            for c in owned:
                if resume and self._plaid_chunk_exists(c):
                    continue
                p0, p1 = c * chunksize, min(n, (c + 1) * chunksize)
                embs, doclens = self._encode_chunk_embs(collection[p0:p1])
                codes, residuals = plaid.encode(embs, centroids, cutoffs, nbits=self.nbits)
                q.put((c, p0, codes.to("cpu", non_blocking=False), residuals.cpu(), doclens))
        finally:
            q.put(None)
            th.join()
        if errors:
            raise errors[0]
        self._barrier()                                              # every rank's chunks are on disk
        if self.rank == 0:
            self._finalize_plaid(num_chunks, n, int(plan["num_partitions"]))
        self._barrier()                                              # nobody returns before metadata.json exists

    def _train_plaid(self, collection, n: int, chunksize: int, num_chunks: int, owned) -> None:
        """CollectionIndexer.setup + train (collection_indexer.py:75-223): every rank encodes the sampled passages of
        its chunks into ``sample.<rank>.pt``; rank 0 concatenates them in pid order (so the index does not depend on
        the number of ranks), holds out 5 % (at most 50k rows), trains the centroids and saves the codec and plan."""
        typical_doclen = 120                               # _sample_pids (collection_indexer.py:100-116)
        n_sample = min(1 + int(16 * np.sqrt(typical_doclen * n)), n)
        sampled = sorted(random.Random(self.seed).sample(range(n), n_sample))
        sampled_np = np.asarray(sampled, dtype=np.int64)
        pieces = []                                        # (chunk, rows, passages) of this rank's sample
        embs_all = []
        for c in owned:
            p0, p1 = c * chunksize, min(n, (c + 1) * chunksize)
            pids = sampled_np[(sampled_np >= p0) & (sampled_np < p1)]
            if len(pids) == 0:
                continue
            embs, doclens = self._encode_chunk_embs([collection[int(p)] for p in pids])
            embs_all.append(embs.cpu())
            pieces.append([c, int(embs.size(0)), len(doclens)])
        local = torch.cat(embs_all) if embs_all else torch.empty((0, 128), dtype=torch.float16)
        torch.save(local.half(), os.path.join(self.index_path, "sample.%d.pt" % self.rank))
        with open(os.path.join(self.index_path, "sample.%d.json" % self.rank), "w") as f:
            json.dump({"pieces": pieces}, f)
        self._barrier()                                    # every rank's sample is on disk
        if self.rank != 0:
            return
        parts = []                                         # (chunk, rows, passages, tensor)
        for r in range(self.nranks):
            sample_r = torch.load(os.path.join(self.index_path, "sample.%d.pt" % r), map_location="cpu")
            with open(os.path.join(self.index_path, "sample.%d.json" % r)) as f:
                row = 0
                for c, rows, n_pass in json.load(f)["pieces"]:
                    parts.append((c, rows, n_pass, sample_r[row:row + rows]))
                    row += rows
            os.remove(os.path.join(self.index_path, "sample.%d.pt" % r))
            os.remove(os.path.join(self.index_path, "sample.%d.json" % r))
        parts.sort(key=lambda t: t[0])                     # pid order: chunks are contiguous pid ranges
        dev = self._device()
        sample = torch.cat([t[3] for t in parts]).to(dev)
        n_sample_passages = sum(t[2] for t in parts)
        avg_doclen_est = sample.size(0) / max(1, n_sample_passages)
        num_embeddings_est = n * avg_doclen_est
        K = int(2 ** np.floor(np.log2(16 * np.sqrt(num_embeddings_est))))
        # _concatenate_and_split_sample: shuffle, hold out 5 % (at most 50k rows)
        g = torch.Generator().manual_seed(self.seed)
        sample = sample[torch.randperm(sample.size(0), generator=g).to(dev)]
        heldout_size = int(min(0.05 * sample.size(0), 50_000))
        train, heldout = sample.split([sample.size(0) - heldout_size, heldout_size], dim=0)
        K = max(1, min(K, train.size(0)))
        niters = int(getattr(self.config, "kmeans_niters", None) or 4)
        centroids = plaid.kmeans(train, K, niters=niters, seed=self.seed)
        cutoffs, weights, avg_residual = plaid.residual_buckets(centroids, heldout if heldout_size else train,
                                                                self.nbits)
        # ResidualCodec.save (residual.py:152-167)
        torch.save(centroids.cpu().half(), os.path.join(self.index_path, "centroids.pt"))
        torch.save((cutoffs, weights), os.path.join(self.index_path, "buckets.pt"))
        torch.save(avg_residual, os.path.join(self.index_path, "avg_residual.pt"))
        with open(os.path.join(self.index_path, "plan.json"), "w") as f:       # _save_plan
            json.dump({"config": self._plaid_config(), "num_chunks": num_chunks, "num_partitions": K,
                       "num_embeddings_est": num_embeddings_est, "avg_doclen_est": avg_doclen_est}, f, indent=4)

    def _plaid_config(self) -> dict:
        return {"nbits": self.nbits, "dim": 128}

    def _finalize_plaid(self, num_chunks: int, n: int, K: int) -> None:
        """CollectionIndexer.finalize (collection_indexer.py:341-444): embedding offsets into each chunk's metadata,
        the IVF, metadata.json."""
        offset = p_offset = 0
        codes, doclens = [], []
        for c in range(num_chunks):
            mp = os.path.join(self.index_path, "%d.metadata.json" % c)
            with open(mp) as f:
                meta = json.load(f)
            if meta["passage_offset"] != p_offset:
                raise RuntimeError("chunk %d starts at passage %d, expected %d" % (c, meta["passage_offset"], p_offset))
            meta["embedding_offset"] = offset
            with open(mp, "w") as f:
                json.dump(meta, f)
            p_offset += meta["num_passages"]
            offset += meta["num_embeddings"]
            codes.append(torch.load(os.path.join(self.index_path, "%d.codes.pt" % c), map_location="cpu"))
            with open(os.path.join(self.index_path, "doclens.%d.json" % c)) as f:
                doclens.extend(json.load(f))
        all_codes = torch.cat(codes).to(self._device())
        ivf, ivf_lengths = plaid.build_ivf(all_codes, doclens, K)
        torch.save((ivf, ivf_lengths), os.path.join(self.index_path, "ivf.pid.pt"))
        with open(os.path.join(self.index_path, "metadata.json"), "w") as f:
            json.dump({"config": self._plaid_config(), "num_chunks": num_chunks, "num_partitions": K,
                       "num_embeddings": offset, "avg_doclen": offset / max(1, n)}, f, indent=4)


class PlaidIndexer(Indexer):
    """``Indexer`` whose default ``index_format`` is ``"plaid"``: what ``integration.patch_colbert(indexer="plaid")``
    puts in place of ``colbert.Indexer``, so the reference's own call lines write a PLAID directory."""

    def __init__(self, *args, index_format: str = "plaid", **kw):
        super().__init__(*args, index_format=index_format, **kw)
