"""``Searcher`` façade with the call surface of the reference's ``colbert.Searcher``
(third_party/ColBERT/colbert/searcher.py:22-132) so ``src/executors/FLMR_executor.py:774-792`` and
``src/models/rag/rag_model_blip.py:297-301, 397`` run unchanged:

    with Run().context(RunConfig(nranks=1, rank=..., root=..., experiment=...)):
        searcher = Searcher(index="temp_index.nbits=8", config=ColBERTConfig(total_visible_gpus=...))
    ._search_all_Q(queries, Q, k, filter_fn=None, progress=True, remove_zero_tensors=False) -> Ranking
    .dense_search(Q[1,Nq,d], k, filter_fn=None, remove_zero_tensors=False) -> (pids, ranks, scores)
    .search(text, k) / .search_all(queries, k)        (``encode_fn``, or the reference's ``Checkpoint`` built lazily
                                                       from ``checkpoint``: encoders stay PyTorch)
    Ranking.todict() -> {qid: [(pid, rank, score), ...]}   (colbert/data/ranking.py:48)

The index is addressed exactly as the reference does (``<Run().root>/<experiment>/indexes/<index>``,
infra.resolve_index_path) and whatever lives there is opened: a flat index written by this package's
``Indexer`` (index_io.py), or a PLAID directory written by the reference's own ``Indexer`` — decoded on the
GPU into the flat bf16 store (plaid.py).

What differs, by design (SURVEY.md §0): scoring is exhaustive and exact (no PLAID candidate
generation / centroid pruning), all queries of a call go through one batched fused scan instead of
a Python loop of per-query ``rank`` calls, and results always hold exactly ``min(k, n_passages)``
hits (a restricted search, ``pids=`` / ``qid_to_pids=``: ``min(k, allowed live passages)`` per
query).  ``shard_across_ranks=True`` (an extension; needs an initialised ``torch.distributed`` group) keeps
only this rank's passage shard resident and merges the per-shard top-k with one all-gather, where the
reference repeats the whole search on every rank (FLMR_executor.py:778-781).

``residency="host"`` (with ``window_bytes``) opens an index path as a streamed corpus: pinned host memory, copied
through two HBM windows per library call (``FlatCorpus``), for validation inside a training process, where the corpus
does not fit beside the model and optimizer state.  Results are bitwise those of the corpus held in HBM.  Each library
call copies the corpus once, so on a streamed corpus an unrestricted top-k search (k <= 128) hands the whole batch to
one call, and searches with per-query score rows or bitmaps (``filter_fn``, k > 128, ``pids=`` / ``qid_to_pids=``)
take as many queries per call as keep that scratch within ``STREAMED_SCRATCH_BYTES``.  ``residency`` and
``window_bytes`` choose how an index path is loaded; with a ``FlatCorpus`` given, a ``residency`` other than its own
and any ``window_bytes`` are refused.  ``compressed=True`` (with ``residency="host"``, on a PLAID index path) keeps the
index in its compressed form, a centroid code and a packed residual per token, and decodes each window on the GPU
before the scan (``FlatCorpus.from_plaid``); results stay bitwise those of the decoded corpus.  With a ``FlatCorpus``
given, a ``compressed`` that disagrees with it is refused.

``devices=[0, 1, ...]`` (or ``"all"``, every visible device) holds the index in this one process as one token-balanced
shard per device (``sharded.shard_ranges``; shard i loaded on ``devices[i]``, all shards at once, one host thread each),
for a corpus larger than one card searched without a launcher or a process group.  Every search runs each shard's own
top-k, as a one-device Searcher would on that shard, on a stream of the shard's device, and merges the lists on the
home device ``devices[0]`` with one kernel that reads them over peer access (``flmr_topk_merge_devices``); results are
those of the one-device Searcher and come back on the home device.  An fp8 search keeps the one-device shortlist: each
shard hands its e4m3 top-depth to the home device, which selects the global top-depth (the depth and allowed counts
taken over the whole index) and re-ranks those candidates with the one-device code, gathering their bf16 rows from the
shards that own them.  A device may hold several shards (``[0, 0]``).  It
loads an index path only, resident (``residency="host"`` and ``compressed=True`` are refused), and excludes ``device=``
and ``shard_across_ranks``.  ``corpus`` is the first shard, ``shards`` lists them all.

``storage="fp8"`` keeps the corpus as e4m3 in HBM (half the bytes; the exact bf16 rows stay in pinned host memory)
and searches in two stages, as PLAID does (colbert/search/index_storage.py:160-177): the exhaustive e4m3 scan
shortlists ``ndocs / 4`` candidates per query (the reference's exact-scoring depth, filter_pids.cpp:148), which are
gathered from the bf16 master and re-scored exactly.  Returned scores are exact; an id can differ from the bf16
search only where the exact top-k was not inside the shortlist.  With ``shard_across_ranks`` every rank shortlists and
re-ranks its own shard, so its fp8 results need not be those of one device.
"""
from __future__ import annotations

import copy
import json
import os
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from . import _cabi
from .corpus import FlatCorpus, allow_bitmaps
from .index_io import FORMATS as FLAT_FORMATS
from .infra import ColBERTConfig, active_run_config, resolve_index_path
from .maxsim import maxsim_argmax_grouped, maxsim_scores, maxsim_scores_listed, maxsim_topk, topk_select

# bytes of gathered bf16 candidate tokens one re-rank launch may hold: larger batches are split by queries
RERANK_GATHER_BYTES = 1 << 30

# A restricted search scans a plan of its listed passages' rows (maxsim_topk(pids=)) while those rows are at most this
# fraction of the rows its bitmap scan streams (the shard's rows once per scan pass), and tests bitmaps in a full scan
# above it.  tools/listed_scan_probe.py brackets the crossover between 0.12 and 1.2 of this measure on an H100
# (profiles/r09_listed_scan_probe.md).
LISTED_SCAN_MAX_ROW_FRACTION = 0.5

# A streamed corpus (residency="host") copies all of its rows over PCIe once per library call, so its searches hand the
# library as many queries per call as they can: the fused top-k takes a whole batch (the library chunks it by the
# workspace's max_queries inside its window loop), and calls whose per-query scratch grows with the shard (a score row,
# an allow bitmap and the byte per passage it is built from) take as many queries as keep that scratch within this bound.
STREAMED_SCRATCH_BYTES = 1 << 30


def _default_knobs(k: int) -> Tuple[int, float, int]:
    """(ncells, centroid_score_threshold, ndocs) the reference's Searcher.dense_search fills in from k
    (searcher.py:92-118)."""
    return (2, 0.45, 1024) if k <= 100 else (4, 0.4, max(k * 4, 4096))


def shortlist_depth(k: int, ndocs: Optional[int], n_candidates: int) -> int:
    """Candidates per query the e4m3 scan hands to the exact re-rank: ``ndocs / 4``, the depth PLAID scores exactly
    (filter_pids.cpp:148), with ``ndocs`` as the reference derives it from k when unset; never below k, at most the
    select kernel's capacity and the candidates there are."""
    if k > _cabi.SELECT_MAX_K:
        raise ValueError("fp8 storage re-ranks at most %d candidates per query; k=%d" % (_cabi.SELECT_MAX_K, k))
    if ndocs is None:
        ndocs = _default_knobs(k)[2]
    return min(max(int(ndocs) // 4, k), _cabi.SELECT_MAX_K, n_candidates)


def _n_live(corpus) -> int:
    """Passages a search on ``corpus`` can return: all but the deleted ones (a corpus type without updates: all)."""
    return corpus.n_live if hasattr(corpus, "n_live") else corpus.n_passages


def _live_pids(corpus) -> torch.Tensor:
    if hasattr(corpus, "live_pids"):
        return corpus.live_pids()
    return torch.arange(corpus.n_passages, device=corpus.device) + corpus.pid_base


def _allowed_live_counts(shards, lists: List) -> np.ndarray:
    """Per query, the live passages of ``shards`` its list of global ids admits, each id counted once (None: every live
    passage): what a restricted fp8 search's shortlist depth follows."""
    out = np.zeros(len(lists), dtype=np.int64)
    for c in shards:
        dead = c.deleted_pids() if hasattr(c, "deleted_pids") else np.empty(0, dtype=np.int64)
        lo, hi = c.pid_base, c.pid_base + c.n_passages
        for b, ids in enumerate(lists):
            if ids is None:
                out[b] += _n_live(c)
                continue
            u = np.unique(torch.as_tensor(ids).reshape(-1).cpu().numpy())
            u = u[(u >= lo) & (u < hi)]
            out[b] += u.size - int(np.isin(u, dead).sum())
    return out


def _popcount_rows(words: torch.Tensor) -> torch.Tensor:
    """Set bits per row of an int32 bitmap ``[B, words]`` (int64 ``[B]``)."""
    x = words.to(torch.int64) & 0xFFFFFFFF
    x = x - ((x >> 1) & 0x55555555)
    x = (x & 0x33333333) + ((x >> 2) & 0x33333333)
    x = (x + (x >> 4)) & 0x0F0F0F0F
    return (((x * 0x01010101) & 0xFFFFFFFF) >> 24).sum(dim=-1)


def _live_words(corpus) -> torch.Tensor:
    """Bitmap ``[words]`` of the passages of ``corpus`` a search can return (not deleted; no bits past the end)."""
    n = corpus.n_passages
    dead = corpus.deleted_pids() if hasattr(corpus, "deleted_pids") else []
    live = ~allow_bitmaps([dead], n, corpus.pid_base, corpus.device)[0]
    if n % 32:
        live[-1] &= (1 << (n % 32)) - 1
    return live


class Ranking:
    """colbert.data.Ranking (colbert/data/ranking.py:25-94): ``data`` maps qid -> [(pid, rank (1-based),
    score), ...]; ``flat_ranking`` / ``tolist`` is the same as (qid, pid, rank, score) rows; ``save`` writes
    the reference's TSV plus a ``.meta`` JSON with the provenance."""

    def __init__(self, path: Optional[str] = None, data=None, metrics=None, provenance=None):
        del metrics
        self._provenance = provenance if provenance is not None else (path or {})
        if data is None:
            if path is None:
                raise ValueError("Ranking needs data= or path=")
            data = self._load_file(path)
        if isinstance(data, dict):
            self.flat_ranking = [(qid, *rest) for qid, sub in data.items() for rest in sub]
            self.data = data
        else:                                       # flat rows: group by qid, order preserved
            self.flat_ranking = [tuple(r) for r in data]
            grouped: Dict = {}
            for qid, *rest in self.flat_ranking:
                grouped.setdefault(qid, []).append(tuple(rest))
            self.data = grouped

    @staticmethod
    def _load_file(path: str):
        def num(v):
            return float(v) if "." in v else int(v)
        with open(path) as f:
            return [list(map(num, line.strip().split("\t"))) for line in f if line.strip()]

    def provenance(self):
        return self._provenance

    def toDict(self):
        return {"provenance": self.provenance()}

    def todict(self):
        return dict(self.data)

    def tolist(self):
        return list(self.flat_ranking)

    def items(self):
        return self.data.items()

    def save(self, new_path: str) -> str:
        """ranking.py:64-82.  The reference resolves ``new_path`` under ``Run().path_`` (a per-script
        timestamped directory); here a relative path is taken as given."""
        assert "tsv" in new_path.strip("/").split("/")[-1].split("."), "TODO: Support .json[l] too."
        os.makedirs(os.path.dirname(os.path.abspath(new_path)), exist_ok=True)
        with open(new_path, "w") as f:
            for items in self.flat_ranking:
                f.write("\t".join(str(int(x) if type(x) is bool else x) for x in items) + "\n")
        prov = self.provenance()
        with open(new_path + ".meta", "w") as f:
            json.dump({"metadata": {}, "provenance": prov.toDict() if hasattr(prov, "toDict") else prov},
                      f, indent=4, default=str)
        return new_path

    @classmethod
    def cast(cls, obj):
        if type(obj) is str:
            return cls(path=obj)
        if isinstance(obj, (dict, list)):
            return cls(data=obj)
        if type(obj) is cls:
            return obj
        assert False, "obj has type %s which is not compatible with cast()" % type(obj)


def _query_keys(queries, n: int) -> List:
    if queries is None:
        return list(range(n))
    if hasattr(queries, "keys"):
        keys = list(queries.keys())
    else:
        keys = list(queries)
    if len(keys) != n:
        raise ValueError("got %d query ids for %d query matrices" % (len(keys), n))
    return keys


def detect_index_kind(path: str) -> str:
    """'flat' (index_io.py) or 'plaid' (the reference's format, SURVEY.md Appendix C) for the directory the
    reference's ``ColBERTConfig.load_from_index`` (base_config.py:71-87) would read its config from."""
    meta_path = os.path.join(path, "metadata.json")
    if os.path.exists(meta_path):
        with open(meta_path) as f:
            meta = json.load(f)
        if meta.get("format") in FLAT_FORMATS:
            return "flat"
        if "nbits" in meta.get("config", {}) and os.path.exists(os.path.join(path, "centroids.pt")):
            return "plaid"
        raise ValueError("%s holds a metadata.json that is neither a %s index nor a PLAID index "
                         "(config.nbits + centroids.pt)" % (path, " / ".join(FLAT_FORMATS)))
    if os.path.exists(os.path.join(path, "plan.json")):
        raise ValueError("%s holds only plan.json: the PLAID index build did not finish "
                         "(collection_indexer.py:428-444 writes metadata.json last)" % path)
    raise FileNotFoundError("no index at %s (no metadata.json)" % path)


class Searcher:
    def __init__(self, index: Union[str, FlatCorpus], checkpoint=None, collection=None, config=None,
                 disable_gpu: bool = True, device: Optional[Union[int, torch.device]] = None,
                 encode_fn: Optional[Callable] = None, index_root: Optional[str] = None,
                 query_batch: int = 64, shard_across_ranks: bool = False, group=None,
                 storage: Optional[str] = None, residency: Optional[str] = None, window_bytes: Optional[int] = None,
                 compressed: Optional[bool] = None, devices=None):
        # `disable_gpu` is part of the reference signature (default True) but dead there: colbert/searcher.py:23
        # never reads it, the device is chosen by config.total_visible_gpus (:40-43), which FLMR_executor.py:778-781
        # zeroes under DDP to force CPU search.  Here the search always runs on the GPU (no CPU path exists);
        # FlatCorpus raises when CUDA is absent.
        del disable_gpu
        if devices is not None:
            if isinstance(index, FlatCorpus):
                raise ValueError("devices= loads the shards of an index path on their devices; a FlatCorpus given "
                                 "lives on one device")
            if shard_across_ranks:
                raise ValueError("devices= shards the index across the devices of this process; it excludes "
                                 "shard_across_ranks=True, which shards it across ranks")
            if device is not None:
                raise ValueError("devices= places every shard; it excludes device=")
            if residency not in (None, "device") or compressed:
                raise ValueError("devices= keeps every shard resident in HBM; residency=%r, compressed=%r are not "
                                 "supported with it" % (residency, compressed))
        self.checkpoint = checkpoint
        self.collection = collection
        self.encode_fn = encode_fn
        self.query_batch = int(query_batch)
        self._sharded = None
        self._sharded_index_size = None
        self._devices = None        # a multi-device Searcher's DeviceShardedSearcher
        self._nccl = None
        self._checkpoint_model = None
        self.index_config = None
        run_cfg = active_run_config(config)
        shards = None
        if isinstance(index, FlatCorpus):
            if storage is not None and storage != index.storage:
                raise ValueError("storage=%r, but the corpus given is stored as %r" % (storage, index.storage))
            if residency is not None and residency != index.residency:
                raise ValueError("residency=%r, but the corpus given has residency %r" % (residency, index.residency))
            if window_bytes is not None:
                raise ValueError("window_bytes applies to an index path opened with residency='host'; the corpus given "
                                 "was created with its own")
            if compressed is not None and bool(compressed) != (index.codec_nbits > 0):
                raise ValueError("compressed=%r, but the corpus given %s a PLAID-coded corpus"
                                 % (compressed, "is" if index.codec_nbits else "is not"))
            self.corpus = index
            self.index = None
            self.index_kind = "resident"
        else:
            # searcher.py:26-30: index path = <index_root_ of from_existing(config, Run().config)>/<index>
            self.index = resolve_index_path(index, config, index_root)
            self.index_kind = detect_index_kind(self.index)
            self.index_config = ColBERTConfig.load_from_index(self.index) if self.index_kind == "plaid" else None
            rank, world = 0, 1
            if shard_across_ranks:
                import torch.distributed as dist
                if not (dist.is_available() and dist.is_initialized()):
                    raise RuntimeError("shard_across_ranks needs an initialised torch.distributed process group")
                rank, world = dist.get_rank(group), dist.get_world_size(group)
            load = FlatCorpus.from_index if self.index_kind == "flat" else FlatCorpus.from_plaid
            # storage None: a flat index keeps its own dtype (fp16 for an "flmr-flat-f16" index), PLAID decodes to bf16
            extra = {"storage": storage} if storage is not None else {}
            if window_bytes is not None and residency != "host":
                raise ValueError("window_bytes=%r applies to residency='host' only" % (window_bytes,))
            if residency is not None:   # "host": a streamed corpus (FlatCorpus residency="host")
                extra["residency"] = residency
                if window_bytes is not None:
                    extra["window_bytes"] = window_bytes
            if compressed:   # a PLAID index kept in its compressed form (FlatCorpus.from_plaid compressed=True)
                if self.index_kind != "plaid":
                    raise ValueError("compressed=True streams a PLAID index's compressed form; %s is a flat index"
                                     % self.index)
                extra["compressed"] = True
            if devices is not None:
                from .sharded import resolve_devices
                devs = resolve_devices(devices)
                _cabi.lib()                              # loaded (built if stale) once, before the loader threads

                def load_shard(i):
                    return load(self.index, device=devs[i], rank=i, world_size=len(devs), **extra)
                with ThreadPoolExecutor(len(devs)) as pool:
                    # a shard is None when there are more devices than passages
                    shards = [c for c in pool.map(load_shard, range(len(devs))) if c is not None]
                self.corpus = shards[0]
            else:
                self.corpus = load(self.index, device=device, rank=rank, world_size=world, **extra)
        # the shards this process holds
        self.shards = shards if shards is not None else ([self.corpus] if self.corpus is not None else [])
        self.storage = getattr(self.corpus, "storage", None) or storage or "bf16"
        # every rank of a sharded Searcher gets the same residency argument, so ranks without a shard batch their
        # collectives as the others do
        self.residency = getattr(self.corpus, "residency", None) or residency or "device"
        self._last_depth = None
        # searcher.py:35: checkpoint config < index config < (config + Run().config); kept for callers that
        # read searcher.config — none of its PLAID knobs influence the exhaustive scan.
        cfg_type = type(config) if (config is not None and hasattr(type(config), "from_existing")) else ColBERTConfig
        try:
            self.config = cfg_type.from_existing(self.index_config if cfg_type is ColBERTConfig else None,
                                                 config, run_cfg)
        except Exception:          # foreign config type with a different constructor: keep what was given
            self.config = config
        if getattr(self.config, "interaction", "colbert") != "colbert":
            # the fused scan reduces with the plain sum of colbert_score_reduce (colbert.py:263); ranking a corpus
            # by the 'flipr' partial top-k sums (:248-261, unused by FLMR) is only available through colbert_score
            raise NotImplementedError("Searcher ranks with interaction='colbert'; got %r"
                                      % (self.config.interaction,))
        if shard_across_ranks:
            import torch.distributed as dist
            from .maxsim import topk_merge
            from .sharded import NcclExchange, ShardedSearcher
            self._sharded = ShardedSearcher(None, lambda s, p, k: topk_merge(s, p, k), group)
            self._group = group
            self._want_nccl = dist.get_backend(group) == "nccl"
        if self.corpus is not None:
            self.device = self.corpus.device
        else:
            self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self._sharded is not None and self._want_nccl:
            from .sharded import NcclExchange
            self._nccl = NcclExchange(self.device, self._group)       # collective: every rank constructs it
        if self._sharded is not None:
            # passages of the whole index, for checking the ids of restricted searches; collective, and fixed: a
            # sharded Searcher cannot be updated
            import torch.distributed as dist
            n = self.corpus.pid_base + self.corpus.n_passages if self.corpus is not None else 0
            t = torch.tensor([n], dtype=torch.int64, device=self.device if self._want_nccl else "cpu")
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self._group)
            self._sharded_index_size = int(t.item())
        if shards is not None:
            from .sharded import DeviceShardedSearcher
            self._devices = DeviceShardedSearcher([c.device.index for c in self.shards], self._shard_search)
            self._sharded_index_size = self.shards[-1].pid_base + self.shards[-1].n_passages
        self._relu = False

    # -- reference-compatible surface ------------------------------------------------------------
    def configure(self, **kw):
        """colbert.Searcher.configure (searcher.py:49-50).  PLAID knobs (ncells,
        centroid_score_threshold, ndocs) are recorded on ``config`` and otherwise ignored: the scan is
        exhaustive.  On an fp8 corpus ``ndocs / 4`` sets the depth of the exact re-rank."""
        self._relu = bool(kw.pop("relu", self._relu))
        if kw and self.config is not None and hasattr(self.config, "configure"):
            self.config.configure(**kw)
        return self

    def _text_encoder(self):
        """The reference's own query encoder, built on first use as searcher.py:31-43 does at construction:
        ``Checkpoint(checkpoint or index_config.checkpoint, colbert_config=self.config)`` from the reference's
        ``colbert`` package (it stays PyTorch; nothing of it is reimplemented here)."""
        if self._checkpoint_model is None:
            name = self.checkpoint or getattr(self.index_config, "checkpoint", None)
            if name is None:
                raise RuntimeError("text search needs encode_fn=... or checkpoint=... (the query encoder stays in "
                                   "PyTorch: FLMR.query / Checkpoint.queryFromText, out of scope here)")
            try:
                from colbert.modeling.checkpoint import Checkpoint
            except ImportError as e:
                raise RuntimeError("text search with checkpoint=%r needs the reference's colbert package on "
                                   "sys.path (third_party/ColBERT), or pass encode_fn=..." % (name,)) from e
            model = Checkpoint(name, colbert_config=self.config)
            self._checkpoint_model = model.cuda() if torch.cuda.is_available() else model
        return self._checkpoint_model

    def encode(self, text, full_length_search=False):
        """searcher.py:52-59.  ``encode_fn`` (queries -> ``[n, Nq, d]``) when given, else the reference's
        ``Checkpoint.queryFromText``; the embeddings stay on the GPU (the reference moves them to the CPU)."""
        queries = text if isinstance(text, list) else [text]
        if self.encode_fn is not None:
            return self.encode_fn(queries)
        model = self._text_encoder()
        bsize = 128 if len(queries) > 128 else None
        maxlen = getattr(self.config, "query_maxlen", None)
        if maxlen is not None and hasattr(model, "query_tokenizer"):
            model.query_tokenizer.query_maxlen = maxlen
        return model.queryFromText(queries, bsize=bsize, to_cpu=False)

    def search(self, text: str, k: int = 10, filter_fn=None, pids=None):
        return self.dense_search(self.encode(text), k, filter_fn=filter_fn, pids=pids)

    def search_all(self, queries, k: int = 10, filter_fn=None, qid_to_pids=None):
        texts = list(queries.values()) if hasattr(queries, "values") else list(queries)
        Q = self.encode(texts)
        if isinstance(Q, (list, tuple)):               # queryFromText with a batch size returns per-batch tensors
            Q = torch.cat(list(Q))
        return self._search_all_Q(queries, Q, k, filter_fn=filter_fn, qid_to_pids=qid_to_pids)

    @staticmethod
    def _drop_zero_rows(Q: torch.Tensor) -> torch.Tensor:
        """``remove_zero_tensors`` (searcher.py:120-126) for a batch: all-zero query rows are dropped and the
        remaining rows of every query packed to the front (order kept), padded with zero rows to the longest
        query of the batch.  A zero row adds ``max_j 0 = 0`` to every passage, so scores are unchanged; the
        scan just has fewer rows to go through (WIT pre-training queries: 32 live rows out of 32 + text)."""
        live = Q.abs().sum(dim=-1) > 0                                   # [B, Nq]
        n_live = int(live.sum(dim=1).max().item()) if Q.numel() else 0
        if n_live == Q.size(1):
            return Q
        order = torch.argsort((~live).to(torch.int8), dim=1, stable=True)[:, :max(n_live, 1)]
        return torch.gather(Q, 1, order.unsqueeze(-1).expand(-1, -1, Q.size(2)))

    def _batch(self, scratch_bytes_per_query: int = 0) -> int:
        """Queries per library call: ``query_batch``, or on a streamed corpus (one copy of its rows per call) as many
        as keep per-query scratch of this size within STREAMED_SCRATCH_BYTES (no bound: every query in one call)."""
        if self.residency != "host":
            return self.query_batch
        if scratch_bytes_per_query <= 0:
            return 1 << 30
        return max(self.query_batch, STREAMED_SCRATCH_BYTES // int(scratch_bytes_per_query))

    def _local_topk(self, Q: torch.Tensor, kk: int, keep: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """Top-``kk`` of this shard: (scores [B, kk'], global pids [B, kk']), kk' = min(kk, candidates)."""
        corpus = self.corpus
        if corpus is None:                               # this rank's shard is empty (more ranks than passages)
            return (torch.empty((Q.size(0), 0), dtype=torch.float32, device=self.device),
                    torch.empty((Q.size(0), 0), dtype=torch.int64, device=self.device))
        if self.storage == "fp8":
            return self._reranked_topk(Q, kk, keep)
        if keep is None and kk <= _cabi.MAX_K:
            kq = min(kk, _n_live(corpus))                # deleted passages are never offered to the fused top-k
            outs, outp = [], []
            step = self._batch()
            for b0 in range(0, Q.size(0), step):
                s, p = maxsim_topk(corpus, Q[b0:b0 + step], kq, relu=self._relu)
                outs.append(s)
                outp.append(p)
            return torch.cat(outs), torch.cat(outp)
        # filtered or very large k: all scores from the fused scan, selection as plain plumbing (deleted passages
        # score -inf, so at most n_live candidates are selected)
        outs, outp = [], []
        n_cand = _n_live(corpus) if keep is None else int(keep.numel())
        kq = min(kk, n_cand)
        if kq == 0:
            return (torch.empty((Q.size(0), 0), dtype=torch.float32, device=corpus.device),
                    torch.empty((Q.size(0), 0), dtype=torch.int64, device=corpus.device))
        step = self._batch(4 * corpus.n_passages)               # one fp32 score row per query
        for b0 in range(0, Q.size(0), step):
            s = maxsim_scores(corpus, Q[b0:b0 + step], relu=self._relu)
            if keep is not None:
                s = s[:, keep]
            if kq <= _cabi.SELECT_MAX_K:
                vals, idx = topk_select(s, kq)                       # radix-select kernel
            else:
                vals, idx = torch.sort(s, dim=1, descending=True, stable=True)
                vals, idx = vals[:, :kq], idx[:, :kq]
            outs.append(vals)
            outp.append((keep[idx] if keep is not None else idx) + corpus.pid_base)
        return torch.cat(outs), torch.cat(outp)

    def _reranked_topk(self, Q: torch.Tensor, kk: int, keep: Optional[torch.Tensor]
                       ) -> Tuple[torch.Tensor, torch.Tensor]:
        """``_local_topk`` of an fp8 corpus: all e4m3 scores, a shortlist of ``shortlist_depth`` candidates (after
        ``keep``), their exact bf16 tokens gathered from the master and re-scored by the grouped rowmax kernel,
        the top ``kk`` of those exact scores (ties: lower pid)."""
        corpus = self.corpus
        n_cand = _n_live(corpus) if keep is None else int(keep.numel())
        kq = min(kk, n_cand)
        if kq == 0:
            return (torch.empty((Q.size(0), 0), dtype=torch.float32, device=corpus.device),
                    torch.empty((Q.size(0), 0), dtype=torch.int64, device=corpus.device))
        depth = shortlist_depth(kk, getattr(self.config, "ndocs", None), n_cand)
        self._last_depth = depth
        outs, outp = [], []
        for b0 in range(0, Q.size(0), self.query_batch):
            Qb = Q[b0:b0 + self.query_batch].to(corpus.device).to(torch.bfloat16)
            vals, pids = self._rerank(Qb, self._shortlist(Qb, depth, keep=keep)[1], kq)
            outs.append(vals)
            outp.append(pids)
        return torch.cat(outs), torch.cat(outp)

    def _shortlist(self, Q: torch.Tensor, depth: int, keep: Optional[torch.Tensor] = None,
                   allow: Optional[torch.Tensor] = None, lists: Optional[List] = None
                   ) -> Tuple[torch.Tensor, torch.Tensor]:
        """The e4m3 stage of an fp8 search on this shard: (scores, global pids) ``[B, min(depth, columns)]``, the top
        ``depth`` e4m3 scores of the bf16 queries ``Q`` (ties: the lower pid) among the passages ``keep`` (local ids, in
        ascending order), ``allow`` (bitmaps) or ``lists`` (global id lists, on the listed scan) admit.  An entry with a
        -inf score (a deleted or disallowed passage, or padding) has pid -1."""
        corpus = self.corpus
        if lists is not None:
            s, ids = self._listed_scores(Q, lists)          # ids ascend along a row
        else:
            s = maxsim_scores(corpus, Q, relu=self._relu, allow=allow)
            if keep is not None:
                s = s[:, keep]
        d = min(depth, s.size(1))
        if d == 0:
            return (torch.empty((Q.size(0), 0), dtype=torch.float32, device=corpus.device),
                    torch.empty((Q.size(0), 0), dtype=torch.int64, device=corpus.device))
        vals, col = topk_select(s, d)
        if lists is not None:
            pids = ids.gather(1, col.clamp_min(0))
        else:
            pids = (keep[col] if keep is not None else col) + corpus.pid_base
        return vals, pids.masked_fill(vals == float("-inf"), -1)

    def _rerank(self, Q: torch.Tensor, cand: torch.Tensor, kq: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """The exact stage of an fp8 search: the top ``kq`` (scores, global pids) of the candidates ``cand`` (global
        pids, -1: none) by their MaxSim over the bf16 rows, ties on the lower pid; short rows end in (-inf, -1)."""
        cand = torch.sort(cand, dim=1).values        # pid order: the select below breaks exact ties by lower pid
        exact = self._exact_scores(Q, cand).masked_fill(cand < 0, float("-inf"))
        vals, col = topk_select(exact, kq)
        return vals, cand.gather(1, col).masked_fill(vals == float("-inf"), -1)

    def _exact_scores(self, Q: torch.Tensor, cand: torch.Tensor) -> torch.Tensor:
        """Exact MaxSim ``[B, depth]`` of query b against its candidates ``cand[b]`` (global pids), from the bf16
        rows of the shards that own them; the gather is split by queries to hold at most RERANK_GATHER_BYTES of
        tokens."""
        depth = cand.size(1)
        nd_max = self._longest(cand)
        per_query = depth * nd_max * _cabi.DIM * 2
        step = max(1, RERANK_GATHER_BYTES // per_query)
        out = []
        for q0 in range(0, Q.size(0), step):
            D, mask = self._gather_padded(cand[q0:q0 + step], nd_max)          # [b, depth, nd_max, d]
            _, rowmax = maxsim_argmax_grouped(Q[q0:q0 + step], D.flatten(0, 1), mask.flatten(0, 1), depth,
                                              return_rowmax=True)
            if self._relu:
                rowmax = rowmax.clamp_min(0.0)
            out.append(rowmax.sum(dim=-1))
        return torch.cat(out)

    def _index_size(self) -> int:
        """Passages of the whole index (every shard, deleted ones included): ids a search may name are below it."""
        if self._sharded_index_size is not None:
            return self._sharded_index_size
        return self.corpus.pid_base + self.corpus.n_passages

    def _restricted_tensors(self, Q: torch.Tensor, k: int, filter_fn, pid_lists: List
                            ) -> Tuple[torch.Tensor, torch.Tensor]:
        """``_search_tensors`` with query b restricted to the SET of global ids ``pid_lists[b]`` (None: the whole
        index).  The whole batch is checked before anything is searched.  Each query's allowed ids become a bitmap
        the scan's reducer tests, so there is no score matrix on the fused path.  Rows are padded with (-inf, -1)."""
        lists = self._pid_lists(pid_lists, filter_fn)
        if self._sharded is not None and k > _cabi.MAX_K:
            raise ValueError("sharded search merges at most k=%d results per query" % _cabi.MAX_K)
        corpus = self.corpus
        B = Q.size(0)
        # the C-level sharded search (scan + exchange in one call) takes bf16 shards; the others exchange below
        c_level = self._nccl is not None and corpus is not None and self.storage != "fp8"
        parts = []
        # per query: the allow bitmap, and the byte per passage allow_bitmaps builds it from; sized by the whole index,
        # so that every rank of a sharded search (one without a shard included) makes the same calls and collectives
        step = self._batch(self._index_size() * 9 // 8 + 1)
        if corpus is not None:
            for b0 in range(0, B, step):
                Qb = Q[b0:b0 + step]
                lb = lists[b0:b0 + step]
                if self._listed_is_cheaper(Qb, lb):
                    # the scan streams the listed passages' rows only; on the C-level sharded path the exchange that
                    # flmr_maxsim_topk_sharded_allowed would make follows, so every rank makes the same collectives
                    s_, p_ = self._listed_topk(Qb, k, lb)
                    if c_level:
                        s_ = torch.cat([s_, s_.new_full((s_.size(0), k - s_.size(1)), float("-inf"))], dim=1)
                        p_ = torch.cat([p_, p_.new_full((p_.size(0), k - p_.size(1)), -1)], dim=1)
                        s_, p_ = self._nccl.exchange(s_, p_, k)
                    parts.append((s_, p_))
                    continue
                allow = corpus.allow_bitmaps(lb)     # built on the device
                if c_level:
                    parts.append(self._nccl.search(corpus, Qb, k, relu=self._relu, allow=allow))
                else:
                    parts.append(self._allowed_topk(Qb, k, allow))
        width = k if self._sharded is not None else max([ps.size(1) for ps, _ in parts], default=0)
        s = torch.full((B, width), float("-inf"), dtype=torch.float32, device=self.device)
        p = torch.full((B, width), -1, dtype=torch.int64, device=self.device)
        b0 = 0
        for ps, pp in parts:
            s[b0:b0 + ps.size(0), :ps.size(1)] = ps
            p[b0:b0 + pp.size(0), :pp.size(1)] = pp
            b0 += ps.size(0)
        if self._sharded is not None and not c_level:
            # one exchange per query batch, as the ranks on the C-level path make (a rank without a shard takes this
            # branch while the others may not)
            ex = self._nccl or self._sharded
            merged = [ex.exchange(s[b0:b0 + step], p[b0:b0 + step], k) for b0 in range(0, B, step)]
            s, p = torch.cat([m[0] for m in merged]), torch.cat([m[1] for m in merged])
        n_valid = int((p >= 0).sum(dim=1).max()) if p.numel() else 0
        return s[:, :n_valid], p[:, :n_valid]

    def _pid_lists(self, pid_lists: List, filter_fn) -> List:
        """The id lists of a restricted search, checked against the whole index before anything is searched, with
        ``filter_fn`` applied to each query's own list (to every live passage of this Searcher's shards for a query
        without one), as the reference applies it to the pids it was given."""
        n_index = self._index_size()
        lists = []
        for ids in pid_lists:
            if ids is not None:
                ids = torch.as_tensor(ids, dtype=torch.int64).reshape(-1).cpu()
                if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= n_index):
                    raise ValueError("passage id %d outside the index [0, %d)"
                                     % (int(ids.min()) if int(ids.min()) < 0 else int(ids.max()), n_index))
            lists.append(ids)
        if filter_fn is not None:
            everything = (torch.cat([_live_pids(c).to(self.device) for c in self.shards]) if self.shards
                          else torch.empty(0, dtype=torch.int64))
            lists = [torch.as_tensor(filter_fn(ids.to(everything.device) if ids is not None else everything)).long()
                     for ids in lists]
        return lists

    def _listed_is_cheaper(self, Q: torch.Tensor, lists: List) -> bool:
        """Whether a batch's restricted search takes the listed scan: every query has a list, and the rows of the
        listed passages of this shard are at most LISTED_SCAN_MAX_ROW_FRACTION of what the bitmap scan streams (the
        shard's rows once per scan pass; a pass holds up to 12 queries of at most 32 tokens, fewer of longer ones)."""
        corpus = self.corpus
        if corpus is None or any(ids is None for ids in lists):
            return False
        if getattr(corpus, "residency", "device") == "host":   # a streamed corpus has no listed scan
            return False
        rbq = (Q.size(1) + 31) // 32
        per_pass = max(1, min(12, 12 // rbq)) if rbq <= 12 else 1
        n_passes = (len(lists) + per_pass - 1) // per_pass
        rows = 0
        for ids in lists:
            local = ids.cpu().numpy() - corpus.pid_base
            local = local[(local >= 0) & (local < corpus.n_passages)]
            rows += int(((corpus.doclens[local].astype(np.int64) + 3) // 4 * 4).sum())
        return rows <= LISTED_SCAN_MAX_ROW_FRACTION * n_passes * int(corpus.info.n_rows)

    def _listed_scores(self, Q: torch.Tensor, lists: List) -> Tuple[torch.Tensor, torch.Tensor]:
        """(scores fp32 ``[B, w]``, global ids ``[B, w]``) of each query against its listed passages of this shard,
        each list made sorted and unique and padded with (-inf, -1) to the longest (``maxsim_scores_listed``)."""
        corpus = self.corpus
        uniq = []
        for ids in lists:
            ids = torch.unique(ids.cpu())
            uniq.append(ids[(ids >= corpus.pid_base) & (ids < corpus.pid_base + corpus.n_passages)])
        lens = torch.tensor([len(x) for x in uniq], dtype=torch.int64)
        B, w = len(uniq), int(lens.max()) if len(uniq) else 0
        flat = torch.cat(uniq).to(corpus.device) if w else torch.empty(0, dtype=torch.int64, device=corpus.device)
        sc = maxsim_scores_listed(corpus, Q, uniq, relu=self._relu)
        rows = torch.repeat_interleave(torch.arange(B), lens).to(corpus.device)
        cols = (torch.arange(int(lens.sum())) - torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens))
        cols = cols.to(corpus.device)
        s = torch.full((B, w), float("-inf"), dtype=torch.float32, device=corpus.device)
        p = torch.full((B, w), -1, dtype=torch.int64, device=corpus.device)
        s[rows, cols] = sc
        p[rows, cols] = flat
        return s, p

    def _listed_topk(self, Q: torch.Tensor, k: int, lists: List) -> Tuple[torch.Tensor, torch.Tensor]:
        """``_allowed_topk`` for queries restricted to id lists, on the listed scan: the same (scores, global pids)."""
        corpus = self.corpus
        kq = min(k, _n_live(corpus))
        n_allowed = None
        if self.storage == "fp8" and kq > 0:
            n_allowed = int(_allowed_live_counts([corpus], lists).max(initial=0))
            kq = min(kq, n_allowed)
        if kq == 0:
            return (torch.empty((Q.size(0), 0), dtype=torch.float32, device=corpus.device),
                    torch.empty((Q.size(0), 0), dtype=torch.int64, device=corpus.device))
        if self.storage != "fp8" and kq <= _cabi.MAX_K:
            return maxsim_topk(corpus, Q, kq, relu=self._relu, pids=lists)
        if self.storage == "fp8":
            depth = shortlist_depth(kq, getattr(self.config, "ndocs", None), n_allowed)
            self._last_depth = depth
            Qb = Q.to(corpus.device).to(torch.bfloat16)
            # a -inf e4m3 score is a deleted passage or padding: it never reaches the exact re-rank
            return self._rerank(Qb, self._shortlist(Qb, depth, lists=lists)[1], kq)
        else:
            s, ids = self._listed_scores(Q, lists)
            if s.size(1) < kq:                           # fewer listed passages than kq in every row
                pad = kq - s.size(1)
                s = torch.cat([s, s.new_full((s.size(0), pad), float("-inf"))], dim=1)
                ids = torch.cat([ids, ids.new_full((ids.size(0), pad), -1)], dim=1)
            if kq <= _cabi.SELECT_MAX_K:
                vals, col = topk_select(s, kq)           # ids ascend along a row: ties go to the lower id
            else:
                vals, col = torch.sort(s, dim=1, descending=True, stable=True)
                vals, col = vals[:, :kq], col[:, :kq]
            pids = ids.gather(1, col.clamp_min(0))
        return vals, pids.masked_fill(vals == float("-inf"), -1)

    def _allowed_topk(self, Q: torch.Tensor, k: int, allow: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Top-k of this shard for queries restricted by ``allow`` (``[B, words]``): (scores, global pids)
        ``[B, min(k, live passages)]`` (fp8: at most the most allowed live passages of a query), short rows ending in
        (-inf, -1)."""
        corpus = self.corpus
        kq = min(k, _n_live(corpus))
        n_allowed = None
        if self.storage == "fp8" and kq > 0:
            # the shortlist depth follows the allowed count (the one host synchronisation of a restricted search
            # before its results)
            n_allowed = int(_popcount_rows(allow & _live_words(corpus)).max())
            kq = min(kq, n_allowed)
        if kq == 0:
            return (torch.empty((Q.size(0), 0), dtype=torch.float32, device=corpus.device),
                    torch.empty((Q.size(0), 0), dtype=torch.int64, device=corpus.device))
        if self.storage == "fp8":
            depth = shortlist_depth(kq, getattr(self.config, "ndocs", None), n_allowed)
            self._last_depth = depth
            Qb = Q.to(corpus.device).to(torch.bfloat16)
            # a -inf e4m3 score is a disallowed or deleted passage: it never reaches the exact re-rank
            return self._rerank(Qb, self._shortlist(Qb, depth, allow=allow)[1], kq)
        elif kq <= _cabi.MAX_K:
            return maxsim_topk(corpus, Q, kq, relu=self._relu, allow=allow)
        else:
            s = maxsim_scores(corpus, Q, relu=self._relu, allow=allow)
            if kq <= _cabi.SELECT_MAX_K:
                vals, pids = topk_select(s, kq, corpus.pid_base)
            else:
                vals, idx = torch.sort(s, dim=1, descending=True, stable=True)
                vals, pids = vals[:, :kq], idx[:, :kq] + corpus.pid_base
        return vals, pids.masked_fill(vals == float("-inf"), -1)

    def _search_tensors(self, Q: torch.Tensor, k: int, filter_fn=None,
                        remove_zero_tensors: bool = False, pid_lists: Optional[List] = None
                        ) -> Tuple[torch.Tensor, torch.Tensor]:
        """(scores [B,k'], pids [B,k']) on the GPU, k' = min(k, passages that pass ``filter_fn``).  With
        ``pid_lists`` (one list of global ids, or None, per query) each query searches its own set, and rows with fewer
        hits end in (-inf, -1) entries."""
        if Q.dim() == 2:
            Q = Q.unsqueeze(0)
        if remove_zero_tensors:
            Q = self._drop_zero_rows(Q)
        if self._devices is not None:
            # every shard's own search, then one merge on the home device (fp8: every shard's shortlist, then one
            # re-rank on the home device); rows end in (-inf, -1) past their hits
            if self.storage == "fp8":
                s, p = self._devices_fp8_tensors(Q, int(k), filter_fn, pid_lists)
            else:
                s, p = self._devices.search(Q, int(k), filter_fn=filter_fn, pid_lists=pid_lists)
            n_valid = int((p >= 0).sum(dim=1).max()) if p.numel() else 0
            return s[:, :n_valid], p[:, :n_valid]
        if pid_lists is not None:
            return self._restricted_tensors(Q, int(k), filter_fn, pid_lists)
        corpus = self.corpus
        keep = None
        if filter_fn is not None and corpus is not None:
            # the filter sees the live candidates only, as the reference's filter only ever sees candidates
            keep = torch.as_tensor(filter_fn(_live_pids(corpus)), device=corpus.device).long() - corpus.pid_base
        if self._sharded is not None and int(k) > _cabi.MAX_K:
            raise ValueError("sharded search merges at most k=%d results per query" % _cabi.MAX_K)
        if self._nccl is not None and keep is None and corpus is not None and self.storage != "fp8":
            # the C-level sharded search: scan + one grouped all-gather + merge per call, no torch glue
            # (fp8 shards re-rank their shortlists first, then exchange exact scores below)
            step = self._batch()
            outs = [self._nccl.search(corpus, Q[b0:b0 + step], int(k), relu=self._relu)
                    for b0 in range(0, Q.size(0), step)]
            s, p = torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])
            n_valid = int((p[0] >= 0).sum()) if p.numel() else 0
            return s[:, :n_valid], p[:, :n_valid]
        s, p = self._local_topk(Q, int(k), keep)
        if self._sharded is not None:
            k_merge = int(k)
            if s.size(1) < k_merge:                      # short shard: pad with empty entries
                s = torch.cat([s, s.new_full((s.size(0), k_merge - s.size(1)), float("-inf"))], dim=1)
                p = torch.cat([p, p.new_full((p.size(0), k_merge - p.size(1)), -1)], dim=1)
            if self._nccl is not None:
                s, p = self._nccl.exchange(s, p, k_merge)
            else:
                s, p = self._sharded.exchange(s.to(self.device), p.to(self.device), k_merge)
            n_valid = int((p[0] >= 0).sum()) if p.numel() else 0    # same for every query: min(k, candidates)
            s, p = s[:, :n_valid], p[:, :n_valid]
        return s, p

    def _shard_search(self, i: int, Q: torch.Tensor, k: int, filter_fn=None, pid_lists: Optional[List] = None
                      ) -> Tuple[torch.Tensor, torch.Tensor]:
        """``_search_tensors`` of shard i of a multi-device Searcher: this Searcher's own code on a view of it that
        holds that shard alone (ids are still checked against the whole index)."""
        return self._shard_view(i)._search_tensors(Q, k, filter_fn, False, pid_lists)

    def _shard_view(self, i: int) -> "Searcher":
        view = copy.copy(self)
        view.corpus, view.device, view._devices = self.shards[i], self.shards[i].device, None
        view.shards = [self.shards[i]]
        return view

    def _shard_shortlist(self, i: int, Q: torch.Tensor, depth: int, keep: Optional[torch.Tensor] = None,
                         lists: Optional[List] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """``_shortlist`` of shard i of a multi-device Searcher, on its device: ``keep`` (global ids, ascending) cut to
        the shard, or the id ``lists`` on the listed scan or as bitmaps, as the one-device search would scan them."""
        view = self._shard_view(i)
        c = view.corpus
        if lists is not None:
            if view._listed_is_cheaper(Q, lists):
                return view._shortlist(Q, depth, lists=lists)
            return view._shortlist(Q, depth, allow=c.allow_bitmaps(lists))
        if keep is not None:
            keep = keep.to(c.device)
            keep = keep[(keep >= c.pid_base) & (keep < c.pid_base + c.n_passages)] - c.pid_base
        return view._shortlist(Q, depth, keep=keep)

    def _devices_fp8_tensors(self, Q: torch.Tensor, k: int, filter_fn, pid_lists: Optional[List]
                             ) -> Tuple[torch.Tensor, torch.Tensor]:
        """The fp8 search of a multi-device Searcher, ranked as the one-device Searcher ranks it: the shortlist depth
        (and the allowed count it follows) over the whole index, every shard's e4m3 top-depth, the global top-depth
        selected from them on the home device, and the one-device re-rank of those candidates, with the same query
        batches, gathered from the shards that own them.  Rows end in (-inf, -1) past their hits."""
        B = Q.size(0)
        n_live = sum(_n_live(c) for c in self.shards)
        ndocs = getattr(self.config, "ndocs", None)
        lists = keep = None
        if pid_lists is not None:
            lists = self._pid_lists(pid_lists, filter_fn)
        else:
            if filter_fn is not None:
                everything = torch.cat([_live_pids(c).to(self.device) for c in self.shards])
                keep = torch.as_tensor(filter_fn(everything), device=self.device).long()
            n_cand = n_live if keep is None else int(keep.numel())
            kq = min(k, n_cand)
            if kq > 0:
                depth = shortlist_depth(k, ndocs, n_cand)
        parts = []
        for b0 in range(0, B, self.query_batch):
            Qb = Q[b0:b0 + self.query_batch].to(self.device).to(torch.bfloat16)
            lb = None
            if lists is not None:
                lb = lists[b0:b0 + self.query_batch]
                n_allowed = int(_allowed_live_counts(self.shards, lb).max(initial=0))
                kq = min(k, n_live, n_allowed)
                if kq > 0:
                    depth = shortlist_depth(kq, ndocs, n_allowed)
            if kq == 0:
                parts.append((Qb.new_empty((Qb.size(0), 0), dtype=torch.float32),
                              Qb.new_empty((Qb.size(0), 0), dtype=torch.int64)))
                continue
            self._last_depth = depth
            _, cand = self._devices.shortlist(self._shard_shortlist, Qb, depth, keep=keep, lists=lb)
            parts.append(self._rerank(Qb, cand, kq))
        width = max([ps.size(1) for ps, _ in parts], default=0)
        s = torch.full((B, width), float("-inf"), dtype=torch.float32, device=self.device)
        p = torch.full((B, width), -1, dtype=torch.int64, device=self.device)
        b0 = 0
        for ps, pp in parts:
            s[b0:b0 + ps.size(0), :ps.size(1)] = ps
            p[b0:b0 + pp.size(0), :pp.size(1)] = pp
            b0 += ps.size(0)
        return s, p

    def _longest(self, p: torch.Tensor) -> int:
        """The most tokens of a passage among global ids ``p`` (-1: none; 1 if there is none)."""
        ids = p.cpu().numpy()
        nd_max = 1
        for c in self.shards:
            local = ids[(ids >= c.pid_base) & (ids < c.pid_base + c.n_passages)] - c.pid_base
            if local.size:
                nd_max = max(nd_max, int(c.doclens[local].max()))
        return nd_max

    def _gather_padded(self, p: torch.Tensor, nd_max: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """``FlatCorpus.gather_padded`` of global ids ``p`` from the shards that own them, on the home device: each
        shard gathers its own hits on its device (``flmr_corpus_gather``) and they are copied over."""
        if len(self.shards) == 1:
            return self.corpus.gather_padded(p, nd_max)
        if nd_max is None:
            nd_max = self._longest(p)
        D = mask = None
        for c in self.shards:
            own = (p >= c.pid_base) & (p < c.pid_base + c.n_passages)
            Dc, mc = c.gather_padded(torch.where(own, p, -1), nd_max)
            Dc, mc = Dc.to(self.device), mc.to(self.device)
            if D is None:
                D, mask = Dc, mc
            else:
                D = torch.where(own[..., None, None], Dc, D)
                mask = torch.where(own[..., None, None], mc, mask)
        return D, mask

    def retrieve_and_rescore(self, Q: torch.Tensor, n_docs: int, generator: Optional[torch.Generator] = None):
        """The retrieval block of ``RagModelForBlip.main_retrieve`` (src/models/rag/rag_model_blip.py:388-443)
        in one call: search ``max(5, n_docs)`` passages per query (:392-397), keep ``n_docs`` of them (a random
        subset when ``n_docs < 5``, as :411-412 does with ``random.sample``), fetch their token embeddings and
        re-score them with the differentiable ``score`` so the gradient reaches the query encoder (:430-435).

        ``Q [B, Nq, d]`` stays on the GPU; the retrieved embeddings are gathered out of the resident corpus
        (no host dictionary, no H2D copy).  Returns a dict with ``doc_scores [B, n_docs]`` (differentiable
        w.r.t. ``Q``), ``retrieved_doc_ids`` (int64 numpy ``[B, n_docs]``, as :441), ``search_scores``, and the
        gathered ``item_embeddings [B, n_docs, Nd, d]`` / ``item_mask [B, n_docs, Nd, 1]``.  On an fp16 corpus
        ``item_embeddings`` are its fp16 rows and the re-score runs the fp16 training kernels on them, with the query
        converted to fp16 as the search converts it: ``doc_scores`` and ``search_scores`` score the same operands."""
        from .modeling import grouped_maxsim
        if Q.dim() != 3:
            raise ValueError("Q must be [B, Nq, d]")
        if self._sharded is not None:
            raise RuntimeError("retrieve_and_rescore gathers embeddings from the local shard only; "
                               "use an unsharded Searcher for the RAG block")
        n_live = sum(_n_live(c) for c in self.shards)
        if n_live < n_docs:
            raise ValueError("the corpus holds %d live passages, fewer than n_docs=%d" % (n_live, n_docs))
        n_retrieve = max(5, int(n_docs))
        Qd = Q.to(self.corpus.device)
        s, p = self._search_tensors(Qd.detach(), n_retrieve)
        if s.size(1) < n_docs:
            raise ValueError("the corpus holds %d passages, fewer than n_docs=%d" % (s.size(1), n_docs))
        if s.size(1) != n_docs:
            pick = torch.rand(s.shape, generator=generator, device="cpu").argsort(dim=1)[:, :n_docs].to(s.device)
            s, p = s.gather(1, pick), p.gather(1, pick)
        D, mask = self._gather_padded(p)                                     # [B, n_docs, Nd, d]
        # one block-diagonal launch: question b against ITS n_docs passages only
        doc_scores = grouped_maxsim(Qd, D.flatten(0, 1), mask.flatten(0, 1), n_docs)
        return {"doc_scores": doc_scores, "retrieved_doc_ids": p.cpu().numpy(), "search_scores": s,
                "item_embeddings": D, "item_mask": mask}

    def _fill_search_knobs(self, k: int) -> None:
        """searcher.py:92-118: the first search fills the PLAID knobs still unset on ``config`` from ``k`` (and later
        searches keep them).  The scan is exhaustive, so they steer nothing on a bf16 corpus — but callers that read
        ``searcher.config.ncells`` etc. after a search find what the reference would have left there.  On an fp8
        corpus ``ndocs / 4`` is the depth of the exact re-rank (``shortlist_depth``)."""
        cfg = self.config
        if cfg is None or not hasattr(cfg, "configure") or not hasattr(cfg, "ncells"):
            return
        ncells, thr, ndocs = _default_knobs(k)
        if cfg.ncells is None:
            cfg.configure(ncells=ncells)
        if cfg.centroid_score_threshold is None:
            cfg.configure(centroid_score_threshold=thr)
        if cfg.ndocs is None:
            cfg.configure(ndocs=ndocs)

    def dense_search(self, Q: torch.Tensor, k: int = 10, filter_fn=None, remove_zero_tensors: bool = False,
                     pids=None):
        """searcher.py:91-132 -> ``(pids[:k], [1..k], scores[:k])`` for ONE query ``Q [1, Nq, d]``.

        ``pids`` (later ColBERT's argument): search only this set of global ids (``filter_fn``, if given, is applied
        to it); an id outside the index raises ValueError, deleted ids are never returned."""
        if Q.dim() == 2:
            Q = Q.unsqueeze(0)
        assert Q.size(0) == 1, "dense_search takes a single query (use _search_all_Q for batches)"
        self._fill_search_knobs(k)
        s, p = self._search_tensors(Q, k, filter_fn, remove_zero_tensors, None if pids is None else [pids])
        hit = p[0] >= 0
        pids, scores = p[0][hit].tolist(), s[0][hit].tolist()
        return pids, list(range(1, len(pids) + 1)), scores

    def _search_all_Q(self, queries, Q: torch.Tensor, k: int, filter_fn=None, progress: bool = True,
                      remove_zero_tensors: bool = False, qid_to_pids=None) -> Ranking:
        """searcher.py:73-89, batched: one fused scan per ``query_batch`` queries instead of a Python
        loop of per-query ``dense_search`` calls (on a streamed corpus: one per call, see the module docstring).

        ``qid_to_pids`` (later ColBERT's argument) maps every qid to the global ids its query may return (None: the
        whole index); a qid missing from it raises KeyError.  Queries may then return fewer than k hits."""
        del progress
        self._fill_search_knobs(k)
        keys = _query_keys(queries, Q.size(0))
        lists = [qid_to_pids[qid] for qid in keys] if qid_to_pids is not None else None
        s, p = self._search_tensors(Q, k, filter_fn, remove_zero_tensors, lists)
        s, p = s.cpu().tolist(), p.cpu().tolist()
        data = {qid: [(pid, rank + 1, score) for rank, (pid, score) in enumerate((pid, sc) for pid, sc in zip(pp, ss)
                                                                                 if pid >= 0)]
                for qid, pp, ss in zip(keys, p, s)}
        prov = {"source": "Searcher::search_all", "k": k,
                "queries": queries.provenance() if hasattr(queries, "provenance") else None,
                "config": self.config.export() if hasattr(self.config, "export") else None,
                "backend": "ravqa_b200 exhaustive fused scan", "index": self.index,
                "index_kind": self.index_kind, "exhaustive": True,
                "n_passages": sum(c.n_passages for c in self.shards),
                "n_live": sum(_n_live(c) for c in self.shards),
                "n_deleted": sum(getattr(c, "n_deleted", 0) for c in self.shards),
                "storage": self.storage, "restricted": qid_to_pids is not None}
        if self.storage == "fp8":
            prov["shortlist_depth"] = self._last_depth
        return Ranking(data=data, provenance=prov)
