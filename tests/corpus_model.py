"""Float64 model of a resident corpus (``FlatCorpus``) through appends, deletions and compactions, and the seeded
operation sequences tests/test_corpus_lifecycle_gpu.py applies to the library and to the model alike.  Pinned on CPU
by tests/test_corpus_lifecycle_host.py before any kernel is judged by it.

The model does not call the library.  It holds every id ever given out (its tokens, as the values the storage holds:
bf16, fp16, or the bf16 master of an fp8 corpus, and its length), the deleted ids and the ids whose rows a compaction
removed, and applies the operations as ``FlatCorpus`` documents them:

  * ``append`` returns the next ids (they continue the id extent, whatever was compacted);
  * ``delete`` of an id outside ``[pid_base, pid_base + n_passages)`` raises and changes nothing; deleting an id that is
    already deleted (compacted away or not) changes nothing;
  * ``compact`` removes the stored deleted passages; nothing happens when there are none, and it raises (changing
    nothing) when every stored passage is deleted.

Scores are scan_fp64.maxsim_packed over every id (e4m3-rounded operands for fp8; fp16 values for fp16, held to the bf16
row coefficient: the fp16 MMA keeps the bf16 accumulator model, DESIGN.md §2), with deleted ids at -inf.
"""
from __future__ import annotations

import numpy as np
import torch

import scan_fp64 as S

STORAGES = ("bf16", "fp16", "fp8")


class ModelError(Exception):
    """An operation the model refuses, as the library refuses it (``FlmrError``)."""


def element_dtype(storage: str) -> torch.dtype:
    return torch.float16 if storage == "fp16" else torch.bfloat16


def scan_storage(storage: str) -> str:
    """The storage whose accumulator model and operand rounding the scan of ``storage`` follows."""
    return "fp8" if storage == "fp8" else "bf16"


def passage_tokens(seed: int, n_rows: int, storage: str, device="cpu") -> torch.Tensor:
    """``[n_rows, 128]`` rows in the storage's element type: gaussian directions with norms 2^-1 .. 2^1."""
    dev = torch.device(device)
    g = torch.Generator(device=dev).manual_seed(int(seed))
    x = torch.nn.functional.normalize(torch.randn(n_rows, 128, generator=g, device=dev), dim=1)
    x *= torch.exp2(2 * torch.rand(n_rows, 1, generator=g, device=dev) - 1)
    return x.to(element_dtype(storage))


def query_rows(seed: int, B: int, nq: int, storage: str, device="cpu") -> torch.Tensor:
    g = torch.Generator().manual_seed(int(seed))
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1)
    return Q.to(element_dtype(storage)).to(device)


class CorpusModel:
    """A shard's ids, tokens and deletions (``tokens`` None: the ids and lengths only, as the generator keeps them)."""

    def __init__(self, tokens, lens, pid_base: int = 0, storage: str = "bf16"):
        assert storage in STORAGES
        self.storage = storage
        self.pid_base = int(pid_base)
        self.lens = np.asarray(lens, dtype=np.int64).copy()
        assert self.lens.ndim == 1 and self.lens.size >= 1 and (self.lens >= 1).all()
        self.tokens = None if tokens is None else tokens.detach().to(element_dtype(storage)).contiguous()
        if self.tokens is not None:
            assert self.tokens.shape == (int(self.lens.sum()), 128)
        self.deleted = np.zeros(self.lens.size, dtype=bool)
        self.compacted = np.zeros(self.lens.size, dtype=bool)   # rows removed by a compaction (always deleted too)
        self.n_compactions = 0           # compactions that removed something
        self.appended_since = np.zeros(self.lens.size, dtype=bool)   # appended after the last such compaction

    # -- operations ------------------------------------------------------------------------------------------------
    def append(self, tokens, lens) -> np.ndarray:
        lens = np.asarray(lens, dtype=np.int64).reshape(-1)
        assert lens.size >= 1 and (lens >= 1).all()
        first = self.pid_base + self.lens.size
        if self.tokens is not None:
            t = tokens.detach().to(device=self.tokens.device, dtype=self.tokens.dtype)
            assert t.shape == (int(lens.sum()), 128)
            self.tokens = torch.cat([self.tokens, t])
        grow = np.zeros(lens.size, dtype=bool)
        self.lens = np.concatenate([self.lens, lens])
        self.deleted = np.concatenate([self.deleted, grow])
        self.compacted = np.concatenate([self.compacted, grow])
        self.appended_since = np.concatenate([self.appended_since, ~grow])
        return np.arange(first, first + lens.size, dtype=np.int64)

    def delete(self, pids) -> int:
        """Returns the number of ids newly deleted."""
        local = np.asarray(pids, dtype=np.int64).reshape(-1) - self.pid_base
        if ((local < 0) | (local >= self.lens.size)).any():
            raise ModelError("id outside [%d, %d)" % (self.pid_base, self.pid_base + self.lens.size))
        new = int((~self.deleted[np.unique(local)]).sum())
        self.deleted[local] = True
        return new

    def compact(self) -> int:
        """Returns the number of passages removed."""
        stored = ~self.compacted
        gone = stored & self.deleted
        if not gone.any():
            return 0
        if gone.sum() == stored.sum():
            raise ModelError("every stored passage is deleted")
        self.compacted |= gone
        self.n_compactions += 1
        self.appended_since[:] = False
        return int(gone.sum())

    # -- id sets ---------------------------------------------------------------------------------------------------
    @property
    def n_passages(self) -> int:
        return int(self.lens.size)

    @property
    def n_deleted(self) -> int:
        return int(self.deleted.sum())

    @property
    def n_live(self) -> int:
        return self.n_passages - self.n_deleted

    @property
    def n_stored(self) -> int:
        return int((~self.compacted).sum())

    def _ids(self, mask) -> np.ndarray:
        return np.flatnonzero(mask).astype(np.int64) + self.pid_base

    def live_ids(self) -> np.ndarray:
        return self._ids(~self.deleted)

    def deleted_ids(self) -> np.ndarray:
        return self._ids(self.deleted)

    def stored_ids(self) -> np.ndarray:
        return self._ids(~self.compacted)

    def compacted_ids(self) -> np.ndarray:
        return self._ids(self.compacted)

    def new_ids(self) -> np.ndarray:
        """Ids appended since the last compaction that removed rows."""
        return self._ids(self.appended_since)

    # -- answers ---------------------------------------------------------------------------------------------------
    def scores(self, Q: torch.Tensor, relu: bool = False):
        """(scores, amax, rabs), float64 ``[B, n_passages]`` on Q's device, every id (deleted ones: score -inf)."""
        Q = Q.to(element_dtype(self.storage))
        s, amax, rabs = S.maxsim_packed(Q, self.tokens.to(Q.device), self.lens, relu=relu,
                                        storage=scan_storage(self.storage))
        dead = torch.from_numpy(self.deleted).to(s.device)
        return s.masked_fill(dead, -torch.inf), amax, rabs

    def bound(self, amax, rabs, nq: int):
        """The scan's error bound of each score."""
        return S.scan_bound(amax, rabs, nq, scan_storage(self.storage))

    def exact_scores(self, Q: torch.Tensor):
        """(scores, amax, rabs) of the exact bf16 operands, no e4m3 rounding: what an fp8 corpus re-ranks with."""
        Q = Q.to(element_dtype(self.storage))
        s, amax, rabs = S.maxsim_packed(Q, self.tokens.to(Q.device), self.lens)
        dead = torch.from_numpy(self.deleted).to(s.device)
        return s.masked_fill(dead, -torch.inf), amax, rabs

    def gather(self, pids, nd_max: int):
        """``gather_padded(pids, nd_max)`` as the model holds it: (tokens ``[n, nd_max, 128]``, mask ``[n, nd_max, 1]``),
        on the tokens' device.  Deleted, compacted-away and out-of-shard ids: all-masked zero rows."""
        pids = np.asarray(pids, dtype=np.int64).reshape(-1)
        dev = self.tokens.device
        out = torch.zeros((pids.size, nd_max, 128), dtype=self.tokens.dtype, device=dev)
        mask = torch.zeros((pids.size, nd_max, 1), dtype=torch.bool, device=dev)
        local = pids - self.pid_base
        inside = (local >= 0) & (local < self.n_passages)
        ok = np.flatnonzero(inside)
        ok = ok[~self.deleted[local[ok]]]
        if ok.size:
            off = np.concatenate([[0], np.cumsum(self.lens)])
            lp = local[ok]
            n = np.minimum(self.lens[lp], nd_max)
            i = np.repeat(np.arange(ok.size), n)
            j = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
            rows = np.repeat(off[lp], n) + j
            ti, tj = torch.from_numpy(ok[i]).to(dev), torch.from_numpy(j).to(dev)
            out[ti, tj] = self.tokens[torch.from_numpy(rows).to(dev)]
            mask[ti, tj] = True
        return out, mask


# ---- seeded operation sequences ----------------------------------------------------------------------------------------
# A sequence is (spec, ops).  spec: {"storage", "pid_base", "adopt", "lens0", "seed"}.  Every op is a dict:
#   {"op": "append", "lens": [...], "src": "cpu" | "gpu", "seed": int}
#   {"op": "delete", "ids": [...], "expect": "ok" | "error"}
#   {"op": "compact", "expect": "ok" | "error"}
# with "tags": the edges the op reaches, as the generator saw the state.  Token rows are drawn from the seeds when a
# sequence is replayed, so a logged op list replays without the generator.

EDGES = ("append 1", "append few", "append past SMs", "len 1", "len <= 4", "len 95-97", "len 1000+", "src cpu",
         "src gpu", "delete one", "delete run", "delete random", "delete appended after compaction",
         "delete already deleted", "delete compacted away", "delete out of range", "compact no-op",
         "compact below SMs", "compact 2nd", "compact 3rd", "compact after append", "compact all deleted",
         "append after compact below SMs")


def _short(rng, n, adopt):
    lens = rng.integers(1, 40, n)
    return (lens + 3) // 4 * 4 if adopt else lens


class _Gen:
    def __init__(self, rng, m: CorpusModel, sms: int):
        self.rng, self.m, self.sms, self.ops = rng, m, sms, []
        self.appended_since_compact = False
        self.below_sms = False

    def _src(self):
        return "gpu" if self.rng.random() < 0.5 else "cpu"

    def append(self, lens, tags):
        lens = [int(x) for x in lens]
        src = self._src()
        tags = list(tags) + ["src " + src]
        if self.below_sms and self.m.n_stored + len(lens) > self.sms:
            tags.append("append after compact below SMs")
        self.m.append(None, lens)
        self.appended_since_compact = True
        self.ops.append({"op": "append", "lens": lens, "src": src, "seed": int(self.rng.integers(1 << 30)),
                         "tags": tags})

    def delete(self, ids, tags=()):
        ids = np.asarray(ids, dtype=np.int64)
        tags = list(tags)
        local = ids - self.m.pid_base
        inside = local[(local >= 0) & (local < self.m.n_passages)]
        if self.m.deleted[inside].any():
            tags.append("delete already deleted")
        if self.m.compacted[inside].any():
            tags.append("delete compacted away")
        if self.m.n_compactions and self.m.appended_since[inside].any():
            tags.append("delete appended after compaction")
        try:
            self.m.delete(ids)
            expect = "ok"
        except ModelError:
            expect = "error"
            tags.append("delete out of range")
        self.ops.append({"op": "delete", "ids": ids.tolist(), "expect": expect, "tags": tags})

    def compact(self):
        tags = []
        if self.appended_since_compact and self.m.n_compactions:
            tags.append("compact after append")
        try:
            removed = self.m.compact()
            expect = "ok"
        except ModelError:
            removed, expect = 0, "error"
            tags.append("compact all deleted")
        if expect == "ok" and removed == 0:
            tags.append("compact no-op")
        if removed:
            self.appended_since_compact = False
            self.below_sms = self.m.n_stored < self.sms
            if self.below_sms:
                tags.append("compact below SMs")
            if self.m.n_compactions in (2, 3):
                tags.append("compact %s" % {2: "2nd", 3: "3rd"}[self.m.n_compactions])
        self.ops.append({"op": "compact", "expect": expect, "tags": tags})

    # -- episodes --------------------------------------------------------------------------------------------------
    def ep_append(self, adopt):
        self.append([1], ["append 1", "len 1"])
        few = [int(self.rng.integers(2, 5)), int(self.rng.integers(95, 98)), int(self.rng.integers(1000, 1101))]
        few += _short(self.rng, int(self.rng.integers(0, 4)), False).tolist()
        self.append(self.rng.permutation(few), ["append few", "len <= 4", "len 95-97", "len 1000+"])

    def ep_delete(self):
        m, rng = self.m, self.rng
        live = m.live_ids()
        if live.size:
            self.delete([rng.choice(live)], ["delete one"])
        a = int(rng.integers(0, m.n_passages))
        self.delete(np.arange(a, min(m.n_passages, a + int(rng.integers(5, 40)))) + m.pid_base, ["delete run"])
        k = max(1, m.n_passages // int(rng.integers(8, 20)))
        self.delete(rng.choice(m.n_passages, k, replace=False) + m.pid_base, ["delete random"])

    def ep_delete_new(self):
        new = self.m.new_ids()
        if new.size:
            self.delete(self.rng.choice(new, max(1, new.size // 3), replace=False))

    def ep_refusals(self):
        m, rng = self.m, self.rng
        live = m.live_ids()
        bad = m.pid_base + m.n_passages if rng.random() < 0.5 else m.pid_base - 1
        self.delete(np.concatenate([live[:3], [bad]]))
        old = np.concatenate([m.compacted_ids()[:4], m.deleted_ids()[-4:]])
        if old.size:
            self.delete(old)

    def ep_compact(self):
        m = self.m
        stored_live = np.setdiff1d(m.stored_ids(), m.deleted_ids())
        if not m.deleted[m.stored_ids() - m.pid_base].any() and stored_live.size > 1:
            self.delete([self.rng.choice(stored_live)], ["delete one"])    # so that this compaction removes a row
        self.compact()
        self.compact()

    def ep_shrink(self):
        m, rng = self.m, self.rng
        stored_live = np.setdiff1d(m.stored_ids(), m.deleted_ids())
        keep = int(rng.integers(self.sms // 4, self.sms // 2))
        if stored_live.size > keep:
            self.delete(rng.choice(stored_live, stored_live.size - keep, replace=False), ["delete random"])
        self.compact()
        self.append(_short(rng, self.sms + int(rng.integers(10, 80)), False), ["append past SMs"])

    def ep_all_deleted(self):
        m = self.m
        stored_live = np.setdiff1d(m.stored_ids(), m.deleted_ids())
        if stored_live.size:
            self.delete(stored_live)
        self.compact()
        self.append(_short(self.rng, int(self.rng.integers(2, 6)), False), [])


# (seed, storage, pid_base, adopted start) of every generated sequence tests/test_corpus_lifecycle_gpu.py runs: each
# storage with pid_base 0 and not 0, started from an adopted CUDA matrix (bf16, fp16) or from a copy
SEQUENCE_CASES = [(11, "bf16", 0, True), (12, "bf16", 1000, False), (13, "bf16", 0, False), (14, "bf16", 333, True),
                  (15, "fp16", 0, True), (16, "fp16", 1000, False), (17, "fp16", 0, False), (18, "fp16", 77, True),
                  (19, "fp8", 0, False), (20, "fp8", 1000, False)]


def initial_lens(rng, n, adopt, long=True):
    """Lengths of a sequence's starting corpus: short ones with a few 95-97 and 1000+ passages (multiples of 4 when the
    token matrix is adopted)."""
    lens = _short(rng, n, adopt)
    lens[rng.choice(n, 8, replace=False)] = rng.integers(95, 98, 8)
    if long:
        lens[rng.choice(n, 2, replace=False)] = rng.integers(1000, 1101, 2)
    if adopt:
        lens = (lens + 3) // 4 * 4
    return lens.astype(np.int64)


def generate(seed: int, storage: str = "bf16", pid_base: int = 0, adopt: bool = False, sms: int = 132):
    """A seeded sequence of about 25 operations that reaches every edge in EDGES: the episodes below in a random order,
    each drawing its ids from the state the earlier ones left."""
    rng = np.random.default_rng(seed)
    lens0 = initial_lens(rng, int(rng.integers(sms + 100, sms + 300)), adopt)
    spec = {"storage": storage, "pid_base": int(pid_base), "adopt": bool(adopt), "lens0": lens0.tolist(),
            "seed": int(seed), "src0": "gpu" if adopt or rng.random() < 0.5 else "cpu"}
    g = _Gen(rng, CorpusModel(None, lens0, pid_base, storage), sms)
    episodes = ["append", "delete", "compact", "delete_new", "refusals", "shrink", "append", "delete", "compact",
                "all_deleted", "delete_new", "compact"]
    order = rng.permutation(len(episodes) - 1)
    for i in list(order) + [len(episodes) - 1]:      # the sequence ends on a compaction
        name = episodes[i]
        if name == "append":
            g.ep_append(adopt)
        else:
            getattr(g, "ep_" + name)()
    return spec, g.ops


def large_sequence(seed: int, sms: int = 132, rows: int = (1 << 30) // 256 + (1 << 18)):
    """A bf16 sequence whose token matrix outgrows one 1 GiB physical piece: its first compaction releases pieces and a
    later append maps them again.  ``rows`` token rows of 60..180-token passages, copied from the GPU."""
    rng = np.random.default_rng(seed)
    lens0 = []
    total = 0
    while total < rows:
        x = int(rng.integers(15, 46)) * 4
        lens0.append(x)
        total += x
    lens0 = np.asarray(lens0, dtype=np.int64)
    n = lens0.size
    spec = {"storage": "bf16", "pid_base": 7, "adopt": False, "lens0": lens0.tolist(), "seed": int(seed),
            "src0": "gpu"}
    g = _Gen(rng, CorpusModel(None, lens0, 7, "bf16"), sms)
    g.delete(np.sort(rng.choice(n, n * 2 // 5, replace=False)) + 7, ["delete random"])
    g.compact()
    big = rng.integers(60, 181, n // 2)
    g.append(big, ["append few"])
    g.delete(rng.choice(g.m.new_ids(), 500, replace=False))
    g.compact()
    g.append([1, 3, 96, 1024], ["append few"])
    return spec, g.ops
