"""Passage-sharded search across the GPUs of one box (SURVEY.md §8e).

The reference does not shard: under DDP every rank repeats the whole search on CPU
(src/executors/FLMR_executor.py:778-796).  Here rank r keeps a contiguous range of passages
resident (token-balanced), every rank scans its shard with the fused kernel, and ONE collective —
an all-gather of the per-shard top-k ``[B, k]`` (fp32 score, int64 pid) — precedes a tiny merge
kernel on every rank.  No data-path collective touches the token matrix.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist


def shard_ranges(doclens: Sequence[int], world_size: int) -> List[Tuple[int, int]]:
    """Contiguous passage ranges balanced by TOKEN count (ragged corpora), one per rank."""
    doclens = np.asarray(doclens, dtype=np.int64)
    n = len(doclens)
    off = np.concatenate([[0], np.cumsum(doclens)])
    bounds = [0]
    for r in range(1, world_size):
        target = off[-1] * r // world_size
        p = int(np.searchsorted(off, target, side="left"))
        bounds.append(min(max(p, bounds[-1]), n))
    bounds.append(n)
    return [(bounds[r], bounds[r + 1]) for r in range(world_size)]


class NcclExchange:
    """This rank's end of the C-level exchange (``flmr_comm_*`` / ``flmr_maxsim_topk_sharded`` /
    ``flmr_topk_exchange``): the library's own NCCL communicator, created from an id that rank 0 obtains and
    ``torch.distributed`` broadcasts once.  Per search: the fused scan, ONE grouped all-gather and the merge
    kernel, all enqueued by one C call on the current stream — no tensor packing or casting on the way."""

    def __init__(self, device: torch.device, group=None):
        import ctypes as C
        from . import _cabi
        L = _cabi.lib()
        self.device = device
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        uid = torch.zeros(128, dtype=torch.uint8)
        if self.rank == 0:
            buf = (C.c_char * 128)()
            _cabi.check(L.flmr_comm_unique_id(C.cast(buf, C.c_void_p)))
            uid = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        backend = dist.get_backend(group)
        uid = uid.to(device) if backend == "nccl" else uid
        dist.broadcast(uid, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        raw = bytes(uid.cpu().numpy().tobytes())
        self._h = C.c_void_p()
        with torch.cuda.device(device):
            _cabi.check(L.flmr_comm_create(C.c_char_p(raw), self.rank, self.world, int(device.index), C.byref(self._h)))

    def search(self, corpus, Q: torch.Tensor, k: int, relu: bool = False,
               allow: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """``flmr_maxsim_topk_sharded``: (scores [B, k], global pids [B, k]) of the MERGED ranking, on every rank.
        ``allow``: this rank's bitmaps of its own shard (``maxsim_topk``'s argument; ``allow_bitmaps`` with the
        shard's ``n_passages`` and ``pid_base`` builds them from global id lists); short lists end in (-inf, -1)."""
        import ctypes as C
        from . import _cabi
        from .maxsim import _prep_allow, _prep_queries
        Qd = _prep_queries(corpus, Q)
        B, nq = Qd.size(0), Qd.size(1)
        allow, stride = _prep_allow(corpus, allow, B)
        s = torch.empty((B, k), dtype=torch.float32, device=self.device)
        p = torch.empty((B, k), dtype=torch.int64, device=self.device)
        flags = _cabi.FLAG_RELU if relu else 0
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        with torch.cuda.device(self.device):
            if allow is None:
                _cabi.check(_cabi.lib().flmr_maxsim_topk_sharded(
                    corpus.handle, corpus.workspace(), self._h, C.c_void_p(Qd.data_ptr()), B, nq, k, flags,
                    C.c_void_p(s.data_ptr()), C.c_void_p(p.data_ptr()), stream))
            else:
                _cabi.check(_cabi.lib().flmr_maxsim_topk_sharded_allowed(
                    corpus.handle, corpus.workspace(), self._h, C.c_void_p(Qd.data_ptr()), B, nq, k, flags,
                    C.c_void_p(allow.data_ptr()), stride, C.c_void_p(s.data_ptr()), C.c_void_p(p.data_ptr()),
                    stream))
        return s, p

    def exchange(self, s: torch.Tensor, p: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """``flmr_topk_exchange`` for lists the caller already has (``[B, k_in]``, pid < 0 = empty entry)."""
        import ctypes as C
        from . import _cabi
        s = s.to(self.device, torch.float32).contiguous()
        p = p.to(self.device, torch.int64).contiguous()
        B, k_in = s.shape
        out_s = torch.empty((B, k), dtype=torch.float32, device=self.device)
        out_p = torch.empty((B, k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _cabi.check(_cabi.lib().flmr_topk_exchange(
                self._h, C.c_void_p(s.data_ptr()), C.c_void_p(p.data_ptr()), B, k_in, k,
                C.c_void_p(out_s.data_ptr()), C.c_void_p(out_p.data_ptr()),
                C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
        return out_s, out_p

    def close(self):
        from . import _cabi
        if self._h is not None:
            torch.cuda.synchronize(self.device)
            _cabi.lib().flmr_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShardedSearcher:
    """``local_topk(Q, k) -> (scores [B,k], pids [B,k])`` runs on this rank's shard (global pids);
    ``merge(scores [R,B,k], pids [R,B,k], k) -> (scores [B,k], pids [B,k])`` merges the gathered
    lists.  The product wiring (``from_corpus``) uses the CUDA scan + merge kernels; the CPU/gloo
    tests inject oracle-backed callables to exercise the sharding and exchange logic without a GPU.
    """

    def __init__(self, local_topk: Callable, merge: Callable, group=None):
        self.local_topk = local_topk
        self.merge = merge
        self.group = group

    @classmethod
    def from_corpus(cls, corpus, group=None, relu: bool = False) -> "ShardedSearcher":
        from .maxsim import maxsim_topk, topk_merge
        return cls(lambda Q, k: maxsim_topk(corpus, Q, k, relu=relu),
                   lambda s, p, k: topk_merge(s, p, k), group)

    def search(self, Q: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
        s, p = self.local_topk(Q, k)
        return self.exchange(s, p, k)

    def exchange(self, s: torch.Tensor, p: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """The one exchange step: all-gather of every rank's ``[B, k_local]`` list, then the merge.  Scores
        travel as their bit patterns next to the pids in ONE pre-shaped int64 buffer (one collective, no
        per-rank tensor list); a shard with fewer than ``k`` passages pads its list with (-inf, -1) entries,
        which the merge ignores."""
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        if world == 1:
            return self.merge(s.unsqueeze(0), p.unsqueeze(0), k)
        B, kl = s.shape
        if kl < k:                                  # short shard (k > its passages, or an empty filter)
            s = torch.cat([s, s.new_full((B, k - kl), float("-inf"))], dim=1)
            p = torch.cat([p, p.new_full((B, k - kl), -1)], dim=1)
        payload = torch.empty((2, B, k), dtype=torch.int64, device=s.device)
        payload[0] = s.contiguous().view(torch.int32)
        payload[1] = p
        gathered = torch.empty((world, 2, B, k), dtype=torch.int64, device=s.device)
        if dist.get_backend(self.group) == "nccl":
            dist.all_gather_into_tensor(gathered, payload, group=self.group)
        else:                                        # gloo (CPU tests) has no flat all-gather
            dist.all_gather(list(gathered.unbind(0)), payload, group=self.group)
        gs = gathered[:, 0].to(torch.int32).view(torch.float32)
        return self.merge(gs, gathered[:, 1], k)


def resolve_devices(devices) -> List[int]:
    """The device ordinals of ``Searcher(devices=...)``: ``"all"`` (every visible device) or a non-empty sequence of
    ordinals or CUDA devices, in shard order; a device may repeat (several shards on one GPU)."""
    if isinstance(devices, str):
        if devices != "all":
            raise ValueError("devices must be 'all' or a sequence of CUDA devices, got %r" % (devices,))
        n = torch.cuda.device_count()
        if n == 0:
            raise RuntimeError("devices='all' found no CUDA device")
        return list(range(n))
    out = []
    for d in devices:
        d = torch.device("cuda", d) if isinstance(d, int) else torch.device(d)
        if d.type != "cuda" or d.index is None:
            raise ValueError("devices takes CUDA device ordinals, got %r" % (d,))
        out.append(d.index)
    if not out:
        raise ValueError("devices needs at least one device")
    return out


def merge_device_lists(lists: List[Tuple[torch.Tensor, torch.Tensor]], streams: List[torch.cuda.Stream], k: int,
                       home: torch.device, select: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """The exchange of shards held on several devices of this process, on the current stream of ``home``: list i,
    (scores fp32, pids int64) ``[B, k]`` on its own device, was written on ``streams[i]``.  k <= MAX_K: one
    ``flmr_topk_merge_devices`` call (its kernel reads the lists in place or over peer access, after waiting for each
    stream's event).  Larger k, or ``select``: the lists, copied to ``home``, are concatenated in shard order and
    selected by score; the shards hold ascending id ranges and each list is sorted with ties on the lower id, so the
    lower column is the lower id on every exact tie, as in the merge kernel."""
    import ctypes as C
    from . import _cabi
    from .maxsim import topk_select
    caller = torch.cuda.current_stream(home)
    B = lists[0][0].size(0)
    for s, p in lists:
        s.record_stream(caller)                    # read on the home stream after the shard's own stream is done
        p.record_stream(caller)
    if k <= _cabi.MAX_K and not select:
        n = len(lists)
        out_s = torch.empty((B, k), dtype=torch.float32, device=home)
        out_p = torch.empty((B, k), dtype=torch.int64, device=home)
        sp = (C.c_void_p * n)(*[s.data_ptr() for s, _ in lists])
        pp = (C.c_void_p * n)(*[p.data_ptr() for _, p in lists])
        dev = (C.c_int * n)(*[s.device.index for s, _ in lists])
        sts = (C.c_void_p * n)(*[st.cuda_stream for st in streams])
        with torch.cuda.device(home):
            _cabi.check(_cabi.lib().flmr_topk_merge_devices(sp, pp, dev, sts, n, B, k, k, C.c_void_p(out_s.data_ptr()),
                                                           C.c_void_p(out_p.data_ptr()),
                                                           C.c_void_p(caller.cuda_stream)))
        return out_s, out_p
    for st in streams:
        caller.wait_stream(st)
    s = torch.cat([s.to(home) for s, _ in lists], dim=1)
    p = torch.cat([p.to(home) for _, p in lists], dim=1)
    if k <= _cabi.SELECT_MAX_K:
        vals, col = topk_select(s, k)
    else:
        vals, col = torch.sort(s, dim=1, descending=True, stable=True)
        vals, col = vals[:, :k], col[:, :k]
    return vals, p.gather(1, col).masked_fill(vals == float("-inf"), -1)


class DeviceShardedSearcher:
    """The single-process counterpart of ``ShardedSearcher``, with the same two parts: shard i of one index lives on
    ``devices[i]`` of this process, ``local_topk(i, Q, k, **kw) -> (scores [B, k_i], global pids [B, k_i])`` searches
    it (on the current stream of its device), and ``merge(lists, streams, k, home)`` merges the per-shard lists on the
    home device ``devices[0]`` (``merge_device_lists``).  There is no collective and no host synchronisation between
    the shards: each shard runs on a stream of its own, ordered after the caller's stream on the home device."""

    def __init__(self, devices: Sequence[int], local_topk: Callable, merge: Callable = merge_device_lists):
        self.devices = [torch.device("cuda", int(d)) for d in devices]
        self.home = self.devices[0]
        self.local_topk = local_topk
        self.merge = merge
        self.streams = [torch.cuda.Stream(device=d) for d in self.devices]

    def search(self, Q: torch.Tensor, k: int, **kw) -> Tuple[torch.Tensor, torch.Tensor]:
        """(scores [B, k], global pids [B, k]) of the merged ranking, on the home device's current stream; entries past
        the candidates are (-inf, -1).  Each shard's stream receives a copy of ``Q`` and the shard's top-k, padded to
        ``k``; for k beyond the merge kernel the padded lists are copied to the home device on that stream."""
        from . import _cabi
        return self.merge(self._lists(self.local_topk, Q, k, k > _cabi.MAX_K, kw), self.streams, k, self.home)

    def shortlist(self, local: Callable, Q: torch.Tensor, depth: int, **kw) -> Tuple[torch.Tensor, torch.Tensor]:
        """The global top-``depth`` (scores [B, depth], global pids [B, depth]) of the shards' own top-``depth`` lists
        ``local(i, Q, depth, **kw)``, selected on the home device by score with ties on the lower id at every depth
        (``merge_device_lists(select=True)``): the first stage of a two-stage search, as one device would select it."""
        return merge_device_lists(self._lists(local, Q, depth, True, kw), self.streams, depth, self.home, select=True)

    def _lists(self, local: Callable, Q: torch.Tensor, k: int, to_home: bool, kw: dict) -> List:
        caller = torch.cuda.current_stream(self.home)
        lists = []
        for i, (dev, st) in enumerate(zip(self.devices, self.streams)):
            st.wait_stream(caller)
            with torch.cuda.device(dev), torch.cuda.stream(st):
                s, p = local(i, Q.to(dev, non_blocking=True), k, **kw)
                if s.size(1) < k:                        # short shard: pad with empty entries
                    s = torch.cat([s, s.new_full((s.size(0), k - s.size(1)), float("-inf"))], dim=1)
                    p = torch.cat([p, p.new_full((p.size(0), k - p.size(1)), -1)], dim=1)
                s, p = s.contiguous(), p.contiguous()
                if to_home:
                    s, p = s.to(self.home), p.to(self.home)
            lists.append((s, p))
        return lists
