"""Functional surface of the hot path: MaxSim scores and fused top-k over a resident corpus, plus
drop-in equivalents of the reference's scoring functions (same names, argument meaning and error
behaviour as third_party/ColBERT/colbert/modeling/colbert.py:235-311) that run on the CUDA path.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from . import _cabi
from .corpus import FlatCorpus


def _prep_queries(corpus: FlatCorpus, Q: torch.Tensor) -> torch.Tensor:
    if Q.dim() == 2:
        Q = Q.unsqueeze(0)
    if Q.dim() != 3 or Q.size(-1) != _cabi.DIM:
        raise ValueError("Q must be [n_queries, nq, %d], got %s" % (_cabi.DIM, tuple(Q.shape)))
    Q = Q.detach()
    if not Q.is_cuda or Q.device != corpus.device:
        Q = Q.to(corpus.device, non_blocking=True)   # H2D of the caller's dtype, cast on the device
    return Q.to(corpus.dtype).contiguous()           # the corpus' query type: fp16 on an fp16 corpus, else bf16


def _stream(corpus: FlatCorpus) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(corpus.device).cuda_stream)


def _prep_allow(corpus: FlatCorpus, allow: Optional[torch.Tensor], B: int) -> Tuple[Optional[torch.Tensor], int]:
    """(bitmaps on the corpus' device, stride in words) for ``allow`` = int32 ``[B, words]`` (one bitmap per query) or
    ``[words]`` (shared, stride 0), ``words = ceil(n_passages / 32)``; ``(None, 0)`` for no restriction."""
    if allow is None:
        return None, 0
    words = (corpus.n_passages + 31) // 32
    if allow.dtype != torch.int32 or allow.shape not in ((B, words), (words,)):
        raise ValueError("allow must be int32 [%d, %d] or [%d] (see allow_bitmaps), got %s %s"
                         % (B, words, words, allow.dtype, tuple(allow.shape)))
    allow = allow.to(corpus.device).contiguous()
    return allow, (words if allow.dim() == 2 else 0)


def _prep_lists(corpus: FlatCorpus, pids, B: int) -> Tuple[np.ndarray, torch.Tensor]:
    """(host CSR offsets int64 ``[B + 1]``, the concatenated ids on the corpus' device) of ``pids``: one sequence or
    tensor of GLOBAL ids per query."""
    if len(pids) != B:
        raise ValueError("pids holds %d lists for %d queries" % (len(pids), B))
    lists = []
    for ids in pids:
        if ids is None:
            raise ValueError("pids= takes one list of ids per query (None: use maxsim_topk without pids)")
        lists.append(torch.as_tensor(ids, dtype=torch.int64).reshape(-1))
    off = np.zeros(B + 1, dtype=np.int64)
    off[1:] = np.cumsum([x.numel() for x in lists])
    flat = (torch.cat([x.to(corpus.device) for x in lists]) if off[-1] else
            torch.empty(0, dtype=torch.int64, device=corpus.device))
    return off, flat.contiguous()


def maxsim_scores_listed(corpus: FlatCorpus, Q: torch.Tensor, pids, relu: bool = False) -> torch.Tensor:
    """Scores of query b against each global id of ``pids[b]``: fp32 ``[sum of the list lengths]``, the lists'
    entries in order (query 0's first).  The scan streams only the listed passages' rows; each score is bitwise the
    ``maxsim_scores(..., allow=...)`` entry of the pair.  An id outside the shard, deleted or compacted away scores -inf;
    duplicates score alike."""
    Qd = _prep_queries(corpus, Q)
    B, nq = Qd.size(0), Qd.size(1)
    off, flat = _prep_lists(corpus, pids, B)
    out = torch.empty(int(off[-1]), dtype=torch.float32, device=corpus.device)
    if B == 0 or out.numel() == 0:
        return out
    with torch.cuda.device(corpus.device):
        _cabi.check(_cabi.lib().flmr_maxsim_scores_listed(
            corpus.handle, corpus.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, _cabi.FLAG_RELU if relu else 0,
            off.ctypes.data_as(C.c_void_p), C.c_void_p(flat.data_ptr()), C.c_void_p(out.data_ptr()),
            _stream(corpus)))
    return out


def maxsim_scores(corpus: FlatCorpus, Q: torch.Tensor, relu: bool = False,
                  out: Optional[torch.Tensor] = None, allow: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out[b, p] = sum_i max_j <Q[b,i], D_p[j]>`` for every passage of the shard (fp32, on GPU).

    ``allow`` (see ``allow_bitmaps``) restricts query b to the local passages whose bit is set in its bitmap: the
    others score -inf, as deleted passages do; allowed scores are bitwise those of the unrestricted call."""
    Qd = _prep_queries(corpus, Q)
    B, nq = Qd.size(0), Qd.size(1)
    allow, stride = _prep_allow(corpus, allow, B)
    if out is None:
        out = torch.empty((B, corpus.n_passages), dtype=torch.float32, device=corpus.device)
    elif out.shape != (B, corpus.n_passages) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError("out must be a contiguous fp32 [n_queries, n_passages] CUDA tensor")
    if B == 0:
        return out
    with torch.cuda.device(corpus.device):
        flags = _cabi.FLAG_RELU if relu else 0
        if allow is None:
            _cabi.check(_cabi.lib().flmr_maxsim_scores(
                corpus.handle, corpus.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, flags,
                C.c_void_p(out.data_ptr()), _stream(corpus)))
        else:
            _cabi.check(_cabi.lib().flmr_maxsim_scores_allowed(
                corpus.handle, corpus.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, flags,
                C.c_void_p(allow.data_ptr()), stride, C.c_void_p(out.data_ptr()), _stream(corpus)))
    return out


def maxsim_topk(corpus: FlatCorpus, Q: torch.Tensor, k: int, relu: bool = False,
                allow: Optional[torch.Tensor] = None, pids=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Fused scan + top-k: ``(scores fp32 [B,k], pids int64 [B,k])`` sorted by descending score.

    ``allow`` (see ``maxsim_scores``): query b ranks only its allowed live passages; a list with fewer than k of them
    is filled with (-inf, -1).  ``pids`` (one sequence or tensor of GLOBAL ids per query, in any order, duplicates and
    ids outside the shard allowed) restricts query b to the ids ``pids[b]`` at the cost of those passages: the scan
    streams only their rows.  The result is bitwise that of ``allow=allow_bitmaps(pids, ...)``."""
    if not 1 <= k <= _cabi.MAX_K:
        raise ValueError("k=%d outside [1, %d]" % (k, _cabi.MAX_K))
    if allow is not None and pids is not None:
        raise ValueError("pass allow= or pids=, not both")
    Qd = _prep_queries(corpus, Q)
    B, nq = Qd.size(0), Qd.size(1)
    allow, stride = _prep_allow(corpus, allow, B)
    lists = _prep_lists(corpus, pids, B) if pids is not None else None
    scores = torch.empty((B, k), dtype=torch.float32, device=corpus.device)
    pids = torch.empty((B, k), dtype=torch.int64, device=corpus.device)
    if B == 0:
        return scores, pids
    with torch.cuda.device(corpus.device):
        flags = _cabi.FLAG_RELU if relu else 0
        if lists is not None:
            off, flat = lists
            _cabi.check(_cabi.lib().flmr_maxsim_topk_listed(
                corpus.handle, corpus.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, k, flags,
                off.ctypes.data_as(C.c_void_p), C.c_void_p(flat.data_ptr()), C.c_void_p(scores.data_ptr()),
                C.c_void_p(pids.data_ptr()), _stream(corpus)))
        elif allow is None:
            _cabi.check(_cabi.lib().flmr_maxsim_topk(
                corpus.handle, corpus.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, k, flags,
                C.c_void_p(scores.data_ptr()), C.c_void_p(pids.data_ptr()), _stream(corpus)))
        else:
            _cabi.check(_cabi.lib().flmr_maxsim_topk_allowed(
                corpus.handle, corpus.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, k, flags,
                C.c_void_p(allow.data_ptr()), stride, C.c_void_p(scores.data_ptr()),
                C.c_void_p(pids.data_ptr()), _stream(corpus)))
    return scores, pids


def topk_merge(scores: torch.Tensor, pids: torch.Tensor, k_out: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Merge ``[n_lists, B, k_in]`` candidate lists into ``[B, k_out]`` (score desc, pid asc)."""
    if scores.shape != pids.shape or scores.dim() != 3:
        raise ValueError("scores/pids must both be [n_lists, n_queries, k_in]")
    dev = scores.device
    s = scores.detach().to(torch.float32).contiguous()
    p = pids.detach().to(torch.int64).contiguous()
    L_, B, k_in = s.shape
    out_s = torch.empty((B, k_out), dtype=torch.float32, device=dev)
    out_p = torch.empty((B, k_out), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(_cabi.lib().flmr_topk_merge(
            C.c_void_p(s.data_ptr()), C.c_void_p(p.data_ptr()), L_, B, k_in, k_out,
            C.c_void_p(out_s.data_ptr()), C.c_void_p(out_p.data_ptr()), int(dev.index),
            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out_s, out_p


def topk_select(scores: torch.Tensor, k: int, pid_base: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Top-k of dense score rows ``[B, n]`` on the GPU for k up to 2048 (radix select kernel): the path
    for k beyond the fused capacity.  Returns (scores [B,k], pids [B,k]) sorted, ties by lower pid."""
    if scores.dim() != 2 or not scores.is_cuda:
        raise ValueError("scores must be a CUDA [n_queries, n] tensor")
    if not 1 <= k <= _cabi.SELECT_MAX_K:
        raise ValueError("k=%d outside [1, %d]" % (k, _cabi.SELECT_MAX_K))
    s = scores.detach().to(torch.float32).contiguous()
    B, n = s.shape
    out_s = torch.empty((B, k), dtype=torch.float32, device=s.device)
    out_p = torch.empty((B, k), dtype=torch.int64, device=s.device)
    if B == 0:
        return out_s, out_p
    with torch.cuda.device(s.device):
        _cabi.check(_cabi.lib().flmr_topk_select(
            C.c_void_p(s.data_ptr()), B, n, k, int(pid_base), C.c_void_p(out_s.data_ptr()),
            C.c_void_p(out_p.data_ptr()), int(s.device.index),
            C.c_void_p(torch.cuda.current_stream(s.device).cuda_stream)))
    return out_s, out_p


def _train_operands(Q: torch.Tensor, D_padded: torch.Tensor):
    """The operands of the arg-max / backward kernels and their element type.  fp16 documents (what the reference's
    ColBERT.doc returns on the GPU, colbert.py:205-206) keep their precision: both operands go to the fp16 kernels,
    the query converted to fp16 as colbert_score converts it to the documents' dtype (:284).  Any other document dtype
    takes the bf16 kernels, both operands rounded to bf16."""
    if not (Q.is_cuda and D_padded.is_cuda):
        raise RuntimeError("the scoring path is CUDA-only (no CPU fallback)")
    if Q.dim() != 3 or D_padded.dim() != 3 or Q.size(2) != _cabi.DIM or D_padded.size(2) != _cabi.DIM:
        raise ValueError("expected Q [B, Nq, %d] and D [n, Nd, %d]" % (_cabi.DIM, _cabi.DIM))
    dtype = torch.float16 if D_padded.dtype == torch.float16 else torch.bfloat16
    return Q.detach().to(dtype).contiguous(), D_padded.detach().to(dtype).contiguous()


def _train_call(name: str, operand: torch.Tensor):
    """The C entry point ``name`` for the element type of ``operand``: its ``_fp16`` form for fp16 operands."""
    return getattr(_cabi.lib(), name + "_fp16" if operand.dtype == torch.float16 else name)


def ib_loss_head(rowmax: torch.Tensor, nway: int, label0: int = 0):
    """``flmr_ib_loss`` on the ``[B, n, Nq]`` row maxima of ``maxsim_argmax``: returns (scores ``[B, n]``, per-query
    losses ``[B]`` — the in-batch-negatives loss is their mean —, d mean-loss / d scores ``[B, n]``)."""
    if rowmax.dim() != 3 or rowmax.dtype != torch.float32 or not rowmax.is_cuda:
        raise ValueError("rowmax must be a CUDA fp32 [B, n, Nq] tensor")
    r = rowmax.contiguous()
    B, n, nq = r.shape
    scores = torch.empty((B, n), dtype=torch.float32, device=r.device)
    loss_q = torch.empty((B,), dtype=torch.float32, device=r.device)
    dscores = torch.empty((B, n), dtype=torch.float32, device=r.device)
    with torch.cuda.device(r.device):
        _cabi.check(_cabi.lib().flmr_ib_loss(
            C.c_void_p(r.data_ptr()), B, n, nq, int(nway), int(label0), C.c_void_p(scores.data_ptr()),
            C.c_void_p(loss_q.data_ptr()), C.c_void_p(dscores.data_ptr()), int(r.device.index),
            C.c_void_p(torch.cuda.current_stream(r.device).cuda_stream)))
    return scores, loss_q, dscores


def maxsim_argmax_grouped(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, docs_per_query: int,
                          return_rowmax: bool = False):
    """Block-diagonal ``maxsim_argmax``: query ``b`` meets only documents ``[b*r, (b+1)*r)``, ``r =
    docs_per_query`` (``D_padded`` holds ``B*r`` documents).  Returns ``arg`` int32 ``[B, r, Nq]`` (and the
    maxima, fp32, same shape): ``rowmax.sum(-1)`` is the aligned score matrix ``[B, r]``."""
    Qb, Db = _train_operands(Q, D_padded)
    B, nq, n, nd = Qb.size(0), Qb.size(1), Db.size(0), Db.size(1)
    r = int(docs_per_query)
    if r < 1 or n != B * r:
        raise ValueError("expected %d x %d documents, got %d" % (B, r, n))
    mask = D_mask.reshape(n, nd).to(device=Qb.device, dtype=torch.uint8).contiguous()
    arg = torch.empty((B, r, nq), dtype=torch.int32, device=Qb.device)
    rowmax = torch.empty((B, r, nq), dtype=torch.float32, device=Qb.device) if return_rowmax else None
    with torch.cuda.device(Qb.device):
        _cabi.check(_train_call("flmr_maxsim_argmax_grouped", Db)(
            C.c_void_p(Qb.data_ptr()), B, nq, C.c_void_p(Db.data_ptr()), C.c_void_p(mask.data_ptr()), r, nd,
            C.c_void_p(arg.data_ptr()), C.c_void_p(rowmax.data_ptr() if return_rowmax else None),
            int(Qb.device.index), C.c_void_p(torch.cuda.current_stream(Qb.device).cuda_stream)))
    return (arg, rowmax) if return_rowmax else arg


def maxsim_backward_grouped(Q: torch.Tensor, D_padded: torch.Tensor, arg: torch.Tensor, grad: torch.Tensor,
                            need_dq: bool = True, need_dd: bool = True):
    """Gradients of the block-diagonal scores ``[B, r]`` (see ``maxsim_argmax_grouped``): returns
    (dQ fp32 ``[B, Nq, d]`` or None, dD fp32 ``[B*r, Nd, d]`` or None)."""
    Qb, Db = _train_operands(Q, D_padded)
    B, nq, n, nd = Qb.size(0), Qb.size(1), Db.size(0), Db.size(1)
    r = arg.size(1) if arg.dim() == 3 else 0
    if arg.shape != (B, r, nq) or arg.dtype != torch.int32 or grad.shape != (B, r) or n != B * r:
        raise ValueError("arg must be int32 [B, r, Nq], grad [B, r] and D hold B*r documents")
    g = grad.detach().to(torch.float32).contiguous()
    a = arg.contiguous()
    dq = torch.empty((B, nq, _cabi.DIM), dtype=torch.float32, device=Qb.device) if need_dq else None
    dd = torch.empty((n, nd, _cabi.DIM), dtype=torch.float32, device=Qb.device) if need_dd else None
    with torch.cuda.device(Qb.device):
        _cabi.check(_train_call("flmr_maxsim_backward_grouped", Db)(
            C.c_void_p(Qb.data_ptr()), B, nq, C.c_void_p(Db.data_ptr()), r, nd, C.c_void_p(a.data_ptr()),
            C.c_void_p(g.data_ptr()), C.c_void_p(dq.data_ptr() if need_dq else None),
            C.c_void_p(dd.data_ptr() if need_dd else None), int(Qb.device.index),
            C.c_void_p(torch.cuda.current_stream(Qb.device).cuda_stream)))
    return dq, dd


def maxsim_argmax(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, return_rowmax: bool = False):
    """``arg[b, p, i]`` = index (into the padded document) of the unmasked token of document ``p`` with
    the largest inner product with query token ``Q[b, i]``; int32 ``[B, n, Nq]``, -1 for a fully masked
    document.  What the backward of the all-pairs MaxSim needs instead of the ``[n, Nd, Nq]`` score tensor
    the reference's autograd keeps (colbert.py:235-286).  ``return_rowmax=True`` also returns the maxima
    themselves (fp32, same shape): ``rowmax.sum(-1)`` is the ``[B, n]`` score matrix."""
    Qb, Db = _train_operands(Q, D_padded)
    B, nq, n, nd = Qb.size(0), Qb.size(1), Db.size(0), Db.size(1)
    mask = D_mask.reshape(n, nd).to(device=Qb.device, dtype=torch.uint8).contiguous()
    arg = torch.empty((B, n, nq), dtype=torch.int32, device=Qb.device)
    rowmax = torch.empty((B, n, nq), dtype=torch.float32, device=Qb.device) if return_rowmax else None
    with torch.cuda.device(Qb.device):
        _cabi.check(_train_call("flmr_maxsim_argmax", Db)(
            C.c_void_p(Qb.data_ptr()), B, nq, C.c_void_p(Db.data_ptr()), C.c_void_p(mask.data_ptr()), n, nd,
            C.c_void_p(arg.data_ptr()), C.c_void_p(rowmax.data_ptr() if return_rowmax else None),
            int(Qb.device.index), C.c_void_p(torch.cuda.current_stream(Qb.device).cuda_stream)))
    return (arg, rowmax) if return_rowmax else arg


def maxsim_backward(Q: torch.Tensor, D_padded: torch.Tensor, arg: torch.Tensor, grad: torch.Tensor,
                    need_dq: bool = True, need_dd: bool = True):
    """Gradients of ``scores[b, p] = sum_i <Q[b, i], D[p, arg[b, p, i]]>`` for upstream ``grad [B, n]``:
    returns (dQ fp32 ``[B, Nq, d]`` or None, dD fp32 ``[n, Nd, d]`` or None)."""
    Qb, Db = _train_operands(Q, D_padded)
    B, nq, n, nd = Qb.size(0), Qb.size(1), Db.size(0), Db.size(1)
    if arg.shape != (B, n, nq) or arg.dtype != torch.int32 or grad.shape != (B, n):
        raise ValueError("arg must be int32 [B, n, Nq] and grad [B, n]")
    g = grad.detach().to(torch.float32).contiguous()
    a = arg.contiguous()
    dq = torch.empty((B, nq, _cabi.DIM), dtype=torch.float32, device=Qb.device) if need_dq else None
    dd = torch.empty((n, nd, _cabi.DIM), dtype=torch.float32, device=Qb.device) if need_dd else None
    with torch.cuda.device(Qb.device):
        _cabi.check(_train_call("flmr_maxsim_backward", Db)(
            C.c_void_p(Qb.data_ptr()), B, nq, C.c_void_p(Db.data_ptr()), n, nd, C.c_void_p(a.data_ptr()),
            C.c_void_p(g.data_ptr()), C.c_void_p(dq.data_ptr() if need_dq else None),
            C.c_void_p(dd.data_ptr() if need_dd else None), int(Qb.device.index),
            C.c_void_p(torch.cuda.current_stream(Qb.device).cuda_stream)))
    return dq, dd


def debug_listed_plan(corpus: FlatCorpus, n_queries: int, nq: int, pids) -> list:
    """Test infrastructure: the plans ``maxsim_topk(..., pids=pids)`` scans for ``n_queries`` queries of ``nq`` tokens
    (``flmr_debug_listed_plan``), one dict per pass: ``q_first``, ``n_q``, ``n_ctas``, ``tile_bound``, ``slots`` (the
    union of the pass's listed slots), ``cta_tile_base``, ``tile_row``, ``tile_mask``, ``tile_first`` (numpy)."""
    off, flat = _prep_lists(corpus, pids, n_queries)
    n = C.c_int64(0)
    L = _cabi.lib()
    args = (corpus.handle, corpus.workspace(), n_queries, nq, off.ctypes.data_as(C.c_void_p), C.c_void_p(flat.data_ptr()))
    with torch.cuda.device(corpus.device):
        _cabi.check(L.flmr_debug_listed_plan(*args, None, 0, C.byref(n)))
        buf = np.zeros(n.value, dtype=np.int64)
        _cabi.check(L.flmr_debug_listed_plan(*args, buf.ctypes.data_as(C.c_void_p), n.value, C.byref(n)))
    out, at = [], 1
    for _ in range(int(buf[0])):
        q_first, n_q, n_ctas, nu, nt, bound = (int(x) for x in buf[at:at + 6])
        at += 6
        d = {"q_first": q_first, "n_q": n_q, "n_ctas": n_ctas, "tile_bound": bound}
        for name, size in (("slots", nu), ("cta_tile_base", n_ctas + 1), ("tile_row", nt), ("tile_mask", nt),
                           ("tile_first", nt)):
            d[name] = buf[at:at + size].copy()
            at += size
        out.append(d)
    return out


def debug_scores_simt(corpus: FlatCorpus, Q: torch.Tensor, relu: bool = False) -> torch.Tensor:
    """Test infrastructure: independent plain-SIMT fp32 kernel (same contract as maxsim_scores)."""
    Qd = _prep_queries(corpus, Q)
    B, nq = Qd.size(0), Qd.size(1)
    out = torch.empty((B, corpus.n_passages), dtype=torch.float32, device=corpus.device)
    with torch.cuda.device(corpus.device):
        _cabi.check(_cabi.lib().flmr_debug_maxsim_scores_simt(
            corpus.handle, C.c_void_p(Qd.data_ptr()), B, nq, _cabi.FLAG_RELU if relu else 0,
            C.c_void_p(out.data_ptr()), _stream(corpus)))
    return out
