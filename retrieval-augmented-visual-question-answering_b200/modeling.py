"""Scoring surface of the reference's models on the CUDA path (SURVEY.md 8f-2):

    colbert_score(Q, D_padded, D_mask)          third_party/ColBERT/colbert/modeling/colbert.py:268-286
    ColBERT.score / FLMR*.score                 colbert.py:217-224  (callers: colbert.py:71-73 training,
                                                src/models/rag/rag_model_blip.py:432-435 RAG re-score,
                                                src/executors/FLMR_executor.py:828-833 exhaustive eval)
    compute_ib_loss_new (in-batch negatives)    colbert.py:82-113

Forward, training-sized batches (the usual case here): ONE launch of ``flmr_maxsim_argmax`` computes, for
every (query token, document) pair, the winning document token and its inner product — the row maxima
summed over query tokens are the all-pairs scores ``[B, n]`` (the aligned ``Q_dup`` form the reference
builds with ``repeat_interleave`` is a gather of that matrix, the in-batch-negatives matrix IS that
matrix), and the winners (4 bytes per pair) are what the backward needs.  Large inputs (exhaustive
evaluation through ``score``): the ``n`` padded documents are packed into a temporary FlatCorpus and
scored by one launch of the wgmma scan kernel; the backward then recomputes the winners.  Either way the
``[n, Nd, Nq]`` score tensor the reference materialises (218 MB per rank at C4, SURVEY 8a) never exists.

Backward: ``flmr_maxsim_backward`` routes the gradient through the winners (``dQ_i += g * D_argmax``
gathered, ``dD_argmax += g * Q_i`` scattered with fp32 atomics).  Both are CUDA kernels behind the C ABI
(csrc/flmr_train_kernels.cuh).  fp16 documents, what the reference's ColBERT.doc returns on the GPU
(colbert.py:205-206), are scored in fp16 forward and backward, the query converted to fp16 as colbert_score does
(:284); documents of any other dtype are rounded to bf16 with the query.  Accumulation is fp32 either way, and the
gradients come back in the inputs' dtypes.
"""
from __future__ import annotations

from typing import Optional

import torch

from .corpus import FlatCorpus
from .maxsim import (_train_operands, ib_loss_head, maxsim_argmax, maxsim_argmax_grouped, maxsim_backward,
                     maxsim_backward_grouped, maxsim_scores)


# The forward is ONE arg-max launch (scores = row maxima summed) that also saves the winners for the backward —
# a warp-MMA kernel for small batches, the wgmma kernel from 16M (query row, token) pairs up (chosen inside
# flmr_maxsim_argmax) — as long as the winners + maxima ([B, n, Nq] x 8 bytes) stay below this budget.  Beyond
# it (an exhaustive evaluation of one query against a whole collection through `score`) the n padded documents
# are packed into a temporary FlatCorpus and scored by the scan kernel, which keeps nothing per pair; the
# backward then recomputes the winners.
_FUSED_MAX_ARG_BYTES = 1 << 30


def _forward_scores(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor):
    """All-pairs scores ``[B, n]``; returns (scores, bool mask [n, Nd], saved arg-max or None)."""
    n, nd = D_padded.size(0), D_padded.size(1)
    mask = D_mask.reshape(n, nd).bool()
    if float(Q.size(0)) * n * Q.size(1) * 8 <= _FUSED_MAX_ARG_BYTES:
        # no host round trip on the training path: a document without any unmasked token scores -inf here
        # (its winners are -1 and it receives no gradient); the reference's padded path gives -9999 * Nq
        arg, rowmax = maxsim_argmax(Q, D_padded, mask, return_rowmax=True)
        return rowmax.sum(dim=-1), mask, arg
    if not bool(mask.any(dim=1).all()):
        raise ValueError("a document has no unmasked token: its MaxSim score is undefined "
                         "(-9999 * Nq on the reference's padded path)")
    packed = D_padded.detach()[mask]
    fp16 = D_padded.dtype == torch.float16                  # the arg-max kernels' rule (_train_operands)
    corpus = FlatCorpus(packed.to(torch.float16 if fp16 else torch.bfloat16), mask.sum(dim=1).cpu(), device=Q.device,
                        adopt=True, storage="fp16" if fp16 else "bf16")
    try:
        scores = maxsim_scores(corpus, Q.detach())
        torch.cuda.current_stream(Q.device).synchronize()   # corpus buffers die with this scope
    finally:
        corpus.close()
    return scores, mask, None


def _flipr_reduce(rowmax: torch.Tensor, arg: torch.Tensor, query_maxlen: int):
    """The ``interaction == 'flipr'`` branch of colbert_score_reduce (colbert.py:248-261) on the per-token maxima
    ``rowmax [..., Nq]``: the sum of the ``K1 = query_maxlen // 2`` largest of the first ``query_maxlen`` tokens
    plus, when at least ``K2 = 8`` tokens follow them, the sum of the 8 largest of the rest.  Returns (scores,
    winners with the unselected tokens set to -1): the gradient reaches the selected tokens only, which is what
    autograd through the reference's ``topk(...).values.sum()`` does, and the backward kernels skip winners < 0."""
    assert query_maxlen == 64, ("for now", query_maxlen)                 # the reference's own restriction (:249)
    K1, K2 = query_maxlen // 2, 8
    keep = torch.zeros_like(rowmax, dtype=torch.bool)
    top, idx = rowmax[..., :query_maxlen].topk(K1, dim=-1)
    keep[..., :query_maxlen].scatter_(-1, idx, True)
    scores = top.sum(dim=-1)
    if K2 <= rowmax.size(-1) - query_maxlen:
        top2, idx2 = rowmax[..., query_maxlen:].topk(K2, dim=-1)
        keep[..., query_maxlen:].scatter_(-1, idx2, True)
        scores = scores + top2.sum(dim=-1)
    return scores, torch.where(keep, arg, torch.full_like(arg, -1))


class _AllPairsMaxSim(torch.autograd.Function):
    """scores[b, p] = sum_i max_{j: mask[p, j]} <Q[b, i], D[p, j]>  for all (b, p)."""

    @staticmethod
    def forward(ctx, Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, flipr_maxlen: int = 0
                ) -> torch.Tensor:
        if flipr_maxlen:
            n, nd = D_padded.size(0), D_padded.size(1)
            if float(Q.size(0)) * n * Q.size(1) * 8 > _FUSED_MAX_ARG_BYTES:
                raise ValueError("interaction='flipr' keeps the per-token maxima of every pair: at most %d "
                                 "(query row, document) pairs per call" % (_FUSED_MAX_ARG_BYTES // 8))
            mask = D_mask.reshape(n, nd).bool()
            arg, rowmax = maxsim_argmax(Q, D_padded, mask, return_rowmax=True)
            scores, arg = _flipr_reduce(rowmax, arg, flipr_maxlen)
        else:
            scores, mask, arg = _forward_scores(Q, D_padded, D_mask)
        ctx.has_arg = arg is not None
        ctx.save_for_backward(Q, D_padded, mask, *([arg] if ctx.has_arg else []))
        return scores

    @staticmethod
    def backward(ctx, grad: torch.Tensor):
        Q, D_padded, mask = ctx.saved_tensors[:3]
        need_dq, need_dd = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_dq or need_dd):
            return None, None, None, None
        arg = ctx.saved_tensors[3] if ctx.has_arg else maxsim_argmax(Q, D_padded, mask)
        dQ, dD = maxsim_backward(Q, D_padded, arg, grad, need_dq=need_dq, need_dd=need_dd)
        return (dQ.to(Q.dtype) if dQ is not None else None,
                dD.to(D_padded.dtype) if dD is not None else None, None, None)


def _equal_run_length(Q: torch.Tensor) -> int:
    """``r`` if ``Q [n, Nq, d]`` consists of consecutive runs of exactly ``r`` identical queries each (what
    ``repeat_interleave(r, dim=0)`` builds; adjacent runs differ), else 0.  Two vectorised passes and two scalar
    read-backs — ``torch.unique_consecutive(Q, dim=0)`` compares whole rows serially in one CUDA thread (~80 ms
    per call for an 832-token query, measured in round 1)."""
    n = Q.size(0)
    if n < 2:
        return 0
    Qd = Q.detach()
    new_run = torch.ones(n, dtype=torch.bool, device=Q.device)
    new_run[1:] = (Qd[1:] != Qd[:-1]).flatten(1).any(dim=1)
    starts = new_run.nonzero().flatten()
    U = int(starts.numel())
    r = n // U
    if U * r != n or r < 2:
        return 0
    return r if bool((starts == torch.arange(U, device=Q.device) * r).all()) else 0


class _GroupedMaxSim(torch.autograd.Function):
    """scores[b, t] = MaxSim(Q[b], D[b*r + t]) for ``Q [B, Nq, d]`` and ``D [B*r, Nd, d]``: query ``b`` against
    ITS ``r`` documents only — the block diagonal of the all-pairs matrix, computed without the off-diagonal
    pairs (one launch of the grouped arg-max kernel forward, saved winners, gather/scatter backward)."""

    @staticmethod
    def forward(ctx, Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, r: int,
                flipr_maxlen: int = 0) -> torch.Tensor:
        n, nd = D_padded.size(0), D_padded.size(1)
        mask = D_mask.reshape(n, nd).bool()
        arg, rowmax = maxsim_argmax_grouped(Q, D_padded, mask, r, return_rowmax=True)
        if flipr_maxlen:
            scores, arg = _flipr_reduce(rowmax, arg, flipr_maxlen)
        else:
            scores = rowmax.sum(dim=-1)                                        # [B, r]
        ctx.save_for_backward(Q, D_padded, arg)
        return scores

    @staticmethod
    def backward(ctx, grad: torch.Tensor):
        Q, D_padded, arg = ctx.saved_tensors
        need_dq, need_dd = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_dq or need_dd):
            return None, None, None, None, None
        dQ, dD = maxsim_backward_grouped(Q, D_padded, arg, grad, need_dq=need_dq, need_dd=need_dd)
        return (dQ.to(Q.dtype) if dQ is not None else None,
                dD.to(D_padded.dtype) if dD is not None else None, None, None, None)


def grouped_maxsim(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, docs_per_query: int
                   ) -> torch.Tensor:
    """``[B, r]`` scores of every query against its own ``r = docs_per_query`` documents (differentiable):
    ``ColBERT.score(Q.repeat_interleave(r, 0), D, D_mask).view(B, r)`` (colbert.py:71-73) without the repeat."""
    return _GroupedMaxSim.apply(Q, D_padded, D_mask, int(docs_per_query), 0)


def _aligned_maxsim(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, flipr_maxlen: int = 0
                    ) -> torch.Tensor:
    """scores[p] = MaxSim(Q[p], D[p]) for ``Q [n, Nq, d]`` aligned with ``D [n, Nd, d]``.

    Callers build ``Q`` with ``repeat_interleave`` (colbert.py:71, rag_model_blip.py:433,
    FLMR_executor.py:828).  Runs of identical consecutive queries are detected on the device; equal-length
    runs (the ``repeat_interleave`` form: U queries x r documents each) become ONE grouped launch over the U
    unique queries, anything else a grouped launch with one document per query.  Either way only the n
    aligned pairs are scored — O(n), where scoring all U x n pairs and gathering would be O(U n)."""
    n = D_padded.size(0)
    r = _equal_run_length(Q)
    if r:
        # differentiable pick of one representative per run; its gradient is the sum over the run's rows
        return _GroupedMaxSim.apply(Q[::r], D_padded, D_mask, r, flipr_maxlen).reshape(n)
    return _GroupedMaxSim.apply(Q, D_padded, D_mask, 1, flipr_maxlen).reshape(n)


class _FusedIBLoss(torch.autograd.Function):
    """compute_ib_loss_new (colbert.py:82-113) in three launches: the arg-max kernel (all-pairs row maxima +
    winners), ``flmr_ib_loss`` (scores, cross-entropy against the positives at column ``label0 + i * nway``, and
    the gradient w.r.t. the scores), and — in backward — the gather/scatter kernels.  Returns (loss, scores)."""

    @staticmethod
    def forward(ctx, Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, nway: int, label0: int):
        n, nd = D_padded.size(0), D_padded.size(1)
        mask = D_mask.reshape(n, nd).bool()
        Qb, Db = _train_operands(Q, D_padded)
        arg, rowmax = maxsim_argmax(Qb, Db, mask, return_rowmax=True)
        scores, loss_q, dscores = ib_loss_head(rowmax, nway, label0)
        ctx.save_for_backward(Qb, Db, arg, dscores)       # converted operands: no second cast in backward
        ctx.dtypes = (Q.dtype, D_padded.dtype)
        ctx.mark_non_differentiable(scores)
        return loss_q.mean(), scores

    @staticmethod
    def backward(ctx, grad_loss: torch.Tensor, _grad_scores):
        Qb, Db, arg, dscores = ctx.saved_tensors
        need_dq, need_dd = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_dq or need_dd):
            return None, None, None, None, None
        dQ, dD = maxsim_backward(Qb, Db, arg, dscores * grad_loss, need_dq=need_dq, need_dd=need_dd)
        return (dQ.to(ctx.dtypes[0]) if dQ is not None else None,
                dD.to(ctx.dtypes[1]) if dD is not None else None, None, None, None)


def all_pairs_maxsim(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor) -> torch.Tensor:
    """``[B, n]`` MaxSim of every query against every padded document (differentiable)."""
    return _AllPairsMaxSim.apply(Q, D_padded, D_mask, 0)


def colbert_score(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, config=None,
                  use_gpu: bool = True) -> torch.Tensor:
    """Drop-in for colbert.modeling.colbert.colbert_score (colbert.py:268-286).

    ``Q.size(0)`` is 1 (compare with all documents) or ``n`` (each query against its aligned
    document — callers build it with ``repeat_interleave``).  Returns ``[n]`` scores, true-max
    semantics of the padded path.  ``config.interaction == 'flipr'`` (colbert.py:248-261; FLMR uses the default
    'colbert') reduces the per-token maxima by partial top-k sums instead of the plain sum: same arg-max launch,
    the selection on its ``[n, Nq]`` output."""
    assert Q.dim() == 3 and D_padded.dim() == 3, (Q.size(), D_padded.size())
    assert Q.size(0) in [1, D_padded.size(0)]
    interaction = getattr(config, "interaction", "colbert") if config is not None else "colbert"
    assert interaction in ["colbert", "flipr"], interaction                  # colbert.py:246
    flipr_maxlen = int(config.query_maxlen) if interaction == "flipr" else 0
    del config, use_gpu          # the reference moves the operands to the GPU when use_gpu is set; here ALWAYS
    if torch.cuda.is_available():   # (without CUDA the kernels below raise: there is no CPU fallback)
        dev = Q.device if Q.is_cuda else (D_padded.device if D_padded.is_cuda
                                          else torch.device("cuda", torch.cuda.current_device()))
        Q, D_padded, D_mask = Q.to(dev), D_padded.to(dev), D_mask.to(dev)
    if Q.size(0) == 1:
        return _AllPairsMaxSim.apply(Q, D_padded, D_mask, flipr_maxlen)[0]
    return _aligned_maxsim(Q, D_padded, D_mask, flipr_maxlen)


class _GatherCat(torch.autograd.Function):
    """``cat(all_gather(x))`` along dim 0 whose backward returns every rank's gradient to the owner of the
    rows (sum over ranks of the owner's slice): the differentiable form of the gather the reference sketches
    and leaves disabled (colbert.py:68-69, 115-163 — there remote rows are detached, so a document never
    receives the gradient of another rank's queries)."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, group):
        import torch.distributed as dist
        world = dist.get_world_size(group)
        ctx.group, ctx.rank, ctx.rows = group, dist.get_rank(group), x.size(0)
        ctx.flat = x.is_cuda and dist.get_backend(group) == "nccl"
        x = x.contiguous()
        if ctx.flat:      # one collective straight into the concatenated tensor (no list of outputs, no cat)
            out = x.new_empty((world * x.size(0),) + tuple(x.shape[1:]))
            dist.all_gather_into_tensor(out, x, group=group)
            return out
        outs = [torch.empty_like(x) for _ in range(world)]
        dist.all_gather(outs, x, group=group)
        return torch.cat(outs, dim=0)

    @staticmethod
    def backward(ctx, g: torch.Tensor):
        import torch.distributed as dist
        g = g.contiguous()
        if ctx.flat:      # every rank needs only the sum over ranks of ITS rows: reduce-scatter, half an all-reduce
            out = g.new_empty((ctx.rows,) + tuple(g.shape[1:]))
            dist.reduce_scatter_tensor(out, g, op=dist.ReduceOp.SUM, group=ctx.group)
            return out, None
        g = g.clone()
        dist.all_reduce(g, op=dist.ReduceOp.SUM, group=ctx.group)
        return g[ctx.rank * ctx.rows:(ctx.rank + 1) * ctx.rows], None


def gather_documents(D_padded: torch.Tensor, D_mask: torch.Tensor, group=None):
    """Every rank's documents (and masks), concatenated in rank order, differentiable w.r.t. the local rows.
    Ranks may hold different padded lengths; all are padded (masked out) to the longest."""
    import torch.distributed as dist
    n, nd = D_padded.size(0), D_padded.size(1)
    nd_max = torch.tensor([nd], dtype=torch.int64, device=D_padded.device)
    dist.all_reduce(nd_max, op=dist.ReduceOp.MAX, group=group)
    pad = int(nd_max.item()) - nd
    mask = D_mask.reshape(n, nd).to(torch.uint8)
    if pad:
        D_padded = torch.nn.functional.pad(D_padded, (0, 0, 0, pad))
        mask = torch.nn.functional.pad(mask, (0, pad))
    return _GatherCat.apply(D_padded, group), _GatherCat.apply(mask, group).bool().unsqueeze(-1)


def in_batch_negatives_loss(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, nway: int,
                            return_scores: bool = False, cross_rank_negatives: bool = False, group=None,
                            all_pairs_fn=None):
    """compute_ib_loss_new (colbert.py:82-113): ``Q [B, Nq, d]``, ``D [B*nway, Nd, d]`` with the positive
    of query i at row ``i*nway`` (colbert.py:103-108); cross-entropy over all ``B*nway`` documents.

    ``cross_rank_negatives=True`` (needs an initialised process group; every rank the same B and nway):
    this rank's queries are scored against the documents of ALL ranks — ``[B, world*B*nway]``, the positive
    of local query i at column ``rank*B*nway + i*nway`` — one all-gather of the document embeddings forward,
    one all-reduce of their gradient backward.  The mean over ranks of the returned losses is the
    cross-entropy of the global batch, and its gradient reaches every document from every rank's queries.
    ``all_pairs_fn`` replaces the CUDA scorer (host-logic tests only)."""
    score_fn = all_pairs_maxsim if all_pairs_fn is None else all_pairs_fn
    B = Q.size(0)
    assert D_padded.size(0) == B * nway, (D_padded.size(), B, nway)
    if (all_pairs_fn is None and not cross_rank_negatives and not return_scores and Q.is_cuda
            and float(B) * D_padded.size(0) * Q.size(1) * 8 <= _FUSED_MAX_ARG_BYTES):
        # single-rank batch, only the loss wanted (what compute_ib_loss_new returns): arg-max kernel + fused loss
        # head.  With return_scores the score matrix itself must stay differentiable: generic route below.
        return _FusedIBLoss.apply(Q, D_padded, D_mask, int(nway), 0)[0]
    first = 0
    if cross_rank_negatives:
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("cross_rank_negatives needs an initialised torch.distributed process group")
        first = dist.get_rank(group) * B * nway
        D_padded, D_mask = gather_documents(D_padded, D_mask, group)
        if (all_pairs_fn is None and not return_scores and Q.is_cuda
                and float(B) * D_padded.size(0) * Q.size(1) * 8 <= _FUSED_MAX_ARG_BYTES):
            # same fused route as the single-rank batch, the positives shifted to this rank's columns
            return _FusedIBLoss.apply(Q, D_padded, D_mask, int(nway), int(first))[0]
    scores = score_fn(Q, D_padded, D_mask)                                # [B, (world*)B*nway]
    labels = first + torch.arange(B, device=scores.device) * nway
    loss = torch.nn.functional.cross_entropy(scores, labels)
    return (loss, scores) if return_scores else loss


def graphed_in_batch_negatives_loss(Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor, nway: int,
                                    num_warmup_iters: int = 3):
    """CUDA-graph form of ``in_batch_negatives_loss`` for a training loop whose batch shape is fixed (the reference's
    is: bsz / nranks queries x nway documents of fixed padded lengths, colbert.py:64-113).

    The eager loss step is host-bound — its three kernels take less than half of the ~0.25 ms the autograd function,
    the casts and the allocator need to launch them — so forward and backward are each captured once
    (``torch.cuda.make_graphed_callables``: every launch of the C ABI goes to the capturing stream, nothing in the
    path synchronises or allocates outside torch's and the library's stream-ordered pools) and replayed afterwards.
    The arguments are samples of the right shape / dtype / ``requires_grad``; returns ``loss_fn(Q, D_padded, D_mask)
    -> loss`` that takes part in autograd like the eager function (the encoders around it stay eager)."""
    if not Q.is_cuda:
        raise RuntimeError("graphed_in_batch_negatives_loss needs CUDA tensors (there is no CPU path)")
    nway = int(nway)

    def loss_fn(q, d, m):
        return in_batch_negatives_loss(q, d, m, nway)

    return torch.cuda.make_graphed_callables(loss_fn, (Q, D_padded, D_mask), num_warmup_iters=num_warmup_iters)


class FLMRModelForRetrieval(torch.nn.Module):
    """Façade with the name the reference announces for its HF API (README.md:25) and the call surface
    of the in-repo ``FLMR*`` classes (src/models/retriever/FLMR.py): ``query`` / ``doc`` delegate to the
    wrapped PyTorch encoders (out of scope here), ``score`` / ``forward`` route into the CUDA path."""

    def __init__(self, query_encoder: Optional[torch.nn.Module] = None,
                 doc_encoder: Optional[torch.nn.Module] = None, nway: int = 2, use_ib_negatives: bool = True,
                 cross_rank_negatives: bool = False):
        super().__init__()
        self.cross_rank_negatives = cross_rank_negatives
        self.query_encoder = query_encoder
        self.doc_encoder = doc_encoder
        self.nway = nway
        self.use_ib_negatives = use_ib_negatives

    def query(self, *args, **kw):
        if self.query_encoder is None:
            raise RuntimeError("no query encoder wrapped: FLMR.query stays in PyTorch (SURVEY 8a, a12)")
        return self.query_encoder(*args, **kw)

    def doc(self, *args, **kw):
        if self.doc_encoder is None:
            raise RuntimeError("no document encoder wrapped: ColBERT.doc stays in PyTorch")
        return self.doc_encoder(*args, **kw)

    def score(self, Q: torch.Tensor, D_padded: torch.Tensor, D_mask: torch.Tensor) -> torch.Tensor:
        """ColBERT.score (colbert.py:217-224).  ``similarity == 'cosine'`` (what FLMR uses, settings.py:118) runs
        on the CUDA path; the ``'l2'`` branch of the reference (:219-222, unused by FLMR: negative squared
        distance, no masking) is kept as the same torch expression so a config that selects it still works."""
        cfg = getattr(self, "colbert_config", None)
        if cfg is not None and getattr(cfg, "similarity", "cosine") == "l2":
            assert getattr(cfg, "interaction", "colbert") == "colbert"
            return (-1.0 * ((Q.unsqueeze(2) - D_padded.unsqueeze(1)) ** 2).sum(-1)).max(-1).values.sum(-1)
        return colbert_score(Q, D_padded, D_mask)

    def forward(self, Q: torch.Tensor, D: torch.Tensor, D_mask: torch.Tensor):
        """ColBERT.forward on pre-computed embeddings (colbert.py:64-80): ``Q [B, Nq, d]``,
        ``D [B*nway, Nd, d]`` -> (scores [B*nway] of the aligned pairs, ib_loss)."""
        loss, S = in_batch_negatives_loss(Q, D, D_mask, self.nway, return_scores=True,
                                          cross_rank_negatives=self.cross_rank_negatives)
        B = Q.size(0)
        first = 0
        if self.cross_rank_negatives:
            first = torch.distributed.get_rank() * B * self.nway
        rows = torch.arange(B, device=S.device).repeat_interleave(self.nway)
        aligned = S[rows, first + torch.arange(B * self.nway, device=S.device)]
        return (aligned, loss) if self.use_ib_negatives else aligned
