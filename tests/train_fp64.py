"""Float64 restatement of the training / re-scoring kernels (csrc/flmr_train_kernels.cuh, flmr_train_tc_kernel.cuh):
the arg-max forward, the gather / scatter backward and the in-batch-negatives loss head, plus the error bounds the
kernels are held to.  Pinned on CPU against the reference's own autograd (tests/test_train_fp64_host.py) before any
kernel is judged by it.

Written with torch float64 ops so that the same code runs on the CPU (where it is pinned) and on the GPU (where the
large shapes of tests/test_train_kernels_fp64_gpu.py would take minutes in numpy).  Products of bf16 values are exact
in float64 and a 128-term sum loses at most ~2^-46 of its magnitude: nine orders of magnitude below the fp32 bounds.
"""
from __future__ import annotations

import itertools
import math

import torch

U = 2.0 ** -24                 # unit roundoff of fp32
C_BOUND = 16                   # safety factor of every bound below
TINY = 2.0 ** -149             # smallest fp32 denormal: absolute floor of an underflowing expf
_CHUNK = 1 << 25               # float64 elements per intermediate [B, docs, Nq, Nd] block


def _doc_rows(D: torch.Tensor, B: int, r, p0: int, p1: int) -> torch.Tensor:
    """Documents [p0, p1) each query meets: ``[1, p1 - p0, ...]`` (all pairs) or ``[B, p1 - p0, ...]`` (grouped)."""
    if r is None:
        return D[p0:p1].unsqueeze(0)
    return D.view(B, r, *D.shape[1:])[:, p0:p1]


def argmax_rowmax(Q: torch.Tensor, D: torch.Tensor, mask: torch.Tensor, docs_per_query=None):
    """``flmr_maxsim_argmax`` (``docs_per_query=None``: every query against every document) or its grouped form (query
    b against documents ``[b r, (b + 1) r)``) in float64.  ``Q [B, Nq, d]``, ``D [n, Nd, d]``, ``mask [n, Nd]``.

    Returns (arg int64, rowmax float64, absmax float64), each ``[B, P, Nq]`` with P = n or r: the lowest index among the
    exact maxima over unmasked tokens (-1 / -inf for a document without one), and ``max_j A[b, p, i, j]`` over unmasked
    j with ``A = sum_k |q_ik d_jk|`` — the magnitude an fp32 dot product's rounding error scales with (0 if empty)."""
    Q, D, mask = Q.double(), D.double(), mask.bool()
    B, nq = Q.shape[:2]
    n, nd = D.shape[:2]
    P = n if docs_per_query is None else int(docs_per_query)
    dev = Q.device
    arg = torch.full((B, P, nq), -1, dtype=torch.int64, device=dev)
    rowmax = torch.full((B, P, nq), -math.inf, dtype=torch.float64, device=dev)
    absmax = torch.zeros((B, P, nq), dtype=torch.float64, device=dev)
    Qa = Q.abs()
    step = max(1, _CHUNK // max(1, B * nq * nd))
    cols = torch.arange(nd, device=dev)
    for p0 in range(0, P, step):
        p1 = min(P, p0 + step)
        Dc = _doc_rows(D, B, docs_per_query, p0, p1)                       # [1 or B, pc, Nd, d]
        mc = _doc_rows(mask, B, docs_per_query, p0, p1)[:, :, None, :]     # [1 or B, pc, 1, Nd]
        S = torch.einsum("bid,xpjd->bpij", Q, Dc) if Dc.size(0) == 1 else torch.einsum("bid,bpjd->bpij", Q, Dc)
        A = (torch.einsum("bid,xpjd->bpij", Qa, Dc.abs()) if Dc.size(0) == 1
             else torch.einsum("bid,bpjd->bpij", Qa, Dc.abs()))
        S = S.masked_fill(~mc, -math.inf)
        best = S.max(dim=-1).values
        first = torch.where(S == best[..., None], cols, nd).min(dim=-1).values
        live = mc.any(dim=-1).expand_as(best)
        arg[:, p0:p1] = torch.where(live, first, -1)
        rowmax[:, p0:p1] = best
        absmax[:, p0:p1] = A.masked_fill(~mc, 0.0).max(dim=-1).values
    return arg, rowmax, absmax


def maxsim_exact(Q: torch.Tensor, D: torch.Tensor, mask: torch.Tensor, docs_per_query=None):
    """Float64 MaxSim scores ``[B, P]`` and their fp32 error bound: the sum of the row bounds ``C u max_j A`` plus
    ``Nq u sum_i |rowmax|`` for the summation of the row maxima."""
    _, rowmax, absmax = argmax_rowmax(Q, D, mask, docs_per_query)
    nq = Q.size(1)
    fin = torch.isfinite(rowmax)
    scores = rowmax.sum(dim=-1)
    bound = C_BOUND * U * absmax.sum(dim=-1) + nq * U * torch.where(fin, rowmax.abs(), 0.0).sum(dim=-1)
    return scores, bound


def backward(Q: torch.Tensor, D: torch.Tensor, arg: torch.Tensor, g: torch.Tensor, docs_per_query=None):
    """``flmr_maxsim_backward`` (or ``_grouped``) in float64 for the winners ``arg [B, P, Nq]`` (< 0: no gradient) and
    upstream ``g [B, P]``:  dQ[b, i] = sum_p g[b, p] D[p, arg[b, p, i]],  dD[p, arg[b, p, i]] += g[b, p] Q[b, i].

    Returns (dQ, dD, dq_abs, dd_abs, dd_count): the sums of the absolute terms (what an fp32 summation's error scales
    with) and, per document token, the number of terms that reach it."""
    Q, D, g = Q.double(), D.double(), g.double()
    arg = arg.long()
    B, nq, d = Q.shape
    n, nd = D.shape[:2]
    P = arg.size(1)
    dev = Q.device
    dQ = torch.zeros((B, nq, d), dtype=torch.float64, device=dev)
    dq_abs = torch.zeros_like(dQ)
    dD = torch.zeros((n * nd, d), dtype=torch.float64, device=dev)
    dd_abs = torch.zeros_like(dD)
    dd_count = torch.zeros((n * nd,), dtype=torch.int64, device=dev)
    step = max(1, _CHUNK // max(1, B * nq * d))
    bidx = torch.arange(B, device=dev)[:, None, None]
    for p0 in range(0, P, step):
        p1 = min(P, p0 + step)
        a = arg[:, p0:p1]                                                  # [B, pc, Nq]
        live = a >= 0
        pg = torch.arange(p0, p1, device=dev)[None, :, None]
        if docs_per_query is not None:
            pg = bidx * P + pg
        pg = pg.expand_as(a)
        flat = pg * nd + a.clamp_min(0)
        rows = D.view(n * nd, d)[flat]                                     # [B, pc, Nq, d]
        gw = (g[:, p0:p1, None] * live)[..., None]                         # [B, pc, Nq, 1]
        dQ += (gw * rows).sum(dim=1)
        dq_abs += (gw.abs() * rows.abs()).sum(dim=1)
        contrib = gw * Q[:, None]                                          # [B, pc, Nq, d]
        sel = live.reshape(-1)
        idx = flat.reshape(-1)[sel]
        dD.index_add_(0, idx, contrib.reshape(-1, d)[sel])
        dd_abs.index_add_(0, idx, contrib.reshape(-1, d)[sel].abs())
        dd_count.index_add_(0, idx, torch.ones_like(idx))
    return (dQ, dD.view(n, nd, d), dq_abs, dd_abs.view(n, nd, d), dd_count.view(n, nd))


def ib_loss(rowmax: torch.Tensor, nway: int, label0: int = 0):
    """``flmr_ib_loss`` in float64 on row maxima ``[B, n, Nq]``: (scores [B, n], per-query losses [B],
    d mean-loss / d scores [B, n]) with the positive of query b at column ``label0 + b * nway``."""
    return ib_loss_from_scores(rowmax.double().sum(dim=-1), nway, label0)


def ib_loss_from_scores(scores: torch.Tensor, nway: int, label0: int = 0):
    """The cross-entropy half of ``ib_loss`` on given scores ``[B, n]`` (float64): a -inf score has probability 0 and
    gradient 0; a -inf positive gives an infinite loss and the finite gradient ``(softmax - onehot) / B``."""
    s = scores.double()
    B, n = s.shape
    labels = label0 + torch.arange(B, device=s.device) * nway
    m = s.max(dim=1, keepdim=True).values
    lse = m + torch.log(torch.exp(s - m).sum(dim=1, keepdim=True))
    loss = lse[:, 0] - s.gather(1, labels[:, None])[:, 0]
    onehot = torch.zeros_like(s)
    onehot[torch.arange(B, device=s.device), labels] = 1.0
    return s, loss, (torch.exp(s - lse) - onehot) / B


def ib_loss_bounds(scores: torch.Tensor, nway: int, label0: int = 0):
    """fp32 error bounds of ``flmr_ib_loss``'s per-query loss and dscores, given the scores it summed (float64 copy of
    the kernel's own fp32 scores: the summation has its own bound).  With x_p = s_p - max s, w = softmax(s),
    k = ceil(n / 256) + 12 (the depth of the kernel's sum of exponentials) and expf / logf within 2 ulp:

        err(lse)     <= u (|lse| + 2 |log sum_p e^x_p| + k + 4 + sum_p w_p |x_p|) + n 2^-149
        err(loss)    <= C (err(lse) + u |loss|)
        err(dscore_p) <= C (w_p (err(lse) + u (|s_p - lse| + 4)) + 2 u |w_p - [p = label]|) / B + C 2^-149
    """
    s = scores.double()
    B, n = s.shape
    fin = torch.isfinite(s)
    ref_s, loss, ds = ib_loss_from_scores(s, nway, label0)
    m = s.max(dim=1, keepdim=True).values
    x = torch.where(fin, s - m, 0.0)
    w = torch.where(fin, torch.exp(s - m), 0.0)
    se = w.sum(dim=1, keepdim=True)
    w = w / se
    lse = m + torch.log(se)
    k = math.ceil(n / 256) + 12
    err_lse = U * (lse.abs() + 2 * torch.log(se).abs() + k + 4 + (w * x.abs()).sum(dim=1, keepdim=True)) + n * TINY
    loss_bound = C_BOUND * (err_lse[:, 0] + U * loss.abs())
    dist = torch.where(fin, (s - lse).abs(), 0.0)
    d_bound = C_BOUND * (w * (err_lse + U * (dist + 4)) + 2 * U * (ds * B).abs()) / B + C_BOUND * TINY
    return loss_bound, d_bound


def winner_scores(Q: torch.Tensor, D: torch.Tensor, mask: torch.Tensor, arg: torch.Tensor, docs_per_query=None):
    """Float64 score ``<Q[b, i], D[p, arg[b, p, i]]>`` of given winners and whether each winner is an unmasked token
    (entries with ``arg < 0``: -inf and False)."""
    Q, D = Q.double(), D.double()
    B, nq, d = Q.shape
    n, nd = D.shape[:2]
    P = arg.size(1)
    arg = arg.long()
    out = torch.full(arg.shape, -math.inf, dtype=torch.float64, device=Q.device)
    unmasked = torch.zeros(arg.shape, dtype=torch.bool, device=Q.device)
    step = max(1, _CHUNK // max(1, B * nq * d))
    for p0 in range(0, P, step):
        p1 = min(P, p0 + step)
        a = arg[:, p0:p1]
        pg = torch.arange(p0, p1, device=Q.device)[None, :, None]
        if docs_per_query is not None:
            pg = torch.arange(B, device=Q.device)[:, None, None] * P + pg
        flat = (pg.expand_as(a) * nd + a.clamp_min(0))
        s = (D.view(n * nd, d)[flat] * Q[:, None]).sum(dim=-1)
        out[:, p0:p1] = torch.where(a >= 0, s, -math.inf)
        unmasked[:, p0:p1] = (a >= 0) & mask.reshape(-1)[flat].bool()
    return out, unmasked


# ---- the arg-max / backward grid of tests/test_train_kernels_fp64_gpu.py ------------------------------------------
MASKS = ("full", "prefix", "holes", "first", "last", "none", "spread128", "spread129")
ARGMAX_FACTORS = {
    "nq": [1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 257, 832],
    "nd": [1, 2, 63, 64, 65, 127, 128, 129, 256, 257, 512],
    "mask": list(MASKS),
    "n_docs": [1, 2, 31, 32, 33, 65, 129],
    "B": [1, 3, 9],
    "norm": ["unit", "wide"],
    "path": [1, 2],
    "form": ["all", "grouped"],
}


def argmax_allowed(case: dict) -> bool:
    """128 / 129 unmasked tokens spread over a longer document need Nd >= 256."""
    return not (str(case.get("mask", "")).startswith("spread") and case.get("nd", 512) < 256)


def argmax_grid():
    return pairwise_cases(ARGMAX_FACTORS, argmax_allowed)


def make_mask(kind: str, n: int, nd: int, generator=None) -> torch.Tensor:
    """bool ``[n, nd]``: every token ('full'), a random-length prefix, random holes (30%), only the first / only the
    last token, no token in every other document ('none': the others full, so one batch mixes -1 winners with real
    ones), or exactly 128 / 129 unmasked tokens at random positions ('spread128' / 'spread129')."""
    if kind == "full":
        return torch.ones((n, nd), dtype=torch.bool)
    if kind == "prefix":
        lens = torch.randint(1, nd + 1, (n,), generator=generator)
        return torch.arange(nd)[None, :] < lens[:, None]
    if kind == "holes":
        return torch.rand((n, nd), generator=generator) > 0.3
    m = torch.zeros((n, nd), dtype=torch.bool)
    if kind == "first":
        m[:, 0] = True
    elif kind == "last":
        m[:, nd - 1] = True
    elif kind == "none":
        m[1::2] = True
    elif kind.startswith("spread"):
        k = int(kind[len("spread"):])
        for p in range(n):
            m[p, torch.randperm(nd, generator=generator)[:k]] = True
    else:
        raise ValueError(kind)
    return m


def bf16_rows(shape, norm=None, generator=None, device="cpu"):
    """Random bf16-representable rows ``[..., 128]`` (as float32): unit rows, or rows of norm uniform in ``norm =
    (lo, hi)``; mixed signs either way."""
    x = torch.randn(*shape, generator=generator).float()
    x = torch.nn.functional.normalize(x, dim=-1)
    if norm is not None:
        lo, hi = norm
        x = x * (lo + (hi - lo) * torch.rand(*shape[:-1], 1, generator=generator))
    return x.to(torch.bfloat16).float().to(device)


def flipr_select(rowmax: torch.Tensor, arg: torch.Tensor, query_maxlen: int = 64):
    """The 'flipr' reduction of colbert_score_reduce (colbert.py:248-261) on row maxima ``[..., Nq]``: the sum of the
    ``query_maxlen // 2`` largest of the first ``query_maxlen`` plus, when at least 8 follow, the 8 largest of the
    rest; returns (scores, winners with the unselected tokens set to -1)."""
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


def docs_per_cta(n_queries: int, nq: int, n_per: int, nd: int, sms: int) -> int:
    """Documents per CTA of the wgmma arg-max kernel: restates the makespan model of ``argmax_tc`` in
    csrc/flmr_maxsim.cu (a fixed set-up of ~17 chunks' worth per CTA, waves of one CTA per SM).  It must track that
    function: the tests assert the split each case gets through it."""
    nd_c = (nd + 127) // 128 * 128
    pairs_q = n_queries * ((nq + 127) // 128)
    dpc, best_t = 1, 1e30
    for d in range(1, min(32, max(1, n_per)) + 1):
        ctas = pairs_q * ((n_per + d - 1) // d)
        t = float((ctas + sms - 1) // sms) * (5.0 + d * 0.3 * (nd_c // 128))
        if t < best_t:
            best_t, dpc = t, d
    return dpc


def pairwise_cases(factors: dict, allowed=lambda case: True):
    """Greedy pairwise covering of ``factors`` (name -> list of values): every pair of values of two factors that some
    case may hold (``allowed`` on the partial assignment) appears in at least one returned case.  Deterministic."""
    names = list(factors)
    todo = set()
    for f1, f2 in itertools.combinations(names, 2):
        for v1, v2 in itertools.product(range(len(factors[f1])), range(len(factors[f2]))):
            if allowed({f1: factors[f1][v1], f2: factors[f2][v2]}):
                todo.add((f1, v1, f2, v2))
    order = {f: i for i, f in enumerate(names)}

    def key(fa, va, fb, vb):
        return (fa, va, fb, vb) if order[fa] < order[fb] else (fb, vb, fa, va)

    cases = []
    while todo:
        f1, v1, f2, v2 = min(todo, key=lambda t: (order[t[0]], t[1], order[t[2]], t[3]))
        pick = {f1: v1, f2: v2}
        for f in sorted(names, key=lambda f: -len(factors[f])):
            if f in pick:
                continue
            best, best_gain = None, -1
            for v in range(len(factors[f])):
                trial = {g: factors[g][i] for g, i in pick.items()}
                trial[f] = factors[f][v]
                if not allowed(trial):
                    continue
                gain = sum(key(f, v, g, i) in todo for g, i in pick.items())
                if gain > best_gain:
                    best, best_gain = v, gain
            if best is None:
                raise ValueError("no allowed value of %s completes %s" % (f, pick))
            pick[f] = best
        for fa, fb in itertools.combinations(names, 2):
            todo.discard(key(fa, pick[fa], fb, pick[fb]))
        cases.append({f: factors[f][pick[f]] for f in names})
    return cases
