"""Float64 restatement of the corpus scan (csrc/flmr_scan_kernel.cuh: ``maxsim_scores`` / ``maxsim_topk`` over a
``FlatCorpus``) for both storages, the error bounds the scan and the SIMT cross-check are held to, the scan's
pass plan as the host builds it, and the grid of tests/test_scan_kernels_fp64_gpu.py.  Pinned on CPU
by tests/test_scan_fp64_host.py before any kernel is judged by it.

Torch float64 ops, as in train_fp64.py: the same code runs on the CPU (where it is pinned) and on the GPU (where the
grid's shapes would take minutes in numpy).  Products of bf16 (or e4m3) values are exact in float64.

Bounds.  Row i of query b against passage p: ``A_ij = sum_k |q_ik d_jk|`` is what a dot product's rounding error
scales with; the row maximum is off by at most the largest error over the passage's tokens, ``c max_j A_ij``, and
the fp32 sum of the row maxima (the reducer's, partial scores of earlier row slices included) by
``Nq u sum_i |rowmax_i|``:

  * SIMT cross-check (sequential fp32 FMA over 128 dims, a fixed-order block sum): rigorously ``gamma(128)`` per row
    and ``gamma(Nq)`` for the sum, with ``gamma(n) = n u / (1 - n u)``.
  * wgmma scan: ``c = ROW_COEF[storage]``, derived from the accumulator model the probes of
    test_scan_kernels_fp64_gpu.py measure on an H100 (DESIGN.md §2).  One MMA k-step (K = 16 bf16 or 32 e4m3
    products) aligns its products and the running accumulator to the largest of them and truncates every term below
    2^-m of that leading bit (bf16: m = 25, e4m3: m = 13 = -log2 U8); the step's sum is then truncated to the
    accumulator's format (bf16: fp32, 2^-23).  Each of the S = 128 / K steps therefore loses less than K 2^-m
    max|term| + 2^-p |sum|, and both are at most A: c = S (K 2^-m + 2^-p).  e4m3 takes p = m (the probes cannot
    tell whether its accumulator keeps more than 13 bits between steps).  The empirical 16 u of maxsim_exact
    (train_fp64.py) fails here: one product plus 127 products just below the cut loses 127 of them, 31.75 u.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

import fp8_oracle as F8
from oracle import maxsim_oracle as O
from train_fp64 import U, bf16_rows, pairwise_cases

ALIGN_BITS = {"bf16": 25, "fp8": 13}   # bits a k-step keeps below its leading bit (measured, see above)
U8 = 2.0 ** -ALIGN_BITS["fp8"]         # accumulator unit of the e4m3 wgmma
ROW_COEF = {"bf16": 8 * (16 * 2.0 ** -25 + 2.0 ** -23),    # 40 x 2^-23 = 80 u
            "fp8": 4 * (32 + 1) * U8}                      # 132 u8
_CHUNK = 1 << 25               # float64 elements per [rows, tokens] intermediate
TILE, SLOTS = 96, 24           # scan tile rows, passage ends per tile (kSlots)
STAGE_MAX_PASSES = 64          # passes one staging launch serves (kStageMaxPasses)
WS_QUERIES = 64                # queries of one call chunk (FlatCorpus.workspace())
THREE_WG_BLOCKS = 5            # occupied 64-row blocks from which variant 0 runs three consumer warpgroups


def gamma(n):
    return n * U / (1.0 - n * U)


def e4m3_round(x: torch.Tensor) -> torch.Tensor:
    """fp8_oracle.e4m3_round on a tensor (any device): round to nearest even e4m3, saturated at +-448."""
    r = F8.e4m3_round(x.detach().float().cpu().numpy())
    return torch.from_numpy(r).to(x.device)


def _segments(doclens: np.ndarray, max_tokens: int):
    """Passage ranges [p0, p1) of at most max_tokens tokens (at least one passage), with their token ranges."""
    off = np.concatenate([[0], np.cumsum(doclens, dtype=np.int64)])
    n, p0 = len(doclens), 0
    while p0 < n:
        p1 = int(np.searchsorted(off, off[p0] + max_tokens, side="right")) - 1
        p1 = min(max(p1, p0 + 1), n)
        yield p0, p1, int(off[p0]), int(off[p1])
        p0 = p1


def maxsim_packed(Q: torch.Tensor, D: torch.Tensor, doclens, relu: bool = False, storage: str = "bf16"):
    """Float64 MaxSim of queries ``Q [B, Nq, 128]`` against packed passages ``D [sum(doclens), 128]``:
    ``out[b, p] = sum_i max_{j < len_p} <Q[b, i], D_p[j]>`` (relu: each maximum clamped at 0), after rounding both
    operands to e4m3 when ``storage == "fp8"``.  Returns (scores, amax, rabs), each float64 ``[B, n]``:
    ``amax = sum_i max_j A_ij`` and ``rabs = sum_i |rowmax_i|`` — the two terms of every bound below."""
    dev = Q.device
    Q, D = Q.double(), D.double().to(dev)
    if storage == "fp8":
        Q, D = e4m3_round(Q).double(), e4m3_round(D).double()
    B, nq = Q.shape[:2]
    dl = np.asarray(doclens, dtype=np.int64)
    n = len(dl)
    rows = Q.reshape(B * nq, -1)
    rows_abs = rows.abs()
    pid = torch.from_numpy(np.repeat(np.arange(n), dl)).to(dev)
    scores = torch.zeros((B, n), dtype=torch.float64, device=dev)
    amax = torch.zeros_like(scores)
    rabs = torch.zeros_like(scores)
    for p0, p1, t0, t1 in _segments(dl, max(1, _CHUNK // max(1, B * nq))):
        Dc = D[t0:t1]
        idx = (pid[t0:t1] - p0)[None, :].expand(B * nq, -1)
        m = torch.full((B * nq, p1 - p0), -torch.inf, dtype=torch.float64, device=dev)
        m.scatter_reduce_(1, idx, rows @ Dc.T, reduce="amax", include_self=True)
        a = torch.zeros((B * nq, p1 - p0), dtype=torch.float64, device=dev)
        a.scatter_reduce_(1, idx, rows_abs @ Dc.abs().T, reduce="amax", include_self=True)
        if relu:
            m = m.clamp_min(0.0)
        scores[:, p0:p1] = m.view(B, nq, -1).sum(dim=1)
        amax[:, p0:p1] = a.view(B, nq, -1).sum(dim=1)
        rabs[:, p0:p1] = m.abs().view(B, nq, -1).sum(dim=1)
    return scores, amax, rabs


def scan_bound(amax: torch.Tensor, rabs: torch.Tensor, nq: int, storage: str = "bf16") -> torch.Tensor:
    """Error bound of a scan score (see the module docstring)."""
    return ROW_COEF[storage] * amax + nq * U * rabs


def simt_bound(amax: torch.Tensor, rabs: torch.Tensor, nq: int) -> torch.Tensor:
    """Rigorous bound of the SIMT kernel: gamma(128) per row maximum, gamma(Nq) for their sum (of computed maxima)."""
    return gamma(128) * amax * (1 + gamma(nq)) + gamma(nq) * rabs


# ---- checks: error / bound ratios and the fused top-k certified by float64 -------------------------------------------
def check_ratio(ratios: dict, name, err, bound):
    """err <= bound elementwise (a zero bound demands an exact zero); records the largest err / bound of `name` in
    `ratios`."""
    err, bound = err.double().reshape(-1), bound.double().reshape(-1)
    assert not torch.isnan(err).any(), name
    if err.numel() == 0:
        return
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    worst = int(ratio.argmax())
    r = float(ratio[worst])
    ratios[name] = max(ratios.get(name, 0.0), r)
    assert r <= 1.0, "%s: error %.3e > bound %.3e (ratio %.3g)" % (name, err[worst], bound[worst], r)


def check_topk(scores, ts, tp, s64, bound, k, tag):
    """The fused top-k: a stable sort of the kernel's own scores, and certified by the float64 scores: no passage left
    out is surely better than a returned one, consecutive returned ones are ordered up to their bounds."""
    rs, rp = O.topk(scores.cpu().numpy(), k)
    assert np.array_equal(tp.cpu().numpy(), rp) and np.array_equal(ts.cpu().numpy(), rs), tag
    lo, hi = s64 - bound, s64 + bound
    n = s64.size(1)
    for b in range(s64.size(0)):
        ids = tp[b][tp[b] >= 0]
        assert ids.numel() == min(k, n), tag
        out = torch.ones(n, dtype=torch.bool, device=s64.device)
        out[ids] = False
        if out.any():
            assert lo[b][out].max() <= hi[b][ids].min(), "%s: query %d, a passage left out beats a returned one" % (
                tag, b)
        assert (hi[b][ids[:-1]] >= lo[b][ids[1:]]).all(), "%s: query %d returned out of order" % (tag, b)


def positions(tp, P, pid_base):
    """Global ids ``tp`` (-1: empty) -> their positions in the sorted local ids ``P``; every id must be one of P."""
    local = tp - pid_base
    if P.numel() == 0:
        assert (tp < 0).all(), "an id returned where none may be"
        return torch.full_like(tp, -1)
    pos = torch.searchsorted(P, local.clamp_min(0).contiguous())
    hit = P[pos.clamp_max(P.numel() - 1)] == local
    assert ((tp < 0) | hit).all(), "a returned id is deleted or not allowed"
    return torch.where(tp >= 0, pos, -1)


def check_topk_subset(scores, ts, tp, s64, bound, P, pid_base, k, tag):
    """check_topk of one query whose candidates are the sorted local ids ``P`` (its allowed or listed live passages):
    ``scores``, ``s64`` and ``bound`` are ``[len(P)]``, the kernel's scores and float64's of those candidates; ``ts`` /
    ``tp`` the query's ``[k]`` top-k (global ids)."""
    check_topk(scores[None], ts[None], positions(tp[None], P, pid_base), s64[None], bound[None], k, tag)


# ---- the scan's pass plan, as the host builds it (the partition: helpers.scan_partition) ---------------------------
def scan_plan(n_queries: int, nq: int, allow_pair: bool = False) -> np.ndarray:
    """``flmr_debug_plan_passes`` of one call chunk: rows of (q_first, n_q, row0, rows, rbq, n_mtiles, flags, slot)."""
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    n = C.c_int()
    _cabi.check(L.flmr_debug_plan_passes(n_queries, nq, int(allow_pair), None, 0, C.byref(n)))
    buf = np.zeros((n.value, 8), np.int32)
    _cabi.check(L.flmr_debug_plan_passes(n_queries, nq, int(allow_pair), buf.ctypes.data_as(C.c_void_p), n.value,
                                         C.byref(n)))
    return buf


def call_plans(B: int, nq: int):
    """Pass plans of every chunk of a call with B queries (chunks of WS_QUERIES queries)."""
    return [scan_plan(min(WS_QUERIES, B - c0), nq) for c0 in range(0, B, WS_QUERIES)]


def occupied_blocks(n_q, rbq):
    return (n_q * rbq * 32 + 63) // 64


# ---- the grid ----------------------------------------------------------------------------------------------------------
LENGTHS = ("1", "le4", "mix", "96", "192", "ragged", "long")
ROWS = ("unit", "norms", "e4m3edge", "negative", "cancel", "ties")
SCAN_FACTORS = {
    "storage": ["bf16", "fp8"],
    "variant": [0, 2, 3, 4],
    "relu": [False, True],
    "nq": [1, 31, 32, 33, 128, 129, 320, 383, 384, 385, 768, 769, 832],
    "B": [1, 12, 13, 65],
    "lengths": list(LENGTHS),
    "n": [1, 3, 131, 132, 133, 2000],
    "rows": list(ROWS),
    "zeros": ["none", "trailing", "query"],
}
# the widest call: 64 queries of 832 rows, one chunk of 139 passes (128 row slices + 11 grouped tail passes)
EXTRA_CASES = [dict(storage="bf16", variant=0, relu=False, nq=832, B=64, lengths="96", n=133, rows="unit",
                    zeros="trailing"),
               dict(storage="fp8", variant=0, relu=True, nq=832, B=64, lengths="le4", n=2000, rows="norms",
                    zeros="none")]


def scan_allowed(case: dict) -> bool:
    """The CTA-pair scan (variant 4) exists for bf16 corpora only."""
    return not (case.get("storage") == "fp8" and case.get("variant") == 4)


def scan_grid():
    return pairwise_cases(SCAN_FACTORS, scan_allowed) + [dict(c) for c in EXTRA_CASES]


def case_doclens(case: dict, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    n, kind = case["n"], case["lengths"]
    if kind == "1":
        dl = np.ones(n)
    elif kind == "le4":
        dl = rng.integers(1, 5, n)
    elif kind == "mix":
        dl = rng.integers(1, 24, n)
    elif kind == "96":
        dl = rng.choice([95, 96, 97], n)
    elif kind == "192":
        dl = rng.integers(191, 194, n)
    elif kind == "ragged":
        dl = rng.integers(90, 181, n)
    elif kind == "long":
        dl = np.ones(n)
        dl[rng.choice(n, size=max(1, min(5, n // 3)), replace=False)] = rng.integers(1000, 5001, max(1, min(5, n // 3)))
    else:
        raise ValueError(kind)
    return dl.astype(np.int32)


def case_seed(ci: int) -> int:
    return 5000 + ci


# ---- read-back fixtures: every finite bf16 value through the scan's conversions ------------------------------------
def finite_bf16_values() -> torch.Tensor:
    """Every finite bf16 value (65,280 of the 65,536 bit patterns), as float32, in bit-pattern order."""
    x = (torch.arange(1 << 16, dtype=torch.int32) << 16).view(torch.float32)
    return x[torch.isfinite(x)]


def readback_values() -> torch.Tensor:
    """``[512, 128]``: the finite bf16 values row by row, the last 256 entries zero."""
    v = finite_bf16_values()
    out = torch.zeros(512 * 128)
    out[:v.numel()] = v
    return out.view(512, 128)


READBACK_COPIES = 16


def readback_corpus():
    """(D [8192, 128], doclens): 16 copies of the 512 value rows, copy r with its dims rotated by r, as 1-token
    passages.  Padded to 4 rows each, 132 CTAs get ~62 passages, so their full 96-row tiles end 24 passages."""
    V = readback_values()
    D = torch.cat([torch.roll(V, shifts=r, dims=1) for r in range(READBACK_COPIES)])
    return D, np.ones(D.size(0), np.int32)


def bf16_is_subnormal(x: torch.Tensor) -> torch.Tensor:
    return (x != 0) & (x.abs() < 2.0 ** -126)


def _bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).float()


def _edge_rows(shape, g):
    """Unit rows with 8 entries of magnitude 448..1024 (above e4m3's largest value) and 16 e4m3-subnormal entries
    (multiples of 2^-10: exact subnormals and ties between two of them), mixed signs."""
    x = bf16_rows(shape, generator=g)
    flat = x.view(-1, 128)
    r = flat.size(0)
    sign = lambda k: torch.where(torch.rand((r, k), generator=g) < 0.5, -1.0, 1.0)
    perm = torch.argsort(torch.rand((r, 128), generator=g), dim=1)
    big = 448.0 + 576.0 * torch.rand((r, 8), generator=g)
    flat.scatter_(1, perm[:, :8], _bf16(big) * sign(8))
    tiny = torch.randint(1, 16, (r, 16), generator=g).float() * 2.0 ** -10
    flat.scatter_(1, perm[:, 8:24], tiny * sign(16))
    return flat.view(shape)


def case_data(case: dict, seed: int):
    """(Q [B, Nq, 128] float32, D [sum(doclens), 128] float32, doclens): bf16-representable inputs of one case."""
    g = torch.Generator().manual_seed(seed)
    dl = case_doclens(case, seed)
    B, nq, kind = case["B"], case["nq"], case["rows"]
    T = int(dl.sum())
    if kind == "unit" or kind == "ties":
        Q, D = bf16_rows((B, nq, 128), generator=g), bf16_rows((T, 128), generator=g)
    elif kind == "norms":   # row norms 2^-6 .. 2^6, log-uniform
        Q = _bf16(bf16_rows((B, nq, 128), generator=g) * 2.0 ** (12 * torch.rand((B, nq, 1), generator=g) - 6))
        D = _bf16(bf16_rows((T, 128), generator=g) * 2.0 ** (12 * torch.rand((T, 1), generator=g) - 6))
    elif kind == "e4m3edge":
        Q, D = _edge_rows((B, nq, 128), g), _edge_rows((T, 128), g)
    elif kind == "negative":   # every dot product < 0: true max and relu differ on every row
        Q, D = bf16_rows((B, nq, 128), generator=g).abs(), -bf16_rows((T, 128), generator=g).abs()
    elif kind == "cancel":
        # query rows in pairs x, -x + e (e ~ 2^-8) and passages of tokens d_p + 2^-8 noise: row maxima of either sign
        # whose sum is a small fraction of their magnitudes
        x = bf16_rows((B, (nq + 1) // 2, 128), generator=g)
        e = bf16_rows((B, (nq + 1) // 2, 128), generator=g) * 2.0 ** -8
        Q = _bf16(torch.stack([x, -x + e], dim=2).reshape(B, -1, 128)[:, :nq])
        base = bf16_rows((len(dl), 128), generator=g)
        D = _bf16(torch.repeat_interleave(base, torch.from_numpy(dl.astype(np.int64)), dim=0)
                  + 2.0 ** -8 * bf16_rows((T, 128), generator=g))
    else:
        raise ValueError(kind)
    if kind == "ties":   # every passage's last token repeats its first; query rows ask for it
        off = np.concatenate([[0], np.cumsum(dl)])
        D[off[1:] - 1] = D[off[:-1]]
        for b in range(B):
            p = b % len(dl)
            Q[b, 0] = D[off[p]]
    if case["zeros"] == "trailing":
        Q[:, nq - max(1, nq // 3):] = 0.0
    elif case["zeros"] == "query":
        Q[0] = 0.0
    return Q.contiguous(), D.contiguous(), dl
