"""Float64 / numpy restatement of the fp8 Searcher's two-stage selection (searcher.py: ``shortlist_depth``,
``Searcher._shortlist`` / ``_rerank`` and the restricted forms' allowed counts), the e4m3 decoy corpora that put the
shortlist's edge in charge of the answer, and the per-shard shortlist merge of a multi-device Searcher.  Pinned on CPU
by tests/test_fp8_two_stage_host.py; tests/test_fp8_two_stage_gpu.py runs it on the kernels' own scores.

The selection, for one query:

  * depth = min(max(ndocs // 4, k), 2048, n), ``ndocs`` derived from k when unset (1024 for k <= 100, else
    max(4 k, 4096)), n the candidates there are: live (and kept by ``filter_fn``) passages, or for a restricted search
    the most allowed live passages of any query of the batch;
  * shortlist: the first ``depth`` of the query's admitted passages ordered by (e4m3 score desc, pid asc), -1 past
    them (a query with fewer admitted passages than depth);
  * re-rank: the first k of the shortlist ordered by (exact score desc, pid asc), -1 past them.

Decoys.  e4m3 keeps 3 mantissa bits, so in [1, 2) it rounds to multiples of 1/8, ties to even.  Against the query row
q = (1, 1, 0, ...), the decoy token d = (1.0703125, 1.0) scores 2.0703125 exactly but 1.125 + 1 = 2.125 in e4m3, the
target t = (1.0625, 1.0625) scores 2.125 exactly but 1.0 + 1.0 = 2.0 in e4m3 (1.0625 is halfway and ties to even), and
the better decoy (1.09375, 1.0) ties d in e4m3 while scoring 2.09375 exactly, and the twin (1.1875, 0.9375) ties t
exactly while leading every e4m3 score (2.1875): placed after t, it ranks below t only if the re-rank breaks exact
ties by pid and not by shortlist order.  Every value and sum is exact in bf16
and fp32, so no error bound enters: with more decoys than the depth, the shortlist misses t and the search returns
decoys; one more candidate of depth and it returns t.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

SELECT_MAX_K = 2048            # the select kernel's capacity: the deepest shortlist
DIM = 128

DECOY = (1.0703125, 1.0)       # exact 2.0703125, e4m3 2.125
BETTER_DECOY = (1.09375, 1.0)  # exact 2.09375,   e4m3 2.125
TARGET = (1.0625, 1.0625)      # exact 2.125,     e4m3 2.0
TWIN = (1.1875, 0.9375)        # exact 2.125,     e4m3 2.1875 (1.1875 ties to even at 1.25): the target's exact tie
KINDS = {"decoy": DECOY, "better": BETTER_DECOY, "target": TARGET, "twin": TWIN}
EXACT = {"decoy": 2.0703125, "better": 2.09375, "target": 2.125, "twin": 2.125, "filler": 0.0}
E4M3 = {"decoy": 2.125, "better": 2.125, "target": 2.0, "twin": 2.1875, "filler": 0.0}


def default_ndocs(k: int) -> int:
    return 1024 if k <= 100 else max(4 * k, 4096)


def shortlist_depth(k: int, ndocs: Optional[int], n: int) -> int:
    if k > SELECT_MAX_K:
        raise ValueError("k=%d above %d" % (k, SELECT_MAX_K))
    if ndocs is None:
        ndocs = default_ndocs(k)
    return min(max(int(ndocs) // 4, k), SELECT_MAX_K, n)


def allowed_counts(lists: Sequence, live: np.ndarray) -> np.ndarray:
    """Per query: the live passages its list of global ids admits, each id once (None: every live passage)."""
    live = np.asarray(live, bool)
    return np.array([int(live.sum()) if ids is None else int(live[np.unique(np.asarray(ids, np.int64))].sum())
                     for ids in lists], dtype=np.int64)


def admitted_rows(lists: Sequence, live: np.ndarray) -> np.ndarray:
    """bool ``[B, n]``: passage p is live and in query b's list (None: every live passage)."""
    live = np.asarray(live, bool)
    out = np.zeros((len(lists), live.size), bool)
    for b, ids in enumerate(lists):
        if ids is None:
            out[b] = live
        else:
            out[b, np.asarray(ids, np.int64)] = True
            out[b] &= live
    return out


def _ranked(scores: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """``ids`` ordered by (score desc, id asc)."""
    return ids[np.lexsort((ids, -scores.astype(np.float64)))]


def shortlist(scores: np.ndarray, admitted: np.ndarray, depth: int) -> np.ndarray:
    """int64 ``[B, depth]``: each query's first ``depth`` admitted pids by (e4m3 score desc, pid asc), -1 past them.
    ``scores`` ``[B, n]`` (the kernel's fp32 e4m3 scores), ``admitted`` bool ``[B, n]``."""
    B = scores.shape[0]
    out = np.full((B, depth), -1, np.int64)
    for b in range(B):
        ids = np.flatnonzero(admitted[b])
        top = _ranked(scores[b, ids], ids)[:depth]
        out[b, :top.size] = top
    return out


def rerank(cand: np.ndarray, exact: np.ndarray, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """(scores, pids) ``[B, k]``: each query's first k candidates (``cand`` ``[B, depth]``, -1: none) by (exact score
    desc, pid asc), with ``exact`` aligned to ``cand``; (-inf, -1) past them."""
    B = cand.shape[0]
    out_s = np.full((B, k), -np.inf, np.float64)
    out_p = np.full((B, k), -1, np.int64)
    for b in range(B):
        ok = cand[b] >= 0
        ids, sc = cand[b][ok], exact[b][ok]
        order = np.lexsort((ids, -sc.astype(np.float64)))[:k]
        out_s[b, :order.size] = sc[order]
        out_p[b, :order.size] = ids[order]
    return out_s, out_p


def merged_shortlist(scores: np.ndarray, admitted: np.ndarray, depth: int,
                     ranges: Sequence[Tuple[int, int]]) -> np.ndarray:
    """The shortlist a multi-device Searcher selects: every shard's own top-``depth`` (its admitted passages, by e4m3
    score desc and pid asc, padded with (-inf, -1)), concatenated in shard order, then the first ``depth`` columns by
    score with the lower column on ties (the home device's select), -1 where the score is -inf."""
    B = scores.shape[0]
    cs, cp = [], []
    for p0, p1 in ranges:
        s = np.full((B, depth), -np.inf)
        p = np.full((B, depth), -1, np.int64)
        for b in range(B):
            ids = p0 + np.flatnonzero(admitted[b, p0:p1])
            top = _ranked(scores[b, ids], ids)[:depth]
            s[b, :top.size] = scores[b, top]
            p[b, :top.size] = top
        cs.append(s)
        cp.append(p)
    s, p = np.concatenate(cs, axis=1), np.concatenate(cp, axis=1)
    col = np.argsort(-s, axis=1, kind="stable")[:, :depth]
    return np.where(np.isneginf(np.take_along_axis(s, col, 1)), -1, np.take_along_axis(p, col, 1))


# ---- decoy corpora ----------------------------------------------------------------------------------------------------
def decoy_corpus(doclens: Sequence[int], plant: Dict[int, str], seed: int = 0):
    """(D float32 ``[sum(doclens), 128]``, doclens int32): passage p's first token carries ``KINDS[plant[p]]`` in dims
    0 and 1 (an unplanted passage: zeros there); every other entry is zero in dims 0 and 1 and a bf16 value of
    magnitude below 1/4 elsewhere, so against ``decoy_queries`` a passage scores exactly ``EXACT[kind]`` (bf16) and
    ``E4M3[kind]`` (e4m3)."""
    dl = np.asarray(doclens, np.int32)
    rng = np.random.default_rng(seed)
    D = rng.uniform(-0.25, 0.25, size=(int(dl.sum()), DIM)).astype(np.float32)
    D = bf16(D)
    D[:, :2] = 0.0
    off = np.concatenate([[0], np.cumsum(dl, dtype=np.int64)])
    for p, kind in plant.items():
        D[off[p], :2] = KINDS[kind]
    return D, dl


def decoy_queries(B: int, nq: int) -> np.ndarray:
    """``[B, nq, 128]``: row 0 of every query is (1, 1, 0, ...), every other row zero."""
    Q = np.zeros((B, nq, DIM), np.float32)
    Q[:, 0, :2] = 1.0
    return Q


def bf16(x: np.ndarray) -> np.ndarray:
    """Round float32 to bf16 (nearest even) and back."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16 << 16
    return u.astype(np.uint32).view(np.float32)


def expected_decoy_ranking(plant: Dict[int, str], n: int, depth: int, k: int, admitted: Optional[np.ndarray] = None
                           ) -> Tuple[np.ndarray, np.ndarray]:
    """(scores, pids) ``[k]`` the two-stage search must return on a decoy corpus of n passages (one query; ``admitted``
    bool ``[n]``, default all): the selection above on the planted scores."""
    adm = np.ones(n, bool) if admitted is None else admitted
    e8 = np.array([E4M3[plant.get(p, "filler")] for p in range(n)])
    ex = np.array([EXACT[plant.get(p, "filler")] for p in range(n)])
    cand = shortlist(e8[None], adm[None], depth)
    c = np.sort(cand, axis=1)
    s, p = rerank(c, np.where(c >= 0, ex[np.maximum(c, 0)], -np.inf), min(k, int(adm.sum())))
    return s[0], p[0]
