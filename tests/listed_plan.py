"""Restatement of the listed scan's plan (csrc/flmr_maxsim.cu: flmr_listed_mark_kernel, flmr_listed_plan_kernel and
the tile bound of plan_listed_chunk) in numpy, and the grid of tests/test_listed_scan_fp64_gpu.py: the cases, the
corpus state each one is searched in and the lists its queries name.  Pinned on CPU by tests/test_listed_plan_host.py
before any plan the GPU makes is judged by it.

A listed search of B queries runs in call chunks of 64 queries (scan_fp64.call_plans); each pass of a chunk scans a
plan of its own over the union of its queries' listed slots:

  * an id names a slot when it lies in ``[pid_base, pid_base + n_ids)`` and its rows are stored (not compacted away);
    duplicates name one slot, and a deleted but stored passage is planned (the reducer's tombstone test drops it);
  * ``u_cum``: each union slot's first row inside the union (its stored rows are padded to 4); ``R`` the union's rows;
  * the union is cut into ``n_ctas`` shares at passage boundaries: CTA c starts at the first slot with
    ``u_cum >= R c // n_ctas`` (``cta_of`` below is the share of a slot's first row);
  * a run starts at a slot whose predecessor in the union is not the previous slot, or lies in another share; a run
    is tiled every 96 rows from its first row, and bit 31 of a tile's mask marks a run's first tile; bit g marks a
    passage of the run whose last row is in 4-row group g of the tile, and ``tile_first`` is the lowest slot ending
    in the tile (0x7fffffff when none does);
  * ``cta_tile_base[c]``: the first tile of CTA c's first run (the total for CTAs past the union's end).
"""
from __future__ import annotations

import numpy as np

import corpus_model as M
import scan_fp64 as S

TILE, GROUP = S.TILE, 4
RUN_START = 1 << 31
NO_END = 0x7FFFFFFF
N_CTAS = 132                  # an H100 SXM's SMs


# ---- the shard as the planner sees it ----------------------------------------------------------------------------
class Shard:
    """Stored passages (slots) of a corpus state: ``rows`` the padded rows of each slot, ``slot_pid`` its global id."""

    def __init__(self, m: M.CorpusModel, sms: int = N_CTAS):
        stored = ~m.compacted
        self.pid_base, self.n_ids = m.pid_base, m.n_passages
        self.slot_pid = np.flatnonzero(stored).astype(np.int64) + m.pid_base
        self.rows = (m.lens[stored] + 3) // 4 * 4
        self.poff = np.concatenate([[0], np.cumsum(self.rows)]).astype(np.int64)
        self.n_slots = int(self.rows.size)
        self.n_rows = int(self.poff[-1])
        self.n_ctas = min(sms, self.n_slots)
        self.max_rows = int(self.rows.max())
        self._slot_of = np.full(m.n_passages, -1, np.int64)
        self._slot_of[np.flatnonzero(stored)] = np.arange(self.n_slots)

    def slots(self, ids) -> np.ndarray:
        """Slots the ids name, in list order (flmr_listed_mark_kernel's listed_slot; -1 dropped)."""
        local = np.asarray(ids, np.int64).reshape(-1) - self.pid_base
        local = local[(local >= 0) & (local < self.n_ids)]
        s = self._slot_of[local]
        return s[s >= 0]


def tile_bound(n_listed: int, sh: Shard) -> int:
    """Tiles plan_listed_chunk reserves for a pass whose queries list ``n_listed`` ids (duplicates and ids outside the
    shard counted)."""
    u = min(n_listed, sh.n_slots)
    return u * ((sh.max_rows + TILE - 1) // TILE + 1) + sh.n_ctas


def plan_pass(u_slot, sh: Shard) -> dict:
    """The plan of one pass over the sorted unique slots ``u_slot`` (see the module docstring), with what the edge
    checks read off it: per slot its rows, first row in the union, share, run start, run tile and end tile."""
    u = np.asarray(u_slot, np.int64)
    n, nc = u.size, sh.n_ctas
    rows = sh.rows[u] if n else np.zeros(0, np.int64)
    u_cum = np.concatenate([[0], np.cumsum(rows)[:-1]]).astype(np.int64) if n else np.zeros(0, np.int64)
    R = int(rows.sum())
    cta = np.minimum(nc - 1, (nc * (u_cum + 1) + R - 1) // R - 1) if n else np.zeros(0, np.int64)
    start = np.ones(n, bool)
    start[1:] = (u[1:] != u[:-1] + 1) | (cta[1:] != cta[:-1])
    rs = np.maximum.accumulate(np.where(start, u_cum, -1)) if n else u_cum
    b = u_cum - rs
    e = b + rows
    t0, t1 = -(-b // TILE), -(-e // TILE)
    cnt = t1 - t0
    T = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64) if n else cnt
    run_tile = T - t0
    n_tiles = int(cnt.sum())
    rep = np.repeat(np.arange(n), cnt)
    t = t0[rep] + (np.arange(n_tiles) - T[rep])
    tile_row = (sh.poff[u][rep] - b[rep] + t * TILE).astype(np.int64)
    tile_mask = np.where(t == 0, RUN_START, 0).astype(np.int64)
    tile_first = np.full(n_tiles, NO_END, np.int64)
    end_tile = run_tile + (e - 1) // TILE
    np.bitwise_or.at(tile_mask, end_tile, np.left_shift(1, ((e - 1) % TILE) // GROUP))
    np.minimum.at(tile_first, end_tile, u)
    base = np.full(nc + 1, n_tiles, np.int64)
    base[0] = 0
    if R > 0:
        first = np.searchsorted(u_cum, R * np.arange(1, nc) // nc, side="left")
        base[1:nc] = np.where(first < n, run_tile[np.minimum(first, n - 1)], n_tiles)
    return {"slots": u, "rows": rows, "u_cum": u_cum, "R": R, "cta": cta, "start": start, "run_tile": run_tile,
            "end_tile": end_tile, "end_group": ((e - 1) % TILE) // GROUP, "cta_tile_base": base,
            "tile_row": tile_row, "tile_mask": tile_mask, "tile_first": tile_first}


def call_plan(lists, nq: int, sh: Shard, pass_plans=None) -> list:
    """Every chunk of a listed call: a list per chunk of pass dicts (plan_pass plus ``q_first``, ``n_q``, ``rbq``
    (the pass's row blocks per query), ``tile_bound``, ``slot_sets``: each query's valid slots).  ``pass_plans``: the
    host's pass plans of the chunks (scan_fp64.call_plans(len(lists), nq), the library's debug entry)."""
    B = len(lists)
    pass_plans = S.call_plans(B, nq) if pass_plans is None else pass_plans
    out = []
    for ci, c0 in enumerate(range(0, B, S.WS_QUERIES)):
        chunk = lists[c0:c0 + S.WS_QUERIES]
        sets = [np.unique(sh.slots(ids)) for ids in chunk]
        passes = []
        for q_first, n_q, _, _, rbq, _, _, _ in pass_plans[ci].tolist():
            qs = range(q_first, q_first + n_q)
            union = np.unique(np.concatenate([sets[q] for q in qs])) if n_q else np.zeros(0, np.int64)
            p = plan_pass(union, sh)
            p.update(q_first=q_first, n_q=n_q, rbq=rbq, slot_sets=[sets[q] for q in qs],
                     tile_bound=tile_bound(sum(len(np.asarray(chunk[q]).reshape(-1)) for q in qs), sh))
            passes.append(p)
        out.append(passes)
    return out


def runs(p: dict):
    """(first, last) union index of each run of a pass plan."""
    st = np.flatnonzero(p["start"])
    return list(zip(st.tolist(), (np.append(st[1:], p["slots"].size) - 1).tolist()))


# ---- the grid ----------------------------------------------------------------------------------------------------
FACTORS = {
    "storage": list(M.STORAGES),
    "variant": [0, 2, 6],
    "relu": [False, True],
    "nq": [1, 32, 33, 320, 383, 385, 832],
    "B": [1, 12, 13, 65, 130],
    "lengths": list(S.LENGTHS),
    "n": [1, 3, 131, 132, 133, 2000],
    "rows": list(S.ROWS),
    "state": ["fresh", "deleted", "compacted", "appended"],
    "pid_base": [0, 1000],
}
EXTRA_CASES = [   # the widest call: one chunk of 139 passes
    dict(storage="bf16", variant=0, relu=False, nq=832, B=64, lengths="96", n=133, rows="unit", state="fresh",
         pid_base=0),
    dict(storage="fp8", variant=0, relu=True, nq=832, B=64, lengths="le4", n=2000, rows="norms", state="compacted",
         pid_base=1000),
    # three chunks, each query of a chunk with another kind of list than its neighbours in the other chunks
    dict(storage="bf16", variant=0, relu=False, nq=32, B=130, lengths="long", n=2000, rows="unit", state="appended",
         pid_base=1000),
]
APPEND_LENS = [1, 4, 96, 97, 5, 300]
KINDS = ("empty", "outside", "deleted", "one", "first+last", "run 96t", "gap runs", "long range", "24 one-token",
         "long passage", "disjoint", "dups+outside", "everything")


def grid():
    return pairwise_cases() + [dict(c) for c in EXTRA_CASES]


def pairwise_cases():
    return S.pairwise_cases(FACTORS)


def case_seed(ci: int) -> int:
    return 9000 + ci


def case_state(case: dict, seed: int):
    """The operations that bring a case's corpus to its state: (deleted ids, compact?, appended lengths), drawn from
    the seed and the case's doclens; applied to a model and to a FlatCorpus alike (apply_state)."""
    rng = np.random.default_rng(seed + 1)
    dl = S.case_doclens(case, seed)
    n, base = dl.size, case["pid_base"]
    dead = np.zeros(0, np.int64)
    if case["state"] != "fresh" and n >= 3:
        a = int(rng.integers(0, n - 1))
        run = np.arange(a, min(n - 1, a + 5))                                # a run, never the last passage
        dead = np.unique(np.concatenate([run, rng.choice(n - 1, max(1, n // 7), replace=False)])) + base
    compact = case["state"] in ("compacted", "appended")
    append = APPEND_LENS if case["state"] == "appended" else []
    return dead, compact, append


def apply_state(m: M.CorpusModel, corpus, case: dict, seed: int):
    """Applies case_state to the model and, when given, to the corpus (appended tokens drawn from the seed)."""
    dead, compact, append = case_state(case, seed)
    for target in (m, corpus):
        if target is None:
            continue
        if dead.size:
            target.delete(dead)
        if compact and dead.size:
            target.compact()
        if append:
            t = M.passage_tokens(seed + 2, int(sum(append)), m.storage)
            target.append(t, np.asarray(append, np.int32))


def state_model(case: dict, seed: int) -> M.CorpusModel:
    """The model of a case's corpus in its state, ids and lengths only."""
    m = M.CorpusModel(None, S.case_doclens(case, seed), case["pid_base"], case["storage"])
    apply_state(m, None, case, seed)
    return m


def _consecutive(mask: np.ndarray, length: int):
    """First index of `length` consecutive True entries, or None."""
    if length > mask.size:
        return None
    c = np.concatenate([[0], np.cumsum(mask)])
    hit = np.flatnonzero(c[length:] - c[:-length] == length)
    return int(hit[0]) if hit.size else None


def case_lists(case: dict, m: M.CorpusModel, seed: int, sh: Shard = None) -> list:
    """One list of global ids per query, of the kinds KINDS (query b of case ci takes kind (b + ci) % 13)."""
    sh = Shard(m) if sh is None else sh
    rng = np.random.default_rng(seed + 3)
    base, n_ids, ns = m.pid_base, m.n_passages, sh.n_slots
    ids = sh.slot_pid                                     # global id of each slot
    outside = np.array([base - 1, base + n_ids, base + n_ids + 57], np.int64)

    def run_96t():
        c = sh.poff
        for t in (1, 2, 3):
            for i in range(ns):
                j = int(np.searchsorted(c, c[i] + 96 * t))
                if j <= ns and c[j] == c[i] + 96 * t:
                    return ids[i:j]
        return ids[:1]

    def gap_runs():
        small = np.flatnonzero(sh.rows <= 4)
        small = small[(small >= 1) & (small < ns - 1)]
        g = int(small[len(small) // 2]) if small.size else ns // 2
        w = int(rng.integers(1, 6))
        return np.concatenate([ids[max(0, g - w):g], ids[g + 1:g + 1 + w]])

    def one_token():
        i = _consecutive(sh.rows == 4, 30)
        i = _consecutive(sh.rows == 4, 24) if i is None else i
        return ids[i:i + 30] if i is not None else ids[:30]

    def disjoint(b):
        sel = np.flatnonzero(np.arange(ns) % 3 == b % 3)
        return ids[rng.choice(sel, min(sel.size, 40), replace=False)] if sel.size else ids[:0]

    kinds = {
        "empty": lambda b: np.zeros(0, np.int64),
        "outside": lambda b: outside,
        "deleted": lambda b: m.deleted_ids(),
        "one": lambda b: ids[[int(rng.integers(ns))]],
        "first+last": lambda b: np.array([base + n_ids - 1, base]),
        "run 96t": lambda b: run_96t(),
        "gap runs": lambda b: gap_runs(),
        "long range": lambda b: ids[ns // 5:ns // 5 + max(1, ns // 3)],
        "24 one-token": lambda b: one_token(),
        "long passage": lambda b: ids[[int(sh.rows.argmax())]],
        "disjoint": disjoint,
        "dups+outside": lambda b: np.concatenate([base + rng.choice(n_ids, 30), base + rng.choice(n_ids, 10),
                                                  outside]),
        "everything": lambda b: np.arange(base, base + n_ids),
    }
    ci = seed - case_seed(0)
    return [rng.permutation(np.asarray(kinds[KINDS[(b + ci) % len(KINDS)]](b), np.int64)) for b in range(case["B"])]


def case_inputs(ci: int, case: dict):
    """(model of the state, shard, lists) of grid case ``ci``."""
    seed = case_seed(ci)
    m = state_model(case, seed)
    sh = Shard(m)
    return m, sh, case_lists(case, m, seed, sh)
