"""CPU: the restatement of the listed scan's plan (tests/listed_plan.py) on hand-worked plans written out literally, its
own invariants, and the grid of tests/test_listed_scan_fp64_gpu.py: a pairwise covering whose plans, on 132 CTAs,
provably reach the planner's edges (run, share, tile and chunk boundaries)."""
import itertools

import numpy as np
import pytest

import corpus_model as M
import listed_plan as LP
import scan_fp64 as S

RS = LP.RUN_START
FULL = (1 << S.SLOTS) - 1


def _shard(rows, n_ctas, deleted=(), compact=False):
    m = M.CorpusModel(None, np.asarray(rows, np.int64), 0, "bf16")
    if len(deleted):
        m.delete(np.asarray(deleted))
        if compact:
            m.compact()
    return LP.Shard(m, sms=n_ctas)


def _literal(p):
    return {k: p[k].tolist() for k in ("slots", "cta_tile_base", "tile_row", "tile_mask", "tile_first")}


# ---- hand-worked plans ---------------------------------------------------------------------------------------------
def test_one_share_runs_across_gaps():
    """One CTA, slots of 4, 8, 4, 96, 4, 4 rows, slots 0, 1, 3, 5 listed: runs {0, 1}, {3}, {5}.  The first run's only
    tile (rows 0-95) reaches into slot 3's rows; slot 3 is a run of exactly 96 rows ending in group 23."""
    sh = _shard([4, 8, 4, 96, 4, 4], 1)
    p = LP.plan_pass([0, 1, 3, 5], sh)
    assert _literal(p) == {"slots": [0, 1, 3, 5], "cta_tile_base": [0, 3], "tile_row": [0, 16, 116],
                           "tile_mask": [RS | 0b101, RS | 1 << 23, RS | 1], "tile_first": [0, 3, 5]}
    assert p["R"] == 112 and p["u_cum"].tolist() == [0, 4, 12, 108]
    assert LP.runs(p) == [(0, 1), (2, 2), (3, 3)]


def test_run_split_at_a_share_boundary_without_gap():
    """Two CTAs, four consecutive 8-row slots (R = 32): CTA 1 starts at row 16, slot 2, which starts a run although its
    predecessor is listed."""
    sh = _shard([8, 8, 8, 8], 2)
    p = LP.plan_pass([0, 1, 2, 3], sh)
    assert _literal(p) == {"slots": [0, 1, 2, 3], "cta_tile_base": [0, 1, 2], "tile_row": [0, 16],
                           "tile_mask": [RS | 0b1010, RS | 0b1010], "tile_first": [0, 2]}
    assert p["cta"].tolist() == [0, 0, 1, 1] and p["start"].tolist() == [True, False, True, False]


def test_passage_longer_than_a_share_leaves_ctas_without_tiles():
    """Three CTAs, slots of 4, 200, 4 rows (R = 208, shares start at rows 0, 69, 138): the 200-row passage spans three
    tiles (the middle one ends nothing), CTA 1 has no tiles, CTA 2 starts at slot 2."""
    sh = _shard([4, 200, 4], 3)
    p = LP.plan_pass([0, 1, 2], sh)
    assert _literal(p) == {"slots": [0, 1, 2], "cta_tile_base": [0, 3, 3, 4], "tile_row": [0, 96, 192, 204],
                           "tile_mask": [RS | 1, 0, 1 << 2, RS | 1], "tile_first": [0, LP.NO_END, 1, 2]}
    assert p["cta"].tolist() == [0, 0, 2]


def test_empty_union_and_compacted_slots():
    """An empty union plans no tile; on a compacted shard ids name the stored slots, and deleted-but-stored ones stay."""
    sh = _shard([4, 4, 4, 4], 4)
    p = LP.plan_pass([], sh)
    assert _literal(p) == {"slots": [], "cta_tile_base": [0] * 5, "tile_row": [], "tile_mask": [], "tile_first": []}
    sh = _shard([4, 8, 12, 16, 20], 5, deleted=[1, 3], compact=True)        # slots: ids 0, 2, 4
    assert sh.slot_pid.tolist() == [0, 2, 4] and sh.n_ctas == 3 and sh.rows.tolist() == [4, 12, 20]
    assert sh.slots([4, 1, -1, 5, 2, 2, 3, 0]).tolist() == [2, 1, 1, 0]
    sh = _shard([4, 8, 12], 3, deleted=[1])                                   # deleted, not compacted
    assert sh.slots([1, 2]).tolist() == [1, 2]
    # 4 + 12 rows over 3 CTAs: shares would start at rows 0, 5 and 10, but no passage starts at or past row 5, so
    # CTA 0 holds both in one tile and CTAs 1 and 2 none
    p = LP.plan_pass([0, 1], _shard([4, 12, 4], 3))
    assert _literal(p) == {"slots": [0, 1], "cta_tile_base": [0, 1, 1, 1], "tile_row": [0],
                           "tile_mask": [RS | 0b1001], "tile_first": [0]}


def test_tile_bound():
    sh = _shard([4, 200, 4], 3)                 # max rows 200: 3 + 1 tiles per union entry, plus one per CTA
    assert LP.tile_bound(2, sh) == 2 * 4 + 3
    assert LP.tile_bound(10, sh) == 3 * 4 + 3   # at most the shard's slots


# ---- invariants ----------------------------------------------------------------------------------------------------
def check_invariants(p, sh):
    """What test_listed_scan_gpu.test_plan_invariants asserts of the GPU's plans, on a restated one."""
    want = p["slots"].tolist()
    rows, mask, first, base = p["tile_row"], p["tile_mask"], p["tile_first"], p["cta_tile_base"]
    n_tiles = len(rows)
    assert base[0] == 0 and base[-1] == n_tiles and (np.diff(base) >= 0).all()
    want_set = set(want)
    poff = sh.poff
    starts_at = {int(poff[s]): s for s in want}
    ends = {}
    for cta in range(sh.n_ctas):
        t0, t1 = int(base[cta]), int(base[cta + 1])
        for t in range(t0, t1):
            m = int(mask[t])
            run_start = t == t0 or (int(rows[t]) in starts_at and starts_at[int(rows[t])] - 1 not in want_set)
            if not run_start:
                assert rows[t] == rows[t - 1] + 96 and not m >> 31, (cta, t)
            k = 0
            for g in range(24):
                if (m >> g) & 1:
                    slot = int(first[t]) + k
                    k += 1
                    assert poff[slot + 1] - 1 == rows[t] + 4 * g + 3, slot
                    assert slot not in ends
                    ends[slot] = t
            if m >> 31:
                assert run_start or t == t0, (cta, t)
    assert sorted(ends) == want
    assert n_tiles <= LP.tile_bound(len(want), sh)


GRID = LP.grid()


@pytest.fixture(scope="module")
def plans():
    """(case, shard, call plan) of every grid case."""
    out = []
    for ci, c in enumerate(GRID):
        m, sh, lists = LP.case_inputs(ci, c)
        out.append((c, sh, lists, LP.call_plan(lists, c["nq"], sh)))
    return out


def test_restated_plans_keep_their_invariants(plans):
    n = 0
    for c, sh, lists, chunks in plans:
        for passes in chunks:
            for p in passes:
                check_invariants(p, sh)
                n += 1
    assert n > 1000


# ---- the grid --------------------------------------------------------------------------------------------------------
def test_grid_is_a_pairwise_covering():
    cases = LP.pairwise_cases()
    F = LP.FACTORS
    for f1, f2 in itertools.combinations(F, 2):
        seen = {(c[f1], c[f2]) for c in cases}
        for v1, v2 in itertools.product(F[f1], F[f2]):
            assert (v1, v2) in seen, (f1, v1, f2, v2)
    assert len(GRID) < 70


EDGES = ("run ends in group 23", "run of 96t rows", "run's last tile reaches the next run", "run split at a share "
         "boundary without a gap", "tile with 24 ends", "passage longer than R / n_ctas", "CTA with zero tiles",
         "union of fewer rows than CTAs", "empty pass next to non-empty ones", "shard's last passage, tile past n_rows",
         "disjoint lists in a pass", "2 chunks", "3 chunks", "chunk of > 64 passes", ">= 5 blocks", "< 5 blocks")


def edges(c, sh, chunks):
    seen = set()
    seen.add({1: None, 2: "2 chunks", 3: "3 chunks"}[len(chunks)])
    for passes in chunks:
        if len(passes) > S.STAGE_MAX_PASSES:
            seen.add("chunk of > 64 passes")
        empty = [p["slots"].size == 0 for p in passes]
        if any(empty) and not all(empty):
            seen.add("empty pass next to non-empty ones")
        for p in passes:
            blocks = S.occupied_blocks(p["n_q"], p["rbq"])
            seen.add(">= 5 blocks" if blocks >= S.THREE_WG_BLOCKS else "< 5 blocks")
            n = p["slots"].size
            if n == 0:
                continue
            u, rows, mask = p["slots"], p["rows"], p["tile_mask"]
            if 0 < p["R"] < sh.n_ctas:
                seen.add("union of fewer rows than CTAs")
            if sh.n_ctas > 1 and (rows > p["R"] / sh.n_ctas).any():
                seen.add("passage longer than R / n_ctas")
            if (np.diff(p["cta_tile_base"]) == 0).any():
                seen.add("CTA with zero tiles")
            if ((mask & FULL) == FULL).any():
                seen.add("tile with 24 ends")
            if (p["start"][1:] & (u[1:] == u[:-1] + 1)).any():
                seen.add("run split at a share boundary without a gap")
            rl = LP.runs(p)
            for i, (a, z) in enumerate(rl):
                if p["end_group"][z] == 23:
                    seen.add("run ends in group 23")
                if int(rows[a:z + 1].sum()) % LP.TILE == 0:
                    seen.add("run of 96t rows")
                if i + 1 < len(rl):
                    nxt = rl[i + 1][0]
                    last_tile = p["end_tile"][z]
                    if (u[nxt] == u[z] + 2 and sh.rows[u[z] + 1] <= 4
                            and p["tile_row"][last_tile] + LP.TILE > sh.poff[u[nxt]]
                            and p["cta"][nxt] == p["cta"][z]):
                        seen.add("run's last tile reaches the next run")
            if u[-1] == sh.n_slots - 1 and p["tile_row"][p["end_tile"][-1]] + LP.TILE > sh.n_rows:
                seen.add("shard's last passage, tile past n_rows")
            sets = [s for s in p["slot_sets"] if s.size]
            if any(np.intersect1d(x, y).size == 0 for x, y in itertools.combinations(sets, 2)):
                seen.add("disjoint lists in a pass")
    seen.discard(None)
    return seen


def test_grid_reaches_every_planner_edge(plans):
    seen = set()
    for c, sh, lists, chunks in plans:
        seen |= edges(c, sh, chunks)
    assert set(EDGES) <= seen, sorted(set(EDGES) - seen)
