"""CPU: the float64 restatement of the fp8 two-stage search (tests/fp8_two_stage.py) before any kernel is judged by
it: the decoy arithmetic through the e4m3 oracle, the depth rule against the Searcher's own, and that merging every
shard's own top-depth, then cutting at the global depth, gives the one-device shortlist for any split."""
import itertools

import numpy as np
import pytest

import fp8_oracle as F8
import fp8_two_stage as T
from oracle import maxsim_oracle as O


def test_decoy_arithmetic_is_exact_in_e4m3_and_bf16():
    assert F8.e4m3_round(np.float32(1.0703125)) == 1.125            # rounds up
    assert F8.e4m3_round(np.float32(1.0625)) == 1.0                 # halfway: ties to even
    assert F8.e4m3_round(np.float32(1.09375)) == 1.125
    assert F8.e4m3_round(np.float32(1.1875)) == 1.25                # halfway: ties to even
    for kind, (x0, x1) in T.KINDS.items():
        assert T.bf16(np.array([x0, x1], np.float32)).tolist() == [x0, x1]
        assert np.float32(x0) + np.float32(x1) == T.EXACT[kind]
        assert F8.e4m3_round(np.float32(x0)) + F8.e4m3_round(np.float32(x1)) == T.E4M3[kind]
    assert T.E4M3["target"] < T.E4M3["decoy"] == T.E4M3["better"]
    assert T.EXACT["decoy"] < T.EXACT["better"] < T.EXACT["target"] == T.EXACT["twin"]
    assert T.E4M3["twin"] > T.E4M3["decoy"]


@pytest.mark.parametrize("nq", [1, 32])
def test_decoy_corpus_scores_are_the_planted_ones(nq):
    rng = np.random.default_rng(3)
    dl = rng.integers(1, 40, 60).astype(np.int32)
    plant = {0: "decoy", 7: "better", 33: "target", 41: "twin", 59: "decoy"}
    D, dl = T.decoy_corpus(dl, plant, seed=1)
    Q = T.decoy_queries(2, nq)
    want = np.array([T.EXACT[plant.get(p, "filler")] for p in range(60)])
    want8 = np.array([T.E4M3[plant.get(p, "filler")] for p in range(60)])
    assert np.array_equal(O.maxsim_scores(Q, D, dl)[0], want)
    assert np.array_equal(F8.maxsim_scores_fp8(Q, D, dl)[0], want8)
    assert np.array_equal(T.bf16(D), D)


def test_depth_rule_is_the_searchers():
    from ravqa_b200.searcher import shortlist_depth
    for k, ndocs, n in itertools.product([1, 10, 100, 101, 128, 129, 1024, 2048], [None, 4, 1200, 1204, 9000],
                                         [1, 300, 301, 2047, 2048, 5000]):
        assert T.shortlist_depth(k, ndocs, n) == shortlist_depth(k, ndocs, n), (k, ndocs, n)
    with pytest.raises(ValueError):
        shortlist_depth(2049, None, 5000)
    with pytest.raises(ValueError):
        T.shortlist_depth(2049, None, 5000)


def test_decoys_hide_the_target_until_the_depth_reaches_it():
    n = 400
    plant = {p: "decoy" for p in range(300)}
    plant[350] = "target"
    s, p = T.expected_decoy_ranking(plant, n, 300, 10)
    assert p.tolist() == list(range(10)) and (s == T.EXACT["decoy"]).all()
    s, p = T.expected_decoy_ranking(plant, n, 301, 10)
    assert p[0] == 350 and s[0] == T.EXACT["target"] and p[1:].tolist() == list(range(9))
    plant[360] = "twin"                          # leads the shortlist, ties the target exactly, after it by pid
    s, p = T.expected_decoy_ranking(plant, n, 300, 3)
    assert p.tolist() == [360, 0, 1]
    s, p = T.expected_decoy_ranking(plant, n, 302, 3)
    assert p.tolist() == [350, 360, 0] and s[0] == s[1]


def test_allowed_counts_and_admitted_rows():
    live = np.ones(10, bool)
    live[[2, 5]] = False
    lists = [[1, 1, 2, 3], None, [], [9, 5, 0, 9]]
    assert T.allowed_counts(lists, live).tolist() == [2, 8, 0, 2]
    adm = T.admitted_rows(lists, live)
    assert adm.sum(axis=1).tolist() == [2, 8, 0, 2] and not adm[:, [2, 5]].any()


def _merge_case(rng, B, n, ties):
    """Scores from a few values (ties everywhere, across every boundary) or distinct ones, and random admitted sets of
    every size down to none."""
    s = (rng.integers(0, 4, (B, n)) * 0.5 if ties else rng.standard_normal((B, n))).astype(np.float32)
    adm = rng.random((B, n)) < rng.uniform(0.0, 1.0, (B, 1))
    adm[0] = True
    if B > 1:
        adm[1] = False
    return s, adm


@pytest.mark.parametrize("seed", range(6))
def test_merged_shard_shortlists_are_the_one_device_shortlist(seed):
    from ravqa_b200.sharded import shard_ranges
    rng = np.random.default_rng(seed)
    n = int(rng.integers(5, 120))
    dl = rng.integers(1, 200, n)
    for ties in (True, False):
        s, adm = _merge_case(rng, 4, n, ties)
        for world in (1, 2, 3, 5, 8):
            ranges = shard_ranges(dl, world)
            for depth in sorted({1, 2, n // 3 + 1, n // 2, n - 1, n, int(adm.sum(axis=1).max())} - {0}):
                one = T.shortlist(s, adm, depth)
                many = T.merged_shortlist(s, adm, depth, ranges)
                assert np.array_equal(one, many), (seed, ties, world, depth)
                # a query's shortlist holds its admitted passages only, each once
                for b in range(4):
                    got = one[b][one[b] >= 0]
                    assert got.size == min(depth, adm[b].sum()) and np.unique(got).size == got.size
                    assert adm[b, got].all()


def test_merge_keeps_the_lower_pid_across_a_shard_boundary_tie():
    """Equal e4m3 scores on both sides of a shard boundary, the depth cutting inside the run: the lower pids win, as on
    one device, and a shard with fewer admitted passages than the depth pads its list."""
    s = np.zeros((1, 10), np.float32)
    s[0, 3:8] = 2.0
    adm = np.ones((1, 10), bool)
    adm[0, 8:] = False
    for depth in (1, 3, 4, 6):
        want = T.shortlist(s, adm, depth)
        assert np.array_equal(T.merged_shortlist(s, adm, depth, [(0, 5), (5, 9), (9, 10)]), want)
    assert T.shortlist(s, adm, 3)[0].tolist() == [3, 4, 5]


def test_rerank_breaks_exact_ties_on_the_lower_pid_and_drops_empty_entries():
    cand = np.array([[-1, -1, 2, 5, 9]])
    exact = np.array([[7.0, 7.0, 1.0, 3.0, 3.0]])      # the -1 entries would win if they were candidates
    s, p = T.rerank(cand, exact, 4)
    assert p[0].tolist() == [5, 9, 2, -1] and s[0, :3].tolist() == [3.0, 3.0, 1.0] and np.isneginf(s[0, 3])
