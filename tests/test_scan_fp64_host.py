"""CPU: the float64 restatement of the corpus scan (tests/scan_fp64.py) against the reference-generated goldens and
the fp32 oracles, its e4m3 rounding against torch on every finite bf16 value, and the scan grid of
tests/test_scan_kernels_fp64_gpu.py: a pairwise covering that provably reaches the scan's structural edges (tile,
slot, CTA and pass boundaries), as the host builds the partition and the pass plan."""
import itertools

import numpy as np
import pytest
import torch

import fp8_oracle as F8
import scan_fp64 as S
from helpers import golden_names, load_golden, scan_partition
from oracle import maxsim_oracle as O

N_CTAS = 132                  # an H100 SXM's SMs
FULL = (1 << S.SLOTS) - 1     # a tile in which all 24 four-token groups end a passage
PASS_FINAL = 4


def _within(got, want, bound, tag):
    err = (torch.as_tensor(np.asarray(got, dtype=np.float64)) - want).abs()
    worst = float((err / bound.clamp_min(1e-300)).max())
    assert (err <= bound).all(), "%s: error / bound %.3g" % (tag, worst)
    return worst


@pytest.mark.parametrize("name", golden_names())
@pytest.mark.parametrize("relu", [False, True])
def test_restatement_matches_goldens_and_fp32_oracle(name, relu):
    """The reference's own outputs and the numpy fp32 oracle, both fp32 computations: within gamma(128) A per row and
    gamma(Nq) for the sum.  A token dropped from a passage moves the restatement far outside that bound."""
    g = load_golden(name)
    Q, D, dl = torch.from_numpy(g["Q"]), torch.from_numpy(g["D"]), g["doclens"]
    s64, amax, rabs = S.maxsim_packed(Q, D, dl, relu=relu)
    bound = S.simt_bound(amax, rabs, Q.size(1))
    _within(g["scores_relu" if relu else "scores_true_max"], s64, bound, name)
    _within(O.maxsim_scores(g["Q"], g["D"], dl, relu=relu), s64, bound, name + " oracle")
    assert (amax >= rabs - 1e-12).all() and (bound > 0).all()
    # e4m3: the fp8 oracle (fp32 over rounded operands) within the same rigorous bound over the rounded operands
    s8, a8, r8 = S.maxsim_packed(Q, D, dl, relu=relu, storage="fp8")
    _within(F8.maxsim_scores_fp8(g["Q"], g["D"], dl, relu=relu), s8, S.simt_bound(a8, r8, Q.size(1)), name + " fp8")
    # sensitivity: passage 0 without its best token for query 0's row 0
    off = np.concatenate([[0], np.cumsum(dl)])
    if dl[0] > 1:
        j = int((D[off[0]:off[1]].double() @ Q[0, 0].double()).argmax())
        keep = np.ones(len(D), bool)
        keep[off[0] + j] = False
        dl2 = dl.copy()
        dl2[0] -= 1
        s2 = S.maxsim_packed(Q[:1], D[torch.from_numpy(keep)], dl2, relu=relu)[0]
        assert (s2[0, 0] - s64[0, 0]).abs() > 10 * bound[0, 0] or relu


def test_e4m3_round_matches_torch_on_every_finite_bf16():
    """fp8_oracle.e4m3_round against torch's float8_e4m3fn (round to nearest even) on all 65,280 finite bf16 values,
    clamped to +-448 first (torch does not saturate): equal values and equal signs of every nonzero result."""
    x = S.finite_bf16_values()
    assert x.numel() == 65536 - 256
    ours = S.e4m3_round(x)
    ref = x.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()
    assert torch.equal(ours, ref)
    nz = ref != 0
    assert torch.equal(torch.signbit(ours[nz]), torch.signbit(ref[nz]))
    # the edges the device conversion is read back on: ties to even, saturation, the 2^-9 subnormal steps
    t = torch.tensor([1.0625, 1.1875, 464.0, 480.0, 1e30, -1e30, 2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -9, 2.0 ** -11])
    assert S.e4m3_round(t).tolist() == [1.0, 1.25, 448.0, 448.0, 448.0, -448.0, 0.0, 2.0 ** -8, 2.0 ** -9, 0.0]


def test_restatement_runs_the_long_and_empty_shapes():
    """One-token passages next to a 5,000-token one, a chunk boundary inside a passage, zero query rows."""
    g = torch.Generator().manual_seed(3)
    dl = np.array([1, 5000, 1, 3], np.int32)
    D = S.bf16_rows((int(dl.sum()), 128), generator=g)
    Q = S.bf16_rows((2, 33, 128), generator=g)
    Q[1] = 0.0
    s, a, r = S.maxsim_packed(Q, D, dl)
    ref = O.maxsim_scores(Q.numpy(), D.numpy(), dl)
    _within(ref, s, S.simt_bound(a, r, 33), "long")
    assert (s[1] == 0).all() and (a[1] == 0).all()
    old = S._CHUNK
    try:
        S._CHUNK = 66 * 700          # 700 tokens per chunk: the 5,000-token passage is split
        s2 = S.maxsim_packed(Q, D, dl)[0]
    finally:
        S._CHUNK = old
    assert torch.equal(s, s2)


def test_grid_is_a_pairwise_covering():
    cases = S.pairwise_cases(S.SCAN_FACTORS, S.scan_allowed)
    F = S.SCAN_FACTORS
    for f1, f2 in itertools.combinations(F, 2):
        seen = {(c[f1], c[f2]) for c in cases}
        for v1, v2 in itertools.product(F[f1], F[f2]):
            if S.scan_allowed({f1: v1, f2: v2}):
                assert (v1, v2) in seen, (f1, v1, f2, v2)
    assert all(S.scan_allowed(c) for c in S.scan_grid())
    assert len(S.scan_grid()) < 140


def test_readback_corpus_uses_every_reducer_slot():
    """The read-back corpus puts values in all 24 slots of a tile: 0-3 summed by the reducer from parked row maxima,
    4-23 from the consumer warps' 16-row sums."""
    D, dl = S.readback_corpus()
    part = scan_partition(dl, N_CTAS)
    assert part["n_ctas"] == N_CTAS and D.size(0) == 8192
    assert set(part["slot"].tolist()) == set(range(S.SLOTS))
    assert (part["end_mask"] == FULL).sum() >= N_CTAS
    # every finite bf16 bit pattern sits in each copy once (+0 and -0 compare equal: 65,279 distinct values)
    assert S.readback_values().flatten()[:65280].unique().numel() == 65279
    assert torch.equal(D[512:1024], torch.roll(D[:512], shifts=1, dims=1))


def _edges():
    """Which structural edges the grid's cases reach on 132 CTAs."""
    seen = set()
    for ci, c in enumerate(S.scan_grid()):
        dl = S.case_doclens(c, S.case_seed(ci))
        part = scan_partition(dl, N_CTAS)
        em = part["end_mask"]
        assert part["n_ctas"] == min(N_CTAS, c["n"])
        if (em == FULL).any():
            seen.add("tile with 24 ends")
        if ((em >> 23) & 1).any():
            seen.add("end in group 23")
        if ((part["last_tile"] - part["first_tile"]) >= 2).any():
            seen.add("passage open across 3+ tiles")
        if (part["cta_tiles"] == 1).any():
            seen.add("single-tile CTA")
        cta_of_passage = np.searchsorted(part["row_begin"][1:], np.concatenate([[0], np.cumsum(part["rows"])])[:-1],
                                         side="right")
        if (np.bincount(cta_of_passage, minlength=part["n_ctas"]) == 1).any():
            seen.add("single-passage CTA")
        if (part["rows"] > part["n_rows"] / part["n_ctas"]).any() and part["n_ctas"] > 1:
            seen.add("passage longer than its CTA's share")
        if part["cta_rows"][-1] % S.TILE:
            seen.add("last tile past n_rows")
        seen.add("n %s SMs" % ("<" if c["n"] < N_CTAS else "=" if c["n"] == N_CTAS else ">"))
        for plan in S.call_plans(c["B"], c["nq"]):
            if len(plan) > S.STAGE_MAX_PASSES:
                seen.add("chunk of > 64 passes")
            final = plan[(plan[:, 6] & PASS_FINAL) != 0]
            if (final[:, 4] <= 4).any():
                seen.add("lane mode")
            if (final[:, 4] > 4).any():
                seen.add("warp mode")
            if ((plan[:, 2] > 0) & (plan[:, 1] > 1)).any():
                seen.add("grouped tail pass")
            blocks = S.occupied_blocks(plan[:, 1], plan[:, 4])
            if (blocks >= S.THREE_WG_BLOCKS).any():
                seen.add(">= 5 blocks")
            if (blocks < S.THREE_WG_BLOCKS).any():
                seen.add("< 5 blocks")
            if (plan[:, 1] == 12).any():
                seen.add("12 queries in a pass")
        if c["B"] > S.WS_QUERIES:
            seen.add("two call chunks")
        if c["B"] == 13:
            seen.add("13 queries in a call")
    return seen


def test_grid_reaches_every_structural_edge():
    seen = _edges()
    want = {"tile with 24 ends", "end in group 23", "passage open across 3+ tiles", "single-tile CTA",
            "single-passage CTA", "passage longer than its CTA's share", "last tile past n_rows", "n < SMs",
            "n = SMs", "n > SMs", "chunk of > 64 passes", "lane mode", "warp mode", "grouped tail pass",
            ">= 5 blocks", "< 5 blocks", "12 queries in a pass", "two call chunks", "13 queries in a call"}
    assert want <= seen, sorted(want - seen)


def test_single_passage_ctas_at_the_sm_count():
    """131 / 132 passages: one passage per CTA; 133: every CTA still has at least one, one CTA has two."""
    for n in (131, 132, 133):
        part = scan_partition(np.full(n, 50, np.int32), N_CTAS)
        per_cta = np.bincount(np.searchsorted(part["row_begin"][1:], np.arange(n) * 52, side="right"),
                              minlength=part["n_ctas"])
        assert part["n_ctas"] == min(n, N_CTAS) and (per_cta >= 1).all()
        assert per_cta.max() == (1 if n <= N_CTAS else 2)
