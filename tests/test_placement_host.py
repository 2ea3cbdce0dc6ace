"""The placement fixture of tests/test_placement_and_ties_gpu.py is not vacuous (no GPU needed).

The scan's reducer receives a passage's score in one of two forms: the first 4 passages to end in a 96-token tile
park per-row maxima, later ones arrive as the consumer warps' 16-row sums.  Both must add up in the same order, so
that a score does not depend on where the passage is stored.  The GPU tests move passages between the two forms by
prepending a passage, sharding and appending; here the partition builder the scan uses shows that each of those
moves at least a quarter of the tracked passages across the slot-4 line (for 132 CTAs, an H100's SM count).
"""
import numpy as np
import pytest

from helpers import placement_doclens, placement_tracked, scan_slots

N_CTAS = 132


@pytest.fixture(scope="module")
def base():
    dl = placement_doclens()
    return dl, scan_slots(dl, N_CTAS) >= 4


def _moved(base_cls, cls, n):
    return (base_cls != cls)[placement_tracked(n)].mean()


def test_fixture_holds_both_slot_classes(base):
    dl, cls = base
    tr = placement_tracked(len(dl))
    assert 0.25 < cls[tr].mean() < 0.75, cls[tr].mean()
    assert (dl < 24).mean() > 0.9


def test_prepended_shim_moves_passages(base):
    dl, cls = base
    moved_any = np.zeros(len(dl), bool)
    for groups in range(1, 6):
        shifted = scan_slots(np.concatenate([[4 * groups], dl]), N_CTAS)[1:] >= 4
        assert (shifted != cls).any(), groups
        moved_any |= shifted != cls
    assert moved_any[placement_tracked(len(dl))].mean() >= 0.25


@pytest.mark.parametrize("world", [2, 4])
def test_shards_move_passages(base, world):
    from ravqa_b200.sharded import shard_ranges
    dl, cls = base
    sharded = np.empty(len(dl), bool)
    for p0, p1 in shard_ranges(dl, world):
        sharded[p0:p1] = scan_slots(dl[p0:p1], N_CTAS) >= 4
    assert _moved(cls, sharded, len(dl)) >= 0.25


def test_append_moves_passages(base):
    dl, cls = base
    extra = placement_doclens(500, seed=1)
    grown = scan_slots(np.concatenate([dl, extra]), N_CTAS)[:len(dl)] >= 4
    assert _moved(cls, grown, len(dl)) >= 0.25
