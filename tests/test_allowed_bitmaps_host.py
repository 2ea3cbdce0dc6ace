"""Per-query allow bitmaps, CPU side: the pure-torch builder against numpy.packbits, and the new exports."""
import numpy as np
import pytest
import torch

from ravqa_b200 import _cabi, allow_bitmaps


def _packed(rows, n):
    """numpy restatement: one bool row per query -> little-endian bits -> int32 words."""
    words = (n + 31) // 32
    dense = np.zeros((len(rows), words * 32), dtype=bool)
    for b, r in enumerate(rows):
        dense[b, r] = True
    return np.packbits(dense, axis=1, bitorder="little").view("<u4").view(np.int32).reshape(len(rows), words)


@pytest.mark.parametrize("n,pid_base", [(1, 0), (32, 0), (33, 7), (1000, 0), (1000, 5000), (4099, 123)])
def test_builder_matches_packbits(n, pid_base):
    rng = np.random.default_rng(n + pid_base)
    lists, want = [], []
    for b in range(9):
        size = int(rng.integers(0, 3 * n // 2 + 2))
        # global ids spanning the shard and both sides of it, with repeats
        ids = rng.integers(pid_base - n // 2 - 3, pid_base + n + n // 2 + 3, size=size)
        if b % 3 == 0 and size:
            ids = np.concatenate([ids, ids[: size // 2]])
        lists.append(ids.tolist() if b % 2 else torch.from_numpy(ids))
        local = ids - pid_base
        want.append(np.unique(local[(local >= 0) & (local < n)]))
    lists.append([])
    want.append(np.array([], dtype=np.int64))
    got = allow_bitmaps(lists, n, pid_base)
    assert got.dtype == torch.int32 and got.shape == (len(lists), (n + 31) // 32)
    np.testing.assert_array_equal(got.numpy(), _packed(want, n))


def test_none_is_every_passage_and_out_of_shard_ids_drop():
    got = allow_bitmaps([None, [10**12, -1], [3, 3, 3]], 40, pid_base=2)
    assert (got[0] == -1).all()                        # bits past n_passages are ignored by the scan
    assert (got[1] == 0).all()
    np.testing.assert_array_equal(got[2].numpy(), _packed([[1]], 40)[0])


def test_allowed_entry_points_are_exported_and_bound():
    L = _cabi.lib()
    for name in _cabi.ALLOWED_SYMBOLS:
        assert name in _cabi.SYMBOLS
        assert hasattr(L, name) and getattr(L, name).argtypes, name
