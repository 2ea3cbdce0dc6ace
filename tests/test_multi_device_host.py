"""CPU: the multi-device Searcher (``Searcher(devices=...)``) and its merge, ``flmr_topk_merge_devices`` — the C
declaration, export and binding, the merge's argument refusals before any CUDA call, the Searcher's refusals, and the
shard split of ``devices=[...]`` against ``shard_ranges``."""
from __future__ import annotations

import ctypes as C
import os
import re
import types

import numpy as np
import pytest
import torch

from helpers import ROOT
from ravqa_b200 import _cabi, sharded
from ravqa_b200.corpus import FlatCorpus
from ravqa_b200.index_io import save_flat_index
from ravqa_b200.searcher import Searcher
from ravqa_b200.updater import IndexUpdater

INVALID, UNSUPPORTED = 1, 3


def test_header_declares_and_cabi_binds_the_merge():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "flmr_maxsim.h")).read(), flags=re.S)
    L = _cabi.lib()
    for name, n_params in (("flmr_topk_merge_devices", 11), ("flmr_debug_set_merge_path", 1)):
        m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, src)
        assert m, name
        assert m.group(1).count(",") + 1 == n_params, name
        assert name in _cabi.SYMBOLS and name in _cabi.MULTI_DEVICE_SYMBOLS
        assert hasattr(L, name) and len(getattr(L, name).argtypes) == n_params, name
    assert L.flmr_abi_version() == 2


def test_merge_refuses_bad_arguments_before_any_cuda_call():
    """Each refusal returns its code with a message; a call that reached CUDA on this machine would fail with
    FLMR_ERR_CUDA instead.  n_queries == 0 touches no device."""
    L = _cabi.lib()
    buf = np.zeros(64, dtype=np.int64)
    p = buf.ctypes.data                                        # a host address, never dereferenced

    def call(n_lists=2, n_queries=3, k_in=4, k_out=4, scores=True, pids=True, devices=True, streams=True,
             out=True, null_list=None):
        n = max(n_lists, 1)
        sp = (C.c_void_p * n)(*[None if i == null_list else p for i in range(n)])
        pp = (C.c_void_p * n)(*[p] * n)
        dev = (C.c_int * n)(*[0] * n)
        sts = (C.c_void_p * n)(*[None] * n)
        return L.flmr_topk_merge_devices(sp if scores else None, pp if pids else None, dev if devices else None,
                                         sts if streams else None, n_lists, n_queries, k_in, k_out,
                                         p if out else None, p if out else None, None)

    for kw in (dict(scores=False), dict(pids=False), dict(devices=False), dict(streams=False), dict(out=False),
               dict(n_lists=0), dict(n_lists=-1), dict(n_queries=-1), dict(k_in=0), dict(k_out=0),
               dict(k_out=_cabi.MAX_K + 1, k_in=200), dict(n_lists=2, k_in=4, k_out=9), dict(n_lists=1, k_in=1, k_out=2),
               dict(null_list=1)):
        assert call(**kw) == INVALID, kw
        assert L.flmr_last_error(), kw
    assert b"k_out=9" in (call(k_out=9), L.flmr_last_error())[1]
    assert b"null" in (call(null_list=0), L.flmr_last_error())[1]
    # the kernel's capacity: 20480 candidates per query, 128 lists
    assert call(n_lists=2, k_in=10241, k_out=8) == UNSUPPORTED
    assert call(n_lists=129, k_in=1, k_out=8) == UNSUPPORTED
    # nothing to merge: no device is touched
    assert call(n_queries=0) == 0
    assert call(n_lists=1, k_in=8, k_out=8, n_queries=0) == 0


def test_debug_merge_path_switch():
    L = _cabi.lib()
    assert L.flmr_debug_set_merge_path(2) == INVALID and L.flmr_debug_set_merge_path(-1) == INVALID
    assert L.flmr_debug_set_merge_path(1) == 0 and L.flmr_debug_set_merge_path(0) == 0


@pytest.mark.parametrize("kw", [dict(shard_across_ranks=True), dict(device=0), dict(device="cuda:1"),
                                dict(residency="host"), dict(residency="host", window_bytes=1 << 20),
                                dict(compressed=True)])
def test_searcher_refuses_devices_with_conflicting_options(kw):
    with pytest.raises(ValueError, match="devices="):
        Searcher(index="/nonexistent/index", devices=[0, 0], **kw)


def test_searcher_refuses_devices_with_a_corpus_object():
    corpus = FlatCorpus.__new__(FlatCorpus)             # no device work: the refusal comes first
    with pytest.raises(ValueError, match="index path"):
        Searcher(index=corpus, devices=[0, 1])


def test_resolve_devices_refusals():
    for bad in ("some", [], ["cpu"]):
        with pytest.raises(ValueError):
            sharded.resolve_devices(bad)
    assert sharded.resolve_devices([1, 0, 1]) == [1, 0, 1]
    assert sharded.resolve_devices([torch.device("cuda", 2), "cuda:0"]) == [2, 0]


@pytest.fixture
def ragged_index(tmp_path):
    rng = np.random.default_rng(7)
    dl = rng.integers(1, 40, size=97).astype(np.int32)
    dl[40:44] = 300                                      # a run of long passages around a shard boundary
    path = str(tmp_path / "flat")
    save_flat_index(path, torch.zeros((int(dl.sum()), _cabi.DIM), dtype=torch.bfloat16), dl)
    return path, dl


@pytest.mark.parametrize("devices", [[0, 0], [0, 1, 0], [3, 2, 1, 0], [0] * 7])
def test_shard_split_of_devices_equals_shard_ranges(ragged_index, monkeypatch, devices):
    """Shard i is loaded on devices[i] as rank i of len(devices) (FlatCorpus.from_index splits by shard_ranges), the
    shards are loaded together, and the Searcher sees the whole index."""
    path, dl = ragged_index
    calls = []

    def fake_load(p, device=None, rank=0, world_size=1, **kw):
        calls.append((rank, world_size, device))
        p0, p1 = sharded.shard_ranges(dl, world_size)[rank]
        return types.SimpleNamespace(pid_base=p0, n_passages=p1 - p0, device=torch.device("cuda", device),
                                     storage="bf16", residency="device", doclens=dl[p0:p1])

    built = {}

    class FakeDeviceSharded:
        def __init__(self, devs, local_topk):
            built["devices"], built["local_topk"] = devs, local_topk
    monkeypatch.setattr(FlatCorpus, "from_index", staticmethod(fake_load))
    monkeypatch.setattr(sharded, "DeviceShardedSearcher", FakeDeviceSharded)
    s = Searcher(index=path, devices=devices)
    n = len(devices)
    assert sorted(calls) == [(i, n, devices[i]) for i in range(n)]
    assert [(c.pid_base, c.pid_base + c.n_passages) for c in s.shards] == sharded.shard_ranges(dl, n)
    assert built["devices"] == devices and s.corpus is s.shards[0] and s.device == torch.device("cuda", devices[0])
    assert s._index_size() == len(dl)
    with pytest.raises(NotImplementedError, match="devices"):
        IndexUpdater(searcher=s)
