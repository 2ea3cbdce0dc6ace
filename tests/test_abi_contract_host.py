"""The C boundary's host outputs with a capacity, and the guard-band helper of the contract tests (no GPU needed).

* ``flmr_debug_plan_passes`` and ``flmr_debug_compact_plan``: at exactly the needed capacity they write exactly that
  many entries; one short is rejected and writes nothing past the capacity.
* ``abi_contract.Guarded`` (tests/abi_contract.py): every sentinel is the documented pattern (a NaN for the float
  types), the guard bands are large enough, and ``check`` catches a write into either guard, an element of the output
  range left unwritten and a write outside a partial range.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import abi_contract as A


@pytest.fixture(scope="module")
def L():
    from ravqa_b200 import _cabi
    return _cabi.lib()


SENT32 = np.int32(0x5A5A5A5A)
SENT64 = np.int64(0x5A5A5A5A5A5A5A5A)


@pytest.mark.parametrize("n_queries,nq,pair", [(1, 32, 0), (12, 32, 0), (70, 97, 1), (3, 832, 0), (200, 320, 1)])
def test_plan_passes_capacity(L, n_queries, nq, pair):
    n = C.c_int(-1)
    assert L.flmr_debug_plan_passes(n_queries, nq, pair, None, 0, C.byref(n)) == 0
    need = n.value
    assert need >= 1
    for cap, ok in ((need, True), (need - 1, False)):
        buf = np.full(8 * need + 64, SENT32, np.int32)
        m = C.c_int(-1)
        rc = L.flmr_debug_plan_passes(n_queries, nq, pair, buf.ctypes.data_as(C.c_void_p), cap, C.byref(m))
        assert m.value == need
        if ok:
            assert rc == 0
            assert (buf[8 * need:] == SENT32).all(), "written past the plan"
            assert not (buf[:8 * need].reshape(need, 8) == SENT32).all(axis=1).any()
        else:
            assert rc == 1 and "capacity" in L.flmr_last_error().decode()
            assert (buf[8 * cap:] == SENT32).all(), "written past the capacity of a rejected call"


@pytest.mark.parametrize("n,dead_every,chunk_rows", [(50, 3, 0), (400, 7, 64), (1000, 2, 100), (30, 1000, 0)])
def test_compact_plan_capacity(L, n, dead_every, chunk_rows):
    dl = (np.arange(n) % 37 + 1).astype(np.int32)
    dead = np.arange(0, n, dead_every, dtype=np.int64)
    args = (dl.ctypes.data_as(C.c_void_p), n, dead.ctypes.data_as(C.c_void_p), dead.size, chunk_rows)
    m = C.c_int64(-1)
    assert L.flmr_debug_compact_plan(*args, None, 0, C.byref(m)) == 0
    need = m.value
    assert need >= 1
    for cap, ok in ((need, True), (need - 1, False)):
        buf = np.full(5 * need + 64, SENT64, np.int64)
        m = C.c_int64(-1)
        rc = L.flmr_debug_compact_plan(*args, buf.ctypes.data_as(C.c_void_p), cap, C.byref(m))
        assert m.value == need
        if ok:
            assert rc == 0
            assert (buf[5 * need:] == SENT64).all(), "written past the plan"
            moves = buf[:5 * need].reshape(need, 5)
            assert (moves[:, 2] > 0).all() and np.isin(moves[:, 3], (0, 1)).all()
        else:
            assert rc == 1 and "capacity" in L.flmr_last_error().decode()
            assert (buf[5 * cap:] == SENT64).all(), "written past the capacity of a rejected call"


# ---- the guard-band helper -------------------------------------------------------------------------------------------
def test_sentinels_are_the_documented_patterns():
    assert A.SENTINEL_BITS[torch.float32] == 0x7FBADBAD
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        x = torch.empty(4, dtype=dt)
        A.bits(x).fill_(A.SENTINEL_BITS[dt])
        assert torch.isnan(x).all(), dt
        assert A.bits(x)[0].item() == A.SENTINEL_BITS[dt]
    for dt, v in ((torch.int64, 0x5A5A5A5A5A5A5A5A), (torch.int32, 0x5A5A5A5A), (torch.uint8, 0xA5)):
        x = torch.empty(3, dtype=dt)
        A.bits(x).fill_(A.SENTINEL_BITS[dt])
        assert (x == v).all(), dt


@pytest.mark.parametrize("shape,dtype", [((3, 5), torch.float32), ((100000,), torch.int64), ((7,), torch.uint8),
                                         ((2, 40000), torch.bfloat16)])
def test_guard_bands_are_large_enough(shape, dtype):
    g = A.Guarded(shape, dtype, device="cpu")
    item = g.buf.element_size()
    assert g.g >= g.n and g.g * item >= A.GUARD_MIN_BYTES
    assert g.out.shape == shape and g.out.data_ptr() == g.buf.data_ptr() + g.g * item
    assert (A.bits(g.buf) == A.SENTINEL_BITS[dtype]).all()


def test_guard_check_catches_every_kind_of_stray_write():
    def fresh():
        g = A.Guarded((4, 6), torch.float32, device="cpu")
        g.out.fill_(1.0)
        return g
    fresh().check()
    g = fresh()
    g.buf[g.g - 1] = 0.0                                  # one element before the output
    with pytest.raises(AssertionError, match="before the output"):
        g.check()
    g = fresh()
    g.buf[g.g + g.n] = 0.0                                # one element past the output
    with pytest.raises(AssertionError, match="after the output"):
        g.check()
    g = fresh()
    A.bits(g.out)[3, 5] = A.SENTINEL_BITS[torch.float32]  # one element left unwritten
    with pytest.raises(AssertionError, match="not written"):
        g.check()
    g = fresh()                                           # a partial range: the first row must stay untouched
    w = torch.ones((4, 6), dtype=torch.bool)
    w[0] = False
    with pytest.raises(AssertionError, match="outside the output range"):
        g.check(w)
    A.bits(g.out)[0] = A.SENTINEL_BITS[torch.float32]
    g.check(w)


def test_same_bits_tells_nan_payloads_and_signed_zeros_apart():
    a = torch.tensor([0.0, float("nan")])
    b = a.clone()
    assert A.same_bits(a, b)
    b[0] = -0.0
    assert not A.same_bits(a, b)
    c = a.clone()
    A.bits(c)[1] = A.SENTINEL_BITS[torch.float32]
    assert not A.same_bits(a, c)
