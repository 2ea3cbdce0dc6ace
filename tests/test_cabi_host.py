"""CPU: the C-ABI library builds, loads and exports every symbol include/flmr_maxsim.h declares;
argument validation that happens before any CUDA call; host-side partition logic."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import ROOT
from ravqa_b200 import _cabi


def header_functions():
    text = open(os.path.join(ROOT, "include", "flmr_maxsim.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(flmr_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    L = _cabi.lib()
    names = header_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(L, n), "missing export " + n
    assert set(names) == set(_cabi.SYMBOLS)
    assert L.flmr_abi_version() == 2


def header_prototypes():
    """{name: number of parameters} for every function the header declares."""
    text = open(os.path.join(ROOT, "include", "flmr_maxsim.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for name, params in re.findall(r"\b(flmr_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        params = params.strip()
        out[name] = 0 if params in ("", "void") else params.count(",") + 1
    return out


def test_ctypes_prototypes_match_the_header():
    """Every binding in _cabi.py (and the stub shown in INTEGRATION.md) passes exactly the arguments the
    header declares — a mismatch would corrupt the call silently (ctypes cannot check C prototypes)."""
    L = _cabi.lib()
    protos = header_prototypes()
    assert set(protos) == set(_cabi.SYMBOLS)
    for name, n_params in protos.items():
        argtypes = getattr(L, name).argtypes
        assert argtypes is not None, name + " has no argtypes"
        assert len(argtypes) == n_params, "%s: header has %d parameters, ctypes %d" % (name, n_params, len(argtypes))
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    for name, n_list in re.findall(r"L\.(flmr_[a-z0-9_]+)\.argtypes\s*=\s*\[([^\]]*)\]", doc):
        assert n_list.count(",") + 1 == protos[name], "INTEGRATION.md stub of %s is out of date" % name


def test_library_is_sm90a_wgmma_build():
    import subprocess
    from ravqa_b200 import build
    sass = subprocess.run(["cuobjdump", "-sass", build.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA.64x96x16.F32.BF16", "HGMMA.64x128x16.F32.BF16", "UTMALDG.2D.MULTICAST", "SYNCS"):
        assert mnemonic in sass, mnemonic + " missing: the hot kernels are not wgmma/TMA/mbarrier code"


def test_argument_validation_without_gpu():
    L = _cabi.lib()
    h = C.c_void_p()
    dl = np.array([4, 4], dtype=np.int32)
    tok = np.zeros((8, 128), dtype=np.uint16)
    # wrong dim
    rc = L.flmr_corpus_create(tok.ctypes.data, dl.ctypes.data, 2, 64, 0, 0, 0, C.byref(h))
    assert rc == 3 and b"dim" in L.flmr_last_error()
    # zero-length passage is rejected (SURVEY 8a)
    dl0 = np.array([4, 0], dtype=np.int32)
    rc = L.flmr_corpus_create(tok.ctypes.data, dl0.ctypes.data, 2, 128, 0, 0, 0, C.byref(h))
    assert rc == 1 and b"zero-length" in L.flmr_last_error()
    # null pointers
    assert L.flmr_corpus_create(None, dl.ctypes.data, 2, 128, 0, 0, 0, C.byref(h)) == 1
    # a streamed corpus and its builder: each refused before any device call, with its code and, where two checks
    # could trip, in its order (the corpus checks its flags before dim and the window, the builder its window first)
    row, fp8 = _cabi.DIM * 2, _cabi.CORPUS_FP8
    for args, rc, msg in (((tok.ctypes.data, dl.ctypes.data, 2, 64, 0, 0, 0, 1 << 20), 3, b"dim"),
                          ((None, dl.ctypes.data, 2, 128, 0, 0, 0, 1 << 20), 1, None),
                          ((tok.ctypes.data, None, 2, 128, 0, 0, 0, 1 << 20), 1, None),
                          ((tok.ctypes.data, dl0.ctypes.data, 2, 128, 0, 0, 0, 1 << 20), 1, b"zero-length"),
                          ((tok.ctypes.data, dl.ctypes.data, 2, 128, 0, 0, 0, row - 1), 1, b"holds no row"),
                          ((tok.ctypes.data, dl.ctypes.data, 2, 128, 0, 0, 0, 0), 1, b"holds no row"),
                          ((tok.ctypes.data, dl.ctypes.data, 2, 128, 0, 0, fp8, 1 << 20), 3, b"flags"),
                          ((tok.ctypes.data, dl.ctypes.data, 2, 128, 0, 0, _cabi.CORPUS_ADOPT, 1 << 20), 3, b"flags"),
                          ((tok.ctypes.data, dl.ctypes.data, 2, 128, 0, 0, 0, 3 * row), 3, b"window"),
                          ((tok.ctypes.data, dl.ctypes.data, 2, 64, 0, 0, fp8, 0), 3, b"flags")):
        assert L.flmr_corpus_create_streamed(*args, C.byref(h)) == rc and not h.value, args
        assert msg is None or msg in L.flmr_last_error(), (args, L.flmr_last_error())
    b = C.c_void_p()
    for args, rc, msg in (((dl.ctypes.data, 2, 64, 0, 0, 0, 1 << 20), 3, b"dim"),
                          ((None, 2, 128, 0, 0, 0, 1 << 20), 1, None),
                          ((dl0.ctypes.data, 2, 128, 0, 0, 0, 1 << 20), 1, b"zero-length"),
                          ((dl.ctypes.data, 2, 128, 0, 0, 0, row - 1), 1, b"holds no row"),
                          ((dl.ctypes.data, 2, 128, 0, 0, 0, 0), 1, b"holds no row"),
                          ((dl.ctypes.data, 2, 128, 0, 0, fp8, 1 << 20), 3, b"flags"),
                          ((dl.ctypes.data, 2, 128, 0, 0, 0, 3 * row), 3, b"window"),
                          ((dl.ctypes.data, 2, 64, 0, 0, fp8, 0), 1, b"holds no row")):
        assert L.flmr_corpus_builder_create_streamed(*args, C.byref(b)) == rc and not b.value, args
        assert msg is None or msg in L.flmr_last_error(), (args, L.flmr_last_error())
    assert L.flmr_topk_merge(None, None, 1, 1, 1, 1, None, None, 0, None) == 1
    assert L.flmr_maxsim_topk(None, None, None, 1, 32, 5, 0, None, None, None) == 1
    assert L.flmr_corpus_destroy(None) == 0 and L.flmr_workspace_destroy(None) == 0
    with pytest.raises(_cabi.FlmrError):
        _cabi.check(1)


def _partition(doclens, n_ctas):
    L = _cabi.lib()
    dl = np.ascontiguousarray(doclens, dtype=np.int32)
    nc = min(n_ctas, len(dl))
    rb = np.zeros(nc + 1, np.int32)
    tb = np.zeros(nc + 1, np.int64)
    nt = C.c_int64()
    _cabi.check(L.flmr_debug_build_partition(dl.ctypes.data, len(dl), n_ctas, rb.ctypes.data, tb.ctypes.data,
                                             None, None, 0, C.byref(nt)))
    em = np.zeros(nt.value, np.uint32)
    fp = np.zeros(nt.value, np.int32)
    _cabi.check(L.flmr_debug_build_partition(dl.ctypes.data, len(dl), n_ctas, rb.ctypes.data, tb.ctypes.data,
                                             em.ctypes.data, fp.ctypes.data, nt.value, C.byref(nt)))
    return rb, tb, em, fp


@pytest.mark.parametrize("seed,n,lo,hi,ctas", [(0, 1000, 1, 64, 148), (1, 37, 100, 700, 148),
                                                (2, 5000, 1, 4, 16), (3, 3, 180, 180, 148),
                                                (4, 1, 5, 5, 148), (5, 20000, 180, 180, 148)])
def test_partition_invariants(seed, n, lo, hi, ctas):
    rng = np.random.default_rng(seed)
    dl = rng.integers(lo, hi + 1, size=n)
    rb, tb, em, fp = _partition(dl, ctas)
    plen = (dl + 3) // 4 * 4
    poff = np.concatenate([[0], np.cumsum(plen)])
    nc = len(rb) - 1
    assert rb[0] == 0 and rb[-1] == poff[-1] and np.all(np.diff(rb) >= 0)
    assert set(rb.tolist()) <= set(poff.tolist()), "CTA ranges must start on passage boundaries"
    # every passage end appears exactly once, at the right tile/bit, in order
    ends = []
    for c in range(nc):
        for t in range(tb[c], tb[c + 1]):
            bits = int(em[t])
            slot = 0
            for g in range(_cabi.TILE_TOKENS // 4):
                if bits >> g & 1:
                    row_end = rb[c] + (t - tb[c]) * _cabi.TILE_TOKENS + 4 * g + 4   # exclusive end row
                    ends.append((int(fp[t]) + slot, row_end))
                    slot += 1
            assert bits >> (_cabi.TILE_TOKENS // 4) == 0
    assert [e[0] for e in ends] == list(range(n))
    assert [e[1] for e in ends] == poff[1:].tolist()
    # token balance: no CTA holds more than the ideal share + one passage
    share = poff[-1] / nc
    assert np.all(np.diff(rb) <= share + plen.max() + 1)


# residency of one scan pass (flmr_scan_kernel.cuh): MT_MAX 128-row query tiles = RB_MAX 32-row blocks
MT_MAX = 3
RB_MAX = 4 * MT_MAX
ROWS_MAX = 32 * RB_MAX


def _plan(n_queries, nq, allow_pair=0):
    L = _cabi.lib()
    n = C.c_int(0)
    _cabi.check(L.flmr_debug_plan_passes(n_queries, nq, allow_pair, None, 0, C.byref(n)))
    buf = np.zeros((max(n.value, 1), 8), dtype=np.int32)
    _cabi.check(L.flmr_debug_plan_passes(n_queries, nq, allow_pair, buf.ctypes.data_as(C.c_void_p), n.value,
                                         C.byref(n)))
    return buf[: n.value]


@pytest.mark.parametrize("n_queries,nq", [(1, 32), (16, 32), (64, 32), (21, 32), (16, 320), (5, 320), (3, 45),
                                           (7, 832), (1, 832), (3, 1500), (2, 1280), (40, 641), (0, 64), (13, 640), (13, 384), (5, 385)])
def test_pass_plan_invariants(n_queries, nq):
    """flmr_debug_plan_passes: every (query, row) is resident in exactly one pass, never more than ROWS_MAX rows
    or RB_MAX queries per pass, partial scores are read only after they were written, each query is finalised
    exactly once and last, and the number of passes is the minimum this scheme allows."""
    plan = _plan(n_queries, nq)
    ACC_IN, ACC_OUT, FINAL = 1, 2, 4
    covered = np.zeros((n_queries, nq), dtype=np.int32)
    touched = np.zeros(n_queries, dtype=bool)
    finalised = np.zeros(n_queries, dtype=bool)
    for q_first, n_q, row0, rows, rbq, n_mtiles, flags, acc_first in plan:
        assert 1 <= n_q <= RB_MAX and rbq == (rows + 31) // 32 and n_q * rbq <= RB_MAX
        assert n_mtiles == (n_q * rbq * 32 + 127) // 128 and 1 <= n_mtiles <= MT_MAX
        assert 0 <= row0 and row0 + rows <= nq and row0 % 32 == 0
        qs = slice(q_first, q_first + n_q)
        assert not finalised[qs].any()                        # nothing after the final pass of a query
        assert bool(flags & ACC_IN) == bool(touched[qs].all()) and touched[qs].all() == touched[qs].any()
        if not flags & FINAL:
            assert flags & ACC_OUT                            # a non-final slice must store its partial scores
        covered[qs, row0:row0 + rows] += 1
        touched[qs] = True
        if flags & FINAL:
            finalised[qs] = True
        assert acc_first == q_first                           # partial-score rows are indexed by query
    assert (covered == 1).all() and finalised.all()
    rbq_total = (nq + 31) // 32
    if rbq_total <= RB_MAX:
        per_pass = min(RB_MAX, RB_MAX // rbq_total)
        assert len(plan) == -(-n_queries // per_pass)
        sizes = [p[1] for p in plan]
        assert not sizes or max(sizes) - min(sizes) <= per_pass - 1 and max(sizes) == -(-n_queries // len(plan))
    else:
        n_slices = -(-nq // ROWS_MAX)
        tail_rbq = (nq - (n_slices - 1) * ROWS_MAX + 31) // 32
        group = max(1, min(RB_MAX, RB_MAX // tail_rbq, n_queries))
        assert len(plan) == n_queries * (n_slices - 1) + -(-n_queries // group)


def test_pass_plan_random_shapes():
    """Same invariants as above on a sweep of random (batch, query length) pairs."""
    rng = np.random.default_rng(11)
    for _ in range(60):
        n_queries = int(rng.integers(0, 90))
        nq = int(rng.integers(1, 2100))
        plan = _plan(n_queries, nq)
        covered = np.zeros((n_queries, nq), dtype=np.int32)
        final = np.zeros(n_queries, dtype=np.int32)
        for q_first, n_q, row0, rows, rbq, n_mtiles, flags, _acc in plan:
            assert n_q * rbq <= RB_MAX and n_q <= RB_MAX and rows <= ROWS_MAX
            covered[q_first:q_first + n_q, row0:row0 + rows] += 1
            if flags & 4:
                final[q_first:q_first + n_q] += 1
        assert (covered == 1).all() and (final == 1).all(), (n_queries, nq)


@pytest.mark.parametrize("n_queries,nq", [(4, 320), (16, 320), (5, 320), (3, 320), (64, 32), (40, 32), (41, 32),
                                           (16, 832), (6, 832), (7, 832), (5, 832), (13, 1500), (2, 1280), (9, 641),
                                           (8, 128), (3, 45), (0, 64), (44, 200)])
def test_pass_plan_with_cta_pairs(n_queries, nq):
    """With CTA-pair passes allowed: pair passes (flag 8) cover a PREFIX of the queries, two blocks of n_q queries
    each (CTA r of every pair the r-th block), each CTA with all three 128-row tiles when whole queries are
    resident; the rest of the batch is planned exactly like a batch of that size without pairs; every (query, row)
    is still resident exactly once, partial scores are read only after they were written, and within one group of
    row-sliced queries no two queries share a partial-score row."""
    plan = _plan(n_queries, nq, 1)
    ACC_IN, ACC_OUT, FINAL, PAIR = 1, 2, 4, 8
    covered = np.zeros((n_queries, nq), dtype=np.int32)
    touched = np.zeros(n_queries, dtype=bool)
    finalised = np.zeros(n_queries, dtype=bool)
    acc_row = np.full(n_queries, -1)
    n_pair_q, seen_single = 0, False
    for q_first, n_q, row0, rows, rbq, n_mtiles, flags, acc_first in plan:
        pair = bool(flags & PAIR)
        span = 2 * n_q if pair else n_q
        assert 1 <= n_q <= RB_MAX and rbq == (rows + 31) // 32 and n_q * rbq <= RB_MAX
        assert n_mtiles == (n_q * rbq * 32 + 127) // 128 and 1 <= n_mtiles <= MT_MAX
        assert 0 <= row0 and row0 + rows <= nq and row0 % 32 == 0 and q_first + span <= n_queries
        if pair:
            assert not seen_single                            # pair passes first
            n_pair_q = max(n_pair_q, q_first + span)
            if nq <= ROWS_MAX:
                assert n_mtiles == MT_MAX                     # pairs only where a CTA is tensor-bound on its own
        else:
            seen_single = True
            assert q_first >= n_pair_q
        qs = slice(q_first, q_first + span)
        assert not finalised[qs].any()
        assert bool(flags & ACC_IN) == bool(touched[qs].all()) and touched[qs].all() == touched[qs].any()
        if not flags & FINAL:
            assert flags & ACC_OUT
        rows_here = acc_first + np.arange(span)               # partial-score row of query q_first + i
        assert (acc_row[qs] < 0).all() or (acc_row[qs] == rows_here).all()
        acc_row[qs] = rows_here
        covered[qs, row0:row0 + rows] += 1
        touched[qs] = True
        if flags & FINAL:
            finalised[qs] = True
    assert (covered == 1).all() and finalised.all()
    # the queries after the pair prefix: the plan of a (n_queries - n_pair_q)-query batch, shifted
    rest = _plan(n_queries - n_pair_q, nq, 0)
    tail = np.array([p for p in plan if not p[6] & PAIR]).reshape(-1, 8)
    if len(rest):
        shifted = rest.copy()
        shifted[:, 0] += n_pair_q
        shifted[:, 7] += n_pair_q
        assert np.array_equal(tail, shifted)
    else:
        assert len(tail) == 0
    # pairs halve the corpus passes of the prefix
    if n_pair_q:
        assert len(plan) - len(tail) == len(_plan(n_pair_q, nq, 0)) // 2 or nq > ROWS_MAX
        if nq > ROWS_MAX:
            n_slices = -(-nq // ROWS_MAX)
            g = max(1, min(RB_MAX, RB_MAX // ((nq - (n_slices - 1) * ROWS_MAX + 31) // 32)))
            assert n_pair_q % (2 * g) == 0
            assert len(plan) - len(tail) == (n_pair_q // (2 * g)) * (g * (n_slices - 1) + 1)


def test_comm_entry_points_validate_arguments():
    """The C-level sharded search (flmr_comm_* / flmr_topk_exchange / flmr_maxsim_topk_sharded): argument checks
    need neither a GPU nor NCCL."""
    import ctypes as C
    L = _cabi.lib()
    h = C.c_void_p()
    assert L.flmr_comm_create(None, 0, 1, 0, C.byref(h)) == 1 and b"null" in L.flmr_last_error()
    buf = (C.c_char * 128)()
    assert L.flmr_comm_create(buf, 2, 2, 0, C.byref(h)) == 1 and b"rank" in L.flmr_last_error()
    assert L.flmr_comm_adopt(None, 0, C.byref(h)) == 1
    assert L.flmr_comm_destroy(None) == 0
    assert L.flmr_comm_info(None, None, None) == 1
    assert L.flmr_topk_exchange(None, None, None, 1, 5, 5, None, None, None) == 1
    assert L.flmr_maxsim_topk_sharded(None, None, None, None, 1, 32, 5, 0, None, None, None) == 1
    assert L.flmr_comm_unique_id(None) == 1
