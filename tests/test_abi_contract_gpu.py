"""The C boundary's buffer, stream and threading conventions (include/flmr_maxsim.h), on every device entry point.

Each call goes through ``_cabi.lib()`` with an explicit stream handle and is held bitwise to the same call made plainly
(default stream, fresh buffers, inputs in place); the plain call itself is checked against the float64 references.

(a) caller-owned buffers: outputs inside sentinel-filled guard bands (tests/abi_contract.py), optional outputs passed
    as NULL, partial output ranges; inputs, ``flmr_corpus_info`` and a repeat search unchanged by the call;
(b) the caller's stream: late inputs (the real inputs land on a gated side stream just before the call), an early
    consumer (the legacy default stream gated, the outputs cloned on the side stream right after the call), and no
    hidden host synchronisation (the call returns while the gate still holds; flmr_plaid_decode, synchronous by
    contract, returns only once the gate has ended);
(c) CUDA graph capture and replay of select, merge, gather and the training routes;
(d) two threads, each with its own stream and workspace, enqueueing a mixed script on one shared corpus.

Scans run on a pairwise covering of storage (bf16, fp16, e4m3) x corpus state (fresh, with deletions, compacted then
appended) x pid_base (0, 1000) x shapes that reach each product scan kernel under variant 0.
"""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

import abi_contract as A
import load_fp64 as LF
import scan_fp64 as S64
import train_fp64 as T64
from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu

# The gate: a spin kernel of this many SM clock cycles (about 50 ms at the H100's 1980 MHz) on the stream a call is
# given.  It must outlast the host part of every call below; the measured host times are asserted against it.
GATE_CYCLES = 100_000_000
NEG = float("-inf")
DIM = 128
DTYPE = {"bf16": torch.bfloat16, "fp8": torch.bfloat16, "fp16": torch.float16}

# (storage, state, pid_base): every storage meets every state; pid_base alternates
SHARDS = [("bf16", "fresh", 0), ("bf16", "deleted", 1000), ("bf16", "compacted", 1000),
          ("fp16", "fresh", 1000), ("fp16", "deleted", 0), ("fp16", "compacted", 0),
          ("fp8", "fresh", 0), ("fp8", "deleted", 1000), ("fp8", "compacted", 1000)]
# (queries, Nq): six 32-row blocks of 12 queries (split kernel), two warpgroups, five blocks (split), row slices
SHAPES = [(12, 32), (5, 97), (3, 320), (2, 832)]
# shard i meets shapes i % 4 and (i + 2) % 4: every storage and every state meets every shape
# and k alternates 1 / 128 over each shard's two shapes
COMBOS = [(i, SHAPES[j], (1, 128)[(i + h) % 2]) for i in range(len(SHARDS)) for h, j in enumerate((i % 4, (i + 2) % 4))]
SCAN_KINDS = ["topk", "scores", "topk_allowed", "scores_allowed", "topk_listed", "scores_listed"]
LIST_OFFSET0 = 7          # listed calls start their offsets here: d_list_pids[0:7] and out[0:7] are never touched


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    return ravqa_b200


@pytest.fixture(scope="module")
def L(R):
    from ravqa_b200 import _cabi
    return _cabi.lib()


def _unit(n, g, dtype=torch.bfloat16):
    return torch.nn.functional.normalize(torch.randn(n, DIM, generator=g), dim=-1).to(dtype)


class Shard:
    """A corpus in one state, with the rows, lengths and live ids the float64 references need (over the id extent)."""

    def __init__(self, R, storage, state, pid_base, seed):
        rng = np.random.default_rng(seed)
        g = torch.Generator().manual_seed(seed)
        dt = DTYPE[storage]
        dl = rng.integers(1, 130, 1200).astype(np.int32)
        D = _unit(int(dl.sum()), g, dt)
        self.c = R.FlatCorpus(D, dl, device=0, pid_base=pid_base, storage=storage)
        live = np.ones(len(dl), bool)
        if state != "fresh":
            dead = np.sort(rng.choice(len(dl), len(dl) // 4, replace=False))
            self.c.delete(dead + pid_base)
            live[dead] = False
        if state == "compacted":
            self.c.compact()
            dl2 = rng.integers(1, 130, 300).astype(np.int32)
            D2 = _unit(int(dl2.sum()), g, dt)
            self.c.append(D2, dl2)
            D, dl, live = torch.cat([D, D2]), np.concatenate([dl, dl2]), np.concatenate([live, np.ones(300, bool)])
        self.storage, self.state, self.pid_base, self.dtype = storage, state, pid_base, dt
        self.D, self.dl, self.live = D, dl, live
        self.off = np.concatenate([[0], np.cumsum(dl.astype(np.int64))])
        self.n = len(dl)

    def scores64(self, q):
        """(float64 scores, bound) of queries q against every passage (deleted ones included)."""
        st = "fp8" if self.storage == "fp8" else "bf16"
        s64, amax, rabs = S64.maxsim_packed(q, self.D.cuda(), self.dl, storage=st)
        return s64, S64.scan_bound(amax, rabs, q.size(1), st)


@pytest.fixture(scope="module")
def shards(R):
    out = {}

    def get(i):
        if i not in out:
            out[i] = Shard(R, *SHARDS[i], seed=40 + i)
        return out[i]
    yield get
    for s in out.values():
        s.c.close()


@pytest.fixture(scope="module")
def comm(L):
    uid = (C.c_char * 128)()
    assert L.flmr_comm_unique_id(C.cast(uid, C.c_void_p)) == 0
    h = C.c_void_p()
    assert L.flmr_comm_create(C.cast(uid, C.c_void_p), 0, 1, 0, C.byref(h)) == 0
    yield h
    torch.cuda.synchronize()
    L.flmr_comm_destroy(h)


@pytest.fixture(scope="module")
def side():
    return torch.cuda.Stream()


def _h(stream):
    return C.c_void_p(stream or None)


# ---- scan calls ------------------------------------------------------------------------------------------------------
def _lists(sh, B, rng):
    """Host offsets from LIST_OFFSET0 (query 1's list empty) and a generator of device id lists of that length:
    live, deleted and compacted-away ids, ids on both sides of the shard, duplicates."""
    lens = rng.integers(1, 60, B)
    lens[min(1, B - 1)] = 0
    h_off = np.concatenate([[LIST_OFFSET0], LIST_OFFSET0 + np.cumsum(lens)]).astype(np.int64)

    def ids(seed):
        r = np.random.default_rng(seed)
        x = r.integers(0, sh.n, int(h_off[-1])) + sh.pid_base
        out_lo = sh.pid_base - 1 - r.integers(0, 50, x.size)
        out_hi = sh.pid_base + sh.n + r.integers(0, 50, x.size)
        pick = r.random(x.size)
        x = np.where(pick < 0.1, out_lo, np.where(pick < 0.2, out_hi, x))
        x[LIST_OFFSET0 + 1::7] = x[LIST_OFFSET0::7][:x[LIST_OFFSET0 + 1::7].size]     # duplicates
        return torch.from_numpy(x.astype(np.int64)).cuda()
    return h_off, ids


def _allow(sh, B, seed):
    """Bitmaps [B, words]: query 0 allows nothing, query 1 half the shard, the rest about 40 passages each (fewer than
    k = 128: the top-k fill is exercised)."""
    r = np.random.default_rng(seed)
    dens = np.full(B, 40.0 / sh.n)
    dens[0] = 0.0
    if B > 1:
        dens[1] = 0.5
    m = r.random((B, sh.n)) < dens[:, None]
    return sh.c.allow_bitmaps([np.nonzero(row)[0] + sh.pid_base for row in m])


def _allow_mask(sh, allow):
    """Dense bool [B, n] of bitmaps."""
    b = allow.cpu().numpy().view(np.uint8)
    return torch.from_numpy(np.unpackbits(b, axis=1, bitorder="little")[:, :sh.n].astype(bool)).cuda()


def scan_call(L, sh, kind, B, nq, k, seed, ws=None, comm=None):
    c = sh.c
    ws = c.workspace() if ws is None else ws
    rng = np.random.default_rng(seed)
    h_off, ids = _lists(sh, B, rng) if "listed" in kind else (None, None)

    def make(s):
        g = torch.Generator().manual_seed(s)
        ins = {"q": _unit(B * nq, g, sh.dtype).view(B, nq, DIM).cuda()}
        if "allowed" in kind:
            ins["allow"] = _allow(sh, B, s)
        if "listed" in kind:
            ins["pids"] = ids(s)
        return ins

    hq = C.c_void_p(c.handle.value)
    if kind.startswith("topk") or kind.startswith("sharded"):
        outputs = {"s": ((B, k), torch.float32), "p": ((B, k), torch.int64)}
    elif kind == "scores_listed":
        outputs = {"s": ((int(h_off[-1]),), torch.float32)}
    else:
        outputs = {"s": ((B, sh.n), torch.float32)}
    words = (sh.n + 31) // 32

    def fn(i, o, st):
        q, s = A.ptr(i["q"]), A.ptr(o["s"])
        if kind == "topk":
            return L.flmr_maxsim_topk(hq, ws, q, B, nq, k, 0, s, A.ptr(o["p"]), _h(st))
        if kind == "scores":
            return L.flmr_maxsim_scores(hq, ws, q, B, nq, 0, s, _h(st))
        if kind == "topk_allowed":
            return L.flmr_maxsim_topk_allowed(hq, ws, q, B, nq, k, 0, A.ptr(i["allow"]), words, s, A.ptr(o["p"]),
                                              _h(st))
        if kind == "scores_allowed":
            return L.flmr_maxsim_scores_allowed(hq, ws, q, B, nq, 0, A.ptr(i["allow"]), words, s, _h(st))
        if kind == "topk_listed":
            return L.flmr_maxsim_topk_listed(hq, ws, q, B, nq, k, 0, A.ptr(h_off), A.ptr(i["pids"]), s,
                                             A.ptr(o["p"]), _h(st))
        if kind == "scores_listed":
            return L.flmr_maxsim_scores_listed(hq, ws, q, B, nq, 0, A.ptr(h_off), A.ptr(i["pids"]), s, _h(st))
        if kind == "sharded":
            return L.flmr_maxsim_topk_sharded(hq, ws, comm, q, B, nq, k, 0, s, A.ptr(o["p"]), _h(st))
        if kind == "sharded_allowed":
            return L.flmr_maxsim_topk_sharded_allowed(hq, ws, comm, q, B, nq, k, 0, A.ptr(i["allow"]), words, s,
                                                      A.ptr(o["p"]), _h(st))
        raise ValueError(kind)

    call = A.Call("%s/%s" % (kind, "-".join(map(str, (sh.storage, sh.state, sh.pid_base, B, nq, k)))), fn, make(seed),
                  outputs, make, host={"h_off": h_off} if h_off is not None else {})
    if kind == "scores_listed":
        w = torch.zeros(int(h_off[-1]), dtype=torch.bool, device="cuda")
        w[LIST_OFFSET0:] = True
        call.written = {"s": w}
    call.kind, call.k, call.h_off = kind, k, h_off
    return call


def _restriction(sh, call):
    """Dense bool [B, n]: the passages each query may return (live, and allowed or listed)."""
    q = call.inputs["q"]
    B = q.size(0)
    live = torch.from_numpy(sh.live).cuda()
    m = live.expand(B, -1).clone()
    if "allow" in call.inputs:
        m &= _allow_mask(sh, call.inputs["allow"])
    if "pids" in call.inputs:
        lm = torch.zeros_like(m)
        p = call.inputs["pids"].cpu().numpy() - sh.pid_base
        for b in range(B):
            x = p[call.h_off[b]:call.h_off[b + 1]]
            x = x[(x >= 0) & (x < sh.n)]
            lm[b, torch.from_numpy(x).cuda()] = True
        m &= lm
    return m


def check_scan_reference(L, sh, call, got):
    """The plain call against float64: unrestricted scores within the scan bound; every restricted output is the
    unrestricted scores masked (-inf / top-k of the masked row, ties to the lower id, (-inf, -1) fill)."""
    q = call.inputs["q"]
    B = q.size(0)
    full = torch.empty((B, sh.n), dtype=torch.float32, device="cuda")
    assert L.flmr_maxsim_scores(sh.c.handle, sh.c.workspace(), A.ptr(q), B, q.size(1), 0, A.ptr(full), None) == 0
    torch.cuda.synchronize()
    s64, bound = sh.scores64(q)
    live = torch.from_numpy(sh.live).cuda().expand(B, -1)
    assert torch.isneginf(full[~live]).all(), call.name
    err = (full.double() - s64).abs()[live]
    assert (err <= bound[live]).all(), "%s: unrestricted scores off by %.3e beyond the bound" % (
        call.name, float((err - bound[live]).max()))
    masked = torch.where(_restriction(sh, call), full, NEG)
    if call.kind in ("scores", "scores_allowed"):
        assert A.same_bits(got["s"], masked), call.name
    elif call.kind == "scores_listed":
        p = call.inputs["pids"].cpu().numpy() - sh.pid_base
        want = np.full(p.size, -np.inf, np.float32)
        mc = masked.cpu().numpy()
        for b in range(B):
            for i in range(call.h_off[b], call.h_off[b + 1]):
                if 0 <= p[i] < sh.n:
                    want[i] = mc[b, p[i]]
        assert np.array_equal(got["s"].cpu().numpy()[LIST_OFFSET0:], want[LIST_OFFSET0:]), call.name
    else:
        rs, rp = O.topk(masked.cpu().numpy(), call.k, sh.pid_base)
        rp[np.isneginf(rs)] = -1                                    # the (-inf, -1) fill
        assert np.array_equal(got["p"].cpu().numpy(), rp), call.name
        assert np.array_equal(got["s"].cpu().numpy(), rs), call.name


def _info(L, sh):
    from ravqa_b200 import _cabi
    i = _cabi.CorpusInfo()
    assert L.flmr_corpus_info(sh.c.handle, C.byref(i)) == 0
    return bytes(i)


def run_contract(call, S, want, seed, synchronous=False):
    """(a) guarded outputs and untouched inputs; (b) late inputs, no hidden host synchronisation, early consumer."""
    A.guarded(call, want)
    r = A.gated(call, S, GATE_CYCLES, want, seed)
    if synchronous:
        assert r.gate_done_at_return, "%s: returned before the work queued on its stream had run" % call.name
    else:
        assert not r.gate_done_at_return, (
            "%s: the gate had ended when the call returned after %.1f ms: %s" % (
                call.name, 1e3 * r.call_seconds,
                "a host synchronisation" if r.call_seconds > 0.5 * gate_seconds() else "the gate is too short"))
    A.early_consumer(call, S, GATE_CYCLES, want)
    return r


_GATE_S = []


def gate_seconds():
    """Device time of one gate (measured once)."""
    if not _GATE_S:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        torch.cuda._sleep(GATE_CYCLES)
        b.record()
        b.synchronize()
        _GATE_S.append(a.elapsed_time(b) / 1e3)
    return _GATE_S[0]


# ---- (b) setup: the side stream does not wait for the legacy default stream, nor the reverse -------------------------
def test_side_stream_is_non_blocking(side):
    g = A.gate(side, GATE_CYCLES)
    e = torch.cuda.Event()
    e.record(torch.cuda.default_stream())
    e.synchronize()
    assert not g.query(), "the legacy default stream waited for the side stream"
    torch.cuda.synchronize()
    g = A.gate(torch.cuda.default_stream(), GATE_CYCLES)
    e = torch.cuda.Event()
    e.record(side)
    e.synchronize()
    assert not g.query(), "the side stream waited for the legacy default stream"
    torch.cuda.synchronize()
    print("gate: %d cycles = %.1f ms" % (GATE_CYCLES, 1e3 * gate_seconds()))


# ---- (a) + (b) every scan entry point over the corpus states ---------------------------------------------------------
@pytest.mark.parametrize("combo", range(len(COMBOS)),
                         ids=lambda c: "%s-%s-%d_%dx%d_k%d" % (*SHARDS[COMBOS[c][0]], *COMBOS[c][1], COMBOS[c][2]))
def test_scan_entry_points(L, shards, side, comm, combo):
    si, (B, nq), k = COMBOS[combo]
    sh = shards(si)
    kinds = list(SCAN_KINDS)
    if combo % 6 == 0:
        kinds += ["sharded", "sharded_allowed"]
    times = {}
    for ki, kind in enumerate(kinds):
        call = scan_call(L, sh, kind, B, nq, k, seed=1000 * combo + ki, comm=comm)
        info = _info(L, sh)
        want = call.plain()
        check_scan_reference(L, sh, call, want)
        r = run_contract(call, side, want, seed=7 + ki)
        times[kind] = r.call_seconds
        again = call.plain()
        call.compare(again, want, "repeat")
        assert _info(L, sh) == info, call.name
    print("host ms per call: " + ", ".join("%s %.2f" % (n, 1e3 * t) for n, t in times.items()))


@pytest.mark.parametrize("kind", ["topk_listed", "scores_listed"])
def test_listed_call_with_a_large_offset_table(L, shards, side, kind):
    """8,400 queries in one call chunk (a workspace of that many queries): 67 KB of host offsets and a pass table of
    700 passes, both copied from pageable host memory, and the call still returns while the gate holds."""
    sh = shards(0)
    B = 8400
    ws = C.c_void_p()
    assert L.flmr_workspace_create(sh.c.handle, B, 32, C.byref(ws)) == 0
    try:
        call = scan_call(L, sh, kind, B, 32, 10, seed=77, ws=ws)
        want = call.plain()
        run_contract(call, side, want, seed=78)
    finally:
        torch.cuda.synchronize()
        L.flmr_workspace_destroy(ws)


# ---- (a) + (b) select, merge, exchange -------------------------------------------------------------------------------
def select_call(L, B, n, k, pid_base):
    def make(s):
        g = torch.Generator().manual_seed(s)
        x = torch.randint(0, 40, (B, n), generator=g).float() / 8 - 2          # many ties
        return {"scores": x.cuda()}

    def fn(i, o, st):
        return L.flmr_topk_select(A.ptr(i["scores"]), B, n, k, pid_base, A.ptr(o["s"]), A.ptr(o["p"]), 0, _h(st))
    return A.Call("select/%dx%d/k%d" % (B, n, k), fn, make(1), {"s": ((B, k), torch.float32),
                                                                "p": ((B, k), torch.int64)}, make)


def merge_call(L, n_lists, B, k_in, k_out):
    def make(s):
        r = np.random.default_rng(s)
        sc = np.full((n_lists, B, k_in), -np.inf, np.float32)
        pid = np.full((n_lists, B, k_in), -1, np.int64)
        for b in range(B):
            if b % 3 == 1:
                continue                                             # every input of this row is empty
            ids = r.choice(100000, n_lists * k_in, replace=False)
            v = (r.integers(0, 30, ids.size) / 4).astype(np.float32)
            for li in range(n_lists):
                m = r.integers(0, k_in + 1)                          # a list of m entries, then its (-inf, -1) fill
                sl = slice(li * k_in, li * k_in + m)
                order = np.lexsort((ids[sl], -v[sl]))
                sc[li, b, :m], pid[li, b, :m] = v[sl][order], ids[sl][order]
        return {"scores": torch.from_numpy(sc).cuda(), "pids": torch.from_numpy(pid).cuda()}

    def fn(i, o, st):
        return L.flmr_topk_merge(A.ptr(i["scores"]), A.ptr(i["pids"]), n_lists, B, k_in, k_out, A.ptr(o["s"]),
                                 A.ptr(o["p"]), 0, _h(st))
    return A.Call("merge/%dx%dx%d/k%d" % (n_lists, B, k_in, k_out), fn, make(1),
                  {"s": ((B, k_out), torch.float32), "p": ((B, k_out), torch.int64)}, make)


def _merge_ref(scores, pids, k):
    """Top-k of every query's entries with pid >= 0 over all lists, ties to the lower id, (-inf, -1) fill."""
    sc, pid = scores.cpu().numpy(), pids.cpu().numpy()
    B = sc.shape[1]
    out_s, out_p = np.full((B, k), -np.inf, np.float32), np.full((B, k), -1, np.int64)
    for b in range(B):
        v, p = sc[:, b].reshape(-1), pid[:, b].reshape(-1)
        v, p = v[p >= 0], p[p >= 0]
        o = np.lexsort((p, -v.astype(np.float64)))[:k]
        out_s[b, :o.size], out_p[b, :o.size] = v[o], p[o]
    return out_s, out_p


@pytest.mark.parametrize("B,n,k,pid_base", [(3, 50, 300, 1000), (4, 5000, 1000, 0), (2, 130, 128, 7)])
def test_topk_select(L, side, B, n, k, pid_base):
    call = select_call(L, B, n, k, pid_base)
    want = call.plain()
    rs, rp = O.topk(call.inputs["scores"].cpu().numpy(), k, pid_base)
    assert np.array_equal(want["p"].cpu().numpy(), rp) and np.array_equal(want["s"].cpu().numpy(), rs)
    run_contract(call, side, want, seed=5)


@pytest.mark.parametrize("n_lists,B,k_in,k_out", [(3, 7, 10, 25), (1, 5, 128, 128), (8, 4, 64, 1)])
def test_topk_merge(L, side, n_lists, B, k_in, k_out):
    call = merge_call(L, n_lists, B, k_in, k_out)
    want = call.plain()
    rs, rp = _merge_ref(call.inputs["scores"], call.inputs["pids"], k_out)
    assert np.array_equal(want["p"].cpu().numpy(), rp) and np.array_equal(want["s"].cpu().numpy(), rs)
    run_contract(call, side, want, seed=5)


def test_topk_exchange_one_rank(L, side, comm):
    B, k_in, k_out = 6, 40, 100
    inner = merge_call(L, 1, B, k_in, k_out)

    def fn(i, o, st):
        return L.flmr_topk_exchange(comm, A.ptr(i["scores"]), A.ptr(i["pids"]), B, k_in, k_out, A.ptr(o["s"]),
                                    A.ptr(o["p"]), _h(st))
    call = A.Call("exchange", fn, inner.inputs, inner.outputs, inner.make_inputs)
    want = call.plain()
    rs, rp = _merge_ref(call.inputs["scores"], call.inputs["pids"], k_out)
    assert np.array_equal(want["p"].cpu().numpy(), rp) and np.array_equal(want["s"].cpu().numpy(), rs)
    run_contract(call, side, want, seed=5)


# ---- (a) + (b) gather ------------------------------------------------------------------------------------------------
def gather_call(L, sh, n_pids, nd_max, seed):
    def make(s):
        r = np.random.default_rng(s)
        x = r.integers(0, sh.n, n_pids) + sh.pid_base
        pick = r.random(n_pids)
        x = np.where(pick < 0.1, -1, np.where(pick < 0.15, sh.pid_base + sh.n + 3,
                                              np.where(pick < 0.2, sh.pid_base - 2, x)))
        return {"pids": torch.from_numpy(x.astype(np.int64)).cuda()}

    def fn(i, o, st):
        return L.flmr_corpus_gather(sh.c.handle, A.ptr(i["pids"]), n_pids, nd_max, A.ptr(o["out"]),
                                    A.ptr(o.get("mask")), _h(st))
    return A.Call("gather/%s-%s-%d" % (sh.storage, sh.state, sh.pid_base), fn, make(seed),
                  {"out": ((n_pids, nd_max, DIM), sh.dtype), "mask": ((n_pids, nd_max), torch.uint8)}, make)


def check_gather_reference(sh, call, got):
    p = call.inputs["pids"].cpu().numpy() - sh.pid_base
    n_pids, nd_max = got["mask"].shape
    out = torch.zeros((n_pids, nd_max, DIM), dtype=sh.dtype)
    mask = torch.zeros((n_pids, nd_max), dtype=torch.uint8)
    for i, x in enumerate(p):
        if 0 <= x < sh.n and sh.live[x]:
            m = min(int(sh.dl[x]), nd_max)
            out[i, :m] = sh.D[sh.off[x]:sh.off[x] + m]
            mask[i, :m] = 1
    assert A.same_bits(got["out"].cpu(), out) and torch.equal(got["mask"].cpu(), mask), call.name


@pytest.mark.parametrize("si", [0, 2, 4, 8], ids=lambda i: "-".join(map(str, SHARDS[i])))
def test_corpus_gather(L, shards, side, si):
    sh = shards(si)
    call = gather_call(L, sh, 300, 100, seed=si)
    want = call.plain()
    check_gather_reference(sh, call, want)
    run_contract(call, side, want, seed=9)
    A.guarded(call, {"out": want["out"]}, omit="mask")


# ---- (a) + (b) training routes ---------------------------------------------------------------------------------------
def _train_inputs(B, nq, n_docs, nd, dtype, s, grouped):
    g = torch.Generator().manual_seed(s)
    nt = B * n_docs if grouped else n_docs
    mask = (torch.rand((nt, nd), generator=g) < 0.8).to(torch.uint8)
    mask[0] = 0                                                       # a fully masked document: arg -1
    return {"q": _unit(B * nq, g, dtype).view(B, nq, DIM).cuda(),
            "docs": _unit(nt * nd, g, dtype).view(nt, nd, DIM).cuda(), "mask": mask.cuda()}


ROUTES = [(grouped, f16, path) for grouped in (False, True) for f16 in (False, True) for path in (1, 2)]


def argmax_call(L, grouped, f16, path, B=3, nq=40, n_docs=5, nd=70):
    name = "flmr_maxsim_argmax" + ("_grouped" if grouped else "") + ("_fp16" if f16 else "")
    dtype = torch.float16 if f16 else torch.bfloat16
    P = n_docs

    def fn(i, o, st):
        L.flmr_debug_set_argmax_path(path)
        try:
            return getattr(L, name)(A.ptr(i["q"]), B, nq, A.ptr(i["docs"]), A.ptr(i["mask"]), n_docs, nd,
                                    A.ptr(o["arg"]), A.ptr(o.get("rowmax")), 0, _h(st))
        finally:
            L.flmr_debug_set_argmax_path(0)
    make = lambda s: _train_inputs(B, nq, n_docs, nd, dtype, s, grouped)
    return A.Call("%s/path%d" % (name, path), fn, make(3), {"arg": ((B, P, nq), torch.int32),
                                                            "rowmax": ((B, P, nq), torch.float32)}, make)


def backward_call(L, grouped, f16, B=3, nq=40, n_docs=5, nd=70):
    name = "flmr_maxsim_backward" + ("_grouped" if grouped else "") + ("_fp16" if f16 else "")
    dtype = torch.float16 if f16 else torch.bfloat16
    nt = B * n_docs if grouped else n_docs

    def make(s):
        ins = _train_inputs(B, nq, n_docs, nd, dtype, s, grouped)
        g = torch.Generator().manual_seed(s + 1)
        arg = torch.randint(0, nd, (B, n_docs, nq), generator=g, dtype=torch.int32)
        arg[:, 0] = -1
        del ins["mask"]
        ins["arg"] = arg.cuda()
        ins["grad"] = torch.randn((B, n_docs), generator=g).cuda()
        return ins

    def fn(i, o, st):
        return getattr(L, name)(A.ptr(i["q"]), B, nq, A.ptr(i["docs"]), n_docs, nd, A.ptr(i["arg"]),
                                A.ptr(i["grad"]), A.ptr(o.get("dq")), A.ptr(o.get("dd")), 0, _h(st))
    def dd_close(ins, got, want):
        # dD is accumulated with fp32 atomics: two calls may sum in different orders, so it is held to the summation
        # bound of its float64 value instead of bitwise
        _, dD, _, dd_abs, cnt = T64.backward(ins["q"], ins["docs"], ins["arg"].long(), ins["grad"],
                                             n_docs if grouped else None)
        return ((got.double() - want.double()).abs() <= 2 * (cnt[..., None] + 1) * T64.U * dd_abs).all()
    return A.Call(name, fn, make(4), {"dq": ((B, nq, DIM), torch.float32), "dd": ((nt, nd, DIM), torch.float32)},
                  make, close={"dd": dd_close})


def ib_loss_call(L, B=4, n_docs=12, nq=20, nway=3, label0=0):
    def make(s):
        g = torch.Generator().manual_seed(s)
        return {"rowmax": torch.rand((B, n_docs, nq), generator=g).cuda()}

    def fn(i, o, st):
        return L.flmr_ib_loss(A.ptr(i["rowmax"]), B, n_docs, nq, nway, label0, A.ptr(o["scores"]), A.ptr(o["loss"]),
                              A.ptr(o["dscores"]), 0, _h(st))
    return A.Call("flmr_ib_loss", fn, make(5), {"scores": ((B, n_docs), torch.float32), "loss": ((B,), torch.float32),
                                                "dscores": ((B, n_docs), torch.float32)}, make)


@pytest.mark.parametrize("grouped,f16,path", ROUTES, ids=lambda v: str(v))
def test_argmax_routes(L, side, grouped, f16, path):
    call = argmax_call(L, grouped, f16, path)
    want = call.plain()
    i = call.inputs
    arg64, rowmax64, absmax = T64.argmax_rowmax(i["q"], i["docs"], i["mask"], 5 if grouped else None)
    fin = torch.isfinite(rowmax64)
    assert torch.equal(torch.isfinite(want["rowmax"]), fin) and (want["arg"][~fin] == -1).all(), call.name
    err = (want["rowmax"].double() - rowmax64)[fin].abs()
    assert (err <= T64.C_BOUND * T64.U * absmax[fin]).all(), call.name
    run_contract(call, side, want, seed=6)
    A.guarded(call, {"arg": want["arg"]}, omit="rowmax")


@pytest.mark.parametrize("grouped,f16", [(g, f) for g in (False, True) for f in (False, True)], ids=str)
def test_backward_routes(L, side, grouped, f16):
    call = backward_call(L, grouped, f16)
    want = call.plain()
    i = call.inputs
    dQ, dD, dq_abs, dd_abs, _ = T64.backward(i["q"], i["docs"], i["arg"].long(), i["grad"], 5 if grouped else None)
    assert ((want["dq"].double() - dQ).abs() <= 64 * T64.U * dq_abs + 1e-30).all(), call.name
    assert ((want["dd"].double() - dD).abs() <= 64 * T64.U * dd_abs + 1e-30).all(), call.name
    run_contract(call, side, want, seed=6)
    A.guarded(call, {"dd": want["dd"]}, omit="dq")
    A.guarded(call, {"dq": want["dq"]}, omit="dd")


def test_ib_loss(L, side):
    call = ib_loss_call(L)
    want = call.plain()
    s, loss, ds = T64.ib_loss(call.inputs["rowmax"], 3, 0)
    lb, db = T64.ib_loss_bounds(want["scores"], 3, 0)
    assert ((want["loss"].double() - loss).abs() <= lb + 20 * T64.U * loss.abs()).all()
    assert ((want["scores"].double() - s).abs() <= 20 * T64.U * s.abs()).all()
    run_contract(call, side, want, seed=6)


# ---- (a) + (b) PLAID decode: synchronous on its stream ---------------------------------------------------------------
@pytest.mark.parametrize("f16,nbits", [(False, 2), (True, 4)], ids=["bf16-nbits2", "fp16-nbits4"])
def test_plaid_decode(L, side, f16, nbits):
    n, nc = 3000, 64
    name = "flmr_plaid_decode" + ("_fp16" if f16 else "")
    dtype = torch.float16 if f16 else torch.bfloat16

    def make(s):
        g = torch.Generator().manual_seed(s)
        codes, res = LF.random_codes(n, nc, nbits, g)
        return {"codes": codes.cuda(), "res": res.cuda(), "cent": _unit(nc, g, torch.float32).cuda(),
                "w": LF.fixture_weights(nbits, g).float().cuda()}

    def fn(i, o, st):
        return getattr(L, name)(A.ptr(i["codes"]), A.ptr(i["res"]), n, A.ptr(i["cent"]), nc, A.ptr(i["w"]), nbits,
                                DIM, 1, A.ptr(o["out"]), 0, _h(st))
    call = A.Call(name, fn, make(1), {"out": ((n, DIM), dtype)}, make, synchronous=True)
    want = call.plain()
    i = {k: v.cpu() for k, v in call.inputs.items()}
    LF.check_rounding(want["out"].cpu(), LF.decode_fp64(i["codes"], i["res"], i["cent"], i["w"], nbits), name)
    run_contract(call, side, want, seed=2, synchronous=True)


# ---- (c) graph capture and replay ------------------------------------------------------------------------------------
def test_graph_replay_select_merge(L):
    A.graph_replay(select_call(L, 3, 5000, 700, 1000))
    A.graph_replay(select_call(L, 2, 60, 128, 0))
    A.graph_replay(merge_call(L, 4, 6, 32, 50))


@pytest.mark.parametrize("si", [0, 2, 8], ids=lambda i: "-".join(map(str, SHARDS[i])))
def test_graph_replay_gather(L, shards, si):
    A.graph_replay(gather_call(L, shards(si), 200, 90, seed=3))


@pytest.mark.parametrize("route", ["grouped", "fp16", "path1", "path2"])
def test_graph_replay_training(L, route):
    if route == "grouped":
        calls = [argmax_call(L, True, False, 0), backward_call(L, True, False)]
    elif route == "fp16":
        calls = [argmax_call(L, False, True, 0), backward_call(L, False, True), argmax_call(L, True, True, 0),
                 backward_call(L, True, True)]
    else:
        calls = [argmax_call(L, False, False, int(route[-1])), argmax_call(L, True, True, int(route[-1]))]
    for call in calls:
        A.graph_replay(call)


# ---- (d) one workspace per thread ------------------------------------------------------------------------------------
def _script(L, sh, ws, seed):
    """About 20 mixed calls on one workspace: top-k, scores, allowed, listed and gather."""
    calls = []
    kinds = ["topk", "scores", "topk_allowed", "topk_listed", "scores_allowed", "scores_listed"]
    for j in range(18):
        B, nq = SHAPES[(seed + j) % 3]
        calls.append(scan_call(L, sh, kinds[j % len(kinds)], B, nq, (1, 128, 10)[j % 3], seed * 100 + j, ws=ws))
    calls.append(gather_call(L, sh, 120, 80, seed))
    calls.append(gather_call(L, sh, 50, 200, seed + 1))
    return calls


@pytest.mark.parametrize("si", [0, 6, 5], ids=lambda i: "-".join(map(str, SHARDS[i])))
def test_two_threads_one_corpus(L, shards, si):
    sh = shards(si)
    wss = []
    for _ in range(2):
        ws = C.c_void_p()
        assert L.flmr_workspace_create(sh.c.handle, 64, 1024, C.byref(ws)) == 0
        wss.append(ws)
    try:
        scripts = [_script(L, sh, wss[t], seed=11 + t) for t in range(2)]
        wants = [[call.plain() for call in script] for script in scripts]      # serially, default stream
        guards = [[{n: A.Guarded(s, d) for n, (s, d) in call.outputs.items()} for call in script] for script in scripts]
        streams = [torch.cuda.Stream() for _ in range(2)]
        torch.cuda.synchronize()
        barrier = threading.Barrier(2)
        errors = [None, None]

        def work(t):
            try:
                barrier.wait()
                A.gate(streams[t], GATE_CYCLES)
                for call, gs in zip(scripts[t], guards[t]):
                    call.run(call.inputs, {n: g.out for n, g in gs.items()}, streams[t].cuda_stream)
            except BaseException as e:                                   # reported by the main thread
                errors[t] = e
        th = [threading.Thread(target=work, args=(t,)) for t in range(2)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        torch.cuda.synchronize()
        for e in errors:
            if e is not None:
                raise e
        for t in range(2):
            for call, gs, want in zip(scripts[t], guards[t], wants[t]):
                for n, g in gs.items():
                    g.check(call.written.get(n), "thread %d / %s / %s" % (t, call.name, n))
                call.compare({n: g.out for n, g in gs.items()}, want, "thread %d" % t)
    finally:
        torch.cuda.synchronize()
        for ws in wss:
            L.flmr_workspace_destroy(ws)


def test_last_error_and_scan_variant_are_per_thread(L, shards):
    sh = shards(0)
    q = torch.zeros((2, 32, DIM), dtype=torch.bfloat16, device="cuda")
    s = torch.empty((2, 8), device="cuda")
    p = torch.empty((2, 8), dtype=torch.int64, device="cuda")
    h_off = np.array([0, 3, 5], np.int64)
    ids = torch.arange(5, dtype=torch.int64, device="cuda")
    wss = []
    for _ in range(2):
        ws = C.c_void_p()
        assert L.flmr_workspace_create(sh.c.handle, 64, 1024, C.byref(ws)) == 0
        wss.append(ws)
    barrier = threading.Barrier(2)
    seen = [None, None]

    def listed(t):
        return L.flmr_maxsim_topk_listed(sh.c.handle, wss[t], A.ptr(q), 2, 32, 8, 0, A.ptr(h_off), A.ptr(ids),
                                         A.ptr(s if t == 0 else s.clone()), A.ptr(p if t == 0 else p.clone()), None)

    def work(t):
        try:
            # each thread fails with its own message
            bad = (L.flmr_maxsim_topk(sh.c.handle, wss[t], A.ptr(q), 2, 32, 0, 0, A.ptr(s), A.ptr(p), None) if t == 0
                   else L.flmr_topk_merge(A.ptr(s), A.ptr(p), 0, 2, 8, 8, A.ptr(s), A.ptr(p), 0, None))
            barrier.wait()
            msg = L.flmr_last_error().decode()
            barrier.wait()
            # thread 0 forces variant 3, which has no listed kernel; thread 1 keeps the product's choice
            if t == 0:
                L.flmr_debug_set_scan_variant(3)
            barrier.wait()
            rc = listed(t)
            barrier.wait()
            if t == 0:
                L.flmr_debug_set_scan_variant(0)
            seen[t] = (bad, msg, rc)
        except BaseException as e:
            seen[t] = e
    th = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    torch.cuda.synchronize()
    try:
        for t in range(2):
            if isinstance(seen[t], BaseException):
                raise seen[t]
        assert seen[0][0] == 1 and "k=0" in seen[0][1], seen[0]
        assert seen[1][0] == 1 and "merge shape" in seen[1][1], seen[1]
        assert seen[0][2] == 3, "variant 3 set on this thread: the listed call must be refused"
        assert seen[1][2] == 0, "variant 3 set on the other thread changed this thread's scan"
    finally:
        for ws in wss:
            L.flmr_workspace_destroy(ws)


# ---- (a) host outputs with a capacity that need a device -------------------------------------------------------------
def test_host_outputs_with_capacity(L, R):
    S64_ = np.int64(0x5A5A5A5A5A5A5A5A)
    g = torch.Generator().manual_seed(3)
    dl = (np.arange(700) % 50 + 1).astype(np.int32)
    c = R.FlatCorpus(_unit(int(dl.sum()), g), dl, device=0, pid_base=1000)
    try:
        def deleted():
            n = C.c_int64(-1)
            assert L.flmr_corpus_deleted(c.handle, C.byref(n), None, 0) == 0
            need = n.value
            for cap, ok in ((need, True), (need - 1, False)):
                buf = np.full(need + 64, S64_, np.int64)
                rc = L.flmr_corpus_deleted(c.handle, C.byref(n), buf.ctypes.data_as(C.c_void_p), cap)
                assert n.value == need
                if ok:
                    assert rc == 0 and (buf[need:] == S64_).all()
                    got = buf[:need]
                else:
                    assert rc == 1 and (buf[max(cap, 0):] == S64_).all()
            return got
        c.delete(np.arange(1000, 1700, 5))
        before = deleted()
        assert np.array_equal(before, np.arange(1000, 1700, 5))
        c.compact()                                        # compacted-away ids still count as deleted
        c.delete([1001, 1002])
        assert np.array_equal(deleted(), np.sort(np.concatenate([before, [1001, 1002]])))
        # flmr_debug_listed_plan
        h_off = np.array([0, 40, 40, 90], np.int64)
        ids = torch.from_numpy(np.random.default_rng(1).integers(990, 1710, 90)).cuda()
        n = C.c_int64(-1)
        args = (c.handle, c.workspace(), 3, 97, h_off.ctypes.data_as(C.c_void_p), A.ptr(ids))
        assert L.flmr_debug_listed_plan(*args, None, 0, C.byref(n)) == 0
        need = n.value
        for cap, ok in ((need, True), (need - 1, False)):
            buf = np.full(need + 64, S64_, np.int64)
            rc = L.flmr_debug_listed_plan(*args, buf.ctypes.data_as(C.c_void_p), cap, C.byref(n))
            assert n.value == need
            assert (buf[need:] == S64_).all() if ok else (rc == 1 and (buf[cap:] == S64_).all())
            if ok:
                assert rc == 0 and buf[0] >= 1
    finally:
        c.close()
    # flmr_comm_unique_id writes 128 bytes and no more
    buf = (C.c_uint8 * 256)(*([0xA5] * 256))
    assert L.flmr_comm_unique_id(C.cast(buf, C.c_void_p)) == 0
    assert list(buf[128:]) == [0xA5] * 128
    assert list(buf[:128]) != [0xA5] * 128


def test_sharded_send_buffers_grow_apart_from_the_exchange(L, R, shards):
    """The communicator's send buffers (this rank's lists of flmr_maxsim_topk_sharded) and receive buffers (everybody's
    lists, grown by flmr_topk_exchange) are sized apart: an exchange of many entries followed by sharded searches of
    few and then more entries than the first search held."""
    sh = shards(0)
    uid = (C.c_char * 128)()
    assert L.flmr_comm_unique_id(C.cast(uid, C.c_void_p)) == 0
    comm = C.c_void_p()
    assert L.flmr_comm_create(C.cast(uid, C.c_void_p), 0, 1, 0, C.byref(comm)) == 0
    try:
        big = merge_call(L, 1, 60, 128, 128)
        s = torch.empty((60, 128), device="cuda")
        p = torch.empty((60, 128), dtype=torch.int64, device="cuda")
        assert L.flmr_topk_exchange(comm, A.ptr(big.inputs["scores"]), A.ptr(big.inputs["pids"]), 60, 128, 128,
                                    A.ptr(s), A.ptr(p), None) == 0
        for B, k in ((2, 10), (40, 128), (3, 5)):
            call = scan_call(L, sh, "sharded", B, 32, k, seed=B, comm=comm)
            local = scan_call(L, sh, "topk", B, 32, k, seed=B)
            A.guarded(call, local.plain())
    finally:
        torch.cuda.synchronize()
        L.flmr_comm_destroy(comm)
