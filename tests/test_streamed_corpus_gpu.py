"""GPU: a streamed corpus (FlatCorpus(residency="host"): rows in pinned host memory, copied through two HBM windows per
search) returns BITWISE what the resident corpus built from the same rows returns — scores, top-k, gather, Searcher —
over a pairwise covering of storage, relu, query length, batch, window count, pid_base, deletions and allow bitmaps;
and holds the C boundary's conventions, its refusals and its memory promise."""
from __future__ import annotations

import ctypes as C
import itertools
import os
import threading

import numpy as np
import pytest
import torch

import abi_contract as A
from helpers import GOLDEN_DIR

pytestmark = pytest.mark.gpu

DIM = 128
ROW = DIM * 2
UNSUPPORTED = 3


@pytest.fixture(scope="module")
def R():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import ravqa_b200 as R
    return R


@pytest.fixture(scope="module")
def L(R):
    from ravqa_b200 import _cabi
    return _cabi.lib()


def _rows(n, seed, lo=1, hi=120, dtype=torch.bfloat16):
    rng = np.random.default_rng(seed)
    dl = rng.integers(lo, hi, size=n).astype(np.int32)
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(int(dl.sum()), DIM, generator=g)
    return torch.nn.functional.normalize(t, dim=-1).to(dtype), dl


def _queries(B, nq, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    q = torch.nn.functional.normalize(torch.randn(B, nq, DIM, generator=g), dim=-1)
    if nq > 3:
        q[:, -2:] = 0                      # zero rows, as the encoder's masked tokens
    return q.to(dtype).cuda()


def _n_windows(dl, window_rows):
    """Windows of the greedy plan (as flmr_debug_window_plan cuts them) of window_rows rows."""
    poff = np.concatenate([[0], np.cumsum((dl.astype(np.int64) + 3) // 4 * 4)])
    n, s0 = 0, 0
    while s0 < len(dl):
        s0 = int(np.searchsorted(poff, poff[s0] + window_rows, side="right")) - 1
        n += 1
    return n


def _window_bytes_for(dl, n_windows):
    """The smallest window (in whole 4-row groups) whose plan has at most n_windows windows."""
    rows = (dl.astype(np.int64) + 3) // 4 * 4
    lo, hi = int(rows.max()), int(rows.sum())
    while lo < hi:
        mid = (lo + hi) // 2 // 4 * 4
        if mid < lo:
            mid = lo
        if _n_windows(dl, mid) <= n_windows:
            hi = mid
        else:
            lo = mid + 4
    return hi * ROW


def _pair(R, tokens, dl, storage, pid_base, window_bytes):
    res = R.FlatCorpus(tokens, dl, pid_base=pid_base, storage=storage, adopt=False)
    st = R.FlatCorpus(tokens, dl, pid_base=pid_base, storage=storage, residency="host", window_bytes=window_bytes)
    return res, st


def _windows(L, dl, window_bytes):
    nw = C.c_int64()
    assert L.flmr_debug_window_plan(np.ascontiguousarray(dl).ctypes.data, len(dl), window_bytes, 132, None, 0,
                                    C.byref(nw), None, None, None, None, 0, None) == 0
    table = np.zeros((nw.value, 6), np.int64)
    assert L.flmr_debug_window_plan(np.ascontiguousarray(dl).ctypes.data, len(dl), window_bytes, 132,
                                    table.ctypes.data, nw.value, C.byref(nw), None, None, None, None, 0, None) == 0
    return table


def _want_info(L, dl, storage, window_bytes, sms):
    """(n_ctas, n_tiles, hbm_bytes) flmr_corpus_info reports for a new library-owned corpus of doclens dl: resident
    (window_bytes 0: its rows, one partition and, bf16, the CTA-pair partition) or streamed (its windows' partitions),
    each beside the offsets and lengths.  Every device array takes 4 or 8 B per entry."""
    dl = np.ascontiguousarray(dl, np.int32)
    n, rows = len(dl), int(((dl.astype(np.int64) + 3) // 4 * 4).sum())

    def tiles(n_ctas):
        nt = C.c_int64()
        rb, tb = np.zeros(n_ctas + 1, np.int32), np.zeros(n_ctas + 1, np.int64)
        assert L.flmr_debug_build_partition(dl.ctypes.data, n, n_ctas, rb.ctypes.data, tb.ctypes.data, None, None, 0,
                                            C.byref(nt)) == 0
        return nt.value

    def partition_bytes(n_ctas, n_tiles):
        return (n_ctas + 1) * (4 + 8) + n_tiles * (4 + 4)

    meta = (n + 1) * 8 + n * 4
    if window_bytes:
        nw = C.c_int64()
        assert L.flmr_debug_window_plan(dl.ctypes.data, n, window_bytes, sms, None, 0, C.byref(nw), None, None, None,
                                        None, 0, None) == 0
        table = np.zeros((nw.value, 6), np.int64)
        assert L.flmr_debug_window_plan(dl.ctypes.data, n, window_bytes, sms, table.ctypes.data, nw.value,
                                        C.byref(nw), None, None, None, None, 0, None) == 0
        return (int(table[:, 4].max()), int(table[:, 5].sum()),
                meta + sum(partition_bytes(int(w[4]), int(w[5])) for w in table))
    nc = min(sms, n)
    hbm = rows * ROW + meta + partition_bytes(nc, tiles(nc))
    if storage == "bf16" and nc >= 2:
        hbm += partition_bytes(nc // 2, tiles(nc // 2))
    return nc, tiles(nc), hbm


# storage, relu, Nq, B, windows (24: more than 20), pid_base, deletions, allow bitmaps.  B = 70 exceeds the default
# workspace's 64 queries, so such a call scans each window in two chunks; Nq = 832 is row-sliced (partial scores by slot).
FACTORS = (("bf16", "fp16"), (False, True), (1, 32, 320, 832), (1, 5, 13, 70), (1, 2, 3, 24), (0, 1000),
           ("none", "some", "window"), (False, True))
CASES = [
    ("bf16", False, 832, 70, 24, 1000, "window", True),
    ("bf16", True, 1, 1, 1, 0, "none", False),
    ("fp16", True, 32, 13, 2, 1000, "some", False),
    ("fp16", False, 320, 5, 2, 0, "window", True),
    ("bf16", False, 832, 13, 3, 0, "some", True),
    ("fp16", True, 320, 70, 3, 1000, "none", False),
    ("bf16", False, 32, 5, 24, 0, "none", False),
    ("fp16", False, 32, 1, 1, 1000, "window", True),
    ("fp16", True, 1, 13, 24, 1000, "window", True),
    ("fp16", True, 832, 5, 1, 1000, "some", False),
    ("bf16", False, 1, 70, 2, 0, "some", True),
    ("bf16", True, 320, 1, 24, 1000, "some", False),
    ("fp16", True, 832, 1, 2, 1000, "none", False),
    ("fp16", True, 320, 13, 1, 1000, "none", True),
    ("fp16", True, 1, 5, 3, 1000, "window", False),
    ("fp16", False, 32, 1, 3, 0, "none", False),
    ("bf16", True, 32, 70, 1, 1000, "window", True),
]


def test_cases_cover_every_pair():
    """Every value of every factor meets every value of every other factor in some case."""
    missing = []
    for (i, fi), (j, fj) in itertools.combinations(enumerate(FACTORS), 2):
        for a, b in itertools.product(fi, fj):
            if not any(c[i] == a and c[j] == b for c in CASES):
                missing.append((i, a, j, b))
    assert not missing, missing
    assert all(len(c) == len(FACTORS) and all(v in f for v, f in zip(c, FACTORS)) for c in CASES)
    assert any(c[2] == 832 and c[3] > 64 and c[4] > 20 for c in CASES)


@pytest.mark.parametrize("storage,relu,nq,B,n_windows,pid_base,dels,allow", CASES,
                         ids=["-".join(map(str, c)) for c in CASES])
def test_streamed_is_bitwise_resident(R, L, storage, relu, nq, B, n_windows, pid_base, dels, allow):
    from ravqa_b200.maxsim import maxsim_scores, maxsim_topk
    dtype = torch.float16 if storage == "fp16" else torch.bfloat16
    n = 3000 if nq < 320 else 1200
    tokens, dl = _rows(n, seed=nq * 7 + n_windows, dtype=dtype)
    wb = _window_bytes_for(dl, n_windows)
    res, st = _pair(R, tokens, dl, storage, pid_base, wb)
    table = _windows(L, dl, wb)
    assert (len(table) == n_windows) if n_windows < 20 else (len(table) > 20)
    assert st.residency == "host" and res.residency == "device"
    assert st.residency_info()["window_bytes"] == wb and st.residency_info()["host_bytes"] == st.info.n_rows * ROW
    assert res.residency_info() == {"streamed": False, "window_bytes": 0, "host_bytes": 0}
    sms = torch.cuda.get_device_properties(st.device).multi_processor_count
    for c, w in ((res, 0), (st, wb)):
        assert (c.info.n_ctas, c.info.n_tiles, c.info.hbm_bytes) == _want_info(L, dl, storage, w, sms), c.residency
    rng = np.random.default_rng(B)
    if dels != "none":
        dead = rng.choice(n, size=n // 10, replace=False)
        if dels == "window":       # every passage of one window (the middle one), and a few more
            w = table[len(table) // 2]
            dead = np.union1d(dead, np.arange(w[0], w[1]))
        for c in (res, st):
            c.delete(dead + pid_base)
        assert st.n_deleted == res.n_deleted
    Q = _queries(B, nq, seed=B + nq, dtype=dtype)
    kw = {}
    if allow:
        lists = [None if b % 3 == 0 else rng.choice(n, size=n // 3, replace=False) + pid_base for b in range(B)]
        kw["allow"] = res.allow_bitmaps(lists)
    a = maxsim_scores(res, Q, relu=relu, **kw)
    b = maxsim_scores(st, Q, relu=relu, **kw)
    assert A.same_bits(a, b), "scores"
    for k in (1, 10, 128):
        sa, pa = maxsim_topk(res, Q, k, relu=relu, **kw)
        sb, pb = maxsim_topk(st, Q, k, relu=relu, **kw)
        assert A.same_bits(sa, sb) and torch.equal(pa, pb), "top-%d" % k
    pids = torch.from_numpy(rng.integers(pid_base - 3, pid_base + n + 3, size=(4, 37))).cuda()
    ga, ma = res.gather_padded(pids, nd_max=130)
    gb, mb = st.gather_padded(pids, nd_max=130)
    assert A.same_bits(ga, gb) and torch.equal(ma, mb), "gather"
    torch.cuda.synchronize()
    res.close()
    st.close()


def test_streamed_against_float64_and_simt(R):
    """Independently of the resident path: the scan's scores within the existing float64 bound, the SIMT kernel's
    within its own, on a streamed corpus of many windows."""
    import scan_fp64 as F
    from ravqa_b200.maxsim import debug_scores_simt, maxsim_scores
    tokens, dl = _rows(2500, seed=5)
    st = R.FlatCorpus(tokens, dl, residency="host", window_bytes=_window_bytes_for(dl, 7))
    for nq, B in ((32, 9), (832, 2)):
        Q = _queries(B, nq, seed=nq, dtype=torch.bfloat16)
        s64, amax, rabs = F.maxsim_packed(Q.float(), tokens.float(), dl)
        got = maxsim_scores(st, Q).double()
        assert ((got - s64).abs() <= F.scan_bound(amax, rabs, nq)).all()
        simt = debug_scores_simt(st, Q).double()
        assert ((simt - s64).abs() <= F.simt_bound(amax, rabs, nq)).all()
    st.close()


def test_device_memory_holds_windows_not_tokens(R):
    """A streamed corpus of a few GB with 64 MB windows: creating it and its workspace grows device memory by the two
    windows and the metadata, not by the tokens."""
    n, L_tok = 40_000, 180                              # 7.2M rows: 1.84 GB of bf16 tokens
    dl = np.full(n, L_tok, np.int32)
    tokens = torch.empty(n * L_tok, DIM, dtype=torch.bfloat16)
    tokens.fill_(0.05)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    st = R.FlatCorpus(tokens, dl, residency="host", window_bytes=64 << 20)
    st.workspace()
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    grown = free0 - free1
    token_bytes = n * L_tok * ROW
    assert st.info.hbm_bytes < 16 << 20, st.info.hbm_bytes
    # two windows (128 MB) + layout + workspace scratch (query staging, candidate lists): far below the tokens
    assert grown < (128 << 20) + (96 << 20), "device memory grew by %d B for %d B of tokens" % (grown, token_bytes)
    Q = _queries(3, 32, seed=1, dtype=torch.bfloat16)
    from ravqa_b200.maxsim import maxsim_topk
    s, p = maxsim_topk(st, Q, 10)
    torch.cuda.synchronize()
    assert (p >= 0).all()
    st.close()


def test_refusals_leave_the_corpus_unchanged(R, L):
    from ravqa_b200 import _cabi
    from ravqa_b200.maxsim import maxsim_topk
    tokens, dl = _rows(600, seed=11)
    res, st = _pair(R, tokens, dl, "bf16", 50, _window_bytes_for(dl, 3))
    Q = _queries(4, 32, seed=3, dtype=torch.bfloat16)
    before = maxsim_topk(st, Q, 20)
    info = bytes(st.info)
    # creation: fp8, adopt, a window smaller than the longest passage
    h = C.c_void_p()
    for flags, wb in ((_cabi.CORPUS_FP8, 1 << 20), (_cabi.CORPUS_ADOPT, 1 << 20), (0, ROW * 8)):
        assert L.flmr_corpus_create_streamed(C.c_void_p(tokens.data_ptr()), dl.ctypes.data, len(dl), DIM, 0, 0, flags,
                                             wb, C.byref(h)) == UNSUPPORTED and not h.value
    with pytest.raises(_cabi.FlmrError) as e:
        st.append(tokens[:int(dl[0])], dl[:1])
    assert e.value.code == UNSUPPORTED
    with pytest.raises(_cabi.FlmrError) as e:
        st.compact()
    assert e.value.code == UNSUPPORTED
    with pytest.raises(_cabi.FlmrError) as e:
        maxsim_topk(st, Q, 5, pids=[[50, 51]] * 4)
    assert e.value.code == UNSUPPORTED
    from ravqa_b200.maxsim import maxsim_scores_listed
    with pytest.raises(_cabi.FlmrError) as e:
        maxsim_scores_listed(st, Q, [[50, 51]] * 4)
    assert e.value.code == UNSUPPORTED
    st._refresh()
    assert bytes(st.info) == info
    after = maxsim_topk(st, Q, 20)
    assert A.same_bits(before[0], after[0]) and torch.equal(before[1], after[1])
    want = maxsim_topk(res, Q, 20)
    assert A.same_bits(want[0], after[0]) and torch.equal(want[1], after[1])
    # a streamed Searcher takes the bitmap path, and the updater surfaces the refusal
    s = R.Searcher(index=st, config=R.ColBERTConfig(total_visible_gpus=1))
    assert s.residency == "host"
    assert not s._listed_is_cheaper(Q, [torch.tensor([50, 51])] * 4)
    # a Searcher does not silently ignore what it cannot apply to the corpus it is given
    with pytest.raises(ValueError, match="residency"):
        R.Searcher(index=st, config=R.ColBERTConfig(total_visible_gpus=1), residency="device")
    with pytest.raises(ValueError, match="window_bytes"):
        R.Searcher(index=st, config=R.ColBERTConfig(total_visible_gpus=1), window_bytes=1 << 20)
    assert R.Searcher(index=res, config=R.ColBERTConfig(total_visible_gpus=1)).residency == "device"
    up = R.IndexUpdater(config=None, searcher=s)
    with pytest.raises(_cabi.FlmrError):
        up.add_embeddings(tokens[:int(dl[0])], dl[:1])
    with pytest.raises(_cabi.FlmrError):
        up.compact()
    up.remove([51])
    assert 51 not in maxsim_topk(st, Q, 128)[1].cpu().numpy()
    res.close()
    st.close()


def test_searcher_paths_bitwise(R):
    """_search_all_Q, dense_search(pids=) and retrieve_and_rescore on a streamed corpus: bitwise the resident ones."""
    tokens, dl = _rows(2000, seed=21)
    res, st = _pair(R, tokens, dl, "bf16", 0, _window_bytes_for(dl, 5))
    cfg = R.ColBERTConfig(total_visible_gpus=1)
    sr, ss = R.Searcher(index=res, config=cfg), R.Searcher(index=st, config=cfg)
    Q = _queries(90, 32, seed=9, dtype=torch.bfloat16).float().cpu()
    ra = sr._search_all_Q(None, Q, k=20).todict()
    rb = ss._search_all_Q(None, Q, k=20).todict()
    assert ra == rb
    pids = list(range(0, 2000, 7))
    for i in range(3):
        a = sr.dense_search(Q[i:i + 1], k=10, pids=pids)
        b = ss.dense_search(Q[i:i + 1], k=10, pids=pids)
        assert a == b
    Qg = Q[:6].to(torch.bfloat16).cuda()
    ga = torch.Generator(device="cpu").manual_seed(3)
    gb = torch.Generator(device="cpu").manual_seed(3)
    oa = sr.retrieve_and_rescore(Qg, 5, generator=ga)
    ob = ss.retrieve_and_rescore(Qg, 5, generator=gb)
    assert np.array_equal(oa["retrieved_doc_ids"], ob["retrieved_doc_ids"])
    for name in ("doc_scores", "search_scores", "item_embeddings"):
        assert A.same_bits(oa[name].detach(), ob[name].detach()), name
    assert torch.equal(oa["item_mask"], ob["item_mask"])
    res.close()
    st.close()


def _pinned_copies(fn):
    """fn() under torch.profiler: (its result, the number of pinned host-to-device copies it made)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    return out, sum(1 for n in names if "HtoD" in n and "Pinned" in n)


def test_searcher_streams_the_corpus_once_per_call(R):
    """A Searcher call of more than query_batch queries copies a streamed corpus once: unrestricted (one fused top-k
    call), restricted by qid_to_pids (bitmaps) and filtered (score rows) alike, with the resident results."""
    tokens, dl = _rows(2000, seed=51)
    wb = _window_bytes_for(dl, 4)
    res, st = _pair(R, tokens, dl, "bf16", 0, wb)
    n_windows = len(_windows(R._cabi.lib(), dl, wb))
    assert n_windows == 4
    cfg = R.ColBERTConfig(total_visible_gpus=1)
    sr, ss = R.Searcher(index=res, config=cfg), R.Searcher(index=st, config=cfg)
    B = 150
    assert B > ss.query_batch
    Q = _queries(B, 32, seed=4, dtype=torch.bfloat16).float().cpu()
    rng = np.random.default_rng(0)
    qid_to_pids = {b: rng.choice(2000, size=300, replace=False).tolist() for b in range(B)}
    keep = torch.arange(0, 2000, 3)

    def runs(s):
        return {"plain": lambda: s._search_all_Q(None, Q, k=10).todict(),
                "pids": lambda: s._search_all_Q(None, Q, k=10, qid_to_pids=qid_to_pids).todict(),
                "filter": lambda: s._search_all_Q(None, Q, k=10, filter_fn=lambda p: keep.to(p.device)).todict()}
    for name in ("plain", "pids", "filter"):
        want = runs(sr)[name]()
        runs(ss)[name]()                                  # warm-up: workspaces, scratch
        got, copies = _pinned_copies(runs(ss)[name])
        assert got == want, name
        assert copies == n_windows, "%s: %d window copies for %d windows" % (name, copies, n_windows)
    res.close()
    st.close()


def test_sharded_call_on_one_rank(R, L):
    """flmr_maxsim_topk_sharded(_allowed) on a one-rank communicator: bitwise the resident corpus's."""
    tokens, dl = _rows(1500, seed=61)
    res, st = _pair(R, tokens, dl, "bf16", 300, _window_bytes_for(dl, 3))
    uid = (C.c_char * 128)()
    assert L.flmr_comm_unique_id(C.cast(uid, C.c_void_p)) == 0
    comm = C.c_void_p()
    assert L.flmr_comm_create(C.cast(uid, C.c_void_p), 0, 1, 0, C.byref(comm)) == 0
    B, nq, k = 70, 32, 16
    Q = _queries(B, nq, seed=8, dtype=torch.bfloat16)
    allow = res.allow_bitmaps([np.arange(300, 1800, 2)] * B)
    words = allow.size(1)
    out = {}
    for name, c in (("res", res), ("st", st)):
        s = torch.empty((B, k), dtype=torch.float32, device="cuda")
        p = torch.empty((B, k), dtype=torch.int64, device="cuda")
        s2, p2 = torch.empty_like(s), torch.empty_like(p)
        assert L.flmr_maxsim_topk_sharded(c.handle, c.workspace(), comm, A.ptr(Q), B, nq, k, 0, A.ptr(s), A.ptr(p),
                                          None) == 0
        assert L.flmr_maxsim_topk_sharded_allowed(c.handle, c.workspace(), comm, A.ptr(Q), B, nq, k, 0, A.ptr(allow),
                                                  words, A.ptr(s2), A.ptr(p2), None) == 0
        torch.cuda.synchronize()
        out[name] = (s, p, s2, p2)
    for a, b in zip(out["res"], out["st"]):
        assert A.same_bits(a, b) if a.is_floating_point() else torch.equal(a, b)
    L.flmr_comm_destroy(comm)
    res.close()
    st.close()


@pytest.mark.parametrize("aligned", [True, False])
def test_from_index_and_builder_streamed(R, tmp_path, aligned):
    """A flat index loaded with residency="host" (rows read straight into the pinned matrix; through the staging
    buffer when doclens are not multiples of 4), whole and as shards, searches bitwise like the same index loaded
    into HBM."""
    from ravqa_b200.maxsim import maxsim_topk
    tokens, dl = _rows(1500, seed=31)
    if aligned:
        dl = (dl + 3) // 4 * 4
        tokens = torch.cat([tokens, tokens])[:int(dl.sum())]
    path = str(tmp_path / "flat.idx")
    R.save_flat_index(path, tokens, dl)
    Q = _queries(7, 32, seed=2, dtype=torch.bfloat16)
    for rank, world in ((0, 1), (0, 2), (1, 2)):
        a = R.FlatCorpus.from_index(path, rank=rank, world_size=world)
        b = R.FlatCorpus.from_index(path, rank=rank, world_size=world, residency="host",
                                    window_bytes=_window_bytes_for(dl, 4))
        assert b.residency == "host" and b.pid_base == a.pid_base
        sa, pa = maxsim_topk(a, Q, 50)
        sb, pb = maxsim_topk(b, Q, 50)
        assert A.same_bits(sa, sb) and torch.equal(pa, pb)
        ga, _ = a.gather_padded(pa)
        gb, _ = b.gather_padded(pb)
        assert A.same_bits(ga, gb)
        a.close()
        b.close()


def _streamed_calls(L, st, B, nq, k, seed):
    """topk / scores / topk_allowed / gather on the streamed corpus as abi_contract Calls."""
    hq = C.c_void_p(st.handle.value)
    n = st.n_passages
    words = (n + 31) // 32
    calls = []

    def make(s):
        g = torch.Generator().manual_seed(s)
        q = torch.nn.functional.normalize(torch.randn(B, nq, DIM, generator=g), dim=-1).to(torch.bfloat16).cuda()
        allow = torch.randint(-2**31, 2**31 - 1, (B, words), generator=g, dtype=torch.int64).to(torch.int32).cuda()
        return {"q": q, "allow": allow}

    def topk(i, o, st_):
        return L.flmr_maxsim_topk(hq, ws, A.ptr(i["q"]), B, nq, k, 0, A.ptr(o["s"]), A.ptr(o["p"]), C.c_void_p(st_))

    def scores(i, o, st_):
        return L.flmr_maxsim_scores(hq, ws, A.ptr(i["q"]), B, nq, 0, A.ptr(o["s"]), C.c_void_p(st_))

    def allowed(i, o, st_):
        return L.flmr_maxsim_topk_allowed(hq, ws, A.ptr(i["q"]), B, nq, k, 0, A.ptr(i["allow"]), words, A.ptr(o["s"]),
                                          A.ptr(o["p"]), C.c_void_p(st_))
    ws = st.workspace()
    ins = make(seed)
    calls.append(A.Call("streamed topk", topk, {"q": ins["q"]}, {"s": ((B, k), torch.float32),
                                                                  "p": ((B, k), torch.int64)},
                        lambda s: {"q": make(s)["q"]}))
    calls.append(A.Call("streamed scores", scores, {"q": ins["q"]}, {"s": ((B, n), torch.float32)},
                        lambda s: {"q": make(s)["q"]}))
    calls.append(A.Call("streamed topk_allowed", allowed, ins, {"s": ((B, k), torch.float32),
                                                                "p": ((B, k), torch.int64)}, make))
    return calls


GATE_CYCLES = 100_000_000


def test_c_boundary_conventions(R, L):
    """Guard bands, a gated caller stream (the call returns before the gate opens and reads late inputs), an early
    consumer on another stream; and two threads with their own workspaces get bitwise the serial results."""
    tokens, dl = _rows(2500, seed=41)
    st = R.FlatCorpus(tokens, dl, pid_base=7, residency="host", window_bytes=_window_bytes_for(dl, 5))
    st.delete([7, 100, 2000])
    S = torch.cuda.Stream()
    for call in _streamed_calls(L, st, B=70, nq=32, k=16, seed=1):
        want = call.plain()
        A.guarded(call, want)
        r = A.gated(call, S, GATE_CYCLES, want, seed=5)
        assert not r.gate_done_at_return, call.name
        A.early_consumer(call, S, GATE_CYCLES, want)
    # the gather reads the mapped host rows
    pids = torch.arange(0, 60, dtype=torch.int64).cuda() * 41 + 3
    gcall = A.Call("streamed gather",
                   lambda i, o, s_: L.flmr_corpus_gather(st.handle, A.ptr(i["p"]), 60, 64, A.ptr(o["out"]),
                                                         A.ptr(o["mask"]), C.c_void_p(s_)),
                   {"p": pids}, {"out": ((60, 64, DIM), torch.bfloat16), "mask": ((60, 64), torch.uint8)},
                   lambda s: {"p": (torch.arange(0, 60, dtype=torch.int64) * 37 + s).cuda()})
    want = gcall.plain()
    A.guarded(gcall, want)
    assert not A.gated(gcall, S, GATE_CYCLES, want, seed=2).gate_done_at_return
    # two threads, own workspaces and streams, one shared corpus
    Qs = [_queries(20, 32, seed=60 + t, dtype=torch.bfloat16) for t in range(2)]
    serial = []
    for t in range(2):
        s = torch.empty((20, 10), dtype=torch.float32, device="cuda")
        p = torch.empty((20, 10), dtype=torch.int64, device="cuda")
        assert L.flmr_maxsim_topk(st.handle, st.workspace(), A.ptr(Qs[t]), 20, 32, 10, 0, A.ptr(s), A.ptr(p),
                                  None) == 0
        serial.append((s, p))
    torch.cuda.synchronize()
    got = [None, None]

    def worker(t):
        ws = C.c_void_p()
        assert L.flmr_workspace_create(st.handle, 8, 64, C.byref(ws)) == 0
        stream = torch.cuda.Stream()
        outs = []
        for _ in range(3):
            s = torch.empty((20, 10), dtype=torch.float32, device="cuda")
            p = torch.empty((20, 10), dtype=torch.int64, device="cuda")
            assert L.flmr_maxsim_topk(st.handle, ws, A.ptr(Qs[t]), 20, 32, 10, 0, A.ptr(s), A.ptr(p),
                                      C.c_void_p(stream.cuda_stream)) == 0
            outs.append((s, p))
        stream.synchronize()
        L.flmr_workspace_destroy(ws)
        got[t] = outs
    th = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    for t in range(2):
        for s, p in got[t]:
            assert A.same_bits(s, serial[t][0]) and torch.equal(p, serial[t][1])
    st.close()


def test_executor_lines_on_a_streamed_plaid_directory(R):
    """src/executors/FLMR_executor.py:774-792's Searcher lines on the reference-built PLAID directory opened with
    residency="host" (decoded on the GPU in bounded steps, copied into the pinned matrix): the same ids and scores as
    the resident run."""
    from ravqa_b200 import ColBERTConfig, Queries, Run, RunConfig, Searcher
    from ravqa_b200.plaid import plaid_to_flat, plaid_to_host_chunks
    z = np.load(os.path.join(GOLDEN_DIR, "callsites.npz"))
    ckpt = os.path.join(GOLDEN_DIR, "callsites", "ckpt")
    Qe = torch.from_numpy(z["queries"])
    qids = ["q%d" % i for i in range(Qe.shape[0])]
    k = int(z["k"])
    out = {}
    for residency in ("device", "host"):
        with Run().context(RunConfig(nranks=1, rank=0, root=ckpt, experiment="temp_index_0")):
            config = ColBERTConfig(total_visible_gpus=1)
            extra = {"residency": "host", "window_bytes": 64 * 1024} if residency == "host" else {}
            searcher = Searcher(index="temp_index.nbits=8", config=config, **extra)
            assert searcher.corpus.residency == residency
            queries = Queries(data={q: "question" for q in qids})
            out[residency] = (searcher._search_all_Q(queries, Qe, k=k).todict(),
                              [searcher.dense_search(Qe[i:i + 1], k=k, remove_zero_tensors=True)
                               for i in range(len(qids))])
            del searcher
    assert out["device"] == out["host"]
    with Run().context(RunConfig(nranks=1, rank=0, root=ckpt, experiment="temp_index_0")):
        with pytest.raises(ValueError, match="window_bytes"):
            Searcher(index="temp_index.nbits=8", config=ColBERTConfig(total_visible_gpus=1), window_bytes=1 << 20)
    # the bounded-step host decode is the one-shot GPU decode, row for row
    path = os.path.join(ckpt, "temp_index_0", "indexes", "temp_index.nbits=8")
    tokens, dl = plaid_to_flat(path)
    _dev, dl2, steps = plaid_to_host_chunks(path, rows_per_step=1000)
    host = torch.cat(list(steps))
    assert np.array_equal(dl, dl2) and A.same_bits(tokens.cpu(), host)


def test_plaid_shards_streamed(R):
    """from_plaid(residency="host") with world_size = 2: each rank's streamed shard is bitwise its resident shard."""
    from ravqa_b200.maxsim import maxsim_topk
    path = os.path.join(GOLDEN_DIR, "callsites", "ckpt", "temp_index_0", "indexes", "temp_index.nbits=8")
    Q = _queries(6, 32, seed=12, dtype=torch.bfloat16)
    for rank in range(2):
        a = R.FlatCorpus.from_plaid(path, rank=rank, world_size=2)
        b = R.FlatCorpus.from_plaid(path, rank=rank, world_size=2, residency="host", window_bytes=32 * 1024)
        assert b.residency == "host" and (a.pid_base, a.n_passages) == (b.pid_base, b.n_passages)
        k = min(20, a.n_passages)
        sa, pa = maxsim_topk(a, Q, k)
        sb, pb = maxsim_topk(b, Q, k)
        assert A.same_bits(sa, sb) and torch.equal(pa, pb)
        a.close()
        b.close()
