"""GPU: a PLAID-coded streamed corpus (FlatCorpus.from_plaid(residency="host", compressed=True): codes and residuals in
pinned host memory, each window copied and decoded on the GPU before the scan) returns BITWISE what the resident
from_plaid corpus of the same storage returns — scores, top-k, gather, Searcher — over the golden PLAID directories and
a pairwise covering of storage, nbits, relu, query length, batch, window count, shards, deletions, allow bitmaps and
builder splits; and keeps the streamed corpus's conventions, refusals and memory promise."""
from __future__ import annotations

import ctypes as C
import itertools
import json
import os
import threading

import numpy as np
import pytest
import torch

import abi_contract as A
import load_fp64 as LF
from helpers import GOLDEN_DIR

pytestmark = pytest.mark.gpu

DIM = 128
ROW = DIM * 2
INVALID = 1
UNSUPPORTED = 3
GATE_CYCLES = 100_000_000


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


def _queries(B, nq, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    q = torch.nn.functional.normalize(torch.randn(B, nq, DIM, generator=g), dim=-1)
    if nq > 3:
        q[:, -2:] = 0
    return q.to(dtype).cuda()


def _rows_of(dl):
    return (np.asarray(dl, np.int64) + 3) // 4 * 4


def _window_bytes_for(dl, n_windows):
    """The smallest window (whole 4-row groups) whose greedy plan has at most n_windows windows."""
    rows = _rows_of(dl)
    poff = np.concatenate([[0], np.cumsum(rows)])

    def count(wr):
        n, s0 = 0, 0
        while s0 < len(dl):
            s0 = int(np.searchsorted(poff, poff[s0] + wr, side="right")) - 1
            n += 1
        return n
    lo, hi = int(rows.max()), int(rows.sum())
    while lo < hi:
        mid = max(lo, (lo + hi) // 2 // 4 * 4)
        if count(mid) <= n_windows:
            hi = mid
        else:
            lo = mid + 4
    return hi * ROW


def _n_windows(L, dl, window_bytes):
    nw = C.c_int64()
    d = np.ascontiguousarray(dl, np.int32)
    assert L.flmr_debug_window_plan(d.ctypes.data, len(d), window_bytes, 132, None, 0, C.byref(nw), None, None, None,
                                    None, 0, None) == 0
    return nw.value


def _write_synthetic(path, nbits, n_passages, seed, n_chunks=2, n_centroids=300, lo=1, hi=120):
    """A PLAID directory of seeded random codes and residuals over normalised centroids, in n_chunks chunks."""
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    dl = rng.integers(lo, hi, size=n_passages)
    if hi - lo > 40:
        dl[rng.choice(n_passages, size=max(1, n_passages // 50), replace=False)] = 1
    centroids = torch.nn.functional.normalize(torch.randn(n_centroids, DIM, generator=g), dim=-1)
    weights = LF.fixture_weights(nbits, g)
    cuts = np.linspace(0, n_passages, n_chunks + 1).astype(int)
    chunks = []
    for c in range(n_chunks):
        d = dl[cuts[c]:cuts[c + 1]]
        codes, residuals = LF.random_codes(int(d.sum()), n_centroids, nbits, g)
        chunks.append((codes, residuals, d))
    LF.write_plaid(path, nbits, centroids, torch.zeros((1 << nbits) - 1), weights, chunks)
    return dl.astype(np.int32)


def _pair(R, path, storage, window_bytes, rank=0, world_size=1):
    res = R.FlatCorpus.from_plaid(path, rank=rank, world_size=world_size, storage=storage)
    cmp = R.FlatCorpus.from_plaid(path, rank=rank, world_size=world_size, storage=storage, residency="host",
                                  window_bytes=window_bytes, compressed=True)
    return res, cmp


def _check_all(R, res, cmp, Q, relu=False, allow=None, ks=(1, 10, 128), gather_seed=0):
    from ravqa_b200.maxsim import maxsim_scores, maxsim_topk
    kw = {} if allow is None else {"allow": allow}
    assert A.same_bits(maxsim_scores(res, Q, relu=relu, **kw), maxsim_scores(cmp, Q, relu=relu, **kw)), "scores"
    for k in ks:
        sa, pa = maxsim_topk(res, Q, k, relu=relu, **kw)
        sb, pb = maxsim_topk(cmp, Q, k, relu=relu, **kw)
        assert A.same_bits(sa, sb) and torch.equal(pa, pb), "top-%d" % k
    rng = np.random.default_rng(gather_seed)
    pids = torch.from_numpy(rng.integers(res.pid_base - 3, res.pid_base + res.n_passages + 3, size=(3, 29))).cuda()
    ga, ma = res.gather_padded(pids, nd_max=130)
    gb, mb = cmp.gather_padded(pids, nd_max=130)
    assert A.same_bits(ga, gb) and torch.equal(ma, mb), "gather"


# ---- the golden directories ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
@pytest.mark.parametrize("storage", ["bf16", "fp16"])
def test_golden_directories_bitwise(R, L, nbits, storage):
    from ravqa_b200.plaid import read_plaid_doclens, read_plaid_metadata
    path = os.path.join(GOLDEN_DIR, "plaid_nbits%d" % nbits)
    dl = np.concatenate(read_plaid_doclens(path, read_plaid_metadata(path)["num_chunks"]))
    wb = _window_bytes_for(dl, 3)
    res, cmp = _pair(R, path, storage, wb)
    assert cmp.codec_nbits == nbits and res.codec_nbits == 0
    assert cmp.residency == "host" and cmp.storage == storage
    info = cmp.residency_info()
    assert info == {"streamed": True, "window_bytes": wb, "host_bytes": int(_rows_of(dl).sum()) * (4 + 16 * nbits)}
    dtype = torch.float16 if storage == "fp16" else torch.bfloat16
    _check_all(R, res, cmp, _queries(5, 32, seed=nbits, dtype=dtype), gather_seed=nbits)
    res.close()
    cmp.close()


# ---- the pairwise covering ---------------------------------------------------------------------------------------------
# storage, nbits, relu, Nq, B, windows ("one-passage": a window per passage), shards (world_size, rank), deletions,
# allow bitmaps, builder split (rows per append_plaid call: whole chunks, or pieces that cut passages).  B = 70 exceeds
# the default workspace's 64 queries (two call chunks); Nq = 832 is row-sliced.
FACTORS = (("bf16", "fp16"), (1, 2, 4, 8), (False, True), (32, 320, 832), (1, 13, 70), (1, 2, 9, "one-passage"),
           ((1, 0), (2, 1), (3, 2)), ("none", "some", "window"), (False, True), ("chunks", "split"))
CASES = [
    ("bf16", 1, False, 32, 1, 1, (1, 0), "none", False, "chunks"),
    ("fp16", 2, True, 320, 13, 2, (2, 1), "some", True, "split"),
    ("bf16", 4, True, 832, 70, 9, (3, 2), "window", False, "split"),
    ("fp16", 8, False, 832, 1, "one-passage", (1, 0), "some", True, "chunks"),
    ("fp16", 1, True, 320, 70, "one-passage", (2, 1), "window", False, "chunks"),
    ("bf16", 2, False, 832, 13, 1, (3, 2), "window", True, "split"),
    ("bf16", 8, True, 32, 13, 9, (2, 1), "none", False, "split"),
    ("fp16", 4, False, 32, 70, 2, (3, 2), "none", True, "chunks"),
    ("bf16", 1, False, 320, 1, 9, (1, 0), "window", True, "split"),
    ("fp16", 2, True, 32, 1, "one-passage", (3, 2), "none", False, "split"),
    ("bf16", 4, False, 320, 1, 1, (2, 1), "some", False, "chunks"),
    ("fp16", 8, True, 320, 70, 2, (1, 0), "window", False, "split"),
    ("bf16", 2, True, 832, 70, 2, (1, 0), "some", False, "chunks"),
    ("fp16", 4, True, 832, 13, "one-passage", (1, 0), "none", True, "split"),
    ("bf16", 8, False, 832, 13, 9, (2, 1), "some", True, "chunks"),
    ("fp16", 1, False, 832, 13, 2, (3, 2), "some", False, "split"),
    ("bf16", 1, True, 32, 70, 1, (2, 1), "some", True, "chunks"),
    ("fp16", 2, False, 32, 70, 9, (1, 0), "window", True, "chunks"),
    ("bf16", 4, True, 32, 13, "one-passage", (3, 2), "some", False, "chunks"),
    ("fp16", 8, False, 32, 1, 1, (3, 2), "window", True, "split"),
    ("bf16", 8, True, 320, 1, "one-passage", (2, 1), "none", True, "chunks"),
    ("fp16", 4, False, 320, 13, 9, (1, 0), "none", False, "chunks"),
    ("bf16", 2, False, 320, 1, 2, (2, 1), "window", True, "chunks"),
    ("fp16", 1, True, 832, 1, 9, (2, 1), "none", True, "chunks"),
    ("fp16", 8, True, 32, 13, 2, (1, 0), "none", False, "chunks"),
    ("bf16", 1, False, 32, 13, "one-passage", (1, 0), "some", False, "split"),
    ("bf16", 4, True, 320, 70, 1, (1, 0), "window", True, "chunks"),
    ("fp16", 2, False, 320, 13, 1, (3, 2), "none", False, "chunks"),
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


@pytest.mark.parametrize("storage,nbits,relu,nq,B,windows,shard,dels,allow,split", CASES,
                         ids=["-".join(map(str, c)) for c in CASES])
def test_compressed_is_bitwise_resident(R, L, tmp_path, storage, nbits, relu, nq, B, windows, shard, dels, allow,
                                        split):
    from ravqa_b200 import _cabi
    from ravqa_b200.plaid import plaid_compressed_chunks
    from ravqa_b200.sharded import shard_ranges
    world, rank = shard
    n = 160 if windows == "one-passage" else (1500 if nq < 832 else 700)
    path = str(tmp_path / "plaid")
    dl_all = _write_synthetic(path, nbits, n, seed=nbits * 100 + nq + B)
    p0, p1 = shard_ranges(dl_all, world)[rank] if world > 1 else (0, n)
    dl = dl_all[p0:p1]
    wb = int(_rows_of(dl).max()) * ROW if windows == "one-passage" else _window_bytes_for(dl, windows)
    if split == "chunks":
        res, cmp = _pair(R, path, storage, wb, rank, world)
    else:   # the builder fed in pieces of 37 rows, which cut passages at arbitrary rows
        res = R.FlatCorpus.from_plaid(path, rank=rank, world_size=world, storage=storage)
        nb, cen, w, dl2, chunks = plaid_compressed_chunks(path, passage_range=(p0, p1))
        chunks = list(chunks)
        codes = torch.cat([c for c, _ in chunks])
        resid = torch.cat([r for _, r in chunks])

        def feed(Lb, b):
            for a in range(0, codes.numel(), 37):
                e = min(codes.numel(), a + 37)
                _cabi.check(Lb.flmr_corpus_builder_append_plaid(b, C.c_void_p(codes[a:].data_ptr()),
                                                                C.c_void_p(resid[a:].data_ptr()), e - a))
        flag = _cabi.CORPUS_FP16 if storage == "fp16" else 0
        cmp = R.FlatCorpus._build(np.ascontiguousarray(dl2, np.int32), res.device, p0, flag, "host", wb, feed,
                                  codec=(nb, cen, w))[0]
    assert cmp.pid_base == res.pid_base == p0 and cmp.n_passages == res.n_passages == len(dl)
    nw = _n_windows(L, dl, wb)
    if windows == "one-passage":
        assert nw >= len(dl) // 3
    else:
        assert nw == windows
    rng = np.random.default_rng(B + nq)
    if dels != "none":
        dead = rng.choice(len(dl), size=max(1, len(dl) // 10), replace=False)
        if dels == "window":   # a run of passages as long as a window's share
            a = len(dl) // 3
            dead = np.union1d(dead, np.arange(a, min(len(dl), a + max(1, len(dl) // max(nw, 2)))))
        for c in (res, cmp):
            c.delete(dead + p0)
    dtype = torch.float16 if storage == "fp16" else torch.bfloat16
    Q = _queries(B, nq, seed=B * 3 + nq, dtype=dtype)
    allow_t = None
    if allow:
        lists = [None if b % 3 == 0 else rng.choice(len(dl), size=len(dl) // 3, replace=False) + p0
                 for b in range(B)]
        allow_t = res.allow_bitmaps(lists)
    _check_all(R, res, cmp, Q, relu=relu, allow=allow_t, gather_seed=B)
    torch.cuda.synchronize()
    res.close()
    cmp.close()


# ---- gather ------------------------------------------------------------------------------------------------------------
def test_gather_cuts_masks_replays_and_matches_float64(R, L, tmp_path):
    """The gather's nd_max cut, deleted and out-of-shard ids, eager and as a CUDA-graph replay, bitwise the resident
    corpus's; and its rows within the rounding float64 allows of the decode."""
    path = str(tmp_path / "plaid")
    dl = _write_synthetic(path, 2, 400, seed=7)
    res, cmp = _pair(R, path, "bf16", _window_bytes_for(dl, 3), rank=1, world_size=2)
    p0, n = res.pid_base, res.n_passages
    for c in (res, cmp):
        c.delete([p0 + 1, p0 + 5])
    pids = torch.tensor([p0, p0 + 1, p0 + 2, p0 + 5, p0 - 1, p0 + n, p0 + n - 1, 3, p0 + 7], device="cuda")
    for nd_max in (1, 5, 130):
        ga, ma = res.gather_padded(pids, nd_max=nd_max)
        gb, mb = cmp.gather_padded(pids, nd_max=nd_max)
        assert A.same_bits(ga, gb) and torch.equal(ma, mb), nd_max
        assert not mb[1].any() and not mb[3].any() and not mb[4].any() and not mb[5].any()
        assert (gb[1] == 0).all() and (gb[4] == 0).all()
    # CUDA-graph capture and replay with new ids in the same buffer
    nd = 64
    ids = pids.clone()
    out = torch.empty((ids.numel(), nd, DIM), dtype=torch.bfloat16, device="cuda")
    mask = torch.empty((ids.numel(), nd), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        assert L.flmr_corpus_gather(cmp.handle, A.ptr(ids), ids.numel(), nd, A.ptr(out), A.ptr(mask),
                                    C.c_void_p(s.cuda_stream)) == 0
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert L.flmr_corpus_gather(cmp.handle, A.ptr(ids), ids.numel(), nd, A.ptr(out), A.ptr(mask),
                                    C.c_void_p(s.cuda_stream)) == 0
    new = torch.tensor([p0 + 3, p0 + 5, p0 + n + 9, p0 + 11, p0, p0 + 2, p0 + 1, p0 + 40, p0 + 41], device="cuda")
    ids.copy_(new)
    g.replay()
    torch.cuda.synchronize()
    want, wmask = res.gather_padded(new, nd_max=nd)
    assert A.same_bits(out, want) and torch.equal(mask.bool(), wmask.squeeze(-1))
    # against float64: every real row of every passage within check_rounding's band
    from ravqa_b200.plaid import plaid_compressed_chunks
    nbits, cen, w, dl2, chunks = plaid_compressed_chunks(path, passage_range=(p0, p0 + n))
    chunks = list(chunks)
    codes = torch.cat([c for c, _ in chunks])
    resid = torch.cat([r for _, r in chunks])
    y = LF.decode_fp64(codes, resid, cen, w, nbits)
    live = torch.arange(p0, p0 + n, device="cuda")
    got, m = cmp.gather_padded(live, nd_max=int(dl2.max()))
    got, m = got.cpu(), m.cpu().squeeze(-1)
    real = got[m]                              # [tokens of the live passages, 128] in passage order
    keep = np.ones(n, bool)
    keep[[1, 5]] = False
    off = np.concatenate([[0], np.cumsum(dl2)])
    sel = np.concatenate([np.arange(off[i], off[i + 1]) for i in range(n) if keep[i]])
    LF.check_rounding(real, y[torch.from_numpy(sel)], "gather")
    res.close()
    cmp.close()


# ---- Searcher paths ------------------------------------------------------------------------------------------------------
def test_searcher_paths_bitwise(R, tmp_path):
    """_search_all_Q, dense_search(pids=), filter_fn, k > 128 and retrieve_and_rescore: bitwise the resident ones."""
    path = str(tmp_path / "plaid")
    _write_synthetic(path, 4, 1200, seed=21)
    cfg = R.ColBERTConfig(total_visible_gpus=1)
    sr = R.Searcher(index=path, config=cfg)
    ss = R.Searcher(index=path, config=cfg, residency="host", window_bytes=96 * 1024, compressed=True)
    assert ss.corpus.codec_nbits == 4 and ss.residency == "host" and sr.corpus.codec_nbits == 0
    Q = _queries(90, 32, seed=9, dtype=torch.bfloat16).float().cpu()
    assert sr._search_all_Q(None, Q, k=20).todict() == ss._search_all_Q(None, Q, k=20).todict()
    assert sr._search_all_Q(None, Q[:5], k=200).todict() == ss._search_all_Q(None, Q[:5], k=200).todict()
    keep = torch.arange(0, 1200, 3)
    fa = sr._search_all_Q(None, Q[:7], k=10, filter_fn=lambda p: keep.to(p.device)).todict()
    fb = ss._search_all_Q(None, Q[:7], k=10, filter_fn=lambda p: keep.to(p.device)).todict()
    assert fa == fb
    pids = list(range(0, 1200, 7))
    for i in range(3):
        assert sr.dense_search(Q[i:i + 1], k=10, pids=pids) == ss.dense_search(Q[i:i + 1], k=10, pids=pids)
    Qg = Q[:6].to(torch.bfloat16).cuda()
    oa = sr.retrieve_and_rescore(Qg, 5, generator=torch.Generator(device="cpu").manual_seed(3))
    ob = ss.retrieve_and_rescore(Qg, 5, generator=torch.Generator(device="cpu").manual_seed(3))
    assert np.array_equal(oa["retrieved_doc_ids"], ob["retrieved_doc_ids"])
    for name in ("doc_scores", "search_scores", "item_embeddings"):
        assert A.same_bits(oa[name].detach(), ob[name].detach()), name
    assert torch.equal(oa["item_mask"], ob["item_mask"])
    # a Searcher refuses a compressed= that disagrees with the corpus it is given
    with pytest.raises(ValueError, match="compressed"):
        R.Searcher(index=sr.corpus, config=cfg, compressed=True)
    with pytest.raises(ValueError, match="compressed"):
        R.Searcher(index=ss.corpus, config=cfg, compressed=False)
    assert R.Searcher(index=ss.corpus, config=cfg, compressed=True).residency == "host"


def test_sharded_call_on_one_rank(R, L, tmp_path):
    """flmr_maxsim_topk_sharded(_allowed) on a one-rank communicator: bitwise the resident corpus's."""
    path = str(tmp_path / "plaid")
    dl = _write_synthetic(path, 2, 900, seed=61)
    res, cmp = _pair(R, path, "bf16", _window_bytes_for(dl, 3))
    uid = (C.c_char * 128)()
    assert L.flmr_comm_unique_id(C.cast(uid, C.c_void_p)) == 0
    comm = C.c_void_p()
    assert L.flmr_comm_create(C.cast(uid, C.c_void_p), 0, 1, 0, C.byref(comm)) == 0
    B, nq, k = 70, 32, 16
    Q = _queries(B, nq, seed=8, dtype=torch.bfloat16)
    allow = res.allow_bitmaps([np.arange(0, 800, 2)] * B)
    out = {}
    for name, c in (("res", res), ("cmp", cmp)):
        s = torch.empty((B, k), dtype=torch.float32, device="cuda")
        p = torch.empty((B, k), dtype=torch.int64, device="cuda")
        s2, p2 = torch.empty_like(s), torch.empty_like(p)
        assert L.flmr_maxsim_topk_sharded(c.handle, c.workspace(), comm, A.ptr(Q), B, nq, k, 0, A.ptr(s), A.ptr(p),
                                          None) == 0
        assert L.flmr_maxsim_topk_sharded_allowed(c.handle, c.workspace(), comm, A.ptr(Q), B, nq, k, 0, A.ptr(allow),
                                                  allow.size(1), A.ptr(s2), A.ptr(p2), None) == 0
        torch.cuda.synchronize()
        out[name] = (s, p, s2, p2)
    for a, b in zip(out["res"], out["cmp"]):
        assert A.same_bits(a, b) if a.is_floating_point() else torch.equal(a, b)
    L.flmr_comm_destroy(comm)
    res.close()
    cmp.close()


# ---- copies and memory ---------------------------------------------------------------------------------------------------
def _profiled_copies(path, window_bytes, trace):
    """Run in a child process: one maxsim_topk call on the compressed corpus of ``path`` under torch.profiler, its
    chrome trace written to ``trace``; prints whether it was bitwise the resident corpus's call."""
    import ravqa_b200 as R
    from torch.profiler import ProfilerActivity, profile
    from ravqa_b200.maxsim import maxsim_topk
    res, cmp = _pair(R, path, "bf16", window_bytes)
    Q = _queries(150, 32, seed=4, dtype=torch.bfloat16)
    want = maxsim_topk(res, Q, 10)
    maxsim_topk(cmp, Q, 10)                          # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        got = maxsim_topk(cmp, Q, 10)
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    print(json.dumps({"bitwise": bool(A.same_bits(want[0], got[0]) and torch.equal(want[1], got[1])),
                      "host_bytes": cmp.residency_info()["host_bytes"]}))


def test_each_window_is_copied_once_in_compressed_form(R, L, tmp_path):
    """Under torch.profiler, one call copies every window's codes and residuals once (two pinned host-to-device copies
    per window) and, in all, exactly the corpus's compressed bytes.  The profiled call runs in a child process, so this
    profiler session leaves no state behind for the profiled tests that run after it in this process."""
    import subprocess
    import sys
    from helpers import ROOT
    path = str(tmp_path / "plaid")
    dl = _write_synthetic(path, 2, 1500, seed=51)
    wb = _window_bytes_for(dl, 4)
    assert _n_windows(L, dl, wb) == 4
    trace = str(tmp_path / "trace.json")
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_plaid_streamed_gpu as T; T._profiled_copies(%r, %d, %r)"
            % (ROOT, tests_dir, path, wb, trace))
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    result = json.loads(out.stdout.strip().splitlines()[-1])
    assert result["bitwise"]
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    copies = [e for e in events if e.get("cat") == "gpu_memcpy" and "HtoD" in e.get("name", "")
              and "Pinned" in e.get("name", "")]
    assert len(copies) == 2 * 4, [e["name"] for e in copies]
    compressed = result["host_bytes"]
    assert compressed == int(_rows_of(dl).sum()) * (4 + 32)
    assert sum(int(e["args"]["bytes"]) for e in copies) == compressed


def test_workspace_device_memory(R, L, tmp_path):
    """A workspace of the compressed corpus adds one decoded window and two staging buffers of compressed rows: about
    one window less than a workspace of the bf16-streamed corpus of the same rows."""
    path = str(tmp_path / "plaid")
    dl = _write_synthetic(path, 2, 3000, seed=3, hi=180)
    wb = 8 << 20
    rows = int(_rows_of(dl).sum())
    cmp = R.FlatCorpus.from_plaid(path, residency="host", window_bytes=wb, compressed=True)
    st = R.FlatCorpus.from_plaid(path, residency="host", window_bytes=wb)
    assert _n_windows(L, dl, wb) >= 2
    assert cmp.residency_info()["host_bytes"] == rows * 36 and st.residency_info()["host_bytes"] == rows * ROW
    k_bytes = 300 * DIM * 4 + 4 * 4
    assert cmp.info.hbm_bytes == st.info.hbm_bytes + k_bytes

    def grown(c):
        torch.cuda.synchronize()
        free0, _ = torch.cuda.mem_get_info()
        ws = C.c_void_p()
        assert L.flmr_workspace_create(c.handle, 64, 1024, C.byref(ws)) == 0
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info()
        L.flmr_workspace_destroy(ws)
        return free0 - free1
    window_rows = wb // ROW
    g_cmp, g_st = grown(cmp), grown(st)
    # the two differ by one decoded window less and two staging buffers more (allocation granularity: 2 MiB each)
    want = window_rows * ROW - 2 * window_rows * 36
    assert abs((g_st - g_cmp) - want) <= 8 << 20, (g_st, g_cmp, want)
    cmp.close()
    st.close()


# ---- the C boundary ----------------------------------------------------------------------------------------------------
def test_threads_and_gated_stream(R, L, tmp_path):
    """A gated caller stream (the call returns before the gate opens and reads late inputs); two threads with their own
    workspaces get bitwise the serial results."""
    path = str(tmp_path / "plaid")
    dl = _write_synthetic(path, 4, 1500, seed=41)
    cmp = R.FlatCorpus.from_plaid(path, residency="host", window_bytes=_window_bytes_for(dl, 5), compressed=True)
    cmp.delete([7, 100, 1400])
    hq, B, nq, k = cmp.handle, 70, 32, 16
    ws = cmp.workspace()

    def make(s):
        g = torch.Generator().manual_seed(s)
        return {"q": torch.nn.functional.normalize(torch.randn(B, nq, DIM, generator=g), dim=-1)
                .to(torch.bfloat16).cuda()}
    call = A.Call("compressed topk",
                  lambda i, o, s_: L.flmr_maxsim_topk(hq, ws, A.ptr(i["q"]), B, nq, k, 0, A.ptr(o["s"]),
                                                      A.ptr(o["p"]), C.c_void_p(s_)),
                  make(1), {"s": ((B, k), torch.float32), "p": ((B, k), torch.int64)}, make)
    S = torch.cuda.Stream()
    want = call.plain()
    A.guarded(call, want)
    assert not A.gated(call, S, GATE_CYCLES, want, seed=5).gate_done_at_return
    A.early_consumer(call, S, GATE_CYCLES, want)
    Qs = [_queries(20, 32, seed=60 + t, dtype=torch.bfloat16) for t in range(2)]
    serial = []
    for t in range(2):
        s = torch.empty((20, 10), dtype=torch.float32, device="cuda")
        p = torch.empty((20, 10), dtype=torch.int64, device="cuda")
        assert L.flmr_maxsim_topk(hq, ws, A.ptr(Qs[t]), 20, 32, 10, 0, A.ptr(s), A.ptr(p), None) == 0
        serial.append((s, p))
    torch.cuda.synchronize()
    got = [None, None]

    def worker(t):
        w = C.c_void_p()
        assert L.flmr_workspace_create(hq, 8, 64, C.byref(w)) == 0
        stream = torch.cuda.Stream()
        outs = []
        for _ in range(3):
            s = torch.empty((20, 10), dtype=torch.float32, device="cuda")
            p = torch.empty((20, 10), dtype=torch.int64, device="cuda")
            assert L.flmr_maxsim_topk(hq, w, A.ptr(Qs[t]), 20, 32, 10, 0, A.ptr(s), A.ptr(p),
                                      C.c_void_p(stream.cuda_stream)) == 0
            outs.append((s, p))
        stream.synchronize()
        L.flmr_workspace_destroy(w)
        got[t] = outs
    th = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    for t in range(2):
        for s, p in got[t]:
            assert A.same_bits(s, serial[t][0]) and torch.equal(p, serial[t][1])
    cmp.close()


def test_refusals_leave_the_corpus_unchanged(R, L, tmp_path):
    from ravqa_b200 import _cabi
    from ravqa_b200.maxsim import debug_scores_simt, maxsim_scores_listed, maxsim_topk
    path = str(tmp_path / "plaid")
    dl = _write_synthetic(path, 2, 600, seed=11)
    res, cmp = _pair(R, path, "bf16", _window_bytes_for(dl, 3))
    Q = _queries(4, 32, seed=3, dtype=torch.bfloat16)
    before = maxsim_topk(cmp, Q, 20)
    info = bytes(cmp.info)
    # a bad code is refused at append, and nothing is stored
    cen = torch.nn.functional.normalize(torch.randn(10, DIM), dim=-1).contiguous()
    w = torch.linspace(-0.2, 0.2, 4).contiguous()
    d = np.array([3, 5], np.int32)
    b = C.c_void_p()
    assert L.flmr_corpus_builder_create_plaid(d.ctypes.data, 2, DIM, 0, 0, 0, 1 << 20, 2, A.ptr(cen), 10, A.ptr(w),
                                              C.byref(b)) == 0
    codes = torch.tensor([0, 1, 2, 10, 4, 5, 6, 7], dtype=torch.int32)
    resid = torch.zeros((8, 32), dtype=torch.uint8)
    assert L.flmr_corpus_builder_append_plaid(b, A.ptr(codes), A.ptr(resid), 8) == INVALID
    assert b"outside" in L.flmr_last_error()
    codes[3] = -1
    assert L.flmr_corpus_builder_append_plaid(b, A.ptr(codes), A.ptr(resid), 8) == INVALID
    codes[3] = 3
    tok = torch.zeros((8, DIM), dtype=torch.bfloat16)
    assert L.flmr_corpus_builder_append(b, A.ptr(tok), 8) == INVALID        # the wrong feed
    assert L.flmr_corpus_builder_append_plaid(b, A.ptr(codes), A.ptr(resid), 8) == 0
    h = C.c_void_p()
    assert L.flmr_corpus_builder_finish(b, C.byref(h), None) == 0
    nb = C.c_int(-1)
    assert L.flmr_corpus_codec(h, C.byref(nb)) == 0 and nb.value == 2
    L.flmr_corpus_destroy(h)
    assert L.flmr_corpus_codec(res.handle, C.byref(nb)) == 0 and nb.value == 0
    # append_plaid on another builder
    b = C.c_void_p()
    assert L.flmr_corpus_builder_create_streamed(d.ctypes.data, 2, DIM, 0, 0, 0, 1 << 20, C.byref(b)) == 0
    assert L.flmr_corpus_builder_append_plaid(b, A.ptr(codes), A.ptr(resid), 8) == INVALID
    L.flmr_corpus_builder_destroy(b)
    # refusals on the corpus: append, compact, listed calls, the SIMT kernel
    with pytest.raises(_cabi.FlmrError) as e:
        cmp.append(torch.zeros((3, DIM)), [3])
    assert e.value.code == UNSUPPORTED
    with pytest.raises(_cabi.FlmrError) as e:
        cmp.compact()
    assert e.value.code == UNSUPPORTED
    with pytest.raises(_cabi.FlmrError) as e:
        maxsim_scores_listed(cmp, Q, [[0, 1]] * 4)
    assert e.value.code == UNSUPPORTED
    with pytest.raises(_cabi.FlmrError) as e:
        debug_scores_simt(cmp, Q)
    assert e.value.code == UNSUPPORTED
    off = np.array([0, 2], np.int64)
    pl = torch.tensor([0, 1], device="cuda")
    n_out = C.c_int64()
    assert L.flmr_debug_listed_plan(cmp.handle, cmp.workspace(), 1, 32, off.ctypes.data, A.ptr(pl), None, 0,
                                    C.byref(n_out)) == UNSUPPORTED
    cmp._refresh()
    assert bytes(cmp.info) == info
    after = maxsim_topk(cmp, Q, 20)
    assert A.same_bits(before[0], after[0]) and torch.equal(before[1], after[1])
    want = maxsim_topk(res, Q, 20)
    assert A.same_bits(want[0], after[0]) and torch.equal(want[1], after[1])
    # the updater surfaces the refusals of add and compact, and remove works
    s = R.Searcher(index=cmp, config=R.ColBERTConfig(total_visible_gpus=1))
    up = R.IndexUpdater(config=None, searcher=s)
    with pytest.raises(_cabi.FlmrError):
        up.add_embeddings(torch.zeros((3, DIM)), [3])
    with pytest.raises(_cabi.FlmrError):
        up.compact()
    top = int(maxsim_topk(cmp, Q, 1)[1][0, 0])
    up.remove([top])
    assert top not in maxsim_topk(cmp, Q, 128)[1].cpu().numpy()
    res.close()
    cmp.close()
