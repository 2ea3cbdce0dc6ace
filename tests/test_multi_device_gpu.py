"""GPU: a Searcher whose shards one process holds on several devices (``Searcher(devices=...)``) returns BITWISE the
ids and scores of the one-device Searcher on the same index — every search form, flat and PLAID indexes, bf16, fp16
and fp8 storage, shard boundaries inside a run of long passages, equal scores planted in different shards — and its
merge, ``flmr_topk_merge_devices``, equals ``flmr_topk_merge`` on its three read paths (in place, peer reads, staged
copy), writes only its output and orders itself after busy source streams without blocking the host.

``devices=[0, 0]`` and ``[0, 0, 0]`` (several shards on one GPU) run on any GPU; ``[0, 1]`` and every visible device
need at least two."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest
import torch

import abi_contract as A
from helpers import GOLDEN_DIR

pytestmark = pytest.mark.gpu

DIM = 128
N_GPUS = torch.cuda.device_count() if torch.cuda.is_available() else 0
TWO_GPUS = pytest.mark.skipif(N_GPUS < 2, reason="needs at least two GPUs")
DEVICE_SETS = [pytest.param([0, 0], id="0-0"), pytest.param([0, 0, 0], id="0-0-0"),
               pytest.param([0, 1], id="0-1", marks=TWO_GPUS), pytest.param("all", id="all", marks=TWO_GPUS)]
# two copies of the same passage, in different shards for every device set above
TIE_A, TIE_B = 7, 231


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


def _ragged():
    """240 passages: short ones around a run of long ones that holds the token-balanced shard boundaries of 2 and 3
    shards."""
    rng = np.random.default_rng(11)
    dl = rng.integers(1, 31, size=240).astype(np.int32)
    dl[90:150] = rng.integers(120, 181, size=60)
    dl[TIE_B] = dl[TIE_A]
    g = torch.Generator().manual_seed(3)
    D = torch.nn.functional.normalize(torch.randn(int(dl.sum()), DIM, generator=g), dim=-1)
    off = np.concatenate([[0], np.cumsum(dl)])
    D[off[TIE_B]:off[TIE_B + 1]] = D[off[TIE_A]:off[TIE_A + 1]]
    return D.to(torch.bfloat16), dl


@pytest.fixture(scope="module")
def flat_index(R, tmp_path_factory):
    D, dl = _ragged()
    path = str(tmp_path_factory.mktemp("multi") / "flat")
    R.save_flat_index(path, D, dl)
    return path, D, dl


def _index(kind, flat_index):
    return flat_index[0] if kind == "flat" else os.path.join(GOLDEN_DIR, "plaid_nbits2")


def _queries(B, nq, seed, zero_rows=True):
    g = torch.Generator().manual_seed(seed)
    q = torch.nn.functional.normalize(torch.randn(B, nq, DIM, generator=g), dim=-1)
    if zero_rows:
        q[:, -3:] = 0
    return q.to(torch.bfloat16).cuda()


def _same(a, b, tag):
    sa, pa = a
    sb, pb = b
    assert sa.device == pa.device and sa.device.index == sb.device.index, tag
    assert torch.equal(pa.cpu(), pb.cpu()), "%s: ids differ" % tag
    assert torch.equal(sa.cpu().view(torch.int32), sb.cpu().view(torch.int32)), "%s: scores differ" % tag


def _lists(n, n_index, seed):
    rng = np.random.default_rng(seed)
    return [None if b % 4 == 3 else rng.choice(n_index, size=int(rng.integers(1, min(60, n_index) + 1)), replace=False)
            for b in range(n)]


@pytest.mark.parametrize("devices", DEVICE_SETS)
@pytest.mark.parametrize("kind,storage", [("flat", None), ("flat", "fp16"), ("flat", "fp8"), ("plaid", None),
                                          ("plaid", "fp16"), ("plaid", "fp8")])
def test_every_search_form_matches_the_one_device_searcher(R, flat_index, kind, storage, devices):
    path = _index(kind, flat_index)
    kw = {} if storage is None else {"storage": storage}
    one = R.Searcher(index=path, **kw)
    many = R.Searcher(index=path, devices=devices, **kw)
    n_dev = N_GPUS if devices == "all" else len(devices)
    assert len(many.shards) == min(n_dev, one.corpus.n_passages) and many.corpus is many.shards[0]
    assert many.storage == one.storage and many.device == torch.device("cuda", 0 if devices == "all" else devices[0])
    assert [c.pid_base for c in many.shards] == [a for a, _ in R.shard_ranges(one.corpus.doclens, n_dev)][:len(many.shards)]
    n = one.corpus.n_passages
    Q = _queries(9, 32, seed=5)
    lists = _lists(9, n, seed=6)
    keep = (lambda pids: pids[pids % 3 != 0])
    for k in (1, 5, 100, 200):
        tag = "%s/%s/%s/k=%d" % (kind, storage, devices, k)
        _same(one._search_tensors(Q, k), many._search_tensors(Q, k), tag)
        _same(one._search_tensors(Q, k, remove_zero_tensors=True), many._search_tensors(Q, k, remove_zero_tensors=True),
              tag + "/remove_zero_tensors")
        _same(one._search_tensors(Q, k, filter_fn=keep), many._search_tensors(Q, k, filter_fn=keep), tag + "/filter_fn")
        _same(one._search_tensors(Q, k, pid_lists=lists), many._search_tensors(Q, k, pid_lists=lists), tag + "/pids")
        _same(one._search_tensors(Q, k, filter_fn=keep, pid_lists=lists),
              many._search_tensors(Q, k, filter_fn=keep, pid_lists=lists), tag + "/pids+filter_fn")
        for b in (0, 3):
            ids = lists[b]
            assert one.dense_search(Q[b:b + 1], k) == many.dense_search(Q[b:b + 1], k), tag
            assert one.dense_search(Q[b:b + 1], k, pids=ids) == many.dense_search(Q[b:b + 1], k, pids=ids), tag
            assert one.dense_search(Q[b:b + 1], k, filter_fn=keep) == many.dense_search(Q[b:b + 1], k,
                                                                                       filter_fn=keep), tag
        qids = ["q%d" % b for b in range(9)]
        r1 = one._search_all_Q(qids, Q, k, qid_to_pids=dict(zip(qids, lists)))
        r2 = many._search_all_Q(qids, Q, k, qid_to_pids=dict(zip(qids, lists)))
        assert r1.todict() == r2.todict(), tag
        assert one._search_all_Q(qids, Q, k).todict() == many._search_all_Q(qids, Q, k).todict(), tag
    Qr = Q[:4].float().requires_grad_(True)
    for n_docs in (3, 5):
        a = one.retrieve_and_rescore(Qr, n_docs, generator=torch.Generator().manual_seed(1))
        b = many.retrieve_and_rescore(Qr, n_docs, generator=torch.Generator().manual_seed(1))
        assert np.array_equal(a["retrieved_doc_ids"], b["retrieved_doc_ids"])
        for key in ("doc_scores", "search_scores", "item_embeddings", "item_mask"):
            assert torch.equal(a[key].detach().cpu(), b[key].detach().cpu()), key
        assert b["doc_scores"].device == many.device
        b["doc_scores"].sum().backward()
        assert Qr.grad is not None and Qr.grad.abs().sum() > 0
        Qr.grad = None


@pytest.mark.parametrize("devices", DEVICE_SETS)
def test_equal_scores_in_different_shards_rank_the_lower_id_first(R, flat_index, devices):
    path, D, dl = flat_index
    off = np.concatenate([[0], np.cumsum(dl)])
    many = R.Searcher(index=path, devices=devices)
    owner = [next(i for i, c in enumerate(many.shards) if c.pid_base <= p < c.pid_base + c.n_passages)
             for p in (TIE_A, TIE_B)]
    assert owner[0] != owner[1]
    Q = D[off[TIE_A]:off[TIE_A + 1]][None].cuda()        # the planted passage itself: the two copies tie at the top
    s, p = many._search_tensors(Q, 5)
    assert p[0, :2].tolist() == [TIE_A, TIE_B] and s[0, 0].item() == s[0, 1].item()
    _same(R.Searcher(index=path)._search_tensors(Q, 5), (s, p), "ties")


# ---- the merge kernel ---------------------------------------------------------------------------------------------
def _merge_case(n_lists, B, k_in, seed):
    """Seeded lists: scores from a small set (exact ties across lists), -0.0, -inf, and empty (pid -1) entries; every
    query has fewer live entries than n_lists * k_in."""
    g = torch.Generator().manual_seed(seed)
    s = (torch.randint(0, 6, (n_lists, B, k_in), generator=g).float() * 0.5 - 1.0)
    s[torch.rand(s.shape, generator=g) < 0.05] = -0.0
    s[torch.rand(s.shape, generator=g) < 0.05] = float("-inf")
    p = torch.randint(0, 10_000, (n_lists, B, k_in), generator=g)
    p[torch.rand(p.shape, generator=g) < 0.3] = -1
    p[:, 0, :] = -1                                        # a query with nothing to merge
    return s, p


def _merge(L, lists, k_out, out_s, out_p, stream, src_streams):
    n = len(lists)
    B, k_in = lists[0][0].shape
    rc = L.flmr_topk_merge_devices((C.c_void_p * n)(*[s.data_ptr() for s, _ in lists]),
                                   (C.c_void_p * n)(*[p.data_ptr() for _, p in lists]),
                                   (C.c_int * n)(*[s.device.index for s, _ in lists]),
                                   (C.c_void_p * n)(*[st.cuda_stream for st in src_streams]), n, B, k_in, k_out,
                                   C.c_void_p(out_s.data_ptr()), C.c_void_p(out_p.data_ptr()),
                                   C.c_void_p(stream.cuda_stream))
    return rc


@pytest.mark.parametrize("path", [pytest.param("in_place", id="in_place"),
                                  pytest.param("peer", id="peer", marks=TWO_GPUS),
                                  pytest.param("staged", id="staged")])
@pytest.mark.parametrize("n_lists,B,k_in,k_out", [(1, 3, 5, 5), (2, 17, 128, 128), (3, 5, 40, 100),
                                                   (8, 9, 128, 128)])
def test_merge_equals_topk_merge(R, L, path, n_lists, B, k_in, k_out):
    s, p = _merge_case(n_lists, B, k_in, seed=n_lists * 131 + k_in)
    want_s, want_p = R.topk_merge(s.cuda(), p.cuda(), k_out)
    devs = [(i % 2 if path == "peer" else 0) for i in range(n_lists)]
    lists = [(s[i].to(f"cuda:{d}"), p[i].to(f"cuda:{d}")) for i, d in enumerate(devs)]
    torch.cuda.synchronize()
    gs, gp = A.Guarded((B, k_out), torch.float32), A.Guarded((B, k_out), torch.int64)
    S = torch.cuda.current_stream(0)
    srcs = [torch.cuda.current_stream(d) for d in devs]
    L.flmr_launch_count(1)
    try:
        if path == "staged":
            assert L.flmr_debug_set_merge_path(1) == 0
        assert _merge(L, lists, k_out, gs.out, gp.out, S, srcs) == 0, L.flmr_last_error()
    finally:
        L.flmr_debug_set_merge_path(0)
    assert L.flmr_launch_count(1) == 1
    torch.cuda.synchronize()
    gs.check(tag="scores")
    gp.check(tag="pids")
    assert torch.equal(gp.out.cpu(), want_p.cpu())
    assert torch.equal(gs.out.cpu().view(torch.int32), want_s.cpu().view(torch.int32))
    assert (gp.out[0] == -1).all() and torch.isinf(gs.out[0]).all()


@pytest.mark.parametrize("n_lists,k_in", [(20, 1024), (128, 160)])
def test_merge_at_full_capacity(R, L, n_lists, k_in):
    """The kernel's capacity: n_lists * k_in = 20480 candidates per query, as long lists or as the most lists."""
    s, p = _merge_case(n_lists, 3, k_in, seed=9)
    want = R.topk_merge(s.cuda(), p.cuda(), 128)
    lists = [(s[i].cuda(), p[i].cuda()) for i in range(n_lists)]
    out_s = torch.empty((3, 128), device="cuda")
    out_p = torch.empty((3, 128), dtype=torch.int64, device="cuda")
    S = torch.cuda.current_stream()
    assert _merge(L, lists, 128, out_s, out_p, S, [S] * n_lists) == 0, L.flmr_last_error()
    assert torch.equal(out_p.cpu(), want[1].cpu())
    assert torch.equal(out_s.cpu().view(torch.int32), want[0].cpu().view(torch.int32))


def test_merge_waits_for_busy_source_streams_and_never_blocks_the_host(R, L):
    """Lists written late on two busy source streams, the merge on a third non-default stream: its result is that of
    the finished lists (it waited for both streams' events), the call returned while a source stream was still busy,
    and it launched one kernel."""
    n_lists, B, k_in, k_out = 2, 7, 64, 64
    s, p = _merge_case(n_lists, B, k_in, seed=21)
    want = R.topk_merge(s.cuda(), p.cuda(), k_out)
    srcs = [torch.cuda.Stream(), torch.cuda.Stream()]
    S = torch.cuda.Stream()
    lists = [(torch.zeros(B, k_in, device="cuda"), torch.full((B, k_in), 5, dtype=torch.int64, device="cuda"))
             for _ in range(n_lists)]                   # decoys until the source streams write the real lists
    real = [(s[i].cuda(), p[i].cuda()) for i in range(n_lists)]
    torch.cuda.synchronize()
    gates = [A.gate(st, 50_000_000 * (i + 1)) for i, st in enumerate(srcs)]
    for st, (ds, dp), (rs, rp) in zip(srcs, lists, real):
        with torch.cuda.stream(st):
            ds.copy_(rs)
            dp.copy_(rp)
    out_s = torch.empty((B, k_out), device="cuda")
    out_p = torch.empty((B, k_out), dtype=torch.int64, device="cuda")
    L.flmr_launch_count(1)
    assert _merge(L, lists, k_out, out_s, out_p, S, srcs) == 0, L.flmr_last_error()
    busy_at_return = not gates[1].query()
    assert L.flmr_launch_count(1) == 1
    S.synchronize()
    assert busy_at_return
    assert torch.equal(out_p.cpu(), want[1].cpu()) and torch.equal(out_s.cpu(), want[0].cpu())


@pytest.mark.parametrize("devices", DEVICE_SETS)
def test_searcher_on_a_busy_non_default_stream(R, flat_index, devices):
    """A multi-device search issued on a non-default stream that is still busy: each shard's stream is ordered after
    it, so the queries it writes late are the ones searched."""
    path = flat_index[0]
    one = R.Searcher(index=path)
    many = R.Searcher(index=path, devices=devices)
    Q = _queries(6, 32, seed=8)
    want = one._search_tensors(Q, 20)
    S = torch.cuda.Stream()
    late = torch.zeros_like(Q)
    torch.cuda.synchronize()
    A.gate(S, 50_000_000)
    with torch.cuda.stream(S):
        late.copy_(Q)
        got = many._search_tensors(late, 20)
    torch.cuda.synchronize()
    _same(want, got, "busy stream %s" % devices)
