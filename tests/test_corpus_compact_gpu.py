"""Corpus compaction on the GPU: every call on a compacted corpus returns bitwise what it returned before (and what a
fresh build of the live passages returns, ids mapped), for each storage, deletion pattern, query length and scan
variant; appends and deletes interleaved with compactions; an adopted matrix; the memory released; ordering against
searches already enqueued; the Searcher / IndexUpdater surface with persistence; and a 200k-passage corpus.
The module runs in about 20 s on an H100 80GB HBM3 (700 W)."""
import filecmp
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu

# scan variants each storage has (flmr_debug_set_scan_variant): 0 = the product's choice
VARIANTS = {"bf16": (0, 2, 3, 4, 6), "fp16": (0, 2, 6), "fp8": (0, 2, 3, 6)}
PIECE = 1 << 30        # largest physical allocation behind a token matrix


@pytest.fixture(scope="module")
def R():
    import ravqa_b200 as R
    return R


@pytest.fixture(scope="module")
def L():
    from ravqa_b200 import _cabi
    return _cabi.lib()


def _ragged(n, seed, lo=1, hi=61):
    """Ragged passages, lengths both multiples of 4 and not."""
    rng = np.random.default_rng(seed)
    dl = rng.integers(lo, hi, size=n).astype(np.int32)
    D = rng.standard_normal((int(dl.sum()), 128), dtype=np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    return torch.from_numpy(D), dl


def _queries(B, nq, seed, dtype):
    Q, _, _ = O.synth(1, 4, B, nq, seed=seed)
    return torch.from_numpy(Q).to(dtype).cuda()


def _bits(t):
    """The bit pattern of a tensor as a numpy array (floats compared bit for bit)."""
    if t.dtype in (torch.bfloat16, torch.float16):
        t = t.view(torch.int16)
    elif t.dtype == torch.float32:
        t = t.view(torch.int32)
    elif t.dtype == torch.bool:
        t = t.to(torch.uint8)
    return t.cpu().numpy()


def _stored(L, A):
    import ctypes as C
    n, mapped = C.c_int64(0), C.c_int64(0)
    assert L.flmr_corpus_stored(A.handle, C.byref(n), C.byref(mapped)) == 0
    return n.value, mapped.value


def _observe(R, L, A, storage, Qs, allow, variants, gather_ids):
    """Everything the tests compare, as bit patterns: {call name: array}."""
    out = {}
    try:
        for v in variants:
            assert L.flmr_debug_set_scan_variant(v) == 0
            for nq, Q in Qs.items():
                if v == 4 and nq != 320:
                    continue
                for k in (1, 10, 128):
                    s, p = R.maxsim_topk(A, Q, k)
                    out["topk", v, nq, k] = (_bits(s), _bits(p))
                out["scores", v, nq] = _bits(R.maxsim_scores(A, Q))
            Q = Qs[32]
            out["relu", v] = (_bits(R.maxsim_scores(A, Q, relu=True)), *map(_bits, R.maxsim_topk(A, Q, 10, relu=True)))
            for name, bm in allow.items():
                out["allow_scores", v, name] = _bits(R.maxsim_scores(A, Q, allow=bm))
                out["allow_topk", v, name] = tuple(map(_bits, R.maxsim_topk(A, Q, 10, allow=bm)))
    finally:
        L.flmr_debug_set_scan_variant(0)
    D, mask = A.gather_padded(gather_ids, 64)
    out["gather"] = (_bits(D), _bits(mask))
    out["simt"] = _bits(R.debug_scores_simt(A, Qs[32]))
    out["deleted"] = np.asarray(A.deleted_pids())
    return out


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for key in a:
        x, y = (a[key], b[key]) if isinstance(a[key], tuple) else ((a[key],), (b[key],))
        for u, w in zip(x, y):
            assert u.shape == w.shape and np.array_equal(u, w), key


def _setup(R, storage, n, seed, pid_base):
    t, dl = _ragged(n, seed)
    dtype = torch.float16 if storage == "fp16" else torch.bfloat16
    A = R.FlatCorpus(t.to(dtype), dl, pid_base=pid_base, storage=storage)
    Qs = {32: _queries(4, 32, seed + 1, dtype), 320: _queries(4, 320, seed + 2, dtype),
          832: _queries(3, 832, seed + 3, dtype)}
    rng = np.random.default_rng(seed + 4)
    lists = [pid_base + rng.choice(n, n // 3, replace=False) for _ in range(4)]
    allow = {"shared": A.allow_bitmaps([lists[0]])[0], "per_query": A.allow_bitmaps(lists)}
    ids = torch.cat([torch.arange(n) + pid_base, torch.tensor([-1, pid_base - 1, pid_base + n])])
    return A, t.to(dtype), dl, Qs, allow, ids


def _patterns(n, sms):
    rng = np.random.default_rng(5)
    return {
        "none": [],
        "first": [0],
        "last": [n - 1],
        "ends": [0, n - 1],
        "runs": list(range(40, 260)) + list(range(700, 705)) + list(range(1200, 1500)),
        "random_30": sorted(rng.choice(n, n * 3 // 10, replace=False).tolist()),
        "below_sms": sorted(set(range(n)) - set(rng.choice(n, sms // 2, replace=False).tolist())),
    }


@pytest.mark.parametrize("pattern", ["none", "first", "last", "ends", "runs", "random_30", "below_sms"])
@pytest.mark.parametrize("storage", ["bf16", "fp16", "fp8"])
def test_compacted_corpus_answers_bitwise_as_before(R, L, storage, pattern):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n, base = 1600, 1000
    A, toks, dl, Qs, allow, ids = _setup(R, storage, n, seed=101, pid_base=base)
    dead = np.asarray(_patterns(n, sms)[pattern], dtype=np.int64)
    if dead.size:
        A.delete(dead + base)
    before = _observe(R, L, A, storage, Qs, allow, VARIANTS[storage], ids)
    info0 = (A.info.n_passages, A.info.n_rows, A.info.n_tiles, A.info.hbm_bytes, A.info.n_ctas)
    stats = A.compact()
    assert stats["removed"] == dead.size and stats["rows_before"] == info0[1]
    if not dead.size:                                       # a no-op: the handle is unchanged
        assert (A.info.n_passages, A.info.n_rows, A.info.n_tiles, A.info.hbm_bytes, A.info.n_ctas) == info0
        assert stats["bytes_released"] == 0 and stats["rows_after"] == info0[1]
    live = np.setdiff1d(np.arange(n), dead)
    assert A.n_passages == n and A.n_stored == live.size and A.n_deleted == dead.size
    assert A.info.n_ctas == min(sms, live.size)
    if pattern == "below_sms":
        assert A.info.n_ctas < sms
    after = _observe(R, L, A, storage, Qs, allow, VARIANTS[storage], ids)
    _assert_same(before, after)
    # a fresh build of the live passages scores them bitwise alike, its ids mapped through the live list
    off = np.concatenate([[0], np.cumsum(dl)])
    F = R.FlatCorpus(torch.cat([toks[off[p]:off[p + 1]] for p in live]), dl[live], storage=storage)
    gid = torch.from_numpy(live + base).cuda()
    for nq, Q in Qs.items():
        s, p = R.maxsim_topk(F, Q, 128)
        mapped = torch.where(p >= 0, gid[p.clamp(min=0)], p)
        sa, pa = R.maxsim_topk(A, Q, 128)
        assert np.array_equal(_bits(s), _bits(sa)) and torch.equal(mapped, pa), nq
        assert np.array_equal(_bits(R.maxsim_scores(F, Q)), _bits(R.maxsim_scores(A, Q)[:, torch.from_numpy(live)]))
    assert (A.info.n_rows, A.info.n_tiles, A.info.n_tokens, A.info.n_ctas) == \
        (F.info.n_rows, F.info.n_tiles, F.info.n_tokens, F.info.n_ctas)
    # the stored corpus's HBM: the fresh build's, plus the slot -> id map once a compaction has run
    assert A.info.hbm_bytes == F.info.hbm_bytes + (8 * live.size if dead.size else 0)
    A.close()
    F.close()


def test_compact_append_delete_compact_again(R, L):
    n, base = 900, 50
    A, toks, dl, Qs, _, _ = _setup(R, "bf16", n, seed=201, pid_base=base)
    all_t, all_dl = [toks], [dl]
    dead = set(range(100, 300)) | {0}
    A.delete(np.array(sorted(dead)) + base)
    A.compact()
    t2, dl2 = _ragged(300, 202)
    ids = A.append(t2.to(torch.bfloat16), dl2)
    assert ids.tolist() == list(range(base + n, base + n + 300))      # ids continue from the id extent
    all_t.append(t2.to(torch.bfloat16))
    all_dl.append(dl2)
    from ravqa_b200._cabi import FlmrError
    with pytest.raises(FlmrError):
        A.delete([base + n + 300])                            # out of range: nothing changes
    assert A.n_deleted == len(dead)
    A.delete([base + 150, base + 0])                           # compacted-away ids: nothing changes
    assert A.n_deleted == len(dead) and A.n_stored == n + 300 - len(dead)
    more = {5, 6, 899, 900, 1000, 1199}
    A.delete(np.array(sorted(more)) + base)
    dead |= more
    toks_all, dl_all = torch.cat(all_t), np.concatenate(all_dl)
    live = np.setdiff1d(np.arange(n + 300), sorted(dead))
    off = np.concatenate([[0], np.cumsum(dl_all)])

    def fresh():
        return R.FlatCorpus(torch.cat([toks_all[off[p]:off[p + 1]] for p in live]), dl_all[live])

    def check(F):
        gid = torch.from_numpy(live + base).cuda()
        for nq in (32, 320, 832):
            s, p = R.maxsim_topk(F, Qs[nq], 128)
            sa, pa = R.maxsim_topk(A, Qs[nq], 128)
            assert np.array_equal(_bits(s), _bits(sa))
            assert torch.equal(torch.where(p >= 0, gid[p.clamp(min=0)], p), pa)
            sc = R.maxsim_scores(A, Qs[nq])
            assert np.array_equal(_bits(sc[:, torch.from_numpy(live)]), _bits(R.maxsim_scores(F, Qs[nq])))
            assert torch.isneginf(sc[:, torch.tensor(sorted(dead))]).all()
        D, m = A.gather_padded(torch.from_numpy(live + base), 64)
        Df, mf = F.gather_padded(torch.arange(live.size), 64)
        assert torch.equal(D, Df) and torch.equal(m, mf)
    F = fresh()
    check(F)                                                  # deletions after a compaction sit in the slot bitmap
    assert np.array_equal(A.deleted_pids(), np.array(sorted(dead)) + base)
    stats = A.compact()
    assert stats["removed"] == len(more) and A.n_stored == live.size
    check(F)
    assert A.compact()["removed"] == 0                        # nothing left to remove
    A.delete(live + base)                                     # every stored passage deleted: refused, nothing changes
    with pytest.raises(FlmrError):
        A.compact()
    assert A.n_stored == live.size
    A.close()
    F.close()


def test_adopted_matrix_is_never_written(R, L):
    rng = np.random.default_rng(301)
    dl = (rng.integers(1, 16, size=500) * 4).astype(np.int32)
    D = torch.nn.functional.normalize(torch.randn(int(dl.sum()), 128, device="cuda"), dim=1).to(torch.bfloat16)
    keep = D.clone()
    A = R.FlatCorpus(D, dl)
    assert A.info.adopted == 1
    assert _stored(L, A)[1] == 0                              # nothing of the library's is mapped behind it
    Q = _queries(4, 64, 302, torch.bfloat16)
    A.delete(np.arange(0, 500, 3))
    s0, (t0, p0) = R.maxsim_scores(A, Q), R.maxsim_topk(A, Q, 50)
    g0 = A.gather_padded(torch.arange(500), 64)
    stats = A.compact()
    torch.cuda.synchronize()
    assert torch.equal(D.view(torch.int16), keep.view(torch.int16))
    assert A.info.adopted == 0 and A._keepalive is None and stats["bytes_released"] == 0
    D.fill_(1.0)                                              # no longer referenced
    torch.cuda.synchronize()
    assert torch.equal(R.maxsim_scores(A, Q), s0)
    t1, p1 = R.maxsim_topk(A, Q, 50)
    assert torch.equal(t0, t1) and torch.equal(p0, p1)
    g1 = A.gather_padded(torch.arange(500), 64)
    assert torch.equal(g0[0], g1[0]) and torch.equal(g0[1], g1[1])
    A.close()


@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_search_enqueued_before_compact_sees_the_corpus_as_it_was(R, storage):
    A, _, _, Qs, _, _ = _setup(R, storage, 600, seed=401, pid_base=0)
    A.delete(np.arange(0, 600, 2))
    Q = Qs[32]
    ref_s = R.maxsim_scores(A, Q)
    ref_ts, ref_tp = R.maxsim_topk(A, Q, 10)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                        # keeps the searches below queued while compact runs
        s = R.maxsim_scores(A, Q)
        ts, tp = R.maxsim_topk(A, Q, 10)
    A.compact()
    torch.cuda.synchronize()
    assert torch.equal(s, ref_s) and torch.equal(ts, ref_ts) and torch.equal(tp, ref_tp)
    A.close()


def _text_table(n, seed):
    rng = np.random.default_rng(seed)
    return {"passage %d" % i: _ragged(1, int(rng.integers(1 << 30)), lo=8, hi=40)[0].to(torch.bfloat16)
            for i in range(n)}


@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_searcher_and_updater_rank_alike_and_persist_the_same_index(R, tmp_path, storage):
    table = _text_table(400, 501)

    def enc(passages):
        embs = [table[p] for p in passages]
        return torch.cat(embs), [e.size(0) for e in embs]
    Q = _queries(6, 32, 502, torch.bfloat16)
    collection = ["passage %d" % i for i in range(300)]
    paths = [str(tmp_path / "a"), str(tmp_path / "b")]
    R.Indexer(encode_fn=enc, chunksize=100).index(paths[0], collection, overwrite=True)
    shutil.copytree(paths[0], paths[1])
    results = []
    for i, path in enumerate(paths):
        searcher = R.Searcher(index=path, collection=list(collection), storage=storage)
        updater = R.IndexUpdater(searcher=searcher, encode_fn=enc)
        updater.add(["passage %d" % j for j in range(300, 400)])
        updater.remove(list(range(0, 400, 4)) + [301, 302])
        before = searcher._search_all_Q(None, Q, 20).todict()
        if i == 0:
            stats = updater.compact()
            assert stats["removed"] == 102 and searcher.corpus.n_stored == 298
        after = searcher._search_all_Q(None, Q, 20).todict()
        assert after == before
        updater.persist_to_disk()
        results.append(after)
    assert results[0] == results[1]
    ranked = {q: [(h[0], h[2]) for h in hits] for q, hits in results[0].items()}
    # the compacted corpus persisted byte for byte what the uncompacted one did
    names = sorted(os.listdir(paths[0]))
    assert names == sorted(os.listdir(paths[1]))
    match, mismatch, errors = filecmp.cmpfiles(paths[0], paths[1], names, shallow=False)
    assert not mismatch and not errors
    again = R.Searcher(index=paths[0], storage=storage)
    assert {q: [(h[0], h[2]) for h in hits] for q, hits in again._search_all_Q(None, Q, 20).todict().items()} == ranked


def test_200k_passages_top100_bitwise_and_memory_released(R, L):
    rng = np.random.default_rng(601)
    n = 200_000
    dl = rng.integers(60, 181, size=n).astype(np.int32)
    g = torch.Generator(device="cuda").manual_seed(602)
    D = torch.randn(int(dl.sum()), 128, device="cuda", generator=g, dtype=torch.bfloat16).mul_(128 ** -0.5)
    A = R.FlatCorpus(D, dl, adopt=False)
    del D
    Q = _queries(16, 320, 603, torch.bfloat16)
    dead = np.sort(rng.choice(n, n * 3 // 10, replace=False))
    A.delete(dead)
    s0, p0 = R.maxsim_topk(A, Q, 100)
    _, mapped0 = _stored(L, A)
    stats = A.compact()
    s1, p1 = R.maxsim_topk(A, Q, 100)
    assert np.array_equal(_bits(s0), _bits(s1)) and torch.equal(p0, p1)
    live = np.setdiff1d(np.arange(n), dead)
    need = int(((dl[live] + 3) // 4 * 4).sum()) * 128 * 2
    n_stored, mapped1 = _stored(L, A)
    assert n_stored == live.size and A.info.n_rows * 256 == need and stats["rows_after"] == A.info.n_rows
    assert stats["bytes_released"] == mapped0 - mapped1 > 0
    assert need <= mapped1 < need + PIECE                     # at most one piece stays partly used
    A.close()
