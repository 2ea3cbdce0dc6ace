"""Corpus updates on the GPU: a corpus grown by appends and thinned by deletes against one built in one go, every entry
point on deleted passages, ownership of an adopted matrix, ordering against searches already enqueued, and the Python
surface (IndexUpdater, filter_fn, the fp8 two-stage Searcher, persistence and sharded loading)."""
import numpy as np
import pytest
import torch

from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu

# scores of the same passage can differ between two partitions of the corpus: the reducer sums a passage's row
# partials in an order that depends on whether its end falls in one of a tile's first kFastSlots slots
TOL = {"bf16": dict(rtol=2e-5, atol=1e-6), "fp8": dict(rtol=1e-4, atol=1e-5)}


@pytest.fixture(scope="module")
def R():
    import ravqa_b200 as R
    return R


def _ragged(n, seed, lo=1, hi=61):
    rng = np.random.default_rng(seed)
    dl = rng.integers(lo, hi, size=n).astype(np.int32)
    dl[dl % 4 == 0] += 1                                  # not multiples of 4: padded rows on every passage
    D = rng.standard_normal((int(dl.sum()), 128), dtype=np.float32)
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    return torch.from_numpy(D).to(torch.bfloat16), dl


def _queries(B, nq, seed):
    Q, _, _ = O.synth(1, 4, B, nq, seed=seed)
    return torch.from_numpy(Q).to(torch.bfloat16).cuda()


def _grown(R, storage, sizes, seed, device_source=False):
    """Corpus A built from the first part and grown by appending the others; all tokens and doclens."""
    parts = [_ragged(n, seed + i) for i, n in enumerate(sizes)]
    A = R.FlatCorpus(parts[0][0], parts[0][1], storage=storage)
    first = parts[0][1].shape[0]
    for t, dl in parts[1:]:
        pids = A.append(t.cuda() if device_source else t, dl)
        assert pids.tolist() == list(range(first, first + dl.shape[0]))
        first += dl.shape[0]
    return A, torch.cat([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def _check_topk(s, p, ref_scores, dead, k, tol):
    """Top-k (s, p) of a corpus against the dense scores of a one-go corpus with the deleted columns at -inf."""
    ref = ref_scores.copy()
    ref[:, dead] = -np.inf
    n_live = ref.shape[1] - len(dead)
    for b in range(ref.shape[0]):
        order = np.lexsort((np.arange(ref.shape[1]), -ref[b]))[:min(k, n_live)]
        valid = p[b] >= 0
        assert valid.sum() == min(k, n_live)
        assert not np.isin(p[b][valid], dead).any()
        # every returned id's score is its true score, and the scores rank by rank are the reference's
        np.testing.assert_allclose(s[b][valid], ref[b][p[b][valid]], **tol)
        np.testing.assert_allclose(s[b][valid], ref[b][order], **tol)
        gap = np.abs(np.diff(ref[b][order])) if len(order) > 1 else np.array([])
        for i in range(len(order)):   # ids are identical wherever the neighbouring scores are separated
            near = (i > 0 and gap[i - 1] <= tol["rtol"] * abs(ref[b][order[i]]) + tol["atol"]) or \
                   (i < len(gap) and gap[i] <= tol["rtol"] * abs(ref[b][order[i]]) + tol["atol"])
            if not near:
                assert p[b][i] == order[i], (b, i)
        assert (p[b][~valid] == -1).all() and np.isneginf(s[b][~valid]).all()


@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_grown_corpus_matches_one_built_in_one_go(R, storage):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # 40 passages, two one-passage appends, then one that takes the corpus past the SM count (more CTAs than the
    # workspace was sized for), then a ragged tail
    A, toks, dl = _grown(R, storage, [40], seed=11)
    Q = _queries(4, 32, seed=5)
    R.maxsim_topk(A, Q, 5)                                 # the workspace is created while A is small
    parts = [_ragged(n, 12 + i) for i, n in enumerate([1, 1, sms + 100, 17])]
    for t, d in parts:
        A.append(t, d)
    toks = torch.cat([toks] + [t for t, _ in parts])
    dl = np.concatenate([dl] + [d for _, d in parts])
    assert A.info.n_ctas == sms and A.n_passages == dl.shape[0]
    rng = np.random.default_rng(3)
    dead = np.sort(rng.choice(dl.shape[0], size=dl.shape[0] // 10, replace=False))
    A.delete(dead)
    A.delete(dead[:3])                                     # already deleted: nothing changes
    assert A.n_deleted == len(dead) and A.n_live == dl.shape[0] - len(dead)
    assert np.array_equal(A.deleted_pids(), dead)
    B = R.FlatCorpus(toks, dl, storage=storage)
    tol = TOL[storage]
    sa = R.maxsim_scores(A, Q).cpu().numpy()
    sb = R.maxsim_scores(B, Q).cpu().numpy()
    assert np.isneginf(sa[:, dead]).all()
    live = np.setdiff1d(np.arange(dl.shape[0]), dead)
    np.testing.assert_allclose(sa[:, live], sb[:, live], **tol)
    for k in (1, 5, 128):
        s, p = R.maxsim_topk(A, Q, k)
        _check_topk(s.cpu().numpy(), p.cpu().numpy(), sb, dead, k, tol)
    # reruns on A are bit-identical
    s1, p1 = R.maxsim_topk(A, Q, 128)
    s2, p2 = R.maxsim_topk(A, Q, 128)
    assert torch.equal(s1, s2) and torch.equal(p1, p2)
    assert torch.equal(R.maxsim_scores(A, Q), R.maxsim_scores(A, Q))
    # k beyond the live count: short lists filled with -1 / -inf
    small, st, sdl = _grown(R, storage, [6, 3], seed=21)
    small.delete([0, 2, 7, 8])
    sbig = R.FlatCorpus(st, sdl, storage=storage)
    s, p = R.maxsim_topk(small, Q, 8)
    _check_topk(s.cpu().numpy(), p.cpu().numpy(), R.maxsim_scores(sbig, Q).cpu().numpy(), np.array([0, 2, 7, 8]), 8,
                tol)
    for c in (A, B, small, sbig):
        c.close()


def test_deleted_passages_at_every_entry_point(R):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    A, toks, dl = _grown(R, "bf16", [300, 120], seed=31, device_source=True)
    dead = np.arange(5, A.n_passages, 9)
    A.delete(dead)
    live = np.setdiff1d(np.arange(A.n_passages), dead)
    # row-sliced queries (Nq = 832: partial-score passes, then the final pass)
    Q = _queries(3, 832, seed=7)
    s = R.maxsim_scores(A, Q).cpu().numpy()
    simt = R.debug_scores_simt(A, Q).cpu().numpy()
    assert np.isneginf(s[:, dead]).all() and np.isneginf(simt[:, dead]).all()
    np.testing.assert_allclose(s[:, live], simt[:, live], rtol=1e-4, atol=1e-5)
    ts, tp = R.maxsim_topk(A, Q, 16)
    _check_topk(ts.cpu().numpy(), tp.cpu().numpy(), simt, dead, 16, dict(rtol=1e-4, atol=1e-5))
    # two- and three-warpgroup kernels (bit-identical to each other) and the CTA-pair kernel
    Q = _queries(4, 320, seed=8)
    out = {}
    try:
        for variant in (2, 3, 4):
            _cabi.check(L.flmr_debug_set_scan_variant(variant))
            out[variant] = (R.maxsim_scores(A, Q).cpu().numpy(), *[t.cpu().numpy() for t in R.maxsim_topk(A, Q, 10)])
    finally:
        L.flmr_debug_set_scan_variant(0)
    ref = R.debug_scores_simt(A, Q).cpu().numpy()
    for variant, (sc, ks, kp) in out.items():
        assert np.isneginf(sc[:, dead]).all(), variant
        np.testing.assert_allclose(sc[:, live], ref[:, live], rtol=1e-4, atol=1e-5)
        _check_topk(ks, kp, ref, dead, 10, dict(rtol=1e-4, atol=1e-5))
    assert np.array_equal(out[2][0], out[3][0]) and np.array_equal(out[2][2], out[3][2])
    # gather: a deleted id gives the all-masked zero row of an id outside the shard
    D, mask = A.gather_padded(torch.tensor([int(dead[0]), int(live[0]), -1]), 64)
    assert not mask[0].any() and not (D[0] != 0).any() and not mask[2].any()
    assert int(mask[1].sum()) == min(64, int(dl[live[0]]))
    A.close()


def test_adopted_matrix_is_not_read_after_the_first_append(R):
    rng = np.random.default_rng(41)
    dl = (rng.integers(1, 16, size=200) * 4).astype(np.int32)
    D = torch.randn(int(dl.sum()), 128, device="cuda").to(torch.bfloat16)
    D = torch.nn.functional.normalize(D.float(), dim=1).to(torch.bfloat16)
    A = R.FlatCorpus(D, dl)
    assert A.info.adopted == 1
    A.append(*_ragged(50, 42))
    assert A.info.adopted == 0 and A._keepalive is None
    Q = _queries(2, 64, seed=9)
    before = R.maxsim_scores(A, Q)
    ts, tp = R.maxsim_topk(A, Q, 20)
    D.fill_(1.0)                                            # the caller's buffer is theirs again
    torch.cuda.synchronize()
    assert torch.equal(R.maxsim_scores(A, Q), before)
    ts2, tp2 = R.maxsim_topk(A, Q, 20)
    assert torch.equal(ts, ts2) and torch.equal(tp, tp2)
    A.close()


@pytest.mark.parametrize("mutation", ["append", "delete"])
def test_search_enqueued_before_an_update_sees_the_corpus_as_it_was(R, mutation):
    A, _, _ = _grown(R, "bf16", [500], seed=51)
    Q = _queries(4, 64, seed=10)
    ref_s = R.maxsim_scores(A, Q)
    ref_ts, ref_tp = R.maxsim_topk(A, Q, 10)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                     # keeps the searches below queued while the update runs
        s = R.maxsim_scores(A, Q)
        ts, tp = R.maxsim_topk(A, Q, 10)
    if mutation == "append":
        A.append(*_ragged(200, 52))
    else:
        A.delete(ref_tp[:, 0].cpu().numpy())
    torch.cuda.synchronize()
    assert torch.equal(s, ref_s) and torch.equal(ts, ref_ts) and torch.equal(tp, ref_tp)
    A.close()


def test_delete_validates_the_whole_list_first(R):
    A, _, _ = _grown(R, "bf16", [20], seed=61)
    from ravqa_b200._cabi import FlmrError
    with pytest.raises(FlmrError):
        A.delete([3, 20])
    with pytest.raises(FlmrError):
        A.delete([-1])
    assert A.n_deleted == 0
    A.close()


def _collection_encoder(table):
    def encode(passages):
        embs = [table[p] for p in passages]
        return torch.cat(embs), [e.size(0) for e in embs]
    return encode


def _text_table(n, seed):
    rng = np.random.default_rng(seed)
    table = {}
    for i in range(n):
        t, _ = _ragged(1, int(rng.integers(1 << 30)), lo=8, hi=40)
        table["passage %d" % i] = t
    return table


@pytest.mark.parametrize("storage", ["bf16", "fp8"])
def test_index_updater_end_to_end(R, tmp_path, storage):
    table = _text_table(300, 71)
    Q = _queries(3, 32, seed=12)
    table["planted"] = Q[1].cpu()                          # scores highest for query 1
    enc = _collection_encoder(table)
    collection = ["passage %d" % i for i in range(250)]
    path = str(tmp_path / "idx")
    R.Indexer(encode_fn=enc, chunksize=100).index(path, collection, overwrite=True)
    searcher = R.Searcher(index=path, collection=list(collection), storage=storage)
    updater = R.IndexUpdater(searcher=searcher, encode_fn=enc)
    new = updater.add(["passage %d" % i for i in range(250, 300)] + ["planted"])
    assert new == list(range(250, 301)) and len(searcher.collection) == 301
    pids, _, _ = searcher.dense_search(Q[1:2], 5)
    assert pids[0] == 300
    updater.remove([300, 3, 260])
    pids, _, _ = searcher.dense_search(Q[1:2], 5)
    assert 300 not in pids
    seen = []

    def filt(p):
        seen.append(p.cpu().numpy())
        return p[p % 2 == 0]
    r = searcher._search_all_Q(None, Q, 10, filter_fn=filt)
    assert not np.isin(seen[0], [3, 260, 300]).any() and len(seen[0]) == 298
    assert all(pid % 2 == 0 and pid not in (260, 300) for hits in r.todict().values() for pid, _, _ in hits)
    assert r.provenance()["n_live"] == 298 and r.provenance()["n_deleted"] == 3
    # the two-stage fp8 search returns exact scores: it agrees with a bf16 searcher over the same updated corpus
    ref = R.Searcher(index=R.FlatCorpus(*_all_tokens(table, collection + ["passage %d" % i for i in range(250, 300)]
                                                      + ["planted"]), storage="bf16"))
    ref.corpus.delete([300, 3, 260])
    a, b = searcher._search_all_Q(None, Q, 10).todict(), ref._search_all_Q(None, Q, 10).todict()
    for q in a:
        assert [x[0] for x in a[q]] == [x[0] for x in b[q]]
        np.testing.assert_allclose([x[2] for x in a[q]], [x[2] for x in b[q]], rtol=2e-5)
    if storage == "fp8":
        assert searcher._last_depth == 256
    # persisted, a new Searcher reproduces the rankings; two shards honour the deletions
    meta = updater.persist_to_disk()
    assert meta["format"] == "flmr-flat-v2" and meta["n_passages"] == 301
    again = R.Searcher(index=path, storage=storage)
    assert again.corpus.n_live == 298
    c = again._search_all_Q(None, Q, 10).todict()
    for q in a:
        assert [x[0] for x in c[q]] == [x[0] for x in a[q]]
        np.testing.assert_allclose([x[2] for x in c[q]], [x[2] for x in a[q]], rtol=2e-5)
    shards = [R.FlatCorpus.from_index(path, rank=r, world_size=2, storage=storage) for r in range(2)]
    assert np.array_equal(np.concatenate([s.deleted_pids() for s in shards]), [3, 260, 300])
    merged = [R.maxsim_topk(s, Q, 10) for s in shards]
    ms, mp = R.topk_merge(torch.stack([m[0] for m in merged]), torch.stack([m[1] for m in merged]), 10)
    full_s, full_p = R.maxsim_topk(again.corpus, Q, 10)
    assert not np.isin(mp.cpu().numpy(), [3, 260, 300]).any()
    torch.testing.assert_close(ms, full_s, **TOL[storage])
    for s in shards:
        s.close()


def _all_tokens(table, names):
    embs = [table[n] for n in names]
    return torch.cat(embs), np.array([e.size(0) for e in embs], dtype=np.int32)


def test_persist_is_refused_for_plaid_and_sharded_updates_are_refused(R):
    from ravqa_b200 import IndexUpdater
    t, dl = _ragged(30, 81)
    s = R.Searcher(index=R.FlatCorpus(t, dl))
    u = IndexUpdater(searcher=s)
    u.add_embeddings(*_ragged(2, 82))
    with pytest.raises(ValueError):
        u.persist_to_disk()                                # a resident corpus has no index on disk
    s.index, s.index_kind = "/nonexistent", "plaid"
    with pytest.raises(NotImplementedError):
        u.persist_to_disk()
