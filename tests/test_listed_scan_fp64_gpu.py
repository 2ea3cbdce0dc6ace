"""GPU: the listed scan (``maxsim_scores_listed``, ``maxsim_topk(pids=)``: flmr_listed_plan_kernel and the plan-mode
scan kernels) against float64, over the grid of tests/listed_plan.py (pinned on CPU by tests/test_listed_plan_host.py,
which also shows that the grid reaches the planner's edges).  Each case's corpus is a ``FlatCorpus`` and a
``corpus_model.CorpusModel`` brought to one state (fresh, deletions, compacted, compacted then appended; pid_base 0 or
not), and every case checks

* the exact plan: ``debug_listed_plan`` of every call chunk equals the restatement element by element, within its
  tile bound;
* scores: each listed live entry within the scan bound of float64, ids outside the shard, deleted or compacted away
  exactly -inf, duplicates bitwise alike;
* top-k at k 1, 10, 128: a stable sort of the call's own listed scores (ties to the lower id, (-inf, -1) fill),
  certified by float64 over the query's listed live passages;
* the contract: bitwise the ``allow=`` calls for ``allow_bitmaps`` of the same lists.

Then the widest call, three chunks, the plan buffer regrowing across and within calls, and list offsets that do not
start at 0 through the C ABI.  The module prints the largest error / bound per storage at its end (run with -s)."""
import ctypes as C

import numpy as np
import pytest
import torch

import corpus_model as M
import listed_plan as LP
import scan_fp64 as S

pytestmark = pytest.mark.gpu

RATIOS = {}
GRID = LP.grid()
NEG = float("-inf")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[listed fp64] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[listed fp64]   %-24s %.3e" % (k, RATIOS[k]))


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


@pytest.fixture()
def scan_variant(R):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    yield lambda v: _cabi.check(L.flmr_debug_set_scan_variant(v))
    L.flmr_debug_set_scan_variant(0)


def _bits(x):
    return x.contiguous().view(torch.int32)


def _flat(lists):
    """(query of each entry, the concatenated ids) of per-query id lists."""
    lens = [len(x) for x in lists]
    q = np.repeat(np.arange(len(lists)), lens)
    ids = np.concatenate([np.asarray(x, np.int64) for x in lists]) if sum(lens) else np.zeros(0, np.int64)
    return q, ids


def _check_plan(R, corpus, sh, lists, nq, tag):
    from ravqa_b200.maxsim import debug_listed_plan
    want = LP.call_plan(lists, nq, sh)
    for ci, passes in enumerate(want):
        chunk = lists[ci * S.WS_QUERIES:(ci + 1) * S.WS_QUERIES]
        got = debug_listed_plan(corpus, len(chunk), nq, chunk)
        assert len(got) == len(passes), tag
        for pi, (g, w) in enumerate(zip(got, passes)):
            t = "%s chunk %d pass %d" % (tag, ci, pi)
            assert (g["q_first"], g["n_q"], g["n_ctas"], g["tile_bound"]) == (
                w["q_first"], w["n_q"], sh.n_ctas, w["tile_bound"]), t
            for key in ("slots", "cta_tile_base", "tile_row", "tile_mask", "tile_first"):
                assert np.array_equal(g[key], w[key]), "%s: %s differs" % (t, key)
            assert len(g["tile_row"]) <= g["tile_bound"], t


def _check_listed(R, corpus, m, Q, lists, relu, tag, ks=(1, 10, 128)):
    """Scores, top-k and the allow= contract of one listed call against the model."""
    st = m.storage
    B, nq = Q.size(0), Q.size(1)
    got = R.maxsim_scores_listed(corpus, Q, lists, relu=relu)
    s64, amax, rabs = m.scores(Q, relu=relu)
    bound = m.bound(amax, rabs, nq)
    q, ids = _flat(lists)
    local = ids - m.pid_base
    inside = (local >= 0) & (local < m.n_passages)
    live = inside.copy()
    live[inside] = ~m.deleted[local[inside]]
    qd, ld = torch.from_numpy(q).cuda(), torch.from_numpy(np.clip(local, 0, m.n_passages - 1)).cuda()
    lv = torch.from_numpy(live).cuda()
    assert got.numel() == ids.size, tag
    assert torch.isneginf(got[~lv]).all(), "%s: an id outside the shard, deleted or compacted away scores" % tag
    S.check_ratio(RATIOS, "scores " + st, (got[lv].double() - s64[qd[lv], ld[lv]]).abs(), bound[qd[lv], ld[lv]])
    dense = torch.full((B, m.n_passages), NEG, device="cuda")
    dense[qd[lv], ld[lv]] = got[lv]
    assert torch.equal(_bits(dense[qd[lv], ld[lv]]), _bits(got[lv])), "%s: duplicates score differently" % tag
    # the contract: bitwise the bitmap calls
    allow = corpus.allow_bitmaps(lists)
    full = R.maxsim_scores(corpus, Q, relu=relu, allow=allow)
    want = torch.where(torch.from_numpy(inside).cuda(), full[qd, ld], torch.tensor(NEG, device="cuda"))
    assert torch.equal(_bits(got), _bits(want)), "%s: listed scores differ from the allow= ones" % tag
    cands = [torch.from_numpy(np.unique(local[(q == b) & live])).cuda() for b in range(B)]
    for k in ks:
        ts, tp = R.maxsim_topk(corpus, Q, k, relu=relu, pids=lists)
        ws, wp = R.maxsim_topk(corpus, Q, k, relu=relu, allow=allow)
        assert torch.equal(tp, wp) and torch.equal(_bits(ts), _bits(ws)), "%s k=%d: differs from allow=" % (tag, k)
        for b in range(B):
            P = cands[b]
            S.check_topk_subset(dense[b, P], ts[b], tp[b], s64[b, P], bound[b, P], P, m.pid_base, k,
                                "%s k=%d" % (tag, k))


def _case_corpus(R, c, seed):
    """(FlatCorpus, model, Q on the GPU) of a grid case in its state."""
    Q, D, dl = S.case_data(dict(c, zeros="none"), seed)
    tokens = D.to(M.element_dtype(c["storage"]))
    m = M.CorpusModel(tokens.cuda(), dl, c["pid_base"], c["storage"])
    corpus = R.FlatCorpus(tokens, dl, device=0, pid_base=c["pid_base"], storage=c["storage"])
    LP.apply_state(m, corpus, c, seed)
    return corpus, m, Q.cuda()


@pytest.mark.parametrize("ci", range(len(GRID)), ids=lambda i: "c%03d" % i)
def test_listed_grid(R, scan_variant, ci):
    c = GRID[ci]
    seed = LP.case_seed(ci)
    tag = "case %d %s" % (ci, c)
    corpus, m, Q = _case_corpus(R, c, seed)
    try:
        sh = LP.Shard(m, sms=torch.cuda.get_device_properties(0).multi_processor_count)
        assert corpus.info.n_ctas == sh.n_ctas, tag
        lists = LP.case_lists(c, m, seed, sh)
        _check_plan(R, corpus, sh, lists, c["nq"], tag)
        scan_variant(c["variant"])
        _check_listed(R, corpus, m, Q, lists, c["relu"], tag)
    finally:
        scan_variant(0)
        corpus.close()


# ---- the plan buffer: one workspace through small, large and small plans ------------------------------------------
def _fresh_workspace(corpus):
    from ravqa_b200 import _cabi
    if corpus._ws is not None:
        _cabi.lib().flmr_workspace_destroy(corpus._ws)
        corpus._ws = None


def test_plan_buffer_regrows_across_and_within_calls(R):
    """One workspace plans small lists, then a three-chunk call whose second chunk needs a larger plan buffer than the
    first (regrown between two chunks of one call), then small lists again; every answer is bitwise that of a fresh
    workspace, and the float64 checks hold."""
    from helpers import placement_doclens
    dl = placement_doclens(3000, seed=21)
    tokens = M.passage_tokens(22, int(dl.sum()), "bf16")
    A = R.FlatCorpus(tokens, dl, device=0, pid_base=500)
    F = R.FlatCorpus(tokens, dl, device=0, pid_base=500)
    m = M.CorpusModel(tokens.cuda(), dl, 500, "bf16")
    try:
        rng = np.random.default_rng(3)
        everything = np.arange(500, 3500)
        small = lambda B: [500 + rng.choice(3000, 2) for _ in range(B)]
        big = small(64) + [everything] * 64 + small(2)
        for step, lists in enumerate((small(4), big, small(4), big[64:], small(70))):
            Q = M.query_rows(step, len(lists), 32, "bf16", "cuda")
            got = (R.maxsim_scores_listed(A, Q, lists), *R.maxsim_topk(A, Q, 10, pids=lists))
            _fresh_workspace(F)
            want = (R.maxsim_scores_listed(F, Q, lists), *R.maxsim_topk(F, Q, 10, pids=lists))
            assert torch.equal(_bits(got[0]), _bits(want[0])) and torch.equal(got[2], want[2]), step
            assert torch.equal(_bits(got[1]), _bits(want[1])), step
            _check_listed(R, A, m, Q, lists, False, "regrowth step %d" % step, ks=(10,))
    finally:
        A.close()
        F.close()


# ---- list offsets that start inside a larger id array (C ABI) ---------------------------------------------------------
def test_nonzero_first_list_offset(R):
    """``h_list_offsets[0] > 0``: entry i of the ids lands at index i of the output, across two call chunks; the
    output outside ``[h_off[0], h_off[n])`` keeps its sentinel, and top-k is that of the same lists from offset 0."""
    from ravqa_b200 import _cabi
    from ravqa_b200.maxsim import _prep_queries, _stream
    from helpers import placement_doclens
    dl = placement_doclens(2000, seed=23)
    c = R.FlatCorpus(M.passage_tokens(24, int(dl.sum()), "bf16"), dl, device=0, pid_base=100)
    try:
        rng = np.random.default_rng(5)
        B, nq, lead, tail = 70, 32, 7, 5
        lists = [100 + rng.choice(2100, int(rng.integers(0, 40))) - 50 for _ in range(B)]
        q, ids = _flat(lists)
        h_off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64) + lead
        pids = torch.from_numpy(np.concatenate([rng.integers(0, 2100, lead), ids, rng.integers(0, 2100, tail)])).cuda()
        Q = M.query_rows(6, B, nq, "bf16", "cuda")
        Qd = _prep_queries(c, Q)
        sentinel = 12345.5
        out = torch.full((lead + ids.size + tail,), sentinel, device="cuda")
        L = _cabi.lib()
        _cabi.check(L.flmr_maxsim_scores_listed(c.handle, c.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, 0,
                                                h_off.ctypes.data_as(C.c_void_p), C.c_void_p(pids.data_ptr()),
                                                C.c_void_p(out.data_ptr()), _stream(c)))
        want = R.maxsim_scores_listed(c, Q, lists)
        assert torch.equal(_bits(out[lead:lead + ids.size]), _bits(want))
        assert (out[:lead] == sentinel).all() and (out[lead + ids.size:] == sentinel).all()
        k = 10
        ts = torch.empty((B, k), device="cuda")
        tp = torch.empty((B, k), dtype=torch.int64, device="cuda")
        _cabi.check(L.flmr_maxsim_topk_listed(c.handle, c.workspace(), C.c_void_p(Qd.data_ptr()), B, nq, k, 0,
                                              h_off.ctypes.data_as(C.c_void_p), C.c_void_p(pids.data_ptr()),
                                              C.c_void_p(ts.data_ptr()), C.c_void_p(tp.data_ptr()), _stream(c)))
        ws, wp = R.maxsim_topk(c, Q, k, pids=lists)
        assert torch.equal(tp, wp) and torch.equal(_bits(ts), _bits(ws))
    finally:
        c.close()
