"""GPU: seeded sequences of appends, deletions and compactions applied to a ``FlatCorpus`` and to the float64 model of
tests/corpus_model.py (pinned on CPU by tests/test_corpus_lifecycle_host.py), with every observable call checked after
every operation:

1. bookkeeping (counts, deleted and live ids, ``n_ctas``) equal to the model;
2. ``maxsim_scores`` at Nq 32 and 320 (every fourth state also Nq 832 and relu) within the scan bound of float64, deleted
   and compacted-away ids exactly -inf;
3. ``maxsim_topk`` at k 1 / 10 / 128: a stable sort of the kernel's own scores, certified by float64 over the live ids;
4. allow bitmaps (shared and per query) naming deleted, compacted-away, newly appended and out-of-shard ids: disallowed
   ids -inf, allowed ones bitwise the unrestricted scores, top-k certified over allowed and live ids; a bitmap built
   before an append never admits a passage it did not name;
5. ``gather_padded`` of every id ever issued, ``pid_base - 1`` and one past the end: bitwise the model's rows;
6. the SIMT cross-check within its rigorous bound;
7. ``Searcher`` at k 200 (select kernel) and 3000 (sort) certified by float64; on fp8 the exact re-rank's scores within
   the arg-max bound of their bf16 float64 scores, and no passage surely better than the k-th and surely inside the
   shortlist left out;
   the listed scan (``maxsim_scores_listed``, ``maxsim_topk(pids=)`` at k 10 / 128) on the lists of 4, at Nq 32 and,
   every fourth state, 320: -inf wherever the model has no live passage, within the scan bound elsewhere, bitwise the
   allow observations, top-k certified over each query's listed live ids; and a restricted ``Searcher`` (k 200) on
   its listed and on its bitmap path: bitwise alike, certified (fp8: the re-rank held as above) per query;
8. every call repeated gives bitwise the same answer, and every observation right after a compaction (effective, no-op
   or refused) is bitwise what it was just before.

A failing sequence prints its seed and operation log; ``replay(spec, ops)`` runs a logged sequence again.  The module
prints the largest error / bound per check and the number of operations at its end (run with -s)."""
import json

import numpy as np
import pytest
import torch

import corpus_model as M
import scan_fp64 as S
from train_fp64 import C_BOUND, U

pytestmark = pytest.mark.gpu

RATIOS = {}
COUNT = {"ops": 0, "sequences": 0}
PIECE = 1 << 30            # largest physical allocation behind a token matrix
HEAVY_EVERY = 4            # states between the Nq 832 / relu checks


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[corpus lifecycle] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[corpus lifecycle]   %-28s %.3e" % (k, RATIOS[k]))
    print("[corpus lifecycle] %d operations in %d sequences" % (COUNT["ops"], COUNT["sequences"]))


def _lib():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


def _eq(a, b):
    """Bitwise equality of two tensors (floats compared by bit pattern)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype in (torch.float32, torch.float16, torch.bfloat16):
        w = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}[a.dtype]
        return torch.equal(a.view(w), b.view(w))
    return torch.equal(a, b)


def _same(a: dict, b: dict, tag):
    assert a.keys() == b.keys(), tag
    for key in a:
        x, y = a[key], b[key]
        x, y = (x, y) if isinstance(x, tuple) else ((x,), (y,))
        for u, w in zip(x, y):
            assert _eq(u, w), "%s: %s differs" % (tag, key)


_positions = S.positions


SEARCHER_LISTED_K = 200     # a restricted Searcher's k: past the fused top-k, through the select kernel


def _ranking_tensors(rk, B, k):
    """A Ranking's dict (qid -> [(pid, rank, score)]) as (scores, pids) ``[B, k]``, padded with (-inf, -1)."""
    s = torch.full((B, k), -torch.inf, device="cuda")
    p = torch.full((B, k), -1, dtype=torch.int64, device="cuda")
    for b in range(B):
        hits = rk.get(b, [])
        if hits:
            p[b, :len(hits)] = torch.tensor([h[0] for h in hits])
            s[b, :len(hits)] = torch.tensor([h[2] for h in hits], dtype=torch.float32)
    return s, p


def _same_pair(a, b):
    return _eq(a[0], b[0]) and _eq(a[1], b[1])


def _pad(s, p, k):
    B = s.size(0)
    return (torch.cat([s, s.new_full((B, k - s.size(1)), -torch.inf)], 1),
            torch.cat([p, p.new_full((B, k - p.size(1)), -1)], 1))


class Sequence:
    """One corpus, its model and the inputs its observations use."""

    def __init__(self, R, spec, route="corpus", tmp_path=None):
        self.R, self.spec = R, spec
        self.storage, self.pid_base = spec["storage"], spec["pid_base"]
        self.route = route
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.log = []
        lens0 = np.asarray(spec["lens0"], np.int64)
        src = "cuda" if spec["src0"] == "gpu" else "cpu"
        t0 = M.passage_tokens(spec["seed"], int(lens0.sum()), self.storage, src)
        self.m = M.CorpusModel(t0.cuda(), lens0, self.pid_base, self.storage)
        if route == "corpus":
            self.A = R.FlatCorpus(t0, lens0, device=0, pid_base=self.pid_base, adopt=spec["adopt"],
                                  storage=self.storage)
            assert self.A.info.adopted == int(spec["adopt"])
            self.updater = None
        else:                                  # an index written by Indexer, updated through Searcher + IndexUpdater
            self.table = {}
            names = self._texts(spec["seed"], t0, lens0)
            self.path = str(tmp_path / ("index_%d" % spec["seed"]))
            R.Indexer(encode_fn=self._encode, chunksize=100, storage=self.storage).index(self.path, names,
                                                                                        overwrite=True)
            self.searcher = R.Searcher(index=self.path, collection=list(names))
            self.A = self.searcher.corpus
            assert self.A.storage == self.storage and self.A.pid_base == 0
            self.updater = R.IndexUpdater(searcher=self.searcher, encode_fn=self._encode)
        del t0
        g = torch.Generator().manual_seed(spec["seed"] + 1)
        self.Q = {nq: M.query_rows(int(torch.randint(1 << 30, (1,), generator=g)), B, nq, self.storage, "cuda")
                  for nq, B in ((32, 5), (320, 2), (832, 1))}
        self.rng = np.random.default_rng(spec["seed"] + 2)
        self.state = 0
        self.inp = self._inputs()
        self.obs = None

    # -- the updater route: texts stand for token rows ------------------------------------------------------------
    def _texts(self, seed, tokens, lens):
        off = np.concatenate([[0], np.cumsum(lens)])
        names = []
        for i in range(lens.size):
            name = "s%d p%d" % (seed, i)
            self.table[name] = tokens[off[i]:off[i + 1]].cpu()
            names.append(name)
        return names

    def _encode(self, passages):
        embs = [self.table[p] for p in passages]
        return torch.cat(embs), [e.size(0) for e in embs]

    # -- operations ---------------------------------------------------------------------------------------------
    def apply(self, op):
        from ravqa_b200._cabi import FlmrError
        A, m = self.A, self.m
        kind = op["op"]
        prev = self.obs
        if kind == "append":
            lens = np.asarray(op["lens"], np.int64)
            t = M.passage_tokens(op["seed"], int(lens.sum()), self.storage, "cuda" if op["src"] == "gpu" else "cpu")
            stale_lists = self.inp["lists"]
            stale = A.allow_bitmaps(stale_lists)
            mapped0 = self._mapped()
            if self.updater is not None:
                ids = np.asarray(self.updater.add(self._texts(op["seed"], t, lens)))
            else:
                ids = A.append(t, lens)
            assert np.array_equal(ids, m.append(t, lens)), "append returned other ids"
            self._check_stale(stale, stale_lists)
            assert self._mapped() >= mapped0 and A.info.adopted == 0
        elif kind == "delete":
            ids = np.asarray(op["ids"], np.int64)
            if op["expect"] == "error":
                with pytest.raises(FlmrError):
                    self.updater.remove(ids) if self.updater is not None else A.delete(ids)
                with pytest.raises(M.ModelError):
                    m.delete(ids)
            else:
                self.updater.remove(ids) if self.updater is not None else A.delete(ids)
                m.delete(ids)
        else:
            mapped0, adopted0 = self._mapped(), A.info.adopted
            if op["expect"] == "error":
                with pytest.raises(FlmrError):
                    self.updater.compact() if self.updater is not None else A.compact()
                with pytest.raises(M.ModelError):
                    m.compact()
                stats = {"removed": 0, "bytes_released": 0}
            else:
                stats = self.updater.compact() if self.updater is not None else A.compact()
                assert stats["removed"] == m.compact(), "compaction removed another number of passages"
            # physical memory released: what is no longer mapped (an adopted matrix is copied, nothing released)
            assert stats["bytes_released"] == (0 if adopted0 else mapped0 - self._mapped())
            self.last_compact = stats
        COUNT["ops"] += 1
        self.state += 1
        if kind != "compact":
            self.inp = self._inputs()
        self.obs = self.observe()
        if kind == "compact":
            _same(prev, self.obs, "observations around a compaction")
        self.check()

    def _mapped(self):
        import ctypes as C
        from ravqa_b200 import _cabi
        n, mapped = C.c_int64(0), C.c_int64(0)
        _cabi.check(_cabi.lib().flmr_corpus_stored(self.A.handle, C.byref(n), C.byref(mapped)))
        return mapped.value

    def _check_stale(self, stale, lists):
        """A bitmap built before the append: refused when the word count changed, else the new passages stay out."""
        words = (self.A.n_passages + 31) // 32
        if stale.size(1) != words:
            with pytest.raises(ValueError):
                self.R.maxsim_scores(self.A, self.Q[32], allow=stale)
            return
        got = self.R.maxsim_scores(self.A, self.Q[32], allow=stale)
        named = torch.zeros_like(got, dtype=torch.bool)
        for b, ids in enumerate(lists):
            local = np.asarray(ids, np.int64) - self.pid_base
            local = local[(local >= 0) & (local < self.A.n_passages)]
            named[b, torch.from_numpy(local).cuda()] = True
        assert torch.isneginf(got[~named]).all(), "a bitmap built before an append admits a passage it did not name"

    # -- observations -------------------------------------------------------------------------------------------
    def _inputs(self):
        m, rng = self.m, self.rng
        pools = [m.deleted_ids(), m.compacted_ids(), m.new_ids(), m.live_ids()]
        lists = []
        for _ in range(self.Q[32].size(0)):
            parts = [rng.choice(p, min(p.size, int(rng.integers(1, 40))), replace=False) for p in pools if p.size]
            parts.append(np.array([m.pid_base - 1, m.pid_base + m.n_passages], np.int64))
            lists.append(np.concatenate(parts))
        ids = np.arange(m.pid_base - 1, m.pid_base + m.n_passages + 1)
        if ids.size > 4000:       # the large sequence: a sample, ends included
            ids = np.unique(np.concatenate([ids[:2], ids[-2:], rng.choice(ids, 4000, replace=False)]))
        local = np.clip(ids - m.pid_base, 0, m.n_passages - 1)
        return {"lists": lists, "heavy": self.state % HEAVY_EVERY == 0, "gather": ids,
                "nd_max": int(m.lens[local].max())}

    def _searcher_lists(self):
        """inp["lists"] without the ids a Searcher refuses (below 0, or past the index)."""
        end = self.m.pid_base + self.m.n_passages
        return [ids[(ids >= 0) & (ids < end)] for ids in self.inp["lists"]]

    def _listed_sets(self, lists):
        """(query of each entry, local id of each entry clipped into the shard, live mask of the entries, the sorted
        live local ids of each query) of per-query id lists."""
        m = self.m
        q = np.repeat(np.arange(len(lists)), [len(x) for x in lists])
        local = np.concatenate(lists).astype(np.int64) - m.pid_base
        live = (local >= 0) & (local < m.n_passages)
        live[live] = ~m.deleted[local[live]]
        sets = [torch.from_numpy(np.unique(local[(q == b) & live])).cuda() for b in range(len(lists))]
        return (torch.from_numpy(q).cuda(), torch.from_numpy(np.clip(local, 0, m.n_passages - 1)).cuda(),
                torch.from_numpy(live).cuda(), sets)

    def _searcher(self):
        return self.searcher if self.updater is not None else self.R.Searcher(index=self.A)

    def observe(self):
        R, A, Q, inp = self.R, self.A, self.Q, self.inp
        out = {}
        nqs = (32, 320, 832) if inp["heavy"] else (32, 320)
        for nq in nqs:
            out["scores", nq] = R.maxsim_scores(A, Q[nq])
            for k in (1, 10, 128):
                out["topk", nq, k] = R.maxsim_topk(A, Q[nq], k)
        if inp["heavy"]:
            out["relu"] = R.maxsim_scores(A, Q[32], relu=True)
            out["relu topk"] = R.maxsim_topk(A, Q[32], 128, relu=True)
        bms = {"shared": A.allow_bitmaps(inp["lists"][:1])[0], "per query": A.allow_bitmaps(inp["lists"])}
        for name, bm in bms.items():
            out["allow", name] = R.maxsim_scores(A, Q[32], allow=bm)
            for k in (10, 128):
                out["allow topk", name, k] = R.maxsim_topk(A, Q[32], k, allow=bm)
        for nq in ((32, 320) if inp["heavy"] else (32,)):     # the listed scan on the same lists
            lists = inp["lists"][:Q[nq].size(0)]
            out["listed", nq] = R.maxsim_scores_listed(A, Q[nq], lists)
            for k in (10, 128):
                out["listed topk", nq, k] = R.maxsim_topk(A, Q[nq], k, pids=lists)
        out["gather"] = A.gather_padded(torch.from_numpy(inp["gather"]), inp["nd_max"])
        out["simt"] = R.debug_scores_simt(A, Q[32])
        sr = self._searcher()
        for k in ((200,) if self.storage == "fp8" else (200, 3000)):
            out["searcher", k] = sr._search_tensors(Q[32], k)
        if self.storage == "fp8":      # the shortlist depth (none when no passage is live)
            out["depth"] = torch.tensor([sr._last_depth if self.A.n_live else 0])
        # a restricted Searcher on the listed scan and on the bitmap scan
        import ravqa_b200.searcher as SR
        q2p = dict(enumerate(self._searcher_lists()))
        keep = SR.LISTED_SCAN_MAX_ROW_FRACTION
        try:
            for path, frac in (("listed", float("inf")), ("bitmap", -1.0)):
                SR.LISTED_SCAN_MAX_ROW_FRACTION = frac
                sr._last_depth = 0
                rk = sr._search_all_Q(list(q2p), Q[32], SEARCHER_LISTED_K, qid_to_pids=q2p).todict()
                out["searcher listed", path] = _ranking_tensors(rk, len(q2p), SEARCHER_LISTED_K)
                if self.storage == "fp8":
                    out["depth listed", path] = torch.tensor([sr._last_depth])
        finally:
            SR.LISTED_SCAN_MAX_ROW_FRACTION = keep
        # the same calls again: bitwise the same answers
        assert _eq(R.maxsim_scores(A, Q[32]), out["scores", 32]), "scores differ on a second call"
        again = R.maxsim_topk(A, Q[32], 10)
        assert _eq(again[0], out["topk", 32, 10][0]) and _eq(again[1], out["topk", 32, 10][1]), "top-k differs"
        again = R.maxsim_scores(A, Q[32], allow=bms["per query"])
        assert _eq(again, out["allow", "per query"]), "allowed scores differ on a second call"
        return out

    # -- checks against the model -------------------------------------------------------------------------------
    def check(self):
        A, m, obs, inp = self.A, self.m, self.obs, self.inp
        st = self.storage
        # 1. bookkeeping
        assert (A.n_passages, A.n_deleted, A.n_live, A.n_stored) == (m.n_passages, m.n_deleted, m.n_live,
                                                                      m.n_stored), "counts"
        assert np.array_equal(A.deleted_pids(), m.deleted_ids()), "deleted ids"
        assert np.array_equal(A.live_pids().cpu().numpy(), m.live_ids()), "live ids"
        assert A.info.n_ctas == min(self.sms, m.n_stored), "n_ctas"
        live = torch.from_numpy(~m.deleted).cuda()
        P = torch.from_numpy(np.flatnonzero(~m.deleted)).cuda()
        model = {}
        for key in [k for k in obs if k[0] == "scores"]:
            nq = key[1]
            s64, amax, rabs = m.scores(self.Q[nq])
            model[nq] = (s64, m.bound(amax, rabs, nq), amax, rabs)
        # 2. scores
        for nq, (s64, bound, _, _) in model.items():
            got = obs["scores", nq]
            S.check_ratio(RATIOS, "scores %s" % st, (got[:, live].double() - s64[:, live]).abs(), bound[:, live])
            assert torch.isneginf(got[:, ~live]).all(), "a deleted id scores"
            # 3. fused top-k over the live ids
            for k in (1, 10, 128):
                ts, tp = obs["topk", nq, k]
                S.check_topk(got[:, P], ts, _positions(tp, P, m.pid_base), s64[:, P], bound[:, P], k,
                             "top-k nq=%d k=%d" % (nq, k))
        if inp["heavy"]:
            s64, amax, rabs = m.scores(self.Q[32], relu=True)
            bound = m.bound(amax, rabs, 32)
            got = obs["relu"]
            S.check_ratio(RATIOS, "relu %s" % st, (got[:, live].double() - s64[:, live]).abs(), bound[:, live])
            assert torch.isneginf(got[:, ~live]).all()
            ts, tp = obs["relu topk"]
            S.check_topk(got[:, P], ts, _positions(tp, P, m.pid_base), s64[:, P], bound[:, P], 128, "relu top-k")
        # 4. allow bitmaps
        s64, bound = model[32][:2]
        plain = obs["scores", 32]
        for name in ("shared", "per query"):
            lists = inp["lists"][:1] * 5 if name == "shared" else inp["lists"]
            got = obs["allow", name]
            for b, ids in enumerate(lists):
                local = np.asarray(ids, np.int64) - m.pid_base
                local = np.unique(local[(local >= 0) & (local < m.n_passages)])
                Pb = torch.from_numpy(local[~m.deleted[local]]).cuda()
                ok = torch.zeros(m.n_passages, dtype=torch.bool, device="cuda")
                ok[Pb] = True
                assert torch.isneginf(got[b][~ok]).all(), "%s: a disallowed or deleted id scores" % name
                assert _eq(got[b][ok], plain[b][ok]), "%s: allowed scores differ from unrestricted ones" % name
                for k in (10, 128):
                    ts, tp = obs["allow topk", name, k]
                    S.check_topk(got[b:b + 1, Pb], ts[b:b + 1], _positions(tp[b:b + 1], Pb, m.pid_base),
                                 s64[b:b + 1, Pb], bound[b:b + 1, Pb], k, "allow %s k=%d" % (name, k))
        # 4b. the listed scan: within the bound where the model has a live passage, -inf elsewhere, bitwise the allow
        # observations (allowed scores are bitwise the unrestricted ones); top-k certified over the listed live ids
        for nq in [key[1] for key in obs if key[0] == "listed"]:
            lists = inp["lists"][:self.Q[nq].size(0)]
            q, local, lv, sets = self._listed_sets(lists)
            s64, bound = model[nq][:2]
            got = obs["listed", nq]
            assert torch.isneginf(got[~lv]).all(), "listed: an id without a live passage scores"
            S.check_ratio(RATIOS, "listed %s" % st, (got[lv].double() - s64[q[lv], local[lv]]).abs(),
                          bound[q[lv], local[lv]])
            ref = obs["allow", "per query"] if nq == 32 else obs["scores", nq]
            assert _eq(got[lv], ref[q[lv], local[lv]]), "listed scores differ from the allow observations"
            dense = torch.full_like(ref, -torch.inf)
            dense[q[lv], local[lv]] = got[lv]
            for k in (10, 128):
                ts, tp = obs["listed topk", nq, k]
                if nq == 32:
                    ws, wp = obs["allow topk", "per query", k]
                    assert _eq(ts, ws) and _eq(tp, wp), "listed top-k differs from the allow observation"
                for b, Pb in enumerate(sets):
                    S.check_topk_subset(dense[b, Pb], ts[b], tp[b], s64[b, Pb], bound[b, Pb], Pb, m.pid_base, k,
                                        "listed nq=%d k=%d" % (nq, k))
        # the restricted Searcher: both paths alike, certified over each query's listed live ids
        s64, bound = model[32][:2]
        assert _same_pair(obs["searcher listed", "listed"], obs["searcher listed", "bitmap"]), \
            "the Searcher's listed and bitmap paths differ"
        _, _, _, sets = self._listed_sets(self._searcher_lists())
        s, p = obs["searcher listed", "listed"]
        k = SEARCHER_LISTED_K
        for b, Pb in enumerate(sets):
            n_b = int((p[b] >= 0).sum())
            assert n_b == min(k, Pb.numel()), "restricted Searcher: %d hits of %d" % (n_b, Pb.numel())
            if st != "fp8":
                S.check_topk_subset(plain[b, Pb], s[b], p[b], s64[b, Pb], bound[b, Pb], Pb, m.pid_base, k,
                                    "restricted searcher")
            else:
                self._check_fp8_searcher((s[b:b + 1, :n_b], p[b:b + 1, :n_b]), int(obs["depth listed", "listed"][0]),
                                         k, s64, bound, Pb, row=b)
        # 5. gather, bitwise
        D, mask = obs["gather"]
        Dm, mm = m.gather(inp["gather"], inp["nd_max"])
        assert _eq(D, Dm) and torch.equal(mask, mm), "gather_padded differs from the model"
        # 6. SIMT cross-check
        _, _, amax, rabs = model[32]
        simt = obs["simt"]
        S.check_ratio(RATIOS, "simt %s" % st, (simt[:, live].double() - s64[:, live]).abs(),
                      S.simt_bound(amax, rabs, 32)[:, live])
        assert torch.isneginf(simt[:, ~live]).all()
        # 7. Searcher
        if st != "fp8":
            for k in (200, 3000):
                s, p = obs["searcher", k]
                assert s.size(1) == min(k, m.n_live)
                s, p = _pad(s, p, k)
                S.check_topk(plain[:, P], s, _positions(p, P, m.pid_base), s64[:, P], bound[:, P], k,
                             "searcher k=%d" % k)
        else:
            self._check_fp8_searcher(obs["searcher", 200], int(obs["depth"][0]), 200, s64, bound, P)

    def _check_fp8_searcher(self, result, depth, k, s8, b8, P, row=None):
        """The exact re-rank: scores within the arg-max bound of float64 over the bf16 rows, in order, and no passage
        that surely beats the k-th returned one while surely inside the shortlist left out.  ``row``: the result is
        query ``row``'s alone, over its candidates P (a restricted search), at the depth the search reported."""
        m = self.m
        s, p = result
        Q = self.Q[32]
        if row is not None:
            Q, s8, b8 = Q[row:row + 1], s8[row:row + 1], b8[row:row + 1]
        kq = min(k, m.n_live if row is None else P.numel())
        assert s.size(1) == kq and (p >= 0).all()
        if kq == 0:
            return
        e64, eamax, erabs = m.exact_scores(Q)
        ebound = C_BOUND * U * eamax + Q.size(1) * U * erabs
        local = p - m.pid_base
        assert torch.from_numpy(~m.deleted).cuda()[local].all(), "fp8 searcher returned a deleted id"
        S.check_ratio(RATIOS, "searcher fp8 exact", (s.double() - e64.gather(1, local)).abs(), ebound.gather(1, local))
        assert (s[:, :-1] >= s[:, 1:]).all(), "fp8 searcher out of order"
        if row is None:
            assert depth == min(max(k, 1024), 2048, m.n_live)
        lo8, hi8 = (s8 - b8)[:, P], (s8 + b8)[:, P]
        thr = hi8.sort(dim=1, descending=True).values[:, depth - 1] if depth < P.numel() else \
            torch.full((s.size(0),), -torch.inf, dtype=torch.float64, device="cuda")
        elo = (e64 - ebound)[:, P]
        kth = (e64 + ebound).gather(1, local[:, -1:])
        returned = torch.zeros_like(elo, dtype=torch.bool)
        returned.scatter_(1, _positions(p, P, m.pid_base), True)
        miss = (elo > kth) & (lo8 > thr[:, None]) & ~returned
        assert not miss.any(), "fp8 searcher missed %d passages" % int(miss.sum())

    def run(self, ops):
        COUNT["sequences"] += 1
        self.obs = self.observe()
        self.check()
        for i, op in enumerate(ops):
            self.log.append({k: v for k, v in op.items() if k != "tags"})
            try:
                self.apply(op)
            except BaseException:
                print("\n[corpus lifecycle] sequence seed %d failed at op %d; spec %s; ops so far:\n%s" % (
                    self.spec["seed"], i, json.dumps({k: v for k, v in self.spec.items() if k != "lens0"}),
                    json.dumps(self.log)))
                raise


def replay(spec, ops, route="corpus", tmp_path=None):
    """Run a logged sequence (a spec and its op list, as a failure prints them) against a fresh corpus and model."""
    seq = Sequence(_lib(), spec, route, tmp_path)
    try:
        seq.run(ops)
    finally:
        if route == "corpus":
            seq.A.close()
    return seq


@pytest.mark.parametrize("case", M.SEQUENCE_CASES,
                         ids=lambda c: "%d-%s-base%d-%s" % (c[0], c[1], c[2], "adopted" if c[3] else "copied"))
def test_random_sequence(case):
    seed, storage, pid_base, adopt = case
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    spec, ops = M.generate(seed, storage, pid_base, adopt, sms=sms)
    replay(spec, ops)


def test_large_sequence_releases_and_maps_pieces_again():
    """A bf16 token matrix larger than one 1 GiB piece: compaction returns physical memory, a later append maps it
    again, and every state answers as the model does."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    spec, ops = M.large_sequence(31, sms=sms)
    seq = Sequence(_lib(), spec)
    try:
        COUNT["sequences"] += 1
        seq.obs = seq.observe()
        seq.check()
        mapped = [seq._mapped()]
        released = []
        for op in ops:
            seq.log.append({k: v for k, v in op.items() if k not in ("tags", "ids", "lens")})
            seq.apply(op)
            mapped.append(seq._mapped())
            if op["op"] == "compact":
                released.append(seq.last_compact["bytes_released"])
        # the first compaction unmaps the pieces behind its new end, the append after it maps pieces again
        first_compact = [i for i, op in enumerate(ops) if op["op"] == "compact"][0] + 1
        assert mapped[0] > PIECE and released[0] > 0 and mapped[first_compact] == mapped[0] - released[0], mapped
        assert mapped[first_compact + 1] > mapped[first_compact], mapped
    finally:
        seq.A.close()


@pytest.mark.parametrize("seed,storage", [(41, "bf16"), (42, "fp16")])
def test_indexer_searcher_updater_sequence(tmp_path, seed, storage):
    """An index written by Indexer, updated through Searcher + IndexUpdater, persisted, and searched again by a fresh
    Searcher on the written index: it answers as the model does."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    spec, ops = M.generate(seed, storage, 0, False, sms=sms)
    seq = replay(spec, ops, route="updater", tmp_path=tmp_path)
    seq.updater.persist_to_disk()
    R = seq.R
    fresh = R.Searcher(index=seq.path)
    seq.A, seq.searcher, seq.updater = fresh.corpus, fresh, None
    seq.m.compacted[:] = False                  # a fresh load stores every passage (deleted ones as tombstones)
    assert fresh.corpus.storage == storage and fresh.corpus.n_stored == seq.m.n_passages
    seq.obs = seq.observe()
    m = seq.m
    assert (fresh.corpus.n_passages, fresh.corpus.n_deleted) == (m.n_passages, m.n_deleted)
    assert np.array_equal(fresh.corpus.deleted_pids(), m.deleted_ids())
    seq.check()
