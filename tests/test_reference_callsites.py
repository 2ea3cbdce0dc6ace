"""CPU: the reference's OWN package (/root/reference, build container only) driven through this repository's
host layer — index addressing, PLAID auto-detection, the literal call sites of
src/executors/FLMR_executor.py:774-792 and src/models/rag/rag_model_blip.py:297-301, 397, 430-435,
``ColBERT.score`` / ``ColBERT.compute_ib_loss_new`` after ``integration.patch_colbert()``.

There is no GPU here, so the lowest layer (the C-ABI calls of maxsim.py / corpus.py) is substituted by the
numpy oracle — test infrastructure, tests/oracle_backend.py; everything above it is the product's host code and
everything that calls it is the unmodified reference.  The same lines run on the GPU box against the real
kernels in tests/test_callsites_gpu.py (with the duck-typed ``ravqa_b200.infra`` names, since the reference is
absent there).
"""
import os
import random
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN_DIR

REF = "/root/reference/third_party/ColBERT"
CKPT_DIR = os.path.join(GOLDEN_DIR, "callsites", "ckpt")
needs_reference = pytest.mark.skipif(not os.path.isdir(REF), reason="the reference checkout is absent or not readable")


@pytest.fixture(scope="module")
def ref():
    """The unmodified reference package behind the import shims of SURVEY.md Appendix A."""
    sys.path.insert(0, os.path.join(GOLDEN_DIR))
    from make_golden import import_reference
    import_reference()
    import colbert
    return colbert


@pytest.fixture()
def golden():
    z = np.load(os.path.join(GOLDEN_DIR, "callsites.npz"))
    return {k: z[k] for k in z.files}


# ---------------------------------------------------------------------------------------------------------
# index addressing
# ---------------------------------------------------------------------------------------------------------
@needs_reference
def test_index_path_resolution_equals_reference(ref):
    """infra.resolve_index_path == os.path.join(ColBERTConfig.from_existing(config, Run().config).index_root_, index)
    (colbert/searcher.py:26-30) for the reference's own config / Run objects, and the duck-typed infra classes
    give the same answers in the same situations."""
    from colbert.infra import ColBERTConfig as RC, Run as RRun, RunConfig as RRC
    import ravqa_b200.infra as I

    def reference_path(index, config):
        return os.path.join(RC.from_existing(config, RRun().config).index_root_, index)

    scenarios = [
        # (RunConfig kwargs stack, ColBERTConfig kwargs)
        ([dict(nranks=1, rank=0, root="/ckpt", experiment="temp_index_0")], dict(total_visible_gpus=0)),
        ([dict(nranks=1, rank=3, root="/data/idx", experiment="okvqa")], dict(total_visible_gpus=1)),
        ([dict(root="/a", experiment="b"), dict(experiment="c")], dict()),                  # nested contexts
        ([dict(root="/a", experiment="b")], dict(root="/ignored", experiment="ignored")),   # Run() wins
        ([dict(root="/a", experiment="b")], dict(index_root="/also/ignored")),              # ... even for index_root
        ([dict(index_root="/explicit/root")], dict(total_visible_gpus=0)),
        ([], dict(total_visible_gpus=0)),                                                   # no context at all
    ]
    for stack, ckw in scenarios:
        import contextlib
        with contextlib.ExitStack() as es_ref, contextlib.ExitStack() as es_own:
            for kw in stack:
                es_ref.enter_context(RRun().context(RRC(**kw)))
                es_own.enter_context(I.Run().context(I.RunConfig(**kw)))
            want = reference_path("temp_index.nbits=8", RC(**ckw))
            assert I.resolve_index_path("temp_index.nbits=8", RC(**ckw)) == want, (stack, ckw)
            own = I.resolve_index_path("temp_index.nbits=8", I.ColBERTConfig(**ckw))
            # (without a context both fall back to <cwd at import>/experiments/default/indexes/)
            assert os.path.normpath(own) == os.path.normpath(want), (stack, ckw, own, want)
            # absolute index names win over any root, as os.path.join makes them do in the reference
            assert I.resolve_index_path("/abs/idx", RC(**ckw)) == reference_path("/abs/idx", RC(**ckw)) == "/abs/idx"
    # from_existing / assigned semantics of the stand-ins (core_config.py:20-36, base_config.py:20-35)
    for R_, C_ in ((RRC, RC), (I.RunConfig, I.ColBERTConfig)):
        a = C_(nbits=8, doc_maxlen=None)
        assert set(a.assigned) == {"nbits", "doc_maxlen"} and a.doc_maxlen == 220     # None -> default, still assigned
        b = C_.from_existing(a, R_(root="/r"))
        assert b.nbits == 8 and b.root == "/r" and "experiment" not in b.assigned
        b.configure(ncells=2, bogus=1)
        assert b.ncells == 2 and "ncells" in b.assigned and not hasattr(b, "bogus")
    assert len(I.Run().stack) == 1 and len(RRun().stack) == 1                          # contexts popped


def test_index_kind_detection(tmp_path):
    import ravqa_b200 as R
    from ravqa_b200.searcher import detect_index_kind
    plaid = os.path.join(CKPT_DIR, "temp_index_0", "indexes", "temp_index.nbits=8")
    assert detect_index_kind(plaid) == "plaid"
    flat = str(tmp_path / "flat")
    R.save_flat_index(flat, torch.zeros(6, 128, dtype=torch.bfloat16), [2, 4])
    assert detect_index_kind(flat) == "flat"
    only_plan = tmp_path / "building"
    only_plan.mkdir()
    (only_plan / "plan.json").write_text("{}")
    with pytest.raises(ValueError, match="did not finish"):
        detect_index_kind(str(only_plan))
    with pytest.raises(FileNotFoundError):
        detect_index_kind(str(tmp_path / "missing"))
    # the index config comes from where the reference reads it (base_config.py:71-87)
    cfg = R.ColBERTConfig.load_from_index(plaid)
    assert cfg.nbits == 8 and cfg.dim == 128 and cfg.index_name == "temp_index.nbits=8"


# ---------------------------------------------------------------------------------------------------------
# the literal call sites, reference objects + this repository's Searcher
# ---------------------------------------------------------------------------------------------------------
@needs_reference
def test_executor_search_lines_verbatim_with_patched_colbert(ref, golden, monkeypatch):
    """FLMR_executor.py:774-792, copied line by line, with ``from colbert import Searcher`` resolved AFTER
    ``patch_colbert()``; Run / RunConfig / ColBERTConfig / Queries are the reference's own classes."""
    import oracle_backend
    import ravqa_b200.integration as flmr_b200
    oracle_backend.install(monkeypatch)
    import colbert.searcher
    original = colbert.searcher.Searcher
    # an executor that did `from colbert import Indexer, Searcher` BEFORE the patch (FLMR_executor.py:47)
    import types
    early = types.ModuleType("an_executor_imported_earlier")
    early.Searcher = original
    sys.modules[early.__name__] = early
    try:
        done = flmr_b200.patch_colbert()
        assert done["Searcher"] >= 3 and early.Searcher is flmr_b200.Searcher   # colbert, colbert.searcher, the executor
        from colbert import Searcher
        from colbert.data import Queries
        from colbert.infra import ColBERTConfig, Run, RunConfig
        import ravqa_b200
        assert Searcher is ravqa_b200.Searcher

        # ---- names the executor has in scope at that point ----
        class _Self:
            global_rank = 0
            device = torch.device("cpu")            # (the reference then asks for total_visible_gpus = 0)
            config = type("C", (), {"ckpt_dir": CKPT_DIR})()
            model_config = {"nbits": 8}
        self = _Self()
        dataloader_idx = 0
        question_ids = ["q%d" % i for i in range(golden["queries"].shape[0])]
        questions = ["question %d" % i for i in range(len(question_ids))]
        query_embeddings = torch.from_numpy(golden["queries"])
        Ks = [1, 5, int(golden["k"])]
        get_world_size = lambda: 1                  # noqa: E731

        # ---- FLMR_executor.py:774-792, verbatim (minus logging and the distributed barrier) ----
        with Run().context(RunConfig(nranks=1, rank=self.global_rank, root=self.config.ckpt_dir, experiment=f"temp_index_{dataloader_idx}")):
            if self.device == torch.device('cpu'):
                total_visible_gpus = 0
            else:
                if get_world_size() > 1:
                    total_visible_gpus = 0
                else:
                    total_visible_gpus = 1 #torch.cuda.device_count()

            config = ColBERTConfig(
                total_visible_gpus=total_visible_gpus,
            )
            nbits = self.model_config.get("nbits", 2)
            searcher = Searcher(index=f"temp_index.nbits={nbits}", config=config)
            custom_quries = {question_id: question for question_id, question in zip(question_ids, questions)}
            queries = Queries(data=custom_quries)
            ranking = searcher._search_all_Q(queries, query_embeddings, k=max(Ks))

            ranking_dict = ranking.todict()

            del searcher
        # ---- what the lines after it consume (FLMR_executor.py:851-878) ----
        assert list(ranking_dict.keys()) == question_ids
        want = np.argsort(-golden["exact_scores_bf16"], axis=1, kind="stable")[:, :max(Ks)]
        for qi, (question_id, ranking_list) in enumerate(zip(question_ids, ranking_dict.values())):
            assert len(ranking_list) == max(Ks)
            for rank0, entry in enumerate(ranking_list):
                retrieved_doc_index, rank, retrieved_doc_score = entry
                assert isinstance(retrieved_doc_index, int) and rank == rank0 + 1 and isinstance(retrieved_doc_score, float)
            assert [e[0] for e in ranking_list] == want[qi].tolist()
            np.testing.assert_allclose([e[2] for e in ranking_list], golden["exact_scores_bf16"][qi, want[qi]], rtol=5e-4)
        assert ranking.provenance()["source"] == "Searcher::search_all"
    finally:
        flmr_b200.unpatch_colbert()
        sys.modules.pop(early.__name__, None)
    assert colbert.searcher.Searcher is original and ref.Searcher is original


@needs_reference
def test_rag_retrieval_lines_verbatim_with_patched_colbert(ref, golden, monkeypatch):
    """rag_model_blip.py:288-301 (index opened through the Run context derived from ``index_path``) and
    :390-441 (search, per-question re-score through the reference's OWN ``ColBERT.score``), with the backend
    patched in; result = what the unpatched reference computes for the same retrieved passages."""
    import oracle_backend
    import ravqa_b200.integration as flmr_b200
    oracle_backend.install(monkeypatch)
    from colbert.modeling.colbert import ColBERT
    from colbert.infra import ColBERTConfig as RC
    doclens = golden["doclens"]
    rng = np.random.default_rng(5)
    # host dictionary of item embeddings, as rag_model_blip.py:303-330 loads it: pid -> (emb [Nd, d], mask [Nd, 1])
    nd_max = int(doclens.max())
    item_embeddings = {}
    for pid, n in enumerate(doclens):
        e = np.zeros((nd_max, 128), dtype=np.float32)
        e[:n] = rng.standard_normal((n, 128)).astype(np.float32)
        e[:n] /= np.linalg.norm(e[:n], axis=1, keepdims=True)
        e = torch.from_numpy(e).bfloat16().float().numpy()      # bf16-exact, so both sides see identical operands
        m = np.zeros((nd_max, 1), dtype=np.float32)
        m[:n] = 1
        item_embeddings[pid] = (e, m)

    class _Encoder:          # the reference's ColBERT.score bound to a stand-in `self` (no BERT weights offline)
        colbert_config = RC(total_visible_gpus=0)
        use_gpu = False
        score = ColBERT.score

    def run_lines():
        from colbert import Searcher
        from colbert.data import Queries
        from colbert.infra import ColBERTConfig, Run, RunConfig

        class _Self:
            global_rank = 0
            device = torch.device("cpu")
            question_encoder = _Encoder()
        self = _Self()
        self.item_embeddings = item_embeddings
        index_path = os.path.join(CKPT_DIR, "temp_index_0")
        # ---- rag_model_blip.py:288-301 ----
        index_root = os.path.dirname(index_path)
        index_name = os.path.basename(index_path)
        if self.device == torch.device('cpu'):
            total_visible_gpus = 0
        else:
            total_visible_gpus = 1
        with Run().context(RunConfig(nranks=1, rank=self.global_rank, root=index_root, experiment=index_name)):
            config = ColBERTConfig(
                total_visible_gpus=total_visible_gpus,
            )
            self.index = Searcher(index=f"temp_index.nbits=8", config=config)
        # ---- rag_model_blip.py:388-441 ----
        question_hidden_states = torch.from_numpy(golden["queries"]).clone().requires_grad_(True)
        input_text_sequences = ["question %d" % i for i in range(question_hidden_states.size(0))]
        n_docs = 3
        custom_quries = {i: query for i, query in enumerate(input_text_sequences)}
        queries = Queries(data=custom_quries)
        if n_docs < 5:
            n_docs_retrieve = 5
        else:
            n_docs_retrieve = n_docs
        ranking = self.index._search_all_Q(queries, question_hidden_states.cpu().detach(), k=n_docs_retrieve, progress=False)
        retrieval_results = ranking.todict()
        doc_scores = []
        all_retrieved_doc_indices = []
        for query_index, retrieved_docs in retrieval_results.items():
            retrieved_doc_indices = []
            retrieved_doc_scores = []
            if n_docs != n_docs_retrieve:
                retrieved_docs = random.sample(retrieved_docs, n_docs)
            for doc_index, _, doc_score in retrieved_docs:
                retrieved_doc_indices.append(doc_index)
                retrieved_doc_scores.append(doc_score)
            retrieved_item_embeddings = []
            retrieved_item_embeding_mask = []
            for i in retrieved_doc_indices:
                emb_tuple = self.item_embeddings[i]
                retrieved_item_embeddings.append(torch.Tensor(emb_tuple[0]))
                retrieved_item_embeding_mask.append(torch.Tensor(emb_tuple[1]))
            retrieved_item_embeddings = torch.stack(retrieved_item_embeddings).to(self.device)
            retrieved_item_embeding_mask = torch.stack(retrieved_item_embeding_mask).to(self.device)
            retrieved_query_embedding = question_hidden_states[[query_index]]
            self.question_encoder.colbert_config.nway = len(retrieved_doc_indices)
            Q_duplicated = retrieved_query_embedding.repeat_interleave(self.question_encoder.colbert_config.nway, dim=0).contiguous()
            scores = self.question_encoder.score(Q_duplicated, retrieved_item_embeddings, retrieved_item_embeding_mask)
            doc_scores.append(scores)
            all_retrieved_doc_indices.append(retrieved_doc_indices)
        doc_scores = torch.stack(doc_scores)
        ids = np.array(all_retrieved_doc_indices)
        doc_scores.sum().backward()
        return ids, doc_scores.detach(), question_hidden_states.grad.clone()

    try:
        flmr_b200.patch_colbert()
        random.seed(11)
        ids, doc_scores, dq = run_lines()
    finally:
        flmr_b200.unpatch_colbert()
    # retrieved ids: subsets of the exact top-5 over the reference's decompressed index
    top5 = np.argsort(-golden["exact_scores_bf16"], axis=1, kind="stable")[:, :5]
    assert ids.shape == (golden["queries"].shape[0], 3)
    for b in range(ids.shape[0]):
        assert set(ids[b]).issubset(set(top5[b]))
    # the re-score and its gradient: the UNPATCHED reference ColBERT.score on the same passages (fp32 autograd)
    Qr = torch.from_numpy(golden["queries"]).clone().requires_grad_(True)
    want = []
    for b in range(ids.shape[0]):
        E = torch.stack([torch.Tensor(item_embeddings[i][0]) for i in ids[b]])
        M = torch.stack([torch.Tensor(item_embeddings[i][1]) for i in ids[b]])
        want.append(_Encoder().score(Qr[[b]].repeat_interleave(3, dim=0).contiguous(), E, M))
    want = torch.stack(want)
    want.sum().backward()
    np.testing.assert_allclose(doc_scores.numpy(), want.detach().numpy(), rtol=1e-5)
    np.testing.assert_allclose(dq.numpy(), Qr.grad.numpy(), rtol=1e-5, atol=1e-6)


@needs_reference
def test_reference_colbert_methods_route_into_this_backend(ref, monkeypatch):
    """``ColBERT.score`` (colbert.py:217-224) in its three caller shapes and ``ColBERT.compute_ib_loss_new``
    (colbert.py:82-113) — the reference's own methods — before and after ``patch_colbert()``: same values,
    same gradients, and after the patch every score comes out of this repository's entry points."""
    import oracle_backend
    import ravqa_b200.integration as flmr_b200
    calls = oracle_backend.install(monkeypatch)
    from colbert.infra import ColBERTConfig as RC
    from colbert.modeling.colbert import ColBERT

    class _Model:
        colbert_config = RC(total_visible_gpus=0, nway=2, use_ib_negatives=True)
        use_gpu = False
        loss_fn = torch.nn.CrossEntropyLoss()
        score = ColBERT.score
        compute_ib_loss_new = ColBERT.compute_ib_loss_new

    g = torch.Generator().manual_seed(3)
    B, nway, nq, nd = 3, 2, 40, 24
    Q0 = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).bfloat16().float()
    D0 = torch.nn.functional.normalize(torch.randn(B * nway, nd, 128, generator=g), dim=-1).bfloat16().float()
    M0 = torch.rand(B * nway, nd, 1, generator=g) > 0.3
    M0[:, 0] = True

    def run(model):
        out = {}
        Q, D = Q0.clone().requires_grad_(True), D0.clone().requires_grad_(True)
        # training: colbert.py:71-73 (+ :74-78)
        s = model.score(Q.repeat_interleave(nway, dim=0).contiguous(), D, M0)
        loss = model.compute_ib_loss_new(Q, D, M0)
        (s.sum() + loss).backward()
        out["train"] = (s.detach(), loss.detach(), Q.grad.clone(), D.grad.clone())
        # exhaustive evaluation: FLMR_executor.py:826-833 (items repeated per query, queries interleaved)
        items, imask = D0[:4], M0[:4]
        Qd = Q0.repeat_interleave(4, dim=0).contiguous()
        out["eval"] = model.score(Qd, items.repeat(B, 1, 1), imask.repeat(B, 1, 1)).reshape(B, -1).detach()
        # one query against all documents (Q.size(0) == 1, colbert.py:282)
        out["one"] = model.score(Q0[:1], D0, M0).detach()
        return out

    before = run(_Model())
    n_before = dict(calls)
    try:
        flmr_b200.patch_colbert()

        class _Patched(_Model):
            score = ColBERT.score
            compute_ib_loss_new = ColBERT.compute_ib_loss_new      # now the replacement method
        after = run(_Patched())
    finally:
        flmr_b200.unpatch_colbert()
    assert n_before == {} and calls["argmax_grouped"] >= 2 and calls["argmax"] >= 2 and calls["backward_grouped"] >= 1
    for key in ("eval", "one"):
        np.testing.assert_allclose(after[key].numpy(), before[key].numpy(), rtol=1e-5)
    for a, b in zip(after["train"], before["train"]):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-4, atol=1e-5)
    assert ColBERT.compute_ib_loss_new is _Model.__dict__["compute_ib_loss_new"]   # restored


@needs_reference
@pytest.mark.parametrize("nq", [64, 70, 72, 96])
def test_flipr_interaction_equals_reference(ref, monkeypatch, nq):
    """``config.interaction == 'flipr'`` (colbert_score_reduce, colbert.py:248-261; unused by FLMR): this package's
    ``colbert_score`` against the reference's own — one query vs all documents and aligned pairs, values and
    gradients — with fewer than 8 (no second term), exactly 8 and more tokens beyond ``query_maxlen``."""
    import oracle_backend
    import ravqa_b200 as R
    oracle_backend.install(monkeypatch)
    from colbert.infra import ColBERTConfig as RC
    from colbert.modeling.colbert import colbert_score as ref_score
    cfg = RC(total_visible_gpus=0, interaction="flipr", query_maxlen=64)
    g = torch.Generator().manual_seed(nq)
    n, nd = 5, 30
    Q0 = torch.nn.functional.normalize(torch.randn(n, nq, 128, generator=g), dim=-1).bfloat16().float()
    D0 = torch.nn.functional.normalize(torch.randn(n, nd, 128, generator=g), dim=-1).bfloat16().float()
    M0 = torch.rand(n, nd, 1, generator=g) > 0.3
    M0[:, 0] = True
    w = torch.linspace(0.5, 1.5, n)
    for q_rows in (slice(0, 1), slice(0, n)):
        out = []
        for fn in (ref_score, R.colbert_score):
            Q, D = Q0[q_rows].clone().requires_grad_(True), D0.clone().requires_grad_(True)
            s = fn(Q, D, M0, config=cfg) if fn is R.colbert_score else fn(Q, D * M0, M0, config=cfg, use_gpu=False)
            (s * w).sum().backward()
            out.append((s.detach(), Q.grad.clone(), D.grad.clone()))
        for a, b in zip(*out):
            np.testing.assert_allclose(b.numpy(), a.numpy(), rtol=1e-5, atol=1e-6)
    # and it is not the plain sum
    assert not torch.allclose(R.colbert_score(Q0[:1], D0, M0, config=cfg), R.colbert_score(Q0[:1], D0, M0))
    # packed form (colbert.py:289-311: 'flipr' always takes the padded reduction)
    from colbert.modeling.colbert import colbert_score_packed as ref_packed
    import ravqa_b200.integration as I
    lens = torch.tensor([30, 7, 19, 1, 24])
    packed = torch.cat([D0[i, :l] for i, l in enumerate(lens)])
    want = ref_packed(Q0[:1], packed, lens, cfg)
    got = I.colbert_score_packed(Q0[:1], packed, lens, cfg)
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-5)
    with pytest.raises(NotImplementedError):
        R.Searcher(index=oracle_backend.OracleCorpus(packed, lens), config=cfg)


@needs_reference
def test_text_search_goes_through_the_references_checkpoint(ref, golden, monkeypatch):
    """``Searcher.search`` / ``search_all`` (searcher.py:52-71) with ``checkpoint=``: the query encoder is the
    reference's own ``colbert.modeling.checkpoint.Checkpoint``, constructed lazily with (name, colbert_config=
    searcher.config) and asked through ``queryFromText`` exactly as the reference's ``encode`` does — here a recording
    stand-in with the same constructor and method (no BERT weights offline) that returns the golden query
    embeddings, so the ranking is the exact one."""
    import oracle_backend
    import ravqa_b200 as R
    import colbert.modeling.checkpoint as CK
    from colbert.data import Queries
    from colbert.infra import ColBERTConfig, Run, RunConfig
    oracle_backend.install(monkeypatch)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    seen = {}
    Qg = torch.from_numpy(golden["queries"])
    texts = ["question %d" % i for i in range(Qg.size(0))]

    class FakeCheckpoint:
        def __init__(self, name, colbert_config=None):
            seen["ctor"] = (name, colbert_config)
            self.query_tokenizer = type("T", (), {"query_maxlen": None})()

        def queryFromText(self, queries, bsize=None, to_cpu=False, context=None):
            seen.setdefault("calls", []).append((list(queries), bsize, to_cpu, self.query_tokenizer.query_maxlen))
            return torch.stack([Qg[texts.index(q)] for q in queries])

    monkeypatch.setattr(CK, "Checkpoint", FakeCheckpoint)
    with Run().context(RunConfig(nranks=1, rank=0, root=CKPT_DIR, experiment="temp_index_0")):
        searcher = R.Searcher(index="temp_index.nbits=8", checkpoint="some/checkpoint",
                              config=ColBERTConfig(total_visible_gpus=0, query_maxlen=48))
    assert "ctor" not in seen                                        # nothing is loaded until text arrives
    k = int(golden["k"])
    want = np.argsort(-golden["exact_scores_bf16"], axis=1, kind="stable")[:, :k]
    pids, ranks, scores = searcher.search(texts[3], k=k)
    assert seen["ctor"][0] == "some/checkpoint" and seen["ctor"][1] is searcher.config
    assert seen["calls"][0] == ([texts[3]], None, False, 48)
    assert pids == want[3].tolist() and ranks == list(range(1, k + 1))
    ranking = searcher.search_all(Queries(data=dict(zip(["a%d" % i for i in range(len(texts))], texts))), k=k)
    assert [[e[0] for e in v] for v in ranking.todict().values()] == want.tolist()
    assert len(seen["calls"]) == 2 and seen["calls"][1][0] == texts
    # no checkpoint and no encode_fn: a clear error instead of a silent CPU path
    with Run().context(RunConfig(nranks=1, rank=0, root=CKPT_DIR, experiment="temp_index_0")):
        bare = R.Searcher(index="temp_index.nbits=8", config=ColBERTConfig(total_visible_gpus=0))
    bare.index_config.checkpoint = None
    with pytest.raises(RuntimeError, match="encode_fn"):
        bare.search("text", k=3)


@needs_reference
def test_indexer_with_the_references_checkpoint_and_run_context(ref, monkeypatch, tmp_path):
    """``Indexer(checkpoint=..., config=...).index(name=..., collection=..., overwrite=True)`` as
    FLMR_executor.py:601-617 calls it, inside the reference's ``Run().context``: the document encoder is the
    reference's ``Checkpoint`` (a recording stand-in here: no BERT weights offline) driven with the batching of
    ``CollectionEncoder.encode_passages``; the flat index lands where ``config.index_path_`` points
    (``<root>/<experiment>/indexes/<name>``), and ``Searcher(index=name)`` in the same context opens and ranks it."""
    import zlib
    import oracle_backend
    import ravqa_b200 as R
    import colbert.modeling.checkpoint as CK
    from colbert.infra import ColBERTConfig, Run, RunConfig
    oracle_backend.install(monkeypatch)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    seen = {"batches": []}

    def embed(text):
        g = torch.Generator().manual_seed(zlib.crc32(text.encode()))
        n = 3 + zlib.crc32(text.encode()) % 6
        return torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1)

    class FakeCheckpoint:
        def __init__(self, name, colbert_config=None):
            seen["ctor"] = (name, colbert_config)

        def docFromText(self, docs, bsize=None, keep_dims=True, to_cpu=False, showprogress=False, return_tokens=False):
            assert keep_dims == "flatten" and torch.is_inference_mode_enabled()
            seen["batches"].append((len(docs), bsize))
            embs = [embed(d) for d in docs]
            return torch.cat(embs), [e.size(0) for e in embs]

    monkeypatch.setattr(CK, "Checkpoint", FakeCheckpoint)
    collection = ["passage number %d" % i for i in range(230)]
    with Run().context(RunConfig(nranks=1, rank=0, root=str(tmp_path), experiment="temp_index_0")):
        config = ColBERTConfig(nbits=8, doc_maxlen=512, total_visible_gpus=0, bsize=2)
        indexer = R.Indexer(checkpoint="a/checkpoint", config=config)
        path = indexer.index(name="temp_index.nbits=8", collection=collection, overwrite=True)
        assert path == os.path.join(str(tmp_path), "temp_index_0", "indexes", "temp_index.nbits=8")
        assert path == ColBERTConfig.from_existing(config, Run().config).index_root_ + "temp_index.nbits=8" \
            or os.path.normpath(path) == os.path.normpath(os.path.join(
                ColBERTConfig.from_existing(config, Run().config).index_root_, "temp_index.nbits=8"))
        assert seen["ctor"] == ("a/checkpoint", config)
        assert seen["batches"] == [(100, 2), (100, 2), (30, 2)]           # bsize * 50 passages per docFromText call
        searcher = R.Searcher(index="temp_index.nbits=8", config=ColBERTConfig(total_visible_gpus=0))
    assert searcher.index_kind == "flat" and searcher.corpus.n_passages == len(collection)
    Q = torch.stack([torch.nn.functional.pad(embed(collection[i]), (0, 0, 0, 8 - embed(collection[i]).size(0)))
                     for i in (7, 100, 229)])
    ranking = searcher._search_all_Q(None, Q, k=3).todict()
    assert [v[0][0] for v in ranking.values()] == [7, 100, 229]          # each passage's own tokens find it first
    # opt-in: `from colbert import Indexer` itself becomes the flat-store Indexer; a TSV path is a collection too
    import ravqa_b200.integration as flmr_b200
    import colbert.indexer
    original = colbert.indexer.Indexer
    tsv = tmp_path / "collection.tsv"
    tsv.write_text("".join("%d\t%s\ttitle %d\n" % (i, t, i) for i, t in enumerate(collection[:20])))
    try:
        assert flmr_b200.patch_colbert(searcher=False, scoring=False, ib_loss=False, indexer=True)["Indexer"] >= 2
        from colbert import Indexer
        assert Indexer is R.Indexer
        with Run().context(RunConfig(nranks=1, root=str(tmp_path), experiment="temp_index_1")):
            indexer = Indexer(checkpoint="a/checkpoint", config=ColBERTConfig(nbits=2, bsize=4))
            indexer.index(name="temp_index.nbits=2", collection=str(tsv), overwrite=True)
            index_path = indexer.get_index()
        assert index_path == os.path.join(str(tmp_path), "temp_index_1", "indexes", "temp_index.nbits=2")
        from ravqa_b200.index_io import load_flat_index
        tokens, doclens, meta = load_flat_index(index_path)
        want = [embed("title %d | %s" % (i, t)).size(0) for i, t in enumerate(collection[:20])]
        assert doclens.tolist() == want and tokens.size(0) == sum(want)
    finally:
        flmr_b200.unpatch_colbert()
    assert colbert.indexer.Indexer is original
