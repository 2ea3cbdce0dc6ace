"""CPU: building PLAID indexes (Indexer(index_format="plaid"), plaid.encode / kmeans / residual_buckets / build_ivf).

The encode kernel's argument checks run here; everything else substitutes the numpy restatement of the kernel
(tests/plaid_encode_oracle.py) for ``plaid.encode`` and checks the restatement, the IVF, the k-means loop and the
written directory against the reference's own ResidualCodec, optimize_ivf and IndexScorer where the reference checkout
is present.
"""
import json
import os
import sys
import zlib

import numpy as np
import pytest
import torch

import plaid_encode_oracle as E
from helpers import GOLDEN_DIR
from oracle import maxsim_oracle as O
from ravqa_b200 import _cabi

REF = "/root/reference/third_party/ColBERT"
needs_reference = pytest.mark.skipif(not os.path.isdir(REF), reason="the reference checkout is absent or not readable")


@pytest.fixture(scope="module")
def ref():
    sys.path.insert(0, GOLDEN_DIR)
    from make_golden import import_reference
    import_reference()
    import colbert
    return colbert


def test_encode_refuses_bad_arguments_before_any_cuda_call():
    L = _cabi.lib()
    buf = np.zeros(4096, dtype=np.uint8)
    p = buf.ctypes.data + (-buf.ctypes.data) % 16            # 16-byte aligned host address, never dereferenced
    cut = np.zeros(255, dtype=np.float32)
    ok = dict(x=p, n=10, c=p, K=4, cut=cut.ctypes.data, nbits=2, codes=p, res=p, best=p)

    def call(**kw):
        a = dict(ok, **kw)
        return L.flmr_plaid_encode(a["x"], a["n"], a["c"], a["K"], a["cut"], a["nbits"], a["codes"], a["res"],
                                   a["best"], 0, None)
    for kw in (dict(x=None), dict(c=None), dict(codes=None), dict(cut=None), dict(nbits=0), dict(nbits=3),
               dict(nbits=16), dict(K=0), dict(K=-1), dict(n=-1), dict(x=p + 2), dict(c=p + 8), dict(res=p + 1)):
        assert call(**kw) == 1, kw
    assert b"nbits" in (call(nbits=3), L.flmr_last_error())[1]
    assert call(n=(1 << 31)) == 3                               # beyond the TMA row range: split the call
    # n == 0 does nothing (no device is touched); assignment only needs no cutoffs
    assert call(n=0) == 0 and call(n=0, cut=None, res=None, best=None) == 0


@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
def test_pack_buckets_inverts_the_decode(nbits):
    rng = np.random.default_rng(nbits)
    buckets = rng.integers(0, 1 << nbits, size=(7, 128))
    packed = E.pack_buckets(buckets, nbits)
    assert packed.shape == (7, 16 * nbits)
    weights = np.arange(1 << nbits, dtype=np.float32) * 0.25
    dec = O.plaid_decode(np.zeros(7, np.int32), packed, np.zeros((1, 128), np.float32), weights, nbits,
                         normalize=False)
    assert np.array_equal(dec, weights[buckets])


def _codec_case(nbits, seed, n=900, K=64):
    g = torch.Generator().manual_seed(seed)
    x = torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1).half()
    cents = torch.nn.functional.normalize(torch.randn(K, 128, generator=g), dim=-1).half()
    codes = E.assign(x.numpy(), cents.numpy())
    res = (x.float() - cents.float()[codes.astype(np.int64)]).half().float()
    q = torch.arange(0, 1 << nbits) * (1 / (1 << nbits))
    cutoffs = res.quantile(q[1:])
    weights = res.quantile(q + 0.5 / (1 << nbits))
    return x, cents, cutoffs, weights


@needs_reference
@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
def test_restatement_matches_the_references_compress(ref, nbits):
    """Codes equal ResidualCodec.compress's (CPU); residual bytes equal except on rows where its fp32 residual and
    the fp16-rounded one fall on different sides of a cutoff."""
    from colbert.indexing.codecs.residual import ResidualCodec
    from colbert.infra.config import ColBERTConfig
    x, cents, cutoffs, weights = _codec_case(nbits, 10 + nbits)
    codec = ResidualCodec(config=ColBERTConfig(nbits=nbits, dim=128, total_visible_gpus=0),
                          centroids=cents.float(), avg_residual=0.1, bucket_cutoffs=cutoffs, bucket_weights=weights)
    comp = codec.compress(x.float())
    codes, res = E.encode(x.numpy(), cents.numpy(), cutoffs.numpy(), nbits)
    assert np.array_equal(comp.codes.numpy(), codes)
    straddle = E.straddle_rows(x.numpy(), cents.numpy(), codes, cutoffs.numpy())
    same = (comp.residuals.numpy() == res).all(axis=1)
    assert bool((same | straddle).all()) and same.any()


@needs_reference
def test_ivf_matches_optimize_ivf(ref, tmp_path):
    from colbert.indexing.utils import optimize_ivf
    from ravqa_b200 import plaid
    rng = np.random.default_rng(3)
    doclens = [rng.integers(1, 30, 40).tolist(), rng.integers(1, 30, 25).tolist()]
    for c, dl in enumerate(doclens):
        (tmp_path / ("doclens.%d.json" % c)).write_text(json.dumps(dl))
    K = 50                                                         # some centroids get no token
    codes = torch.from_numpy(rng.integers(0, K - 5, sum(map(sum, doclens))))
    srt = codes.sort()
    want_ivf, want_len = optimize_ivf(srt.indices, torch.bincount(srt.values, minlength=K), str(tmp_path))
    ivf, lengths = plaid.build_ivf(codes, doclens[0] + doclens[1], K)
    assert ivf.dtype == want_ivf.dtype == torch.int32 and lengths.dtype == want_len.dtype
    assert torch.equal(ivf, want_ivf) and torch.equal(lengths, want_len)


def test_kmeans_loop_against_float64_lloyd(monkeypatch):
    """plaid.kmeans with the restatement assigning, against float64 Lloyd iterations from the same initial rows;
    duplicated rows make clusters empty, so the split runs too."""
    from ravqa_b200 import plaid
    monkeypatch.setattr(plaid, "encode", E.encode_torch)
    g = torch.Generator().manual_seed(5)
    base = torch.nn.functional.normalize(torch.randn(12, 128, generator=g), dim=-1)
    dup = base[torch.arange(300) % 12]                                        # 12 distinct rows, 25 copies each
    noisy = torch.nn.functional.normalize(torch.randn(500, 128, generator=g), dim=-1)
    for sample, K in ((dup.half(), 20), (noisy.half(), 37)):
        got16, raw = plaid.kmeans(sample, K, niters=5, seed=7, return_raw=True)
        gi = torch.Generator().manual_seed(7)
        init = sample[torch.randperm(sample.size(0), generator=gi)[:K]].float().numpy()
        want = E.lloyd_float64(sample.numpy(), init, 5)
        assert np.array_equal(raw.numpy(), want)
        assert torch.equal(got16, torch.nn.functional.normalize(torch.from_numpy(want), dim=-1).half())
    counts = np.bincount(E.assign(dup.numpy(), got16.numpy()), minlength=20)
    assert (counts == 0).sum() >= 8                       # only 12 distinct points: the splits were needed and ran


def _embed(text):
    g = torch.Generator().manual_seed(zlib.crc32(text.encode()))
    n = 4 + zlib.crc32(text.encode()) % 9
    return torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1)


def _encode_fn(passages):
    embs = [_embed(p) for p in passages]
    return torch.cat(embs), [e.size(0) for e in embs]


def _build(tmp_path, name, monkeypatch, nbits=2, **kw):
    from ravqa_b200 import plaid
    from ravqa_b200.indexer import Indexer
    monkeypatch.setattr(plaid, "encode", E.encode_torch)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    collection = ["passage %d" % i for i in range(300)]
    ix = Indexer(encode_fn=_encode_fn, index_root=str(tmp_path), chunksize=110, index_format="plaid", nbits=nbits,
                 **kw)
    return ix, ix.index(name, collection, overwrite=True), collection


@needs_reference
@pytest.mark.parametrize("nbits", [2, 4])
def test_indexer_plaid_directory_opens_in_the_reference(ref, tmp_path, monkeypatch, nbits):
    from colbert.indexing.codecs.residual import ResidualCodec
    from colbert.indexing.codecs.residual_embeddings import ResidualEmbeddings
    from colbert.infra.config import ColBERTConfig
    from colbert.search.index_storage import IndexScorer
    ix, path, collection = _build(tmp_path, "idx", monkeypatch, nbits=nbits)
    names = sorted(os.listdir(path))
    for f in ("plan.json", "metadata.json", "centroids.pt", "buckets.pt", "avg_residual.pt", "ivf.pid.pt",
              "0.codes.pt", "2.residuals.pt", "doclens.1.json", "1.metadata.json"):
        assert f in names, (f, names)
    assert not any(f.startswith("sample.") for f in names)
    meta = json.load(open(os.path.join(path, "metadata.json")))
    assert meta["config"]["nbits"] == nbits and meta["num_chunks"] == 3
    codec = ResidualCodec.load(path)
    assert torch.load(os.path.join(path, "centroids.pt")).dtype == torch.float16 and codec.nbits == nbits
    assert torch.load(os.path.join(path, "0.codes.pt")).dtype == torch.int32
    assert torch.load(os.path.join(path, "0.residuals.pt")).dtype == torch.uint8
    cents = codec.centroids.float().numpy()
    weights = codec.bucket_weights.float().numpy()
    want_codes = []
    for c in range(3):
        emb = ResidualEmbeddings.load(path, c)
        dec_ref = codec.decompress(emb).numpy()
        dec_or = O.plaid_decode(emb.codes.numpy(), emb.residuals.numpy(), cents, weights, nbits)
        np.testing.assert_allclose(dec_ref, dec_or, rtol=0, atol=2e-6)
        p0, p1 = c * 110, min(300, (c + 1) * 110)
        x = _encode_fn(collection[p0:p1])[0].half()
        codes, res = E.encode(x.numpy(), codec.centroids.half().numpy(), codec.bucket_cutoffs.numpy(), nbits)
        assert np.array_equal(emb.codes.numpy(), codes) and np.array_equal(emb.residuals.numpy(), res)
        want_codes.append(codes)
    ivf, lengths = torch.load(os.path.join(path, "ivf.pid.pt"))
    assert int(lengths.sum()) == ivf.numel() and lengths.numel() == meta["num_partitions"]
    # the reference's CPU IndexScorer ranks a query planted from passage 123's own rows first
    scorer = IndexScorer(path, use_gpu=False)
    q = _embed(collection[123])
    Q = torch.nn.functional.pad(q, (0, 0, 0, 32 - q.size(0))).unsqueeze(0)
    pids, scores = scorer.rank(ColBERTConfig(ncells=8, centroid_score_threshold=0.0, ndocs=64,
                                             total_visible_gpus=0), Q)
    assert pids[0] == 123


def test_indexer_plaid_is_deterministic_resumable_and_flat_mode_unchanged(tmp_path, monkeypatch):
    ix, path, collection = _build(tmp_path, "a", monkeypatch)
    _, path_b, _ = _build(tmp_path, "b", monkeypatch)

    def files(p):
        return {f: open(os.path.join(p, f), "rb").read() for f in sorted(os.listdir(p))}
    a = files(path)
    assert a == files(path_b)
    # resume: remove one chunk's marker, rebuild only it, same bytes
    os.remove(os.path.join(path, "1.metadata.json"))
    os.remove(os.path.join(path, "1.codes.pt"))
    ix.index("a", collection, overwrite="resume")
    assert files(path) == a
    # erase removes the .pt files of a PLAID build
    deleted = ix.erase()
    assert "centroids.pt" in deleted and "0.codes.pt" in deleted and os.listdir(path) == []
    with pytest.raises(ValueError, match="index_format"):
        from ravqa_b200.indexer import Indexer
        Indexer(index_format="pq")


@needs_reference
def test_patch_colbert_plaid_drives_the_executor_lines(ref, tmp_path, monkeypatch):
    """FLMR_executor.py:601-617 with ``colbert.Indexer`` replaced by ``patch_colbert(indexer="plaid")``: the
    reference's Run context, ColBERTConfig(nbits=...) and Checkpoint (a stand-in: no weights offline)."""
    import colbert.indexer
    import colbert.modeling.checkpoint as CK
    from colbert.infra import ColBERTConfig, Run, RunConfig
    import ravqa_b200.integration as flmr_b200
    from ravqa_b200 import plaid
    from ravqa_b200.indexer import PlaidIndexer
    monkeypatch.setattr(plaid, "encode", E.encode_torch)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)

    class FakeCheckpoint:
        def __init__(self, name, colbert_config=None):
            pass

        def docFromText(self, docs, bsize=None, keep_dims=True, to_cpu=False, showprogress=False, return_tokens=False):
            return _encode_fn(docs)

    monkeypatch.setattr(CK, "Checkpoint", FakeCheckpoint)
    original = colbert.indexer.Indexer
    passage_contents = ["passage %d" % i for i in range(150)]
    try:
        assert flmr_b200.patch_colbert(searcher=False, scoring=False, ib_loss=False, indexer="plaid")["Indexer"] >= 1
        from colbert import Indexer
        assert Indexer is PlaidIndexer
        IndexerClass = Indexer
        with Run().context(RunConfig(nranks=1, root=str(tmp_path), experiment="temp_index_0")):
            nbits = 8
            config = ColBERTConfig(nbits=nbits, doc_maxlen=512)
            indexer = IndexerClass(checkpoint="a/checkpoint", config=config)
            indexer.index(name=f"temp_index.nbits={nbits}", collection=passage_contents, overwrite=True)
            index_path = indexer.get_index()
        assert index_path == os.path.join(str(tmp_path), "temp_index_0", "indexes", "temp_index.nbits=8")
        meta = json.load(open(os.path.join(index_path, "metadata.json")))
        assert meta["config"]["nbits"] == 8
        assert torch.load(os.path.join(index_path, "0.residuals.pt")).shape[1] == 128
    finally:
        flmr_b200.unpatch_colbert()
    assert colbert.indexer.Indexer is original
    with pytest.raises(ValueError):
        flmr_b200.patch_colbert(searcher=False, scoring=False, ib_loss=False, indexer="pq")
