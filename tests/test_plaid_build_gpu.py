"""GPU: flmr_plaid_encode against float64 and the numpy restatement (tests/plaid_encode_oracle.py) at its tile, CTA
and centroid-tile boundaries, and whole PLAID builds (Indexer(index_format="plaid")) opened by this library's three
PLAID paths and its Searcher."""
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest
import torch

import plaid_encode_oracle as E
from abi_contract import SENTINEL_BITS, Guarded, bits, ptr
from helpers import GOLDEN_DIR
from oracle import maxsim_oracle as O

pytestmark = pytest.mark.gpu

ROWS = 256                     # token rows per tile of the kernel (132 CTAs on an H100 SXM)


def _case(n, K, seed, dup=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1).half()
    c = torch.nn.functional.normalize(torch.randn(K, 128, generator=g), dim=-1)
    if dup:                                     # copies of earlier centroids: exact ties the lower index must win
        idx = torch.randint(0, K, (dup,), generator=g)
        c[torch.randint(0, K, (dup,), generator=g)] = c[idx].clone()
    return x, c.half()


def _cutoffs(x, c, nbits):
    codes = E.assign(x.numpy(), c.numpy())
    res = (x.float() - c.float()[codes.astype(np.int64)]).half().float()
    q = torch.arange(0, 1 << nbits) * (1 / (1 << nbits))
    return res.quantile(q[1:]), res.quantile(q + 0.5 / (1 << nbits))


def _f64_check(x, c, codes, best):
    """Codes equal the float64 arg-max wherever the top-two gap exceeds the fp32 accumulation bound; elsewhere the
    winner's float64 score is within that bound of the maximum.  Scores computed on the GPU in float64."""
    xd, cd = x.cuda().double(), c.cuda().double()
    bound = 2 * 128 * 2.0 ** -24 * xd.norm(dim=1) * cd.norm(dim=1).max() + 1e-30
    codes = codes.long()
    for a in range(0, x.size(0), 2048):
        s = xd[a:a + 2048] @ cd.T
        top2 = s.topk(min(2, c.size(0)), dim=1)
        want = s.argmax(dim=1)                                       # first maximum: the lowest index
        gap = top2.values[:, 0] - (top2.values[:, 1] if c.size(0) > 1 else -np.inf)
        b = bound[a:a + 2048]
        mine = s.gather(1, codes[a:a + 2048, None])[:, 0]
        clear = gap > 2 * b
        assert torch.equal(codes[a:a + 2048][clear], want[clear])
        assert bool(((top2.values[:, 0] - mine) <= 2 * b).all())
        assert bool(((best[a:a + 2048].double() - mine).abs() <= b).all())


def _encode(x, c, cutoffs, nbits):
    from ravqa_b200 import plaid
    return plaid.encode(x.cuda(), c.cuda(), None if cutoffs is None else cutoffs.cuda(), nbits=nbits, return_best=True)


# (n, K, nbits): n at and around the token tile and the CTA count, K at and around the centroid tile and large
CASES = [(1, 1, 2), (255, 127, 1), (256, 128, 4), (257, 129, 8), (ROWS * 132 - 1, 300, 2), (ROWS * 132 + 1, 129, 1),
         (3000, 65536, 4), (700, 131072, 8), (ROWS * 133, 1000, 8), (5000, 4096, 2)]


@pytest.mark.parametrize("n,K,nbits", CASES)
def test_encode_against_float64_and_the_restatement(n, K, nbits):
    x, c = _case(n, K, seed=n + K + nbits, dup=min(K // 4, 50))
    cutoffs, weights = _cutoffs(x[:2000], c, nbits)
    codes, res, best = _encode(x, c, cutoffs, nbits)
    torch.cuda.synchronize()
    _f64_check(x, c, codes, best)
    # residual bytes are the restatement's given the kernel's codes
    want = E.residual_bytes(x.numpy(), c.numpy(), codes.cpu().numpy(), cutoffs.numpy(), nbits)
    assert np.array_equal(res.cpu().numpy(), want)
    # the decode of what was encoded is C_code + weight[bucket] exactly
    from ravqa_b200 import _cabi
    dec = torch.empty((n, 128), dtype=torch.float16, device="cuda")
    cf, wf = c.float().cuda(), weights.float().cuda()
    _cabi.check(_cabi.lib().flmr_plaid_decode_fp16(ptr(codes), ptr(res), n, ptr(cf), K, ptr(wf), nbits, 128, 0,
                                                   ptr(dec), 0, None))
    want_dec = O.plaid_decode(codes.cpu().numpy(), res.cpu().numpy(), c.float().numpy(), weights.numpy(), nbits,
                              normalize=False)
    assert np.array_equal(dec.cpu().numpy(), want_dec.astype(np.float16))
    # assignment only: identical codes
    a_codes, a_res, a_best = _encode(x, c, None, nbits)
    assert a_res is None and torch.equal(a_codes, codes) and torch.equal(a_best, best)


def test_duplicate_centroids_go_to_the_lowest_index():
    x, c = _case(600, 300, seed=1)
    c[200:300] = c[0:100]                       # centroids 200..299 repeat 0..99 exactly
    c[150] = c[140]
    codes, _, _ = _encode(x, c, None, 2)
    codes = codes.cpu()
    assert not bool(((codes >= 200) | (codes == 150)).any())
    # a row equal to a duplicated centroid scores the same against both copies
    x2 = c[[0, 140, 250]].clone()
    codes2, _, _ = _encode(x2, c, None, 2)
    assert codes2.cpu().tolist() == [0, 140, 50]


def test_encode_matches_the_reference_codec_golden():
    """The committed golden of the reference's own ResidualCodec (tests/golden/make_golden_plaid_encode.py)."""
    z = np.load(os.path.join(GOLDEN_DIR, "plaid_encode.npz"))
    for nbits in (1, 2, 4, 8):
        x = torch.from_numpy(z["x_%d" % nbits])
        c = torch.from_numpy(z["centroids_%d" % nbits])
        cut = torch.from_numpy(z["cutoffs_%d" % nbits])
        codes, res, _ = _encode(x, c, cut, nbits)
        assert np.array_equal(codes.cpu().numpy(), z["codes_%d" % nbits])
        same = (res.cpu().numpy() == z["residuals_%d" % nbits]).all(axis=1)
        assert bool((same | z["straddle_%d" % nbits]).all()) and same.any()


def test_capture_and_replay_in_a_cuda_graph():
    from ravqa_b200 import plaid
    x, c = _case(3000, 1000, seed=3)
    cut, _ = _cutoffs(x, c, 2)
    xg, cg, cutg = x.cuda(), c.cuda(), cut.cuda()
    want = plaid.encode(xg, cg, cutg, nbits=2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plaid.encode(xg, cg, cutg, nbits=2)                  # sets the kernel's shared-memory limit outside capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = plaid.encode(xg, cg, cutg, nbits=2)
    x2, _ = _case(3000, 1000, seed=4)
    xg.copy_(x2.cuda())
    graph.replay()
    torch.cuda.synchronize()
    direct = plaid.encode(x2.cuda(), cg, cutg, nbits=2)
    assert torch.equal(out[0], direct[0]) and torch.equal(out[1], direct[1])
    assert not torch.equal(out[0], want[0])


def test_stream_conventions_and_guard_bands():
    """Outputs inside guard bands: every element written, nothing outside; the call on a side stream gated behind an
    event gives the bits of the plain call."""
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    n, K, nbits = 1000, 513, 4
    x, c = _case(n, K, seed=9)
    cut, _ = _cutoffs(x, c, nbits)
    xg, cg, cutg = x.cuda(), c.cuda(), cut.cuda()
    outs = [Guarded((n,), torch.int32), Guarded((n, 16 * nbits), torch.uint8), Guarded((n,), torch.float32)]
    side = torch.cuda.Stream()
    gate = torch.cuda.Event()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda._sleep(50_000_000)                               # the current stream is busy when the gate is recorded
    gate.record()
    side.wait_event(gate)
    _cabi.check(L.flmr_plaid_encode(ptr(xg), n, ptr(cg), K, ptr(cutg), nbits, ptr(outs[0].out), ptr(outs[1].out),
                                    ptr(outs[2].out), 0, C.c_void_p(side.cuda_stream)))
    side.synchronize()
    from ravqa_b200 import plaid
    plain = plaid.encode(xg, cg, cutg, nbits=nbits, return_best=True)
    for g, p in zip(outs, plain):
        # a packed residual byte may equal the sentinel: those elements are only compared
        g.check(written=bits(p) != SENTINEL_BITS[p.dtype], tag=str(p.dtype))
        assert torch.equal(g.out, p)


# ---- whole builds ---------------------------------------------------------------------------------------------------
def _embed(text):
    g = torch.Generator().manual_seed(zlib.crc32(text.encode()))
    n = 20 + zlib.crc32(text.encode()) % 40
    # clustered rows: 64 topic directions plus noise, as encoder outputs are
    topics = torch.nn.functional.normalize(torch.randn(64, 128, generator=torch.Generator().manual_seed(0)), dim=-1)
    t = topics[torch.randint(0, 64, (n,), generator=g)]
    return torch.nn.functional.normalize(t + 0.5 * torch.randn(n, 128, generator=g) / 128 ** 0.5, dim=-1)


def _encode_fn(passages):
    embs = [_embed(p) for p in passages]
    return torch.cat(embs), [e.size(0) for e in embs]


COLLECTION = ["passage %d" % i for i in range(2000)]


def _files(p):
    return {f: open(os.path.join(p, f), "rb").read() for f in sorted(os.listdir(p))}


def _build(root, name, **kw):
    from ravqa_b200.indexer import Indexer
    ix = Indexer(encode_fn=_encode_fn, index_root=str(root), chunksize=600, index_format="plaid", nbits=2, **kw)
    return ix, ix.index(name, COLLECTION, overwrite=True)


def _two_rank_worker(rank, port, root):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    torch.cuda.set_device(0)
    from ravqa_b200.indexer import Indexer
    Indexer(encode_fn=_encode_fn, index_root=root, chunksize=600, index_format="plaid", nbits=2, rank=rank,
            nranks=2).index("two", COLLECTION, overwrite=True)
    dist.barrier()
    dist.destroy_process_group()


def test_builds_are_byte_identical_across_runs_ranks_and_resume(tmp_path):
    import socket
    import torch.multiprocessing as mp
    ix, path = _build(tmp_path, "a")
    _, path_b = _build(tmp_path, "b")
    a = _files(path)
    assert a == _files(path_b)
    sock = socket.socket()
    sock.bind(("127.0.0.1", 0))
    port = sock.getsockname()[1]
    sock.close()
    mp.spawn(_two_rank_worker, args=(port, str(tmp_path)), nprocs=2, join=True)
    assert _files(os.path.join(str(tmp_path), "two")) == a
    os.remove(os.path.join(path, "2.metadata.json"))
    os.remove(os.path.join(path, "ivf.pid.pt"))
    ix.index("a", COLLECTION, overwrite="resume")
    assert _files(path) == a


def test_built_index_opens_everywhere_and_finds_planted_queries(tmp_path):
    import ravqa_b200 as R
    from ravqa_b200.corpus import FlatCorpus
    _, path = _build(tmp_path, "idx")
    meta = json.load(open(os.path.join(path, "metadata.json")))
    assert meta["num_embeddings"] == sum(_encode_fn(COLLECTION)[1])
    resident = FlatCorpus.from_plaid(path, device=0)
    host = FlatCorpus.from_plaid(path, device=0, residency="host")
    packed = FlatCorpus.from_plaid(path, device=0, residency="host", compressed=True)
    pids = [3, 777, 1999]
    Q = torch.stack([torch.nn.functional.pad(_embed(COLLECTION[p]), (0, 0, 0, 64 - _embed(COLLECTION[p]).size(0)))
                     for p in pids]).cuda()
    results = []
    for corpus in (resident, host, packed):
        s, p = R.maxsim_topk(corpus, Q, 5)
        assert p[:, 0].cpu().tolist() == pids
        results.append((s.cpu(), p.cpu()))
        corpus.close()
    assert all(torch.equal(results[0][1], r[1]) for r in results[1:])
    searcher = R.Searcher(index=path)
    ranking = searcher._search_all_Q(None, Q.cpu(), k=3).todict()
    assert [v[0][0] for v in ranking.values()] == pids


def test_executor_index_lines_with_the_plaid_indexer(tmp_path):
    """FLMR_executor.py:601-617 with the class patch_colbert(indexer="plaid") installs as colbert.Indexer."""
    from ravqa_b200 import ColBERTConfig, Run, RunConfig
    from ravqa_b200.indexer import PlaidIndexer

    class _Self:
        config = type("C", (), {"ckpt_dir": str(tmp_path)})()
        model_config = {"nbits": 8, }
        IndexerClass = PlaidIndexer
    self = _Self()
    dataloader_idx = 0
    get_world_size = lambda: 1                                          # noqa: E731
    passage_contents = COLLECTION[:300]
    with Run().context(RunConfig(nranks=get_world_size(), root=self.config.ckpt_dir, experiment=f"temp_index_{dataloader_idx}")):
        nbits = self.model_config.get("nbits", 2)
        config = ColBERTConfig(
            nbits=nbits,
            doc_maxlen=512,
        )
        custom_collection = passage_contents
        indexer = self.IndexerClass(checkpoint=None, config=config)
        indexer.encode_fn = _encode_fn                                  # the document encoder stays out of scope
        indexer.index(name=f"temp_index.nbits={nbits}", collection=custom_collection, overwrite=True)
        index_path = indexer.get_index()
        del indexer
    assert index_path == os.path.join(str(tmp_path), "temp_index_0", "indexes", "temp_index.nbits=8")
    assert json.load(open(os.path.join(index_path, "metadata.json")))["config"]["nbits"] == 8
    assert torch.load(os.path.join(index_path, "0.residuals.pt")).shape[1] == 128
