"""GPU: the paths that put a corpus into HBM, each held against its source at the sizes where its loops and buffers
change over (the model, the writer and the designed corpora: tests/load_fp64.py, pinned by
tests/test_corpus_load_host.py).

a. PLAID decode (``flmr_plaid_decode`` / ``_fp16``) for nbits 1, 2, 4, 8 into bf16 and fp16: the bit layout
   exhaustively, values against float64 through the rounding classifier (subnormal, zero, tiny-norm and overflowing
   rows included), every token of three grid strides and a remainder, and out-of-range codes wherever they sit.
b. A multi-chunk PLAID directory, whole and sharded, in every storage: every stored row read back bitwise, the shard
   ranges, and the merged top-k of the shards bitwise that of the whole corpus.
c. The streamed index load (``from_index``, and ``flmr_corpus_builder_append`` driven directly) across its staging
   ring: every row bitwise, and the scan's scores against float64, where a wrong padding row shows.
d. The host-source create and append across the pack chunks, with the same checks.

The module prints the in-band counts, the largest error / bound ratios and the sizes it reached (run with -s).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import load_fp64 as L
import scan_fp64 as S

pytestmark = pytest.mark.gpu

NBITS = [1, 2, 4, 8]
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
RATIOS, BANDS, SIZES = {}, {}, {}

# c. streamed load: corpora of a little more than two staging buffers; name -> (design kind, aligned, index dtype)
STREAM_ROWS = 600_000
STREAM_CORPORA = {"ragged_bf16": ("ends", False, "bfloat16"), "aligned_bf16": ("straddle", True, "bfloat16"),
                  "ragged_fp16": ("straddle", False, "float16")}
STREAM_SEEDS = {"ragged_bf16": 11, "aligned_bf16": 12, "ragged_fp16": 13}
STREAM_WORLDS = (2, 3)
# d. host source: three pack chunks, then an append of more than one
HOST_ROWS, HOST_APPEND_ROWS, HOST_SEED = 2_200_000, 1_100_000, 21


def chunk_cuts(doclens, period: int) -> list:
    """Passage indices where the chunked layout cuts its files: the passage ends nearest to every ``m P - 1``,
    ``m P``, ``m P + 1``."""
    off = L.offsets(doclens)
    cuts = set()
    for b in range(period, int(off[-1]), period):
        for d in (-1, 0, 1):
            p = int(np.abs(off - (b + d)).argmin())
            if 0 < p < len(doclens):
                cuts.add(p)
    return sorted(cuts)


def append_pieces(n_rows: int, period: int) -> list:
    """Row counts of the direct builder appends: 1, P - 1, P + 1 and the rest, so that buffer changes fall inside a
    call and between calls."""
    pieces = [1, period - 1, period + 1]
    return pieces + [n_rows - sum(pieces)]


def decode_tokens(stride: int) -> int:
    return 3 * stride + stride // 3 + 7


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[load fp64] sizes: %s" % ", ".join("%s=%s" % kv for kv in sorted(SIZES.items())))
    print("[load fp64] decode elements inside the rounding band (of all checked):")
    for k in sorted(BANDS):
        print("[load fp64]   %-22s %d / %d" % (k, *BANDS[k]))
    print("[load fp64] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[load fp64]   %-22s %.3e" % (k, RATIOS[k]))


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


def _band(key, got, y, tag):
    n = L.check_rounding(got, y, tag)
    a, b = BANDS.get(key, (0, 0))
    BANDS[key] = (a + n, b + got.numel())


# ---- a. PLAID decode -------------------------------------------------------------------------------------------------
def _decode(codes, residuals, cent, w, nbits, normalize, dtype, stream=None):
    """(status, out) of one decode call; ``out`` starts as NaN so an unwritten token shows."""
    from ravqa_b200 import _cabi
    n = codes.numel()
    out = torch.full((n, 128), float("nan"), dtype=dtype, device="cuda")
    fn = _cabi.lib().flmr_plaid_decode_fp16 if dtype == torch.float16 else _cabi.lib().flmr_plaid_decode
    st = stream if stream is not None else torch.cuda.current_stream()
    torch.cuda.synchronize()                          # the inputs and the NaN fill are in place on any stream
    rc = fn(C.c_void_p(codes.data_ptr()), C.c_void_p(residuals.data_ptr()), n, C.c_void_p(cent.data_ptr()),
            cent.size(0), C.c_void_p(w.data_ptr()), nbits, 128, int(normalize), C.c_void_p(out.data_ptr()), 0,
            C.c_void_p(st.cuda_stream))
    torch.cuda.synchronize()
    return rc, out


def _cuda(*xs):
    return [x.cuda().contiguous() for x in xs]


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nbits", NBITS)
def test_decode_bit_layout_exhaustive(R, nbits, dtype):
    """Centroids 0 and weights 1 .. 2^nbits (exact in both types), no normalisation: every output is the weight its
    field names.  Token t has every byte t, then every byte position rotated through all values."""
    t = torch.arange(256, dtype=torch.int64)
    j = torch.arange(16 * nbits, dtype=torch.int64)
    res = torch.cat([t[:, None].expand(256, j.numel()), (t[:, None] + j[None, :]) % 256,
                     (t[:, None] * 7 + 3 * j[None, :]) % 256]).to(torch.uint8)
    codes = torch.randint(0, 4, (res.size(0),), dtype=torch.int32, generator=torch.Generator().manual_seed(nbits))
    cent = torch.zeros((4, 128))
    w = torch.arange(1, (1 << nbits) + 1, dtype=torch.float32)
    rc, out = _decode(*_cuda(codes, res, cent, w), nbits, False, DTYPES[dtype])
    assert rc == 0
    want = (L.bucket_index(res, nbits) + 1).double()
    assert torch.equal(out.double().cpu(), want)


def _value_cases(nbits, g):
    """(name, codes, residuals, centroids fp32 (fp16 values), weights, normalize) of the value checks."""
    K = 61
    cent = torch.randn((K, 128), generator=g)
    cent = (cent / cent.norm(dim=1, keepdim=True)).half().float()
    w = L.fixture_weights(nbits, g).half().float()
    cent[K - 1] = -w[0]                 # with all-zero residual bytes (bucket 0 in every dim): v = 0
    cases = []
    # main: three grid strides and a remainder, zero rows at the stride edges, first and last code ids used
    stride = L.decode_stride(torch.cuda.get_device_properties(0).multi_processor_count)
    n = decode_tokens(stride)
    SIZES["decode_stride_tokens"] = stride
    SIZES["decode_tokens"] = n
    codes, res = L.random_codes(n, K - 1, nbits, g)
    zero_at = [0, stride - 1, stride, 2 * stride - 1, 2 * stride, 3 * stride - 1, 3 * stride, n - 1]
    codes[zero_at] = K - 1
    res[zero_at] = 0
    codes[1], codes[n - 2] = 0, K - 2
    cases.append(("main", codes, res, cent, w, True))
    # fp16 subnormal outputs: one dominant component, the rest around 1e-6, weights around 1e-8
    m = 512
    cs = ((torch.rand((64, 128), generator=g) + 0.5) * 1e-6 * torch.where(torch.rand((64, 128), generator=g) < .5, -1, 1))
    cs[torch.arange(64), torch.randint(0, 128, (64,), generator=g)] = 1.0
    ws = torch.sort(1e-8 * torch.randn(1 << nbits, generator=g)).values
    codes, res = L.random_codes(m, 64, nbits, g)
    cases.append(("subnormal", codes, res, cs.half().float(), ws, True))
    # norms below 1e-12: out = v / eps, as F.normalize gives
    wt = 1e-16 * torch.arange(1, (1 << nbits) + 1, dtype=torch.float32)
    codes, res = L.random_codes(m, 4, nbits, g)
    cases.append(("tiny_norm", codes, res, torch.zeros((4, 128)), wt, True))
    # no normalisation near the fp16 range's end: 65504 + 16 is the midpoint that rounds to inf
    co = (60000 + 5504 * torch.rand((8, 128), generator=g)).half().float()
    co[0] = 65504.0
    wo = torch.linspace(-32, 32, 1 << nbits) if nbits > 1 else torch.tensor([15.0, 16.0])
    codes, res = L.random_codes(m, 8, nbits, g)
    cases.append(("overflow", codes, res, co, wo.float(), False))
    return cases


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nbits", NBITS)
def test_decode_values_against_fp64(R, nbits, dtype):
    g = torch.Generator().manual_seed(100 + nbits)
    for name, codes, res, cent, w, norm in _value_cases(nbits, g):
        y = L.decode_fp64(codes, res, cent, w, nbits, normalize=norm)
        rc, out = _decode(*_cuda(codes, res, cent, w), nbits, norm, DTYPES[dtype])
        assert rc == 0, name
        _band("nbits%d %s" % (nbits, dtype), out, y.cuda(), "nbits=%d %s %s" % (nbits, dtype, name))
        if name == "main":
            zero = (codes == cent.size(0) - 1).nonzero().flatten()
            assert zero.numel() >= 8 and (out[zero.cuda()] == 0).all()
        if name == "tiny_norm":
            assert (y.norm(dim=1) < 0.5).all() and (out.double().norm(dim=1) < 0.5).all()   # x / eps, not unit rows


@pytest.mark.parametrize("nbits", [2, 8])
def test_decode_rejects_out_of_range_codes(R, nbits):
    from ravqa_b200 import _cabi
    g = torch.Generator().manual_seed(7)
    K = 9
    stride = L.decode_stride(torch.cuda.get_device_properties(0).multi_processor_count)
    n = stride + 100
    codes, res = L.random_codes(n, K, nbits, g)
    cent = (torch.randn((K, 128), generator=g) * 0.1).half().float()
    w = L.fixture_weights(nbits, g)
    codes[0], codes[-1] = 0, K - 1                    # the end ids are accepted
    y = L.decode_fp64(codes, res, cent, w, nbits).cuda()
    dc, dr, dcent, dw = _cuda(codes, res, cent, w)
    side = torch.cuda.Stream()
    for i, (where, bad) in enumerate([(0, -1), (n - 1, K), (stride + 50, -1), (stride + 50, K), (0, K), (n - 1, -1)]):
        c2 = dc.clone()
        c2[where] = bad
        stream = side if i == 2 else None
        rc, _ = _decode(c2, dr, dcent, dw, nbits, True, torch.bfloat16, stream)
        assert rc == _cabi._header_define("FLMR_ERR_INVALID_ARG"), (where, bad)
        assert "centroid code" in _cabi.lib().flmr_last_error().decode()
        rc, out = _decode(dc, dr, dcent, dw, nbits, True, torch.bfloat16, stream)   # the flag resets
        assert rc == 0, (where, bad)
        L.check_rounding(out, y, "after a rejected call")


# ---- b. multi-chunk PLAID directory ----------------------------------------------------------------------------------
PLAID_CHUNK_PASSAGES = [37, 1, 140, 9, 63]


@pytest.fixture(scope="module")
def plaid_dir(tmp_path_factory):
    nbits, K = 4, 57
    g = torch.Generator().manual_seed(31)
    cent = torch.randn((K, 128), generator=g)
    cent = (cent / cent.norm(dim=1, keepdim=True)).half()
    w = L.fixture_weights(nbits, g)
    cut = torch.sort(torch.randn((1 << nbits) - 1, generator=g)).values
    rng = np.random.default_rng(31)
    chunks = []
    for n in PLAID_CHUNK_PASSAGES:
        dl = rng.integers(1, 181, n)
        codes, res = L.random_codes(int(dl.sum()), K, nbits, g)
        chunks.append((codes, res, dl))
    path = str(tmp_path_factory.mktemp("plaid") / "index")
    L.write_plaid(path, nbits, cent, cut, w, chunks)
    codes = torch.cat([c[0] for c in chunks])
    res = torch.cat([c[1] for c in chunks])
    y = L.decode_fp64(codes, res, cent.float(), w, nbits)
    return path, np.concatenate([c[2] for c in chunks]).astype(np.int32), y


def test_plaid_directory_sharded_loads(R, plaid_dir):
    from ravqa_b200.plaid import plaid_to_flat
    path, dl, y = plaid_dir
    off = L.offsets(dl)
    SIZES["plaid_chunks"] = len(PLAID_CHUNK_PASSAGES)
    whole = {}
    for name, dt in DTYPES.items():                     # the whole directory's decode, held against float64
        tok, d = plaid_to_flat(path, dtype=dt)
        assert d.tolist() == dl.tolist()
        _band("plaid dir %s" % name, tok, y.cuda(), "plaid dir %s" % name)
        whole[name] = tok
    whole["fp8"] = whole["bf16"]
    Q = L.design_rows(3 * 32, 5, negative=False).view(3, 32, 128).float()
    for storage in ("bf16", "fp16", "fp8"):
        full = R.FlatCorpus.from_plaid(path, storage=storage)
        ref_s, ref_p = R.maxsim_topk(full, Q.cuda(), 10)
        for ws in (1, 2, 3, 5):
            ranges = R.shard_ranges(dl, ws)
            shards = [full] if ws == 1 else [R.FlatCorpus.from_plaid(path, rank=r, world_size=ws, storage=storage)
                                               for r in range(ws)]
            tops = []
            for sh, (p0, p1) in zip(shards, ranges):
                tag = "%s ws=%d shard %d" % (storage, ws, p0)
                assert sh.pid_base == p0 and sh.n_passages == p1 - p0 and sh.doclens.tolist() == dl[p0:p1].tolist()
                _readback(sh, whole[storage][off[p0]:off[p1]], tag)
                tops.append(R.maxsim_topk(sh, Q.cuda(), 10))
            ms, mp = R.topk_merge(torch.stack([t[0] for t in tops]), torch.stack([t[1] for t in tops]), 10)
            assert torch.equal(ms, ref_s) and torch.equal(mp, ref_p), (storage, ws)
            for sh in shards:
                if sh is not full:
                    sh.close()
        full.close()


# ---- c / d. read-back and float64 scores of a loaded corpus ----------------------------------------------------------
def _readback(corpus, src: torch.Tensor, tag: str, first: int = 0, rows_per_call: int = 1 << 20):
    """Every stored row of passages ``first ..`` of ``corpus`` (local ids) bitwise ``src`` (their packed rows, in
    the corpus' element type), through ``gather_padded`` in pid chunks."""
    dl = corpus.doclens[first:]
    off = L.offsets(dl)
    src = src.to(corpus.device)
    assert src.size(0) == off[-1], tag
    p = 0
    while p < len(dl):
        nd = 1
        q = p
        while q < len(dl) and (q - p + 1) * max(nd, int(dl[q])) <= rows_per_call:
            nd = max(nd, int(dl[q]))
            q += 1
        q = max(q, p + 1)
        pids = torch.arange(p, q, dtype=torch.int64) + corpus.pid_base + first
        out, mask = corpus.gather_padded(pids)
        got = out[mask.squeeze(-1)]
        want = src[off[p]:off[q]]
        assert got.dtype == want.dtype and torch.equal(got.view(torch.int16), want.view(torch.int16)), (
            "%s: passages %d..%d read back wrong" % (tag, p + first, q + first))
        p = q


def _scores_fp64(Q, D, dl, storage):
    """Float64 scores, amax, rabs of ``Q`` against the packed rows ``D`` (on the GPU, in passage segments of at most
    2^19 rows); fp8: both rounded to e4m3 (torch's conversion, pinned against fp8_oracle on the host)."""
    Q = Q.cuda()
    if storage == "fp8":
        Q = Q.to(torch.float8_e4m3fn).float()
    elif storage == "fp16":
        Q = Q.half().float()
    off = L.offsets(dl)
    parts = []
    for p0, p1, t0, t1 in S._segments(np.asarray(dl), 1 << 19):
        Dc = D[t0:t1].cuda()
        if storage == "fp8":
            Dc = Dc.to(torch.float8_e4m3fn)
        parts.append(S.maxsim_packed(Q, Dc.float().double(), dl[p0:p1]))
        del Dc
    assert off[-1] == D.size(0)
    return [torch.cat([p[i] for p in parts], dim=1) for i in range(3)]


def _check_scores(R, corpus, D, tag):
    """The scan's scores (relu off) of the probe queries within the scan bound of float64: query 0's rows -e0 make
    every stored product negative, so a padding row that is not the passage's last token shows."""
    Q = L.probe_queries()
    s64, amax, rabs = _scores_fp64(Q, D, corpus.doclens, corpus.storage)
    got = R.maxsim_scores(corpus, Q.cuda()).double()
    assert (got[0] < 0).all(), "%s: a passage scores >= 0 against -e0 (a zero padding row?)" % tag
    key = "scan %s" % corpus.storage
    # the fp16 scan keeps the bf16 accumulator model (tests/corpus_model.py)
    bound = S.scan_bound(amax, rabs, Q.size(1), "fp8" if corpus.storage == "fp8" else "bf16")
    S.check_ratio(RATIOS, key, (got - s64).abs(), bound)


# ---- c. streamed builder -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def stream_indexes(tmp_path_factory):
    from ravqa_b200.index_io import finalize_chunked_index, save_flat_chunk, save_flat_index, FORMAT
    P = L.load_constants()["buf_rows"]
    SIZES["stream_buf_rows"] = P
    SIZES["stream_rows"] = STREAM_ROWS
    base = tmp_path_factory.mktemp("stream")
    out = {}
    for name, (kind, aligned, dtype) in STREAM_CORPORA.items():
        dl = L.design_doclens(STREAM_ROWS, P, kind, STREAM_SEEDS[name], aligned)
        tok = L.design_rows(STREAM_ROWS, STREAM_SEEDS[name])
        if dtype == "float16":
            tok = tok.half()
        single = save_flat_index(str(base / name), tok, dl, dtype=dtype)
        out[name] = (dl, tok, {"single": single})
    # the chunked layout of the ragged bf16 corpus: file ends at and +-1 of the buffer multiples
    dl, tok, paths = out["ragged_bf16"]
    cuts = [0] + chunk_cuts(dl, P) + [len(dl)]
    off = L.offsets(dl)
    path = str(base / "ragged_bf16_chunked")
    for c, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        save_flat_chunk(path, c, a, tok[off[a]:off[b]], dl[a:b])
    finalize_chunked_index(path, len(cuts) - 1, FORMAT)
    paths["chunked"] = path
    SIZES["stream_chunk_files"] = len(cuts) - 1
    return out


STREAM_LOADS = [(name, layout, storage)
                for name, (_, _, dtype) in STREAM_CORPORA.items()
                for storage in (("fp16",) if dtype == "float16" else ("bf16", "fp8"))
                for layout in (("single", "chunked") if name == "ragged_bf16" else ("single",))]


@pytest.mark.parametrize("name,layout,storage", STREAM_LOADS)
def test_streamed_index_load(R, stream_indexes, name, layout, storage):
    dl, tok, paths = stream_indexes[name]
    off = L.offsets(dl)
    for ws in (1,) + STREAM_WORLDS:
        ranges = R.shard_ranges(dl, ws)
        for rank, (p0, p1) in enumerate(ranges):
            tag = "%s %s %s ws=%d rank=%d" % (name, layout, storage, ws, rank)
            c = R.FlatCorpus.from_index(paths[layout], rank=rank, world_size=ws, storage=storage)
            assert c.storage == storage and c.pid_base == p0 and c.doclens.tolist() == dl[p0:p1].tolist(), tag
            src = tok[off[p0]:off[p1]]
            _readback(c, src, tag)
            _check_scores(R, c, src, tag)
            c.close()


@pytest.mark.parametrize("name,storage", [("ragged_bf16", "bf16"), ("ragged_bf16", "fp8"),
                                          ("aligned_bf16", "bf16"), ("ragged_fp16", "fp16")])
def test_builder_direct_host_appends(R, stream_indexes, name, storage):
    """``flmr_corpus_builder_append`` from host memory in pieces of 1, P - 1, P + 1 rows and the rest."""
    from ravqa_b200 import _cabi
    from ravqa_b200.corpus import _storage_flag
    Lb = _cabi.lib()
    dl, tok, _ = stream_indexes[name]
    dl = np.ascontiguousarray(dl, dtype=np.int32)
    src = tok.contiguous()
    b = C.c_void_p()
    _cabi.check(Lb.flmr_corpus_builder_create_ex(dl.ctypes.data_as(C.c_void_p), len(dl), 128, 0, 0,
                                                 _storage_flag(storage), C.byref(b)))
    try:
        r0 = 0
        for rows in append_pieces(STREAM_ROWS, L.load_constants()["buf_rows"]):
            _cabi.check(Lb.flmr_corpus_builder_append(b, C.c_void_p(src.data_ptr() + r0 * 256), rows))
            r0 += rows
        h = C.c_void_p()
        _cabi.check(Lb.flmr_corpus_builder_finish(b, C.byref(h), None))
        b = None
    finally:
        if b is not None:
            Lb.flmr_corpus_builder_destroy(b)
    c = R.FlatCorpus._from_handle(h, dl, torch.device("cuda", 0), 0)
    tag = "direct %s %s" % (name, storage)
    _readback(c, src, tag)
    _check_scores(R, c, src, tag)
    c.close()


# ---- d. host-source create and append ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_corpus():
    C_ = L.load_constants()["host_chunk_rows"]
    SIZES["host_chunk_rows"] = C_
    SIZES["host_rows"] = HOST_ROWS
    SIZES["host_append_rows"] = HOST_APPEND_ROWS
    dl = L.design_doclens(HOST_ROWS, C_, "straddle", seed=HOST_SEED)
    dla = L.design_doclens(HOST_APPEND_ROWS, C_, "straddle", seed=HOST_SEED + 1)
    return dl, L.design_rows(HOST_ROWS, HOST_SEED), dla, L.design_rows(HOST_APPEND_ROWS, HOST_SEED + 1)


@pytest.mark.parametrize("storage", ["bf16", "fp16", "fp8"])
def test_host_source_create_and_append(R, host_corpus, storage):
    dl, tok, dla, toka = host_corpus
    dt = torch.float16 if storage == "fp16" else torch.bfloat16
    src, srca = tok.to(dt), toka.to(dt)
    c = R.FlatCorpus(tok, dl, device=0, storage=storage)
    tag = "host %s" % storage
    _readback(c, src, tag)
    _check_scores(R, c, src, tag)
    ids = c.append(toka, dla)
    assert ids.tolist() == list(range(len(dl), len(dl) + len(dla)))
    assert c.n_passages == len(dl) + len(dla)
    _readback(c, torch.cat([src, srca]), tag + " after append")
    _check_scores(R, c, torch.cat([src, srca]), tag + " after append")
    c.close()
