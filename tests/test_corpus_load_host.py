"""CPU: the float64 load model of tests/load_fp64.py pinned before any kernel is judged by it.

* the decode model against the reference's own decode of the four PLAID goldens, bit for bit before normalisation,
  and the reference's fp32 normalised rows inside the band the classifier allows the kernel;
* the PLAID writer reproduces the goldens' files;
* the rounding classifier on hand-picked bf16 / fp16 cases;
* the staging sizes read from the CUDA source, and the designed corpora putting boundaries where the GPU tests
  (tests/test_corpus_load_gpu.py) say they do.
"""
import json
import os

import numpy as np
import pytest
import torch

import load_fp64 as L
import scan_fp64 as S
from helpers import GOLDEN_DIR

NBITS = [1, 2, 4, 8]


def _golden(nbits):
    z = np.load(os.path.join(GOLDEN_DIR, "plaid_nbits%d.npz" % nbits))
    return {k: z[k] for k in z.files}, os.path.join(GOLDEN_DIR, "plaid_nbits%d" % nbits)


@pytest.mark.parametrize("nbits", NBITS)
def test_decode_model_matches_reference(nbits):
    g, _ = _golden(nbits)
    args = (g["codes"], g["residuals"], g["centroids"], g["bucket_weights"], nbits)
    raw = L.decode_fp64(*args, normalize=False)
    assert torch.equal(raw, torch.from_numpy(g["decoded_cpp_raw"]).double())      # decompress_residuals_cpp
    y = L.decode_fp64(*args)
    ref = torch.from_numpy(g["decoded_ref"]).double()                               # fp32 + F.normalize
    assert ((ref - y).abs() <= L.BAND * y.abs()).all()


@pytest.mark.parametrize("nbits", NBITS)
def test_plaid_writer_reproduces_golden_directory(nbits, tmp_path):
    from ravqa_b200.plaid import read_plaid_doclens, read_plaid_metadata
    _, src = _golden(nbits)
    ld = lambda d, n: torch.load(os.path.join(d, n), map_location="cpu")
    cutoffs, weights = ld(src, "buckets.pt")
    with open(os.path.join(src, "doclens.0.json")) as f:
        doclens = json.load(f)
    dst = str(tmp_path / "plaid")
    L.write_plaid(dst, nbits, ld(src, "centroids.pt"), cutoffs, weights,
                  [(ld(src, "0.codes.pt"), ld(src, "0.residuals.pt"), doclens)])
    for name in ("centroids.pt", "0.codes.pt", "0.residuals.pt"):
        a, b = ld(src, name), ld(dst, name)
        assert a.dtype == b.dtype and torch.equal(a, b), name
    for a, b in zip(ld(src, "buckets.pt"), ld(dst, "buckets.pt")):
        assert a.dtype == b.dtype and torch.equal(a, b)
    for name in ("metadata.json", "0.metadata.json", "doclens.0.json"):
        with open(os.path.join(src, name)) as f1, open(os.path.join(dst, name)) as f2:
            assert json.load(f1) == json.load(f2), name
    assert read_plaid_metadata(src) == read_plaid_metadata(dst)
    assert [d.tolist() for d in read_plaid_doclens(src, 1)] == [d.tolist() for d in read_plaid_doclens(dst, 1)]


def _check(got, y, dtype):
    return L.check_rounding(torch.tensor(got, dtype=torch.float64).to(dtype), torch.tensor(y, dtype=torch.float64))


def _fails(got, y, dtype):
    with pytest.raises(AssertionError):
        _check(got, y, dtype)


def test_classifier_hand_cases():
    bf, hf = torch.bfloat16, torch.float16
    # ties to even: 1 + 2^-8 lies halfway between bf16 1 and 1 + 2^-7 (odd); 1 + 3 2^-8 between odd and 1 + 2^-6
    assert _check([1.0], [1 + 2 ** -8], bf) == 1            # a midpoint is inside its own band
    assert _check([1 + 2 ** -7], [1 + 2 ** -8], bf) == 1    # ... so either neighbour passes
    assert _check([1 + 2 ** -6], [1 + 3 * 2 ** -8], bf) == 1
    assert _check([1.0], [1 + 2 ** -11], hf) == 1
    # just inside / just outside the band of the midpoint 1 + 2^-8
    m = 1 + 2 ** -8
    assert _check([1 + 2 ** -7], [m - 0.99 * L.BAND * m], bf) == 1
    _fails([1 + 2 ** -7], [m - 1.01 * L.BAND * m], bf)
    assert _check([1.0], [m - 1.01 * L.BAND * m], bf) == 0
    assert _check([1.0], [m + 0.99 * L.BAND * m], bf) == 1
    _fails([1.0], [m + 1.01 * L.BAND * m], bf)
    _fails([1.0 + 2 ** -6], [1 + 2 ** -7], bf)               # a whole ulp off
    assert _check([-1.5], [-1.5], hf) == 0                    # exact, of either sign
    # fp16 subnormals: steps of 2^-24; a flush to zero fails
    s = 2.0 ** -24
    assert _check([3 * s], [3.2 * s], hf) == 0
    _fails([0.0], [3.2 * s], hf)
    _fails([4 * s], [3.2 * s], hf)
    assert _check([2 * s], [2.5 * s], hf) == 1                # tie to even (inside the band either way)
    assert _check([0.0], [0.4 * s], hf) == 0
    _fails([0.0], [0.6 * s], hf)
    assert _check([2.0 ** -14], [2.0 ** -14 - 0.3 * s], hf) == 0     # largest subnormal rounds up to the normal
    # overflow: 65504 is the largest fp16, 65520 the midpoint to "65536", which rounds to inf (nearest even)
    assert _check([65504.0], [65504.0], hf) == 0
    assert _check([65504.0], [65519.0], hf) == 0
    _fails([float("inf")], [65519.0], hf)
    assert _check([float("inf")], [65520.0], hf) == 1
    assert _check([float("inf")], [65536.0], hf) == 0
    assert _check([-float("inf")], [-65540.0], hf) == 0
    _fails([65504.0], [65540.0], hf)
    assert _check([65536.0], [65520.0], bf) == 0              # bf16 reaches far beyond
    # several elements: the count is the number inside the band
    assert _check([1.0, 1.0, 2.0], [1 + 2 ** -8, 1.0, 2.0], bf) == 1


def test_rounding_neighbours_agree_with_torch_outside_the_band():
    """RN(y) of the classifier equals torch's conversion wherever y is not within the band of a midpoint."""
    g = torch.Generator().manual_seed(3)
    y = torch.randn(200_000, generator=g, dtype=torch.float64) * 10.0 ** torch.randint(-9, 5, (200_000,), generator=g)
    for dt in (torch.bfloat16, torch.float16):
        lo, hi, rn, mid = L.rounding_neighbours(y, dt)
        far = (y - mid).abs() > L.BAND * y.abs()
        assert torch.equal(rn[far], y[far].to(dt).double())
        assert ((lo <= y) & (y < hi) | hi.isinf() | lo.isinf()).all()


def test_torch_e4m3_agrees_with_oracle():
    """The GPU test rounds large corpora to e4m3 with torch's conversion: it equals fp8_oracle's rounding for every
    finite bf16 value within +-448."""
    v = S.finite_bf16_values()
    v = v[v.abs() <= 448]
    assert torch.equal(v.to(torch.float8_e4m3fn).float(), S.e4m3_round(v))


def test_staging_constants():
    k = L.load_constants()
    assert k["dim"] == 128
    assert k["buf_rows"] == 262_144 and k["host_chunk_rows"] == 1_048_576
    assert k["decode_threads"] == 256 and k["decode_blocks_per_sm"] == 16
    assert L.decode_stride(132) == 16_896


def _ends(doclens):
    return set(L.offsets(doclens).tolist())


def _straddles(doclens, b):
    o = L.offsets(doclens)
    p = int(np.searchsorted(o, b, side="right")) - 1
    return o[p] <= b - 2 and o[p + 1] >= b + 2


@pytest.mark.parametrize("kind", ["ends", "straddle"])
@pytest.mark.parametrize("aligned", [False, True])
def test_designed_corpora(kind, aligned):
    import test_corpus_load_gpu as G
    period = L.load_constants()["buf_rows"]
    dl = L.design_doclens(G.STREAM_ROWS, period, kind, seed=1, aligned=aligned)
    assert dl.min() >= 1 and int(dl.sum()) == G.STREAM_ROWS
    assert G.STREAM_ROWS > 2 * period                       # the ring fills both buffers and wraps
    ends, step = _ends(dl), 4 if aligned else 1
    for b in range(period, G.STREAM_ROWS, period):
        if kind == "ends":
            assert {b - step, b, b + step} <= ends
        else:
            assert _straddles(dl, b)
    if aligned:
        assert (dl % 4 == 0).all()
    else:
        assert set((dl % 4).tolist()) == {0, 1, 2, 3}
        assert dl[0] == 1 and dl[-3:].tolist() == [1, 2, 3]


def test_gpu_test_corpora_reach_their_boundaries():
    """What tests/test_corpus_load_gpu.py claims about its corpora holds for the sizes in the CUDA source."""
    import test_corpus_load_gpu as G
    k = L.load_constants()
    P, C = k["buf_rows"], k["host_chunk_rows"]
    # streamed: every corpus spans more than two staging buffers; the chunked layout's file ends sit at and +-1 of
    # buffer multiples
    for name, (kind, aligned, _dt) in G.STREAM_CORPORA.items():
        dl = L.design_doclens(G.STREAM_ROWS, P, kind, G.STREAM_SEEDS[name], aligned)
        assert int(dl.sum()) > 2 * P
        cuts = G.chunk_cuts(dl, P)
        rows = L.offsets(dl)[cuts]
        if kind == "ends" and not aligned:
            assert {P - 1, P, P + 1, 2 * P - 1, 2 * P, 2 * P + 1} <= set(rows.tolist())
        for ws in G.STREAM_WORLDS:
            from ravqa_b200.sharded import shard_ranges
            r = shard_ranges(dl, ws)
            assert all(p1 > p0 for p0, p1 in r)
            starts = L.offsets(dl)[[p0 for p0, _ in r[1:]]]
            files = set(rows.tolist()) | {0}
            assert not set(starts.tolist()) <= files         # some shard starts inside a file: a non-zero offset
    # direct appends: buffer changes inside and between calls
    pieces = G.append_pieces(G.STREAM_ROWS, P)
    assert pieces[:3] == [1, P - 1, P + 1] and sum(pieces) == G.STREAM_ROWS and pieces[3] > 0
    # host source: three pack chunks, each boundary straddled; the appended block alone spans a chunk and more
    dl = L.design_doclens(G.HOST_ROWS, C, "straddle", seed=G.HOST_SEED)
    assert int(dl.sum()) > 2 * C
    for b in range(C, G.HOST_ROWS, C):
        assert _straddles(dl, b)
    dla = L.design_doclens(G.HOST_APPEND_ROWS, C, "straddle", seed=G.HOST_SEED + 1)
    assert int(dla.sum()) > C
    # decode: three full grid strides and a remainder, on any device the test meets
    for sms in (114, 132):
        s = L.decode_stride(sms)
        n = G.decode_tokens(s)
        assert 3 * s < n < 4 * s
