"""GPU: the training / re-scoring path on fp16 documents — the _fp16 arg-max (warp-MMA and wgmma) and backward kernels
against the float64 restatement of tests/train_fp64.py, applied to the fp16 operands, and every consumer that reaches
them through the selection rule of ``maxsim._train_operands`` (fp16 documents: both operands in fp16).

* Exact read-backs: every finite fp16 value as documents and as queries against one-hot rows; winners are the planted
  tokens.  The fp16 subnormals kept are counted.
* The float64 grid: the pairwise covering of the bf16 training grid's factors, with full 11-bit mantissas.
* Cross-type identity: on inputs exact in bf16 and fp16, the fp16 route is bitwise the bf16 route.
* End to end: colbert_score (all pairs, aligned, flipr), in_batch_negatives_loss (fused and return_scores), cross-rank
  negatives on two gloo ranks, a graphed loss step, the exhaustive FlatCorpus branch, the reference's operands (fp16
  D, fp32 Q) against float64 compute_ib_loss_new on both routes, and retrieve_and_rescore on an fp16 Searcher.

With a debug library (``FLMR_MAXSIM_LIB=.../libflmr_maxsim_debug.so``) the read-backs and the grid also run the SIMT
twin (``FLMR_ARGMAX_SIMT=1``).  Largest error / bound ratios and the recorded numbers print at the end (run with -s)."""
import os
import socket

import numpy as np
import pytest
import torch

import scan_fp64 as S
import train_fp64 as T

pytestmark = pytest.mark.gpu

RATIOS = {}
REPORT = []
C, U = T.C_BOUND, T.U
DEBUG_LIB = os.environ.get("FLMR_MAXSIM_LIB", "").endswith("_debug.so")
# (arg-max path, SIMT twin): path 1 = warp-MMA kernel, 2 = wgmma kernel; the SIMT twin needs a debug library
PATHS = [(1, False), (2, False)] + ([(1, True)] if DEBUG_LIB else [])


def _check(name, err, bound):
    err, bound = err.double().reshape(-1), bound.double().reshape(-1)
    assert not torch.isnan(err).any(), name
    if err.numel() == 0:
        return
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    worst = int(ratio.argmax())
    r = float(ratio[worst])
    RATIOS[name] = max(RATIOS.get(name, 0.0), r)
    assert r <= 1.0, "%s: error %.3e > bound %.3e (ratio %.3g)" % (name, err[worst], bound[worst], r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\n[fp16 train] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[fp16 train]   %-30s %.3e" % (k, RATIOS[k]))
    for line in REPORT:
        print("[fp16 train] " + line)


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


@pytest.fixture()
def path(R, monkeypatch):
    """``path((kernel, simt))`` selects the arg-max kernel (and the SIMT twin) for the rest of the test."""
    from ravqa_b200 import _cabi
    L = _cabi.lib()

    def select(p):
        kernel, simt = p
        _cabi.check(L.flmr_debug_set_argmax_path(kernel))
        if simt:
            monkeypatch.setenv("FLMR_ARGMAX_SIMT", "1")
        else:
            monkeypatch.delenv("FLMR_ARGMAX_SIMT", raising=False)
    yield select
    L.flmr_debug_set_argmax_path(0)


def f16_rows(shape, norm=None, generator=None):
    """Random fp16 rows ``[..., 128]`` (fp16 tensor): unit rows, or rows of norm uniform in ``norm = (lo, hi)``, rounded
    to fp16 — full 11-bit mantissas, mixed signs."""
    x = torch.nn.functional.normalize(torch.randn(*shape, generator=generator).float(), dim=-1)
    if norm is not None:
        lo, hi = norm
        x = x * (lo + (hi - lo) * torch.rand(*shape[:-1], 1, generator=generator))
    return x.half()


def _make(B, nq, n_total, nd, mask_kind, norm, seed):
    g = torch.Generator().manual_seed(seed)
    nrm = None if norm == "unit" else (4.0, 30.0)
    Q, D = f16_rows((B, nq, 128), nrm, g), f16_rows((n_total, nd, 128), nrm, g)
    mask = T.make_mask(mask_kind, n_total, nd, g)
    tie = None
    live = torch.nonzero(mask[0]).flatten()
    if live.numel() >= 2:
        a, b = int(live[0]), int(live[-1])       # an exact tie: query 0's row 0 asks for document 0's token a, twice
        D[0, b] = D[0, a]
        Q[0, 0] = D[0, a]
        tie = (a, b)
    return Q.cuda(), D.cuda(), mask.cuda(), tie


def _check_forward(Q, D, mask, arg, rowmax, r, tie, tag):
    a64, r64, A = T.argmax_rowmax(Q, D, mask, r)
    empty = torch.isinf(r64)
    assert (arg[empty] == -1).all() and torch.isneginf(rowmax[empty]).all(), tag
    assert (arg[~empty] >= 0).all(), tag
    bound, fin = C * U * A, ~empty
    _check("argmax rowmax", (rowmax.double() - r64).abs()[fin], bound[fin])
    s_win, unmasked = T.winner_scores(Q, D, mask, arg, r)
    assert unmasked[fin].all(), "%s: a winner on a masked token" % tag
    _check("argmax winner score", (r64 - s_win)[fin], bound[fin])
    if tie is not None:
        first = arg[:, 0] if r is None else arg[0, 0]
        assert (first != tie[1]).all(), "%s: the later copy of a tied token won" % tag


def _check_backward(Q, D, mask, arg, r, need, seed, tag):
    from ravqa_b200.maxsim import maxsim_backward, maxsim_backward_grouped
    B, P = arg.shape[:2]
    g = torch.randn((B, P), generator=torch.Generator().manual_seed(seed)).float()
    g[:, ::3] = 0.0
    g = g.cuda()
    need_dq, need_dd = need in ("both", "dq"), need in ("both", "dd")
    fn = maxsim_backward if r is None else maxsim_backward_grouped
    dq, dd = fn(Q, D, arg, g, need_dq=need_dq, need_dd=need_dd)
    assert (dq is None) == (not need_dq) and (dd is None) == (not need_dd), tag
    dQ64, dD64, dq_abs, dd_abs, cnt = T.backward(Q, D, arg, g, r)
    if need_dq:
        assert dq.dtype == torch.float32
        _check("dQ", (dq.double() - dQ64).abs(), C * U * P * dq_abs)
    if need_dd:
        _check("dD", (dd.double() - dD64).abs(), C * U * cnt[..., None] * dd_abs)
        assert (dd[~mask] == 0).all() and (dd[cnt == 0] == 0).all(), "%s: gradient on a masked / losing token" % tag


def test_selection_rule(R):
    """fp16 documents take the fp16 kernels with the query converted to fp16; bf16 and fp32 documents the bf16 ones."""
    from ravqa_b200.maxsim import _train_operands
    Q = torch.randn(2, 3, 128, device="cuda")
    for dt, want in ((torch.float16, torch.float16), (torch.bfloat16, torch.bfloat16), (torch.float32, torch.bfloat16)):
        q, d = _train_operands(Q, torch.randn(4, 5, 128, device="cuda").to(dt))
        assert q.dtype == d.dtype == want and torch.equal(q, Q.to(want)), dt
    q, d = _train_operands(Q.half(), torch.randn(4, 5, 128, device="cuda", dtype=torch.bfloat16))
    assert q.dtype == d.dtype == torch.bfloat16


# ---- read-backs ----------------------------------------------------------------------------------------------------
def finite_f16_values() -> torch.Tensor:
    """Every finite fp16 value (63,488 bit patterns = 496 rows of 128), as float32, in bit-pattern order."""
    x = torch.arange(1 << 16, dtype=torch.int32).to(torch.int16).view(torch.float16).float()
    return x[torch.isfinite(x)].view(496, 128)


def _bits(x):
    return x.float().contiguous().view(torch.int32)


def _readback(tag, got, src):
    """``got`` is bitwise ``src``, but for a zero, which may read back as either zero (the sign of a sum of zero products
    is the accumulator's business); an fp16 subnormal comes back as itself or +-0.  Returns the subnormals kept."""
    got, want = got.cpu(), src.clone()
    sub = (src != 0) & (src.abs() < 2.0 ** -14)
    same = (_bits(got) == _bits(want)) | ((want == 0) & (got == 0))
    bad = ~same & ~sub
    assert not bad.any(), "%s: %d values differ, e.g. %s -> %s" % (tag, int(bad.sum()), src[bad][:4].tolist(),
                                                                     got[bad][:4].tolist())
    kept, flushed = int((sub & same).sum()), int((sub & (got == 0)).sum())
    assert kept + flushed == int(sub.sum()), "%s: a subnormal came back as neither itself nor +0" % tag
    REPORT.append("%s: fp16 subnormals kept %d of %d" % (tag, kept, int(sub.sum())))
    return kept


@pytest.mark.parametrize("p", PATHS, ids=lambda p: "path%d%s" % (p[0], "-simt" if p[1] else ""))
def test_readback_every_f16_value_as_documents(R, path, p):
    """Document i holds row i of the values at token i % 5 (its other tokens masked, holding 60000); query token k is
    the one-hot e_k: rowmax[0, i, k] is the value, the winner token i % 5."""
    from ravqa_b200.maxsim import maxsim_argmax
    V = finite_f16_values()
    n, nd = V.size(0), 5
    D = torch.full((n, nd, 128), 60000.0)
    mask = torch.zeros((n, nd), dtype=torch.bool)
    planted = torch.arange(n) % nd
    D[torch.arange(n), planted] = V
    mask[torch.arange(n), planted] = True
    path(p)
    arg, rowmax = maxsim_argmax(torch.eye(128, device="cuda").half()[None], D.half().cuda(), mask.cuda(),
                                return_rowmax=True)
    assert (arg[0].cpu() == planted[:, None]).all()
    kept = _readback("documents path%d%s" % p, rowmax[0], V)
    assert kept == int(((V != 0) & (V.abs() < 2.0 ** -14)).sum())     # products with 1.0 keep every subnormal


@pytest.mark.parametrize("p", PATHS, ids=lambda p: "path%d%s" % (p[0], "-simt" if p[1] else ""))
def test_readback_every_f16_value_as_queries(R, path, p):
    """Query rows are the values; document k is the one-hot e_k at token k % 3 (the others masked): rowmax[0, k, i] is
    value [i, k], the winner token k % 3."""
    from ravqa_b200.maxsim import maxsim_argmax
    V = finite_f16_values()
    nd = 3
    D = torch.full((128, nd, 128), -60000.0)
    mask = torch.zeros((128, nd), dtype=torch.bool)
    planted = torch.arange(128) % nd
    D[torch.arange(128), planted] = torch.eye(128)
    mask[torch.arange(128), planted] = True
    path(p)
    arg, rowmax = maxsim_argmax(V.half().cuda()[None], D.half().cuda(), mask.cuda(), return_rowmax=True)
    assert (arg[0].cpu() == planted[:, None]).all()
    kept = _readback("queries path%d%s" % p, rowmax[0].T, V)
    assert kept == int(((V != 0) & (V.abs() < 2.0 ** -14)).sum())


# ---- the float64 grid ------------------------------------------------------------------------------------------------
GRID = T.argmax_grid()


@pytest.mark.parametrize("ci", range(len(GRID)), ids=lambda i: "c%03d" % i)
def test_argmax_and_backward_grid(R, path, ci):
    """One case of the bf16 grid's pairwise covering, on fp16 operands: both kernels (forced), both forms, every mask
    kind, unit and wide rows; the backward on the kernel's own winners."""
    from ravqa_b200.maxsim import maxsim_argmax, maxsim_argmax_grouped
    c = GRID[ci]
    B, nq, nd, n = c["B"], c["nq"], c["nd"], c["n_docs"]
    grouped = c["form"] == "grouped"
    Q, D, mask, tie = _make(B, nq, B * n if grouped else n, nd, c["mask"], c["norm"], seed=5000 + ci)
    for p in [(c["path"], False)] + ([(1, True)] if DEBUG_LIB and c["path"] == 1 else []):
        path(p)
        if grouped:
            arg, rowmax = maxsim_argmax_grouped(Q, D, mask, n, return_rowmax=True)
        else:
            arg, rowmax = maxsim_argmax(Q, D, mask, return_rowmax=True)
        tag = "case %d %s simt=%s" % (ci, c, p[1])
        assert arg.shape == (B, n, nq), tag
        r = n if grouped else None
        _check_forward(Q, D, mask, arg, rowmax, r, tie, tag)
        _check_backward(Q, D, mask, arg, r, ("both", "dq", "dd")[ci % 3], ci, tag)


# ---- cross-type identity ---------------------------------------------------------------------------------------------
def _exact_rows(shape, g):
    """k / 256 for integers |k| <= 255: exact in bf16 and fp16 (normal range), and every 128-term dot product of two such
    rows is exact in fp32, whatever the order of its additions."""
    return torch.randint(-255, 256, shape, generator=g).float() / 256


@pytest.mark.parametrize("kernel", [1, 2])
def test_fp16_route_is_bitwise_the_bf16_route_on_exact_inputs(R, path, kernel):
    from ravqa_b200.maxsim import ib_loss_head, maxsim_argmax, maxsim_backward
    g = torch.Generator().manual_seed(kernel)
    B, nq, n, nd, nway = 4, 130, 8, 140, 2
    Q, D = _exact_rows((B, nq, 128), g).cuda(), _exact_rows((n, nd, 128), g).cuda()
    D[:, 7] = D[:, 3]                                          # ties: the lower token must win on both routes
    mask = T.make_mask("holes", n, nd, g).cuda()
    grad = (torch.randint(-8, 9, (B, n), generator=g).float() / 8).cuda()    # exact: dD's atomics add exactly
    path((kernel, False))
    out = {}
    for dt in (torch.bfloat16, torch.float16):
        arg, rowmax = maxsim_argmax(Q.to(dt), D.to(dt), mask, return_rowmax=True)
        dq, dd = maxsim_backward(Q.to(dt), D.to(dt), arg, grad)
        _, loss, ds = ib_loss_head(rowmax, nway)
        out[dt] = (arg, rowmax, dq, dd, loss, ds)
    for name, a, b in zip(("arg", "rowmax", "dQ", "dD", "loss", "dscores"), out[torch.bfloat16], out[torch.float16]):
        assert torch.equal(a, b), name


# ---- end to end --------------------------------------------------------------------------------------------------------
def _grads_and_scores(fn, Q, D, m):
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    out = fn(Qg, Dg, m)
    return out, Qg, Dg


def test_colbert_score_all_pairs_aligned_and_flipr(R):
    """Values against float64 of the fp16 operands (the fp32 query converted to fp16), gradients in the inputs' dtypes."""
    from types import SimpleNamespace
    from ravqa_b200.maxsim import maxsim_argmax
    g = torch.Generator().manual_seed(11)
    n, nd = 6, 90
    Q = f16_rows((1, 80, 128), None, g).float().cuda()
    D = f16_rows((n, nd, 128), None, g).cuda()
    mask = T.make_mask("prefix", n, nd, g).cuda()
    w = torch.linspace(-1, 1, n, device="cuda")
    for form in ("all", "aligned", "flipr"):
        Qf = Q.expand(n, -1, -1).contiguous() if form == "aligned" else Q
        cfg = SimpleNamespace(interaction="flipr", query_maxlen=64) if form == "flipr" else None
        Qg, Dg = Qf.clone().requires_grad_(True), D.clone().requires_grad_(True)
        s = R.colbert_score(Qg, Dg, mask.unsqueeze(-1), cfg)
        (s * w).sum().backward()
        assert Qg.grad.dtype == torch.float32 and Dg.grad.dtype == torch.float16, form
        Q16 = Q.half()
        _, rowmax, A = T.argmax_rowmax(Q16, D, mask)
        karg, krow = maxsim_argmax(Q16, D, mask, return_rowmax=True)     # the kernel's own winners and selection
        if form == "flipr":
            _, sel = T.flipr_select(krow[0], karg[0])
            keep = (sel >= 0).double()
            s64 = (rowmax[0] * keep).sum(-1)
            bound = C * U * (A[0] * keep).sum(-1) + 80 * U * rowmax[0].abs().sum(-1)
        else:
            s64, bound = T.maxsim_exact(Q16, D, mask)
            s64, bound, sel = s64[0], bound[0], karg[0]
        _check("colbert_score " + form, (s.detach().double() - s64).abs(), bound)
        dQ64, dD64, dq_abs, dd_abs, cnt = T.backward(Q16, D, sel[None], w[None])
        dq = Qg.grad.sum(0, keepdim=True) if form == "aligned" else Qg.grad
        # the returned gradients are rounded once to the inputs' dtypes (fp16 for dD)
        _check("colbert_score dQ " + form, (dq.double() - dQ64).abs(), C * U * n * dq_abs)
        _check("colbert_score dD " + form, (Dg.grad.double() - dD64).abs(),
               C * U * cnt[..., None] * dd_abs + 2.0 ** -11 * dD64.abs() + 2.0 ** -25)


def _ib_reference(Q, D, mask, nway, label0=0):
    """Float64 compute_ib_loss_new on the operands ``Q`` (as given: fp16 for the fp16 route) and fp16 ``D``, through the
    fp16 kernels' own winners (ties cannot blur the check).  Returns (loss, scores, their bound, loss bound, dQ, its
    bound, dD, its bound), the bounds as in tests/test_train_kernels_fp64_gpu.py's fused check."""
    from ravqa_b200.maxsim import maxsim_argmax
    B = Q.size(0)
    arg = maxsim_argmax(Q, D, mask)
    s64, sb = T.maxsim_exact(Q, D, mask)
    _, loss, ds = T.ib_loss_from_scores(s64, nway, label0)
    lb, db = T.ib_loss_bounds(s64, nway, label0)
    w = ds.abs() + (torch.arange(s64.size(1), device=s64.device)[None] == (label0 + torch.arange(
        B, device=s64.device) * nway)[:, None]) / B          # |softmax| / B bounds the sensitivity to the scores
    db = db + 2 * w * sb.max()
    dQ64, dD64, dq_abs, dd_abs, cnt = T.backward(Q, D, arg, ds)
    _, _, dqb, ddb, _ = T.backward(Q, D, arg, db)
    return (loss.mean(), s64, sb, (lb + 2 * sb.max()).mean(), dQ64, C * U * s64.size(1) * dq_abs + dqb,
            dD64, C * U * cnt[..., None] * dd_abs + ddb + C * U * dD64.abs())


@pytest.mark.parametrize("return_scores", [False, True])
def test_in_batch_negatives_loss(R, path, return_scores):
    """Fused route (arg-max + loss head + backward) and the generic route (return_scores=True), both arg-max kernels."""
    B, nway, nq, nd = 4, 2, 200, 150
    Q, D, mask, _ = _make(B, nq, B * nway, nd, "holes", "unit", seed=21)
    for kernel in (1, 2):
        path((kernel, False))
        Qg, Dg = Q.float().clone().requires_grad_(True), D.clone().requires_grad_(True)
        out = R.in_batch_negatives_loss(Qg, Dg, mask.unsqueeze(-1), nway, return_scores=return_scores)
        loss = out[0] if return_scores else out
        loss.backward()
        assert Qg.grad.dtype == torch.float32 and Dg.grad.dtype == torch.float16
        loss64, s64, sb, lb, dQ64, dqb, dD64, ddb = _ib_reference(Q, D, mask, nway)
        tag = "ib loss%s" % (" scores" if return_scores else "")
        _check(tag, (loss.detach().double() - loss64).abs(), lb)
        if return_scores:
            _check(tag + " scores", (out[1].detach().double() - s64).abs(), sb)
        _check(tag + " dQ", (Qg.grad.double() - dQ64).abs(), dqb)
        # dD comes back in fp16, the documents' dtype: one more rounding
        _check(tag + " dD", (Dg.grad.double() - dD64).abs(), ddb + 2.0 ** -11 * dD64.abs() + 2.0 ** -25)


def _gloo_worker(rank, world, port, root, ret):
    import torch.distributed as dist
    import ravqa_b200 as R
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    z = torch.load(os.path.join(root, "batch.pt"))
    Q, D, m = z["Q"][rank].cuda().requires_grad_(True), z["D"][rank].cuda().requires_grad_(True), z["M"][rank].cuda()
    loss = R.in_batch_negatives_loss(Q, D, m.unsqueeze(-1), z["nway"], cross_rank_negatives=True)
    loss.backward()
    ret[rank] = {"loss": loss.detach().cpu(), "dq": Q.grad.cpu(), "dd": D.grad.cpu()}
    dist.barrier()
    dist.destroy_process_group()


def test_cross_rank_negatives_two_gloo_ranks_on_one_gpu(R, tmp_path):
    """Two gloo ranks sharing cuda:0 with fp16 documents of different padded lengths: the gathered documents keep fp16,
    so every rank's fused loss runs the fp16 kernels; loss and dQ against float64 of the global batch."""
    import torch.multiprocessing as mp
    B, nway, nq, world = 3, 2, 70, 2
    Qs, Ds, Ms = [], [], []
    for r, nd in enumerate((50, 83)):
        Q, D, m, _ = _make(B, nq, B * nway, nd, "holes", "unit", seed=300 + r)
        Qs.append(Q.float().cpu())
        Ds.append(D.cpu())
        Ms.append(m.cpu())
    torch.save({"Q": Qs, "D": Ds, "M": Ms, "nway": nway}, tmp_path / "batch.pt")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_gloo_worker, args=(world, port, str(tmp_path), ret), nprocs=world, join=True)
    Dg = torch.cat([torch.nn.functional.pad(d, (0, 0, 0, 83 - d.size(1))) for d in Ds]).cuda()
    Mg = torch.cat([torch.nn.functional.pad(m, (0, 83 - m.size(1))) for m in Ms]).cuda()
    for r in range(world):
        out = ret[r]
        assert out["dd"].dtype == torch.float16 and out["dq"].dtype == torch.float32
        loss64, _, _, lb, dQ64, dqb, _, _ = _ib_reference(Qs[r].half().cuda(), Dg, Mg, nway, r * B * nway)
        _check("gloo loss", (out["loss"].double().cuda() - loss64).abs(), lb)
        _check("gloo dQ", (out["dq"].double().cuda() - dQ64).abs(), dqb)


def test_graphed_loss_step_replays_eager(R):
    B, nway, nq, nd = 4, 2, 96, 64
    Q, D, mask, _ = _make(B, nq, B * nway, nd, "holes", "unit", seed=31)
    Qs, Ds = Q.float().clone().requires_grad_(True), D.clone().requires_grad_(True)
    fn = R.graphed_in_batch_negatives_loss(Qs, Ds, mask.unsqueeze(-1), nway)
    Q2, D2, _, _ = _make(B, nq, B * nway, nd, "holes", "unit", seed=32)
    Qe, De = Q2.float().clone().requires_grad_(True), D2.clone().requires_grad_(True)
    le = R.in_batch_negatives_loss(Qe, De, mask.unsqueeze(-1), nway)
    le.backward()
    Qr, Dr = Q2.float().clone().requires_grad_(True), D2.clone().requires_grad_(True)
    lr = fn(Qr, Dr, mask.unsqueeze(-1))
    lr.backward()
    torch.cuda.synchronize()
    assert torch.equal(lr.detach(), le.detach()) and torch.equal(Qr.grad, Qe.grad)
    # dD accumulates with fp32 atomics in varying order: equal to within one fp16 rounding
    assert torch.allclose(Dr.grad.float(), De.grad.float(), rtol=2.0 ** -10, atol=2.0 ** -24)


def test_exhaustive_branch_packs_an_fp16_corpus(R, monkeypatch):
    """Beyond the arg-max budget the documents are scored by the scan over an fp16 FlatCorpus; the backward recomputes
    the winners with the fp16 arg-max kernels."""
    from ravqa_b200 import modeling
    monkeypatch.setattr(modeling, "_FUSED_MAX_ARG_BYTES", 64)
    g = torch.Generator().manual_seed(41)
    n, nd = 9, 70
    Q = f16_rows((1, 40, 128), None, g).float().cuda().requires_grad_(True)
    D = f16_rows((n, nd, 128), None, g).cuda().requires_grad_(True)
    mask = T.make_mask("prefix", n, nd, g).cuda()
    s = R.colbert_score(Q, D, mask.unsqueeze(-1))
    w = torch.linspace(-1, 1, n, device="cuda")
    (s * w).sum().backward()
    assert Q.grad.dtype == torch.float32 and D.grad.dtype == torch.float16
    Q16, Dd = Q.detach().half(), D.detach()
    packed = Dd[mask]
    s64, amax, rabs = S.maxsim_packed(Q16, packed, mask.sum(1).cpu().numpy())
    # the fp16 scan keeps bf16's accumulator model (25 bits per k-step), so it takes bf16's row bound
    _check("exhaustive scores", (s.detach().double() - s64[0]).abs(), S.scan_bound(amax[0], rabs[0], 40))
    arg = T.argmax_rowmax(Q16, Dd, mask)[0]
    dQ64, _, dq_abs, _, _ = T.backward(Q16, Dd, arg, w[None])
    _check("exhaustive dQ", (Q.grad.double() - dQ64).abs(), C * U * n * dq_abs)


def test_reference_operands_precision_gain(R):
    """The reference's training operands — fp16 documents (normalize(randn).half(), ColBERT.doc) and fp32 queries —
    against float64 compute_ib_loss_new on those exact operands.  The fp16 route rounds only the query (to fp16); the
    bf16 route rounds both to bf16.  The fp16 route's loss is held to the bound of a query rounded to fp16; both
    routes' errors are recorded."""
    g = torch.Generator().manual_seed(51)
    B, nway, nq, nd = 8, 2, 128, 180
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).cuda()
    D = torch.nn.functional.normalize(torch.randn(B * nway, nd, 128, generator=g), dim=-1).half().cuda()
    mask = torch.ones(B * nway, nd, dtype=torch.bool, device="cuda")
    _, rowmax, A = T.argmax_rowmax(Q, D, mask)                # the exact fp32 queries against the fp16 documents
    s64, A = rowmax.sum(-1), A.sum(-1)                        # A: sum_i max_j sum_k |q_ik d_jk|
    _, loss64, ds = T.ib_loss_from_scores(s64, nway)
    loss64 = loss64.mean()
    dQ64 = T.backward(Q, D, T.argmax_rowmax(Q, D, mask)[0], ds)[0]
    sb = C * U * A + nq * U * rowmax.abs().sum(-1)
    errs = {}
    for name, Dr in (("fp16", D), ("bf16", D.to(torch.bfloat16))):
        Qg = Q.clone().requires_grad_(True)
        loss = R.in_batch_negatives_loss(Qg, Dr, mask.unsqueeze(-1), nway)
        loss.backward()
        errs[name] = (abs(float(loss) - float(loss64)), float((Qg.grad.double() - dQ64).abs().max()))
    # rounding Q to fp16 moves each score by at most 2^-11 A; the loss moves by at most twice the largest score change
    bound = 2 * (2.0 ** -11 * A + sb).max() + T.ib_loss_bounds(s64, nway)[0].mean()
    _check("reference operands fp16 loss", torch.tensor(errs["fp16"][0]), bound.cpu())
    REPORT.append("reference operands: |loss - float64| fp16 route %.3e, bf16 route %.3e; max |dQ - float64| fp16 "
                  "route %.3e, bf16 route %.3e" % (errs["fp16"][0], errs["bf16"][0], errs["fp16"][1], errs["bf16"][1]))


def test_retrieve_and_rescore_on_an_fp16_searcher(R):
    """doc_scores and dQ of the RAG block within the float64 bounds on the gathered fp16 rows (the query in fp16), and
    doc_scores within the scan bound plus the arg-max bound of the search scores of the same passages."""
    from ravqa_b200.maxsim import maxsim_argmax
    g = torch.Generator().manual_seed(61)
    dl = torch.randint(1, 60, (300,), generator=g).numpy().astype(np.int32)
    D = f16_rows((int(dl.sum()), 128), None, g)
    Q = f16_rows((3, 33, 128), None, g).float().cuda().requires_grad_(True)
    corpus = R.FlatCorpus(D, dl, device=0, storage="fp16")
    try:
        out = R.Searcher(index=corpus).retrieve_and_rescore(Q, 5, generator=torch.Generator().manual_seed(0))
        ids = out["retrieved_doc_ids"]
        assert out["item_embeddings"].dtype == torch.float16
        w = torch.linspace(-1.0, 1.0, 15, device="cuda").view(3, 5)
        (out["doc_scores"] * w).sum().backward()
        Q16 = Q.detach().half()
        off = np.concatenate([[0], np.cumsum(dl)])
        for b in range(3):
            nd = int(dl[ids[b]].max())
            Dp = torch.zeros((5, nd, 128), dtype=torch.float16)
            m = torch.zeros((5, nd), dtype=torch.bool)
            for i, p in enumerate(ids[b]):
                Dp[i, :dl[p]] = D[off[p]:off[p + 1]]
                m[i, :dl[p]] = True
            Dp, m = Dp.cuda(), m.cuda()
            assert torch.equal(out["item_embeddings"][b][:, :nd], Dp)
            s64, bound = T.maxsim_exact(Q16[b:b + 1], Dp, m)
            _check("rescore doc_scores", (out["doc_scores"][b].detach().double() - s64[0]).abs(), bound[0])
            _, amax, rabs = S.maxsim_packed(Q16[b:b + 1], Dp[m], m.sum(1).cpu().numpy())
            _check("rescore vs search", (out["doc_scores"][b].detach() - out["search_scores"][b]).double().abs(),
                   bound[0] + S.scan_bound(amax[0], rabs[0], 33))
            karg = maxsim_argmax(Q16[b:b + 1], Dp, m)
            dQ64, _, dq_abs, _, _ = T.backward(Q16[b:b + 1], Dp, karg, w[b:b + 1])
            _check("rescore dQ", (Q.grad[b].double() - dQ64[0]).abs(), C * U * 5 * dq_abs[0])
    finally:
        corpus.close()
