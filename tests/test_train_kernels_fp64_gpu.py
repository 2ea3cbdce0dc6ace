"""GPU: the arg-max, backward and loss-head kernels against the float64 restatement of tests/train_fp64.py (pinned on
CPU by tests/test_train_fp64_host.py), at their tile, batch and label boundaries, and the consumers that re-score
with them (the fp8 Searcher's exact re-rank, retrieve_and_rescore, the cross-rank fused loss on one GPU).

Every tolerance is a bound in u = 2^-24 (see train_fp64.py); each check records its largest error / bound ratio and
the module prints them all at the end (run with -s)."""
import os
import socket

import numpy as np
import pytest
import torch

import train_fp64 as T

pytestmark = pytest.mark.gpu

RATIOS = {}
C, U = T.C_BOUND, T.U


def _check(name, err, bound):
    """err <= bound elementwise (a zero bound demands an exact zero); records the largest err / bound of `name`."""
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
    print("\n[fp64] largest error / bound per check:")
    for k in sorted(RATIOS):
        print("[fp64]   %-28s %.3e" % (k, RATIOS[k]))


@pytest.fixture(scope="module")
def R():
    import ravqa_b200
    torch.cuda.set_device(0)
    return ravqa_b200


@pytest.fixture()
def argmax_path(R):
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    yield lambda path: _cabi.check(L.flmr_debug_set_argmax_path(path))
    L.flmr_debug_set_argmax_path(0)


def ib_loss_head(rowmax, nway, label0):
    from ravqa_b200.maxsim import ib_loss_head as head
    return head(rowmax, nway, label0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _make(B, nq, n_total, nd, mask_kind, norm, seed):
    g = torch.Generator().manual_seed(seed)
    nrm = None if norm == "unit" else (4.0, 30.0)
    Q = T.bf16_rows((B, nq, 128), nrm, g)
    D = T.bf16_rows((n_total, nd, 128), nrm, g)
    mask = T.make_mask(mask_kind, n_total, nd, g)
    tie = None
    live = torch.nonzero(mask[0]).flatten()
    if live.numel() >= 2:
        # an exact tie: document 0's last unmasked token repeats its first, which query 0's row 0 asks for
        a, b = int(live[0]), int(live[-1])
        D[0, b] = D[0, a]
        Q[0, 0] = D[0, a]
        tie = (a, b)
    return Q.cuda(), D.cuda(), mask.cuda(), tie


def _check_forward(Q, D, mask, arg, rowmax, r, tie, tag):
    a64, r64, A = T.argmax_rowmax(Q, D, mask, r)
    empty = torch.isinf(r64)
    assert (arg[empty] == -1).all() and torch.isneginf(rowmax[empty]).all(), tag
    assert (arg[~empty] >= 0).all(), tag
    bound = C * U * A
    fin = ~empty
    _check("argmax rowmax", (rowmax.double() - r64).abs()[fin], bound[fin])
    s_win, unmasked = T.winner_scores(Q, D, mask, arg, r)
    assert unmasked[fin].all(), "%s: a winner on a masked token" % tag
    _check("argmax winner score", (r64 - s_win)[fin], bound[fin])
    if tie is not None:
        first = arg[:, 0] if r is None else arg[0, 0]
        assert (first != tie[1]).all(), "%s: the later copy of a tied token won" % tag
    return a64


def _check_backward(R, Q, D, mask, arg, r, need, seed, tag):
    from ravqa_b200.maxsim import maxsim_backward, maxsim_backward_grouped
    B, P = arg.shape[:2]
    g = torch.randn((B, P), generator=torch.Generator().manual_seed(seed)).float()
    g[:, ::3] = 0.0                                       # exact zeros: the dD kernel's early exit
    g = g.cuda()
    need_dq, need_dd = need in ("both", "dq"), need in ("both", "dd")
    if r is None:
        dq, dd = maxsim_backward(Q, D, arg, g, need_dq=need_dq, need_dd=need_dd)
    else:
        dq, dd = maxsim_backward_grouped(Q, D, arg, g, need_dq=need_dq, need_dd=need_dd)
    assert (dq is None) == (not need_dq) and (dd is None) == (not need_dd), tag
    dQ64, dD64, dq_abs, dd_abs, cnt = T.backward(Q, D, arg, g, r)
    if need_dq:
        _check("dQ", (dq.double() - dQ64).abs(), C * U * P * dq_abs)
    if need_dd:
        _check("dD", (dd.double() - dD64).abs(), C * U * cnt[..., None] * dd_abs)
        assert (dd[~mask] == 0).all() and (dd[cnt == 0] == 0).all(), "%s: gradient on a masked / losing token" % tag


GRID = T.argmax_grid()


@pytest.mark.parametrize("ci", range(len(GRID)), ids=lambda i: "c%03d" % i)
def test_argmax_and_backward_grid(R, argmax_path, ci):
    """One case of the pairwise covering: both kernels (forced), both forms, every mask kind, unit and wide rows;
    the backward on the kernel's own winners with dQ only / dD only / both and an upstream gradient with zeros."""
    from ravqa_b200.maxsim import maxsim_argmax, maxsim_argmax_grouped
    c = GRID[ci]
    B, nq, nd, n = c["B"], c["nq"], c["nd"], c["n_docs"]
    grouped = c["form"] == "grouped"
    Q, D, mask, tie = _make(B, nq, B * n if grouped else n, nd, c["mask"], c["norm"], seed=1000 + ci)
    argmax_path(c["path"])
    if grouped:
        arg, rowmax = maxsim_argmax_grouped(Q, D, mask, n, return_rowmax=True)
    else:
        arg, rowmax = maxsim_argmax(Q, D, mask, return_rowmax=True)
    tag = "case %d %s" % (ci, c)
    assert arg.shape == (B, n, nq), tag
    r = n if grouped else None
    _check_forward(Q, D, mask, arg, rowmax, r, tie, tag)
    _check_backward(R, Q, D, mask, arg, r, ("both", "dq", "dd")[ci % 3], ci, tag)


def test_wgmma_argmax_docs_per_cta_split(R, argmax_path):
    """The widest split of the wgmma kernel: 32 documents per CTA with a partial last CTA (127 = 3 x 32 + 31 documents
    for a 132-SM H100), all-pairs and grouped, ragged masks with holes."""
    B, nq, nd = 9, 832, 128
    n = next((k for k in (127, 126, 95, 63) if T.docs_per_cta(B, nq, k, nd, _sms()) == 32 and k % 32), None)
    assert n is not None, "no 32-document split with a partial last CTA on %d SMs" % _sms()
    from ravqa_b200.maxsim import maxsim_argmax, maxsim_argmax_grouped
    argmax_path(2)
    for grouped in (False, True):
        n_total = B * n if grouped else n
        assert T.docs_per_cta(B, nq, n, nd, _sms()) == 32
        Q, D, mask, tie = _make(B, nq, n_total, nd, "holes", "wide", seed=77 + grouped)
        if grouped:
            arg, rowmax = maxsim_argmax_grouped(Q, D, mask, n, return_rowmax=True)
        else:
            arg, rowmax = maxsim_argmax(Q, D, mask, return_rowmax=True)
        _check_forward(Q, D, mask, arg, rowmax, n if grouped else None, tie, "split grouped=%s" % grouped)
        _check_backward(R, Q, D, mask, arg, n if grouped else None, "both", 5, "split")


@pytest.mark.parametrize("n,path", [(1953, 1), (1954, 2)])
def test_auto_path_threshold(R, n, path):
    """Path 0 picks the wgmma kernel from 16e6 (query row, token) pairs with Nq >= 64 and Nd >= 128: one shape on each
    side (1 x 64 x n x 128 pairs), told apart by the launches (the wgmma route compacts the documents first)."""
    from ravqa_b200 import _cabi
    from ravqa_b200.maxsim import maxsim_argmax
    L = _cabi.lib()
    _cabi.check(L.flmr_debug_set_argmax_path(0))
    Q, D, mask, tie = _make(1, 64, n, 128, "prefix", "unit", seed=n)
    torch.cuda.synchronize()
    L.flmr_launch_count(1)
    arg, rowmax = maxsim_argmax(Q, D, mask, return_rowmax=True)
    launches = L.flmr_launch_count(1)
    assert launches == path, (n, launches)
    _check_forward(Q, D, mask, arg, rowmax, None, tie, "auto n=%d" % n)


def test_backward_without_documents_zeroes_dq(R):
    """n_per == 0: dQ is a memset (and dD empty), even over memory that held NaNs."""
    from ravqa_b200.maxsim import maxsim_backward
    B, nq, nd = 3, 65, 40
    Q = T.bf16_rows((B, nq, 128)).cuda()
    D = torch.zeros((0, nd, 128), device="cuda")
    junk = torch.full((B, nq, 128), float("nan"), device="cuda")
    del junk                                                  # the allocator hands this block to dQ below
    dq, dd = maxsim_backward(Q, D, torch.zeros((B, 0, nq), dtype=torch.int32, device="cuda"),
                             torch.zeros((B, 0), device="cuda"))
    assert dq.shape == (B, nq, 128) and (dq == 0).all() and dd.shape == (0, nd, 128)


def test_backward_with_flipr_deselected_and_empty_documents(R, argmax_path):
    """Winners of -1 from both sources in one batch: a document without tokens and the tokens the 'flipr' reduction
    leaves out; both kernels' winners."""
    from ravqa_b200.maxsim import maxsim_argmax
    B, nq, n, nd = 3, 96, 7, 130
    Q, D, mask, _ = _make(B, nq, n, nd, "holes", "unit", seed=3)
    mask[2] = False
    for path in (1, 2):
        argmax_path(path)
        arg, rowmax = maxsim_argmax(Q, D, mask, return_rowmax=True)
        _, sel = T.flipr_select(rowmax, arg)
        assert (sel[:, 2] == -1).all() and ((sel == -1).sum() > B * nq) and (sel >= 0).any()
        for need in ("both", "dq", "dd"):
            _check_backward(R, Q, D, mask, sel.contiguous(), None, need, path, "flipr path=%d" % path)


# ---- the loss head --------------------------------------------------------------------------------------------------
def _rowmax(B, n, nq, spread, seed, neg_inf=()):
    """Synthetic fp32 row maxima whose per-document sums spread over ~`spread`; documents in `neg_inf` score -inf
    (one -inf row maximum, as a fully masked document gives)."""
    g = torch.Generator().manual_seed(seed)
    target = (torch.rand((B, n, 1), generator=g) - 0.5) * spread
    r = target / nq + 0.3 * torch.randn((B, n, nq), generator=g)
    for b, p in neg_inf:
        r[b, p, nq // 2] = -torch.inf
    return r.float().cuda()


def _check_loss(R, rowmax, nway, label0, tag):
    s, loss, ds = ib_loss_head(rowmax, nway, label0)
    r64 = rowmax.double()
    fin = torch.isfinite(r64)
    s64 = r64.sum(dim=-1)
    inf = torch.isinf(s64)
    assert torch.equal(torch.isneginf(s), inf), tag
    bound = rowmax.size(-1) * U * torch.where(fin, r64.abs(), 0.0).sum(dim=-1)
    _check("scores", (s.double() - s64).abs()[~inf], bound[~inf])
    # loss and dscores against float64 on the kernel's own scores (their summation is checked just above)
    _, loss64, ds64 = T.ib_loss_from_scores(s.double(), nway, label0)
    lb, db = T.ib_loss_bounds(s.double(), nway, label0)
    _check("loss", (loss.double() - loss64).abs(), lb)
    _check("dscores", (ds.double() - ds64).abs(), db)
    assert (ds[inf] == 0).all(), tag                       # a -inf negative: zero probability, zero gradient
    return s, loss, ds


LOSS_CASES = [  # (B, n_docs, nway, Nq, spread)
    (1, 1, 1, 33, 10.0), (1, 1, 16, 1, 10.0),
    (4, 255, 2, 832, 300.0), (16, 256, 16, 1, 200.0), (3, 257, 1, 33, 400.0),
    (2, 12288, 16, 33, 300.0), (5, 12289, 2, 1, 100.0), (1, 12289, 1, 832, 300.0),
    (3, 51200, 16, 33, 300.0), (2, 51200, 2, 1, 500.0),
]


@pytest.mark.parametrize("B,n,nway,nq,spread", LOSS_CASES)
def test_ib_loss_head(R, B, n, nway, nq, spread):
    """Positives at label0 = 0, an interior offset and the last valid column; the FLMR_ERR_INVALID_ARG one past it.
    12,288 documents fill exactly the 48 KiB of shared memory a launch gets without opting in, which the kernel's
    static reduction buffer overflows (this case failed to launch before flmr_ib_loss opted in there too); 12,289 and
    up take the raised limit; 51,200 is the widest batch the kernel takes."""
    from ravqa_b200 import _cabi
    last = n - 1 - (B - 1) * nway
    labels0 = sorted({0, last // 2, last})
    positives = {l0 + b * nway for l0 in labels0 for b in range(B)}
    neg = [p for p in range(n) if p not in positives][:1]     # a -inf negative wherever one fits
    rowmax = _rowmax(B, n, nq, spread, seed=n + nq, neg_inf=[(b, p) for b in range(B) for p in neg])
    for label0 in labels0:
        _check_loss(R, rowmax, nway, label0, (B, n, nway, nq, label0))
    with pytest.raises(_cabi.FlmrError) as e:
        ib_loss_head(rowmax, nway, last + 1)
    assert e.value.code == 1


def test_ib_loss_head_rejects_wider_batches(R):
    from ravqa_b200 import _cabi
    with pytest.raises(_cabi.FlmrError) as e:
        ib_loss_head(torch.zeros((1, 51201, 1), device="cuda"), 1, 0)
    assert e.value.code == 3


def test_ib_loss_head_minus_inf_positive(R):
    """A fully masked positive scores -inf on the fused route (the reference's padded path gives -9999 Nq): the loss is
    +inf and dscores is the finite (softmax - onehot) / B — float64 cross_entropy's value and gradient."""
    B, n, nway, nq = 3, 12, 4, 33
    rowmax = _rowmax(B, n, nq, 50.0, seed=9)
    rowmax[1, 1 * nway + 2] = -torch.inf                        # positive of query 1 (label0 = 2)
    s, loss, ds = ib_loss_head(rowmax, nway, 2)
    x = s.double().cpu().clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(x, 2 + torch.arange(B) * nway, reduction="none")
    ref.mean().backward()
    assert torch.isposinf(loss[1]) and torch.isposinf(ref[1])
    assert torch.isfinite(loss[[0, 2]]).all() and torch.isfinite(ds).all()
    lb, db = T.ib_loss_bounds(s.double(), nway, 2)
    _check("dscores", (ds.double().cpu() - x.grad).abs(), db.cpu())
    _check("loss", (loss.double().cpu() - ref.detach())[[0, 2]].abs(), lb.cpu()[[0, 2]])
    assert ds[1, 1 * nway + 2].item() == pytest.approx(-1.0 / B, rel=4 * U)


def test_fused_loss_step_end_to_end(R, argmax_path):
    """in_batch_negatives_loss on the fused route (arg-max + loss head + backward) against float64 on the kernel's own
    winners, both arg-max kernels, a 832-row query batch."""
    B, nway, nq, nd = 4, 2, 832, 180
    Q, D, mask, _ = _make(B, nq, B * nway, nd, "holes", "unit", seed=41)
    for path in (1, 2):
        argmax_path(path)
        _fused_check(R, [Q], [D], [mask], 0, nway, "fused path=%d" % path)


def _fused_check(R, Qs, Ds, masks, rank, nway, tag, loss=None, dq=None, dd=None):
    """Float64 restatement of the (global) in-batch-negatives batch of `len(Qs)` ranks; checks rank `rank`'s loss, dQ
    and dD (computed here on one rank if not given)."""
    from ravqa_b200.maxsim import maxsim_argmax
    world, B = len(Qs), Qs[0].size(0)
    nd_max = max(d.size(1) for d in Ds)
    Dg = torch.cat([torch.nn.functional.pad(d, (0, 0, 0, nd_max - d.size(1))) for d in Ds])
    Mg = torch.cat([torch.nn.functional.pad(m, (0, nd_max - m.size(1))) for m in masks])
    if loss is None:
        Qg, Dgg = Qs[0].clone().requires_grad_(True), Dg.clone().requires_grad_(True)
        loss = R.in_batch_negatives_loss(Qg, Dgg, Mg.unsqueeze(-1), nway)
        loss.backward()
        dq, dd = Qg.grad, Dgg.grad
    dD64 = torch.zeros(Dg.shape, dtype=torch.float64, device=Dg.device)
    ddb = torch.zeros_like(dD64)
    for r in range(world):
        arg = maxsim_argmax(Qs[r], Dg, Mg)                    # the kernel's own winners: ties cannot blur the check
        s64, sb = T.maxsim_exact(Qs[r], Dg, Mg)
        _, loss64, ds64 = T.ib_loss_from_scores(s64, nway, r * B * nway)
        lb, db = T.ib_loss_bounds(s64, nway, r * B * nway)
        w = ds64.abs() + (torch.arange(s64.size(1), device=s64.device)[None] == (r * B * nway + torch.arange(
            B, device=s64.device) * nway)[:, None]) / B      # |softmax| / B bounds the sensitivity to the scores
        db = db + 2 * w * sb.max()
        dQ64, dDr, dq_abs, dd_abs, cnt = T.backward(Qs[r], Dg, arg, ds64)
        _, _, dqb, ddbr, _ = T.backward(Qs[r], Dg, arg, db)
        dD64 += dDr
        ddb += C * U * cnt[..., None] * dd_abs + ddbr
        if r == rank:
            _check("fused loss", (loss.detach().double() - loss64.mean()).abs(), (lb + 2 * sb.max()).mean())
            _check("fused dQ", (dq.double() - dQ64).abs(), C * U * s64.size(1) * dq_abs + dqb)
    rows = slice(rank * B * nway, (rank + 1) * B * nway)
    nd_r = Ds[rank].size(1)
    _check("fused dD", (dd.double() - dD64[rows, :nd_r]).abs(),
           ddb[rows, :nd_r] + C * U * dD64[rows, :nd_r].abs())


def _gloo_ib_worker(rank, world, port, root, ret):
    import torch.distributed as dist
    import ravqa_b200 as R
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    z = torch.load(os.path.join(root, "batch.pt"))
    Q, D, m = z["Q"][rank].cuda(), z["D"][rank].cuda(), z["M"][rank].cuda()
    Q.requires_grad_(True)
    D.requires_grad_(True)
    loss = R.in_batch_negatives_loss(Q, D, m.unsqueeze(-1), z["nway"], cross_rank_negatives=True)
    loss.backward()
    ret[rank] = {"loss": loss.detach().cpu(), "dq": Q.grad.cpu(), "dd": D.grad.cpu()}
    dist.barrier()
    dist.destroy_process_group()


def test_cross_rank_fused_loss_two_gloo_ranks_on_one_gpu(R, tmp_path):
    """Two gloo ranks sharing cuda:0, ragged padded lengths per rank: each rank's loss takes the fused route with its
    positives at label0 = rank * B * nway; loss, dQ and dD against a float64 restatement of the global batch."""
    import torch.multiprocessing as mp
    B, nway, nq, world = 3, 2, 70, 2
    nds = [50, 83]
    Qs, Ds, Ms = [], [], []
    for r in range(world):
        Q, D, m, _ = _make(B, nq, B * nway, nds[r], "holes", "unit", seed=300 + r)
        Qs.append(Q.cpu())
        Ds.append(D.cpu())
        Ms.append(m.cpu())
    torch.save({"Q": Qs, "D": Ds, "M": Ms, "nway": nway}, tmp_path / "batch.pt")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_gloo_ib_worker, args=(world, port, str(tmp_path), ret), nprocs=world, join=True)
    for r in range(world):
        out = ret[r]
        _fused_check(R, [q.cuda() for q in Qs], [d.cuda() for d in Ds], [m.cuda() for m in Ms], r, nway,
                     "gloo rank %d" % r, loss=out["loss"].cuda(), dq=out["dq"].cuda(), dd=out["dd"].cuda())


# ---- the re-score consumers -------------------------------------------------------------------------------------------
def _flat_corpus_case(n, seed):
    g = torch.Generator().manual_seed(seed)
    dl = torch.randint(1, 60, (n,), generator=g).numpy().astype(np.int32)
    D = T.bf16_rows((int(dl.sum()), 128), generator=g)
    return D, dl


def _padded(D, dl, pids):
    off = np.concatenate([[0], np.cumsum(dl)])
    nd = int(dl[pids].max())
    out = torch.zeros((len(pids), nd, 128))
    m = torch.zeros((len(pids), nd), dtype=torch.bool)
    for i, p in enumerate(pids):
        out[i, :dl[p]] = D[off[p]:off[p + 1]]
        m[i, :dl[p]] = True
    return out, m


def test_fp8_searcher_scores_are_exact_bf16_maxsim(R):
    """The fp8 Searcher re-ranks its shortlist with the bf16 rows: every returned score is the float64 MaxSim of the
    bf16 query and passage rows, within the fp32 bound."""
    D, dl = _flat_corpus_case(700, 5)
    Q = T.bf16_rows((4, 40, 128), generator=torch.Generator().manual_seed(6))
    c8 = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0, storage="fp8")
    try:
        s, p = R.Searcher(index=c8, storage="fp8")._search_tensors(Q, 20)
        s, p = s.cpu(), p.cpu()
        for b in range(Q.size(0)):
            Dp, m = _padded(D, dl, p[b].numpy())
            s64, bound = T.maxsim_exact(Q[b:b + 1], Dp, m)
            _check("fp8 searcher score", (s[b].double() - s64[0]).abs(), bound[0])
    finally:
        c8.close()


def test_retrieve_and_rescore_scores_and_dq(R):
    """doc_scores of the RAG block and the gradient reaching the queries against float64 MaxSim of the gathered rows."""
    from ravqa_b200.maxsim import maxsim_argmax
    D, dl = _flat_corpus_case(300, 7)
    Q = T.bf16_rows((3, 33, 128), generator=torch.Generator().manual_seed(8)).cuda().requires_grad_(True)
    corpus = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0)
    try:
        out = R.Searcher(index=corpus).retrieve_and_rescore(Q, 5, generator=torch.Generator().manual_seed(0))
        ids = out["retrieved_doc_ids"]
        w = torch.linspace(-1.0, 1.0, 15, device="cuda").view(3, 5)
        (out["doc_scores"] * w).sum().backward()
        Qd = Q.detach()
        for b in range(3):
            Dp, m = _padded(D, dl, ids[b])
            Dp, m = Dp.cuda(), m.cuda()
            assert torch.equal(out["item_embeddings"][b].float()[:, :Dp.size(1)], Dp)
            s64, bound = T.maxsim_exact(Qd[b:b + 1], Dp, m)
            _check("rescore doc_scores", (out["doc_scores"][b].detach().double() - s64[0]).abs(), bound[0])
            karg = maxsim_argmax(Qd[b:b + 1], Dp, m)        # the winners the re-score's backward used
            dQ64, _, dq_abs, _, _ = T.backward(Qd[b:b + 1], Dp, karg, w[b:b + 1])
            _check("rescore dQ", (Q.grad[b].double() - dQ64[0]).abs(), C * U * 5 * dq_abs[0])
    finally:
        corpus.close()


def test_fp8_gather_after_append_and_delete(R):
    """gather_padded on an fp8 corpus reads the pinned bf16 master, which the append reallocates: gathered rows are
    bitwise the source rows, deleted ids give all-masked zero rows."""
    D, dl = _flat_corpus_case(200, 11)
    D2, dl2 = _flat_corpus_case(150, 12)
    c8 = R.FlatCorpus(D.to(torch.bfloat16), dl, device=0, storage="fp8")
    try:
        new = c8.append(D2.to(torch.bfloat16), dl2)
        assert new[0] == 200 and len(new) == 150
        dead = np.array([0, 57, 199, 200, 333, 349])
        c8.delete(dead)
        Dall, dlall = torch.cat([D, D2]), np.concatenate([dl, dl2])
        pids = np.array([0, 1, 57, 58, 198, 199, 200, 201, 260, 333, 348, 349])
        E, M = c8.gather_padded(torch.from_numpy(pids))
        ref, rm = _padded(Dall, dlall, pids)
        for i, p in enumerate(pids):
            if p in dead:
                assert not M[i].any() and (E[i] == 0).all(), p
            else:
                nd = ref.size(1)
                assert torch.equal(E[i, :nd].float().cpu(), ref[i]) and torch.equal(M[i, :nd, 0].cpu(), rm[i]), p
                assert not M[i, nd:].any() and (E[i, nd:] == 0).all()
    finally:
        c8.close()
