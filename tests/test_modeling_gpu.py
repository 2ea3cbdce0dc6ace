"""GPU: differentiable scoring surface (SURVEY 8f-2) — colbert_score / model.score / in-batch negatives —
against a plain torch fp32 restatement of the reference (colbert.py:82-113, 235-286) on the same
bf16-rounded inputs: forward scores and gradients."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref_all_pairs(Q, D, mask):
    """colbert_score semantics for every (query, document) pair, autograd-capable torch fp32."""
    S = torch.einsum("bqd,pkd->bpqk", Q, D)
    S = S.masked_fill(~mask[None, :, None, :], -9999.0)              # colbert_score_reduce (colbert.py:240)
    return S.max(dim=-1).values.sum(dim=-1)                           # [B, n]


def _inputs(B, nq, n, nd, seed):
    g = torch.Generator().manual_seed(seed)
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).bfloat16().float().cuda()
    D = torch.nn.functional.normalize(torch.randn(n, nd, 128, generator=g), dim=-1).bfloat16().float().cuda()
    lens = torch.randint(max(1, nd // 3), nd + 1, (n,), generator=g)
    mask = (torch.arange(nd)[None, :] < lens[:, None]).cuda()
    return Q, D * mask[..., None], mask


def test_colbert_score_forms_and_grads():
    import ravqa_b200 as R
    Q, D, mask = _inputs(6, 40, 6, 50, seed=0)
    # Q.size(0) == 1: one query against all documents
    s1 = R.colbert_score(Q[:1], D, mask.unsqueeze(-1))
    np.testing.assert_allclose(s1.cpu().numpy(), _ref_all_pairs(Q[:1], D, mask)[0].cpu().numpy(), rtol=2e-5)
    # Q.size(0) == n: aligned pairs (the repeat_interleave form of the callers)
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    s = R.colbert_score(Qg, Dg, mask.unsqueeze(-1))
    Qr, Dr = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    sr = _ref_all_pairs(Qr, Dr, mask).diagonal()
    np.testing.assert_allclose(s.detach().cpu().numpy(), sr.detach().cpu().numpy(), rtol=2e-5)
    w = torch.linspace(0.5, 1.5, s.numel(), device="cuda")
    (s * w).sum().backward()
    (sr * w).sum().backward()
    np.testing.assert_allclose(Qg.grad.cpu().numpy(), Qr.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(Dg.grad.cpu().numpy(), Dr.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)


def test_in_batch_negatives_loss_and_model_facade():
    import ravqa_b200 as R
    B, nway = 5, 2
    Q, D, mask = _inputs(B, 64, B * nway, 70, seed=1)
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    model = R.FLMRModelForRetrieval(nway=nway)
    aligned, loss = model(Qg, Dg, mask)
    Qr, Dr = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    S = _ref_all_pairs(Qr, Dr, mask)
    labels = torch.arange(B, device="cuda") * nway                  # positive of query i at column i*nway
    loss_r = torch.nn.functional.cross_entropy(S, labels)
    np.testing.assert_allclose(loss.item(), loss_r.item(), rtol=1e-5)
    rows = torch.arange(B, device="cuda").repeat_interleave(nway)
    np.testing.assert_allclose(aligned.detach().cpu().numpy(),
                               S[rows, torch.arange(B * nway, device="cuda")].detach().cpu().numpy(), rtol=2e-5)
    loss.backward()
    loss_r.backward()
    np.testing.assert_allclose(Qg.grad.cpu().numpy(), Qr.grad.cpu().numpy(), rtol=1e-3, atol=1e-6)
    np.testing.assert_allclose(Dg.grad.cpu().numpy(), Dr.grad.cpu().numpy(), rtol=1e-3, atol=1e-6)
    with pytest.raises(RuntimeError):
        model.query(None)
    # a document with no unmasked token: -inf here, without a host round trip on the training path (the
    # reference's padded path gives -9999 * Nq); documents with tokens are unaffected
    m2 = mask.clone()
    m2[1] = False
    s2 = R.colbert_score(Q[:1], D, m2.unsqueeze(-1))
    assert torch.isinf(s2[1]) and s2[1] < 0 and torch.isfinite(s2[[0, 2]]).all()
    np.testing.assert_allclose(s2[[0, 2]].cpu().numpy(), R.colbert_score(Q[:1], D, mask.unsqueeze(-1))[[0, 2]].cpu().numpy())


def test_argmax_kernel_matches_torch_with_punctuation_style_mask():
    """flmr_maxsim_argmax vs torch argmax on the same bf16 inputs; the mask has holes (ColBERT.doc masks
    punctuation anywhere in the passage, colbert.py:199-203), sizes not multiples of the 64-wide tiles."""
    from ravqa_b200.maxsim import maxsim_argmax
    g = torch.Generator().manual_seed(5)
    B, nq, n, nd = 3, 70, 5, 83
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).bfloat16().cuda()
    D = torch.nn.functional.normalize(torch.randn(n, nd, 128, generator=g), dim=-1).bfloat16().cuda()
    mask = (torch.rand(n, nd, generator=g) > 0.3).cuda()
    mask[:, 0] = True
    mask[1, 64:] = False                                   # a whole trailing tile masked out
    arg = maxsim_argmax(Q, D, mask)
    S = torch.einsum("bqd,pkd->bpqk", Q.float(), D.float()).masked_fill(~mask[None, :, None, :], float("-inf"))
    ref = S.argmax(dim=-1)
    assert arg.dtype == torch.int32 and arg.shape == (B, n, nq)
    same = arg.long() == ref
    # differing picks must be numerical ties of the fp32 accumulation order, never masked tokens
    picked = S.gather(-1, arg.long().unsqueeze(-1)).squeeze(-1)
    assert torch.isfinite(picked).all()
    assert (S.max(dim=-1).values - picked).abs().max().item() < 1e-5
    assert same.float().mean().item() > 0.999
    # fully masked document -> -1
    mask2 = mask.clone()
    mask2[2] = False
    assert (maxsim_argmax(Q, D, mask2)[:, 2] == -1).all()


def test_backward_kernels_match_autograd_at_training_shape():
    """One rank of the C4 contrastive step (SURVEY 8a a6): 8 queries x 16 documents, Nq=832 would need
    218 MB of scores in the reference; here a reduced Nq/Nd keeps the torch restatement small."""
    import ravqa_b200 as R
    B, nway = 8, 2
    Q, D, mask = _inputs(B, 200, B * nway, 130, seed=3)
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    loss = R.in_batch_negatives_loss(Qg, Dg, mask.unsqueeze(-1), nway)
    Qr, Dr = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    loss_r = torch.nn.functional.cross_entropy(_ref_all_pairs(Qr, Dr, mask),
                                               torch.arange(B, device="cuda") * nway)
    np.testing.assert_allclose(loss.item(), loss_r.item(), rtol=1e-5)
    loss.backward()
    loss_r.backward()
    np.testing.assert_allclose(Qg.grad.cpu().numpy(), Qr.grad.cpu().numpy(), rtol=1e-3, atol=1e-6)
    np.testing.assert_allclose(Dg.grad.cpu().numpy(), Dr.grad.cpu().numpy(), rtol=1e-3, atol=1e-6)
    assert (Dg.grad[~mask] == 0).all()                     # masked tokens never receive gradient


def test_aligned_score_with_repeat_interleaved_queries():
    """model.score(Q.repeat_interleave(nway), D, D_mask) — the callers' form (colbert.py:71-73,
    rag_model_blip.py:433): unique queries are scored once; values and gradients as the reference."""
    import ravqa_b200 as R
    B, nway = 4, 3
    Q, D, mask = _inputs(B, 48, B * nway, 40, seed=4)
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    s = R.FLMRModelForRetrieval(nway=nway).score(Qg.repeat_interleave(nway, dim=0).contiguous(), Dg,
                                                 mask.unsqueeze(-1))
    Qr, Dr = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    sr = _ref_all_pairs(Qr.repeat_interleave(nway, dim=0), Dr, mask).diagonal()
    np.testing.assert_allclose(s.detach().cpu().numpy(), sr.detach().cpu().numpy(), rtol=2e-5)
    w = torch.linspace(-1.0, 1.0, s.numel(), device="cuda")
    (s * w).sum().backward()
    (sr * w).sum().backward()
    np.testing.assert_allclose(Qg.grad.cpu().numpy(), Qr.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(Dg.grad.cpu().numpy(), Dr.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)


def test_fused_small_forward_and_scan_kernel_forward_agree(monkeypatch):
    """Batches whose winners fit the memory budget take the one-launch arg-max forward, larger ones the scan kernel
    over a packed temporary corpus: same scores (fp32 accumulation of the same bf16 products), same gradients."""
    import ravqa_b200 as R
    from ravqa_b200 import modeling
    Q, D, mask = _inputs(5, 96, 9, 77, seed=6)
    outs = []
    for limit in (modeling._FUSED_MAX_ARG_BYTES, 0):
        monkeypatch.setattr(modeling, "_FUSED_MAX_ARG_BYTES", limit)
        Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
        S = R.all_pairs_maxsim(Qg, Dg, mask.unsqueeze(-1))
        (S * torch.linspace(-1, 1, S.numel(), device="cuda").view_as(S)).sum().backward()
        outs.append((S.detach(), Qg.grad, Dg.grad))
    np.testing.assert_allclose(outs[0][0].cpu().numpy(), outs[1][0].cpu().numpy(), rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(outs[0][1].cpu().numpy(), outs[1][1].cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(outs[0][2].cpu().numpy(), outs[1][2].cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(outs[0][0].cpu().numpy(), _ref_all_pairs(Q, D, mask).cpu().numpy(), rtol=2e-5)


# ---- cross-rank in-batch negatives over NCCL (needs >= 2 GPUs; skipped on a single-GPU box) ---------------
def _nccl_ib_worker(rank, world, port, ret):
    import os
    import torch.distributed as dist
    import ravqa_b200 as R
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    B, nway, nq = 3, 2, 40
    nds = [30 + 9 * r for r in range(world)]                   # ranks pad their documents differently

    def make(r):
        g = torch.Generator().manual_seed(200 + r)
        Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).bfloat16().float()
        D = torch.nn.functional.normalize(torch.randn(B * nway, nds[r], 128, generator=g), dim=-1).bfloat16().float()
        lens = torch.randint(4, nds[r] + 1, (B * nway,), generator=g)
        m = torch.arange(nds[r])[None, :] < lens[:, None]
        return Q.cuda(rank), (D * m[..., None]).cuda(rank), m.cuda(rank)

    Q, D, m = make(rank)
    Q.requires_grad_(True)
    D.requires_grad_(True)
    loss, S = R.in_batch_negatives_loss(Q, D, m.unsqueeze(-1), nway, return_scores=True, cross_rank_negatives=True)
    loss.backward()
    # single-process torch restatement of the global batch
    parts = [make(r) for r in range(world)]
    Qs = [p[0].clone().requires_grad_(True) for p in parts]
    Ds = [p[1].clone().requires_grad_(True) for p in parts]
    nd_max = max(nds)
    Dg = torch.cat([torch.nn.functional.pad(d, (0, 0, 0, nd_max - d.size(1))) for d in Ds])
    Mg = torch.cat([torch.nn.functional.pad(p[2], (0, nd_max - p[2].size(1))) for p in parts])
    losses = []
    for r in range(world):
        losses.append(torch.nn.functional.cross_entropy(
            _ref_all_pairs(Qs[r], Dg, Mg), r * B * nway + torch.arange(B, device=Dg.device) * nway))
    sum(losses).backward()
    ok = (S.shape == (B, world * B * nway)
          and torch.allclose(loss.detach(), losses[rank].detach(), rtol=1e-5, atol=1e-6)
          and torch.allclose(Q.grad, Qs[rank].grad, rtol=1e-3, atol=1e-6)
          and torch.allclose(D.grad, Ds[rank].grad, rtol=1e-3, atol=1e-6))
    # the loss-only call takes the fused route (arg-max kernel + loss head with this rank's label offset,
    # all-gather straight into the concatenated tensor, reduce-scatter of the document gradient)
    Q2, D2 = Q.detach().clone().requires_grad_(True), D.detach().clone().requires_grad_(True)
    loss2 = R.in_batch_negatives_loss(Q2, D2, m.unsqueeze(-1), nway, cross_rank_negatives=True)
    loss2.backward()
    ok = (ok and torch.allclose(loss2.detach(), losses[rank].detach(), rtol=1e-5, atol=1e-6)
          and torch.allclose(Q2.grad, Qs[rank].grad, rtol=1e-3, atol=1e-6)
          and torch.allclose(D2.grad, Ds[rank].grad, rtol=1e-3, atol=1e-6))
    ret[rank] = bool(ok)
    dist.barrier()
    dist.destroy_process_group()


def test_cross_rank_negatives_nccl():
    import socket
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_nccl_ib_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {r: True for r in range(world)}


def test_training_path_matches_reference_autograd_golden():
    """Loss, aligned scores and gradients vs tests/golden/train_ib_loss.npz — outputs of the reference's own
    compute_ib_loss_new / ColBERT.score and torch autograd (tests/golden/make_golden_train.py); the mask has
    punctuation-style holes."""
    import os
    import ravqa_b200 as R
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "train_ib_loss.npz"))
    f32 = lambda bits: torch.from_numpy((bits.astype(np.uint32) << 16).view(np.float32).copy())
    Q, D, nway = f32(z["Q_bf16"]).cuda(), f32(z["D_bf16"]).cuda(), int(z["nway"])
    mask = torch.from_numpy(z["mask"]).cuda().unsqueeze(-1)
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    loss = R.in_batch_negatives_loss(Qg, Dg, mask, nway)
    loss.backward()
    np.testing.assert_allclose(loss.item(), float(z["ib_loss"]), rtol=5e-6)
    np.testing.assert_allclose(Qg.grad.cpu().numpy(), z["ib_dQ"], rtol=1e-3, atol=1e-6)
    np.testing.assert_allclose(Dg.grad.cpu().numpy(), z["ib_dD"], rtol=1e-3, atol=1e-6)
    Q2, D2 = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    s = R.FLMRModelForRetrieval(nway=nway).score(Q2.repeat_interleave(nway, dim=0).contiguous(), D2, mask)
    np.testing.assert_allclose(s.detach().cpu().numpy(), z["scores"], rtol=2e-5)
    (s * torch.from_numpy(z["score_weights"]).cuda()).sum().backward()
    np.testing.assert_allclose(Q2.grad.cpu().numpy(), z["score_dQ"], rtol=1e-3, atol=1e-6)
    np.testing.assert_allclose(D2.grad.cpu().numpy(), z["score_dD"], rtol=1e-3, atol=1e-6)


@pytest.fixture()
def argmax_path():
    """Force flmr_maxsim_argmax onto one of its two kernels for a test (1 = warp-MMA, 2 = wgmma)."""
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    yield lambda path: _cabi.check(L.flmr_debug_set_argmax_path(path))
    L.flmr_debug_set_argmax_path(0)


@pytest.mark.parametrize("shape", [(3, 70, 5, 83), (2, 320, 7, 300), (1, 832, 9, 512), (4, 129, 3, 128)])
def test_tcgen05_argmax_kernel_equals_warp_mma_kernel_and_torch(shape, argmax_path):
    """The wgmma arg-max kernel (documents compacted to their unmasked tokens, TMA/wgmma pipeline) against the
    warp-MMA kernel and torch on the same bf16 inputs: hole-y masks, a fully masked document, a document whose
    only token sits at the end, sizes off the 128 tiles, several documents per CTA."""
    from ravqa_b200.maxsim import maxsim_argmax, maxsim_argmax_grouped
    B, nq, n, nd = shape
    g = torch.Generator().manual_seed(sum(shape))
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).bfloat16().cuda()
    D = torch.nn.functional.normalize(torch.randn(n, nd, 128, generator=g), dim=-1).bfloat16().cuda()
    mask = (torch.rand(n, nd, generator=g) > 0.3).cuda()
    mask[:, 0] = True
    mask[1] = False                                         # no token at all
    mask[2] = False
    mask[2, nd - 1] = True                                  # one token, the last one
    S = torch.einsum("bqd,pkd->bpqk", Q.float(), D.float()).masked_fill(~mask[None, :, None, :], float("-inf"))
    argmax_path(1)
    a1, m1 = maxsim_argmax(Q, D, mask, return_rowmax=True)
    argmax_path(2)
    a2, m2 = maxsim_argmax(Q, D, mask, return_rowmax=True)
    assert a2.dtype == torch.int32 and a2.shape == (B, n, nq)
    assert (a2[:, 1] == -1).all() and torch.isinf(m2[:, 1]).all() and (a2[:, 2] == nd - 1).all()
    live = [p for p in range(n) if p != 1]
    picked = S[:, live].gather(-1, a2[:, live].long().unsqueeze(-1)).squeeze(-1)
    assert torch.isfinite(picked).all()                                          # never a masked token
    assert (S[:, live].max(dim=-1).values - picked).abs().max().item() < 1e-5      # ties of the accumulation order at most
    np.testing.assert_allclose(m2[:, live].cpu().numpy(), S[:, live].max(dim=-1).values.cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(m2[:, live].cpu().numpy(), m1[:, live].cpu().numpy(), rtol=1e-6, atol=1e-6)
    assert (a1 == a2).float().mean().item() > 0.999
    # block-diagonal form: query b against documents [b*r, (b+1)*r)
    if n >= 2 * B:
        r = n // B
        Dg, Mg = D[: B * r], mask[: B * r]
        argmax_path(1)
        g1, gm1 = maxsim_argmax_grouped(Q, Dg, Mg, r, return_rowmax=True)
        argmax_path(2)
        g2, gm2 = maxsim_argmax_grouped(Q, Dg, Mg, r, return_rowmax=True)
        fin = torch.isfinite(gm1)
        assert torch.equal(torch.isfinite(gm2), fin) and (g1 == g2).float().mean().item() > 0.999
        np.testing.assert_allclose(gm2[fin].cpu().numpy(), gm1[fin].cpu().numpy(), rtol=1e-6, atol=1e-6)


def test_training_step_on_the_tcgen05_path_matches_golden(argmax_path):
    """The reference-generated training golden (loss, scores, dQ, dD of compute_ib_loss_new) with the forward
    forced onto the wgmma kernel."""
    import ravqa_b200 as R
    from helpers import GOLDEN_DIR
    import os
    z = np.load(os.path.join(GOLDEN_DIR, "train_ib_loss.npz"))
    from helpers import bf16_bits_to_f32
    Q = torch.from_numpy(bf16_bits_to_f32(z["Q_bf16"])).cuda().requires_grad_(True)
    D = torch.from_numpy(bf16_bits_to_f32(z["D_bf16"])).cuda().requires_grad_(True)
    mask = torch.from_numpy(z["mask"]).cuda()
    argmax_path(2)
    loss = R.in_batch_negatives_loss(Q, D, mask.unsqueeze(-1), int(z["nway"]))
    loss.backward()
    np.testing.assert_allclose(loss.item(), float(z["ib_loss"]), rtol=5e-6)
    np.testing.assert_allclose(Q.grad.cpu().numpy(), z["ib_dQ"], rtol=1e-3, atol=1e-6)
    np.testing.assert_allclose(D.grad.cpu().numpy(), z["ib_dD"], rtol=1e-3, atol=1e-6)


def test_tcgen05_argmax_many_documents_per_cta_back_to_back(argmax_path):
    """The global-batch shape (8 queries x 832 rows against 128 ragged documents of up to 512 tokens: 12 documents
    per CTA, each consumer warpgroup on half of the query tile) launched back to back without synchronisation:
    same winners and maxima as the warp-MMA kernel every time."""
    from ravqa_b200.maxsim import maxsim_argmax
    g = torch.Generator().manual_seed(12)
    B, nq, n, nd = 8, 832, 128, 512
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).bfloat16().cuda()
    D = torch.nn.functional.normalize(torch.randn(n, nd, 128, generator=g), dim=-1).bfloat16().cuda()
    lens = torch.randint(1, nd + 1, (n,), generator=g)
    lens[:4] = torch.tensor([1, 128, 129, 512])
    mask = (torch.arange(nd)[None, :] < lens[:, None]).cuda()
    argmax_path(1)
    a1, m1 = maxsim_argmax(Q, D, mask, return_rowmax=True)
    argmax_path(2)
    outs = [maxsim_argmax(Q, D, mask, return_rowmax=True) for _ in range(12)]
    torch.cuda.synchronize()
    for a2, m2 in outs:
        assert torch.equal(m2, m1)
        assert (a2 == a1).float().mean().item() > 0.9999


def test_graphed_loss_step_replays_the_eager_step(argmax_path):
    """graphed_in_batch_negatives_loss (forward and backward captured as CUDA graphs): on NEW inputs of the captured
    shape the replayed loss and gradients equal the eager step's — both kernels of the forward (warp-MMA for the
    C4 rank shape, wgmma forced) are capturable: no host synchronisation, stream-ordered scratch only."""
    import ravqa_b200 as R
    B, nway, nq, nd = 8, 2, 832, 512
    Q, D, mask = _inputs(B, nq, B * nway, nd, seed=31)
    m3 = mask.unsqueeze(-1)
    for path in (0, 2):
        argmax_path(path)
        Qs, Ds = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
        graphed = R.graphed_in_batch_negatives_loss(Qs, Ds, m3, nway)
        for seed in (32, 33):
            Q2, D2, mask2 = _inputs(B, nq, B * nway, nd, seed=seed)
            Qa, Da = Q2.clone().requires_grad_(True), D2.clone().requires_grad_(True)
            Qb, Db = Q2.clone().requires_grad_(True), D2.clone().requires_grad_(True)
            la = R.in_batch_negatives_loss(Qa, Da, mask2.unsqueeze(-1), nway)
            (la * 1.7).backward()
            lb = graphed(Qb, Db, mask2.unsqueeze(-1))
            (lb * 1.7).backward()
            assert torch.equal(la.detach(), lb.detach())
            assert torch.equal(Qa.grad, Qb.grad)
            # dD is scattered with fp32 atomics: equal up to the order of the additions
            np.testing.assert_allclose(Da.grad.cpu().numpy(), Db.grad.cpu().numpy(), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("nq", [96, 70])
def test_flipr_interaction_matches_reference_golden(nq):
    """``interaction == 'flipr'`` (colbert_score_reduce, colbert.py:248-261): scores and gradients of both caller
    shapes against what the reference's own ColBERT.score + autograd produced (tests/golden/make_golden_flipr.py)."""
    import os
    import types
    import ravqa_b200 as R
    from helpers import GOLDEN_DIR, bf16_bits_to_f32
    z = np.load(os.path.join(GOLDEN_DIR, "flipr.npz"))
    k = "nq%d_" % nq
    cfg = types.SimpleNamespace(interaction="flipr", query_maxlen=64)
    r = int(z["docs_per_query"])
    w = torch.from_numpy(z["weights"]).cuda()
    mask = torch.from_numpy(z[k + "mask"]).cuda().unsqueeze(-1)
    for shape in ("aligned", "one"):
        Q = torch.from_numpy(bf16_bits_to_f32(z[k + "Q_bf16"])).cuda().requires_grad_(True)
        D = torch.from_numpy(bf16_bits_to_f32(z[k + "D_bf16"])).cuda().requires_grad_(True)
        Qin = Q.repeat_interleave(r, dim=0).contiguous() if shape == "aligned" else Q[:1]
        s = R.colbert_score(Qin, D, mask, config=cfg)
        (s * w).sum().backward()
        np.testing.assert_allclose(s.detach().cpu().numpy(), z[k + shape], rtol=2e-5)
        np.testing.assert_allclose(Q.grad.cpu().numpy(), z[k + shape + "_dQ"], rtol=1e-3, atol=1e-6)
        np.testing.assert_allclose(D.grad.cpu().numpy(), z[k + shape + "_dD"], rtol=1e-3, atol=1e-6)
