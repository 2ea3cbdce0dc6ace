"""CPU: the float64 restatement of the training kernels (tests/train_fp64.py) against outputs of the reference's own
autograd — tests/golden/train_ib_loss.npz (compute_ib_loss_new, aligned ColBERT.score) and tests/golden/flipr.npz
(the 'flipr' reduction) — and against torch's float64 cross-entropy, so that it is known to be right before
tests/test_train_kernels_fp64_gpu.py judges any kernel by it.  Also pins the test grid itself: pairwise covering,
and the docs_per_cta splits it reaches."""
import itertools
import os

import numpy as np
import pytest
import torch

import train_fp64 as T
from helpers import GOLDEN_DIR, bf16_bits_to_f32

# The goldens are fp32 autograd on CPU: what separates them from float64 is their own rounding (~1e-6 relative).
# A stride that drops one document's share of a gradient moves it by ~1e-2 of its magnitude.
RTOL = 2e-5


def _t(bits):
    return torch.from_numpy(bf16_bits_to_f32(bits))


def _close(got, want, rtol=RTOL):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * np.abs(want).max())


def test_ib_loss_and_grads_match_reference_autograd():
    z = np.load(os.path.join(GOLDEN_DIR, "train_ib_loss.npz"))
    Q, D, mask, nway = _t(z["Q_bf16"]), _t(z["D_bf16"]), torch.from_numpy(z["mask"]), int(z["nway"])
    arg, rowmax, absmax = T.argmax_rowmax(Q, D, mask)
    assert arg.shape == (Q.size(0), D.size(0), Q.size(1)) and (arg >= 0).all()
    assert mask[torch.arange(D.size(0))[None, :, None].expand_as(arg), arg].all()
    assert (absmax >= rowmax.abs()).all()
    s, loss, ds = T.ib_loss(rowmax, nway)
    _close(loss.mean().item(), float(z["ib_loss"]))
    dQ, dD, dq_abs, dd_abs, cnt = T.backward(Q, D, arg, ds)
    _close(dQ.numpy(), z["ib_dQ"])
    _close(dD.numpy(), z["ib_dD"])
    assert (dD[~mask] == 0).all() and (cnt[~mask] == 0).all()
    assert (dq_abs >= dQ.abs()).all() and (dd_abs >= dD.abs()).all()
    # sensitivity: the positive one column off moves the loss far outside the tolerance
    assert abs(T.ib_loss(rowmax, nway, 1)[1].mean().item() - float(z["ib_loss"])) > 1e-2


def test_aligned_scores_and_grads_match_reference_autograd():
    z = np.load(os.path.join(GOLDEN_DIR, "train_ib_loss.npz"))
    Q, D, mask, nway = _t(z["Q_bf16"]), _t(z["D_bf16"]), torch.from_numpy(z["mask"]), int(z["nway"])
    B = Q.size(0)
    arg, rowmax, _ = T.argmax_rowmax(Q, D, mask, docs_per_query=nway)
    _close(rowmax.sum(-1).reshape(-1).numpy(), z["scores"])
    s64, bound = T.maxsim_exact(Q, D, mask, docs_per_query=nway)
    assert torch.equal(s64, rowmax.sum(-1)) and (bound > 0).all()
    g = torch.from_numpy(z["score_weights"]).double().view(B, nway)
    dQ, dD = T.backward(Q, D, arg, g, docs_per_query=nway)[:2]
    _close(dQ.numpy(), z["score_dQ"])
    _close(dD.numpy(), z["score_dD"])


@pytest.mark.parametrize("nq", [96, 70])
def test_flipr_scores_and_grads_match_reference_autograd(nq):
    """Winners of -1 (tokens the 'flipr' reduction does not select) next to real ones, in both forms."""
    z = np.load(os.path.join(GOLDEN_DIR, "flipr.npz"))
    k = "nq%d_" % nq
    Q, D, mask = _t(z[k + "Q_bf16"]), _t(z[k + "D_bf16"]), torch.from_numpy(z[k + "mask"])
    r, w = int(z["docs_per_query"]), torch.from_numpy(z["weights"]).double()
    B = Q.size(0)
    arg, rowmax, _ = T.argmax_rowmax(Q, D, mask, docs_per_query=r)
    s, sel = T.flipr_select(rowmax, arg)
    assert (sel < 0).any() and (sel >= 0).any()
    _close(s.reshape(-1).numpy(), z[k + "aligned"])
    dQ, dD = T.backward(Q, D, sel, w.view(B, r), docs_per_query=r)[:2]
    _close(dQ.numpy(), z[k + "aligned_dQ"])
    _close(dD.numpy(), z[k + "aligned_dD"])
    arg1, rowmax1, _ = T.argmax_rowmax(Q[:1], D, mask)
    s1, sel1 = T.flipr_select(rowmax1, arg1)
    _close(s1[0].numpy(), z[k + "one"])
    dQ1, dD1 = T.backward(Q[:1], D, sel1, w[None])[:2]
    dQ_full = np.zeros_like(z[k + "one_dQ"])
    dQ_full[:1] = dQ1.numpy()
    _close(dQ_full, z[k + "one_dQ"])
    _close(dD1.numpy(), z[k + "one_dD"])


@pytest.mark.parametrize("label0", [0, 3, 10])
def test_ib_loss_matches_float64_cross_entropy(label0):
    """Positive columns shifted by label0 (the cross-rank route), a -inf negative, logit spreads of hundreds."""
    g = torch.Generator().manual_seed(label0)
    B, nway, n = 3, 2, 16
    scores = (torch.rand((B, n), generator=g, dtype=torch.float64) - 0.5) * 600
    scores[0, label0 + 1] = -torch.inf
    s, loss, ds = T.ib_loss_from_scores(scores, nway, label0)
    x = scores.clone().requires_grad_(True)
    labels = label0 + torch.arange(B) * nway
    ref = torch.nn.functional.cross_entropy(x, labels, reduction="none")
    ref.mean().backward()
    np.testing.assert_allclose(loss.numpy(), ref.detach().numpy(), rtol=1e-14, atol=1e-12)
    np.testing.assert_allclose(ds.numpy(), x.grad.numpy(), rtol=1e-12, atol=1e-14)
    assert ds[0, label0 + 1] == 0
    lb, db = T.ib_loss_bounds(scores, nway, label0)
    assert torch.isfinite(lb).all() and (lb > 0).all() and torch.isfinite(db).all() and (db > 0).all()


def test_ib_loss_with_minus_inf_positive_matches_cross_entropy():
    """A fully masked positive document scores -inf on the fused route: the loss is +inf and the gradient stays the
    finite (softmax - onehot) / B, which is what float64 cross_entropy gives."""
    scores = torch.tensor([[-torch.inf, 1.0, 3.0], [0.5, 2.0, -1.0]], dtype=torch.float64)
    s, loss, ds = T.ib_loss_from_scores(scores, 1, 0)
    x = scores.clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(x, torch.tensor([0, 1]), reduction="none")
    ref.mean().backward()
    assert torch.isposinf(loss[0]) and torch.isposinf(ref[0])
    np.testing.assert_allclose(loss[1].item(), ref[1].item(), rtol=1e-14)
    np.testing.assert_allclose(ds.numpy(), x.grad.numpy(), rtol=1e-12, atol=1e-14)
    assert ds[0, 0] == -0.5


def test_argmax_ties_take_the_lowest_index():
    D = T.bf16_rows((1, 6, 128), generator=torch.Generator().manual_seed(1))
    D[0, 4] = D[0, 1]
    Q = D[:, 1:2].clone()
    mask = torch.ones((1, 6), dtype=torch.bool)
    assert T.argmax_rowmax(Q, D, mask)[0].item() == 1
    mask[0, 1] = False
    assert T.argmax_rowmax(Q, D, mask)[0].item() == 4
    mask[:] = False
    arg, rowmax, absmax = T.argmax_rowmax(Q, D, mask)
    assert arg.item() == -1 and rowmax.item() == -np.inf and absmax.item() == 0


def test_grid_is_a_pairwise_covering():
    cases = T.argmax_grid()
    F = T.ARGMAX_FACTORS
    for f1, f2 in itertools.combinations(F, 2):
        seen = {(c[f1], c[f2]) for c in cases}
        for v1, v2 in itertools.product(F[f1], F[f2]):
            if T.argmax_allowed({f1: v1, f2: v2}):
                assert (v1, v2) in seen, (f1, v1, f2, v2)
    assert all(T.argmax_allowed(c) for c in cases)
    assert len(cases) < 200


def test_grid_reaches_every_docs_per_cta_regime():
    """On a 132-SM H100 the grid's wgmma cases split their documents one per CTA and into interior counts with a
    partial last CTA; the extra split case of the GPU test takes the 32 maximum with a partial last CTA."""
    splits = set()
    for c in T.argmax_grid():
        if c["path"] == 2:
            d = T.docs_per_cta(c["B"], c["nq"], c["n_docs"], c["nd"], 132)
            splits.add((d, c["n_docs"] % d != 0))
    assert (1, False) in splits
    assert any(1 < d < 32 and partial for d, partial in splits)
    assert T.docs_per_cta(9, 832, 127, 128, 132) == 32 and 127 % 32
