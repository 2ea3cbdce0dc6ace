"""GPU probe of the training path (SURVEY.md 8a a6 / 8f-2): the in-batch-negatives loss, forward + backward.

    python tools/train_step_probe.py                       # one GPU: one rank of the C4 step and its global batch
    torchrun --nproc-per-node N tools/train_step_probe.py --torchrun     # N ranks, cross-rank negatives (C4: N = 8)

Shapes (CB/modeling/colbert.py:64-113): per rank 8 queries x 16 documents (nway = 2), Nq = 832, Nd = 512, d = 128,
ragged masks.  "global" = the same 8 queries against the documents of all 8 ranks (128 documents): the matrix
cross-rank negatives produce (colbert.py:115-163).

Reported: the arg-max forward alone under both of its kernels (warp-MMA / wgmma) with TFLOP/s, the three kernels
of a step (forward, loss head, backward) timed alone, the whole step through `in_batch_negatives_loss(...).backward()`,
and a torch restatement of the reference's compute_ib_loss_new (fp32, materialises [B, B*nway, Nd, Nq]).
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ravqa_b200 as R  # noqa: E402
from ravqa_b200 import _cabi  # noqa: E402
from ravqa_b200.maxsim import ib_loss_head, maxsim_argmax, maxsim_backward  # noqa: E402


def ref_loss(Q, D, mask, nway):
    scores = (D.float().unsqueeze(0) @ Q.float().permute(0, 2, 1).unsqueeze(1)).flatten(0, 1)   # colbert.py:89
    m = mask.repeat(Q.size(0), 1, 1)
    scores = scores.masked_fill(~m, -9999.0)                                                     # :240
    scores = scores.max(1).values.sum(-1).reshape(Q.size(0), -1)                                 # :241,263
    return torch.nn.functional.cross_entropy(scores, torch.arange(Q.size(0), device=Q.device) * nway)


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def make(B, n, nq, nd, seed, dev):
    g = torch.Generator().manual_seed(seed)
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).to(dev)
    D = torch.nn.functional.normalize(torch.randn(n, nd, 128, generator=g), dim=-1).to(dev)
    lens = torch.randint(nd // 2, nd + 1, (n,), generator=g)
    mask = (torch.arange(nd)[None, :] < lens[:, None]).to(dev)
    return Q, D, mask, int(lens.sum())


def single_gpu():
    dev = torch.device("cuda", 0)
    L = _cabi.lib()
    B, nway, nq, nd = 8, 2, 832, 512
    print("| shape | kernel | ms | TFLOP/s (unmasked tokens) |\n|---|---|---:|---:|")
    for name, n in (("one rank: 8 q x 16 docs", B * nway), ("global batch: 8 q x 128 docs", 8 * B * nway),
                    ("64 q x 128 docs (whole global batch on one GPU)", 8 * B * nway)):
        Bq = 64 if name.startswith("64") else B
        Q, D, mask, tok = make(Bq, n, nq, nd, 0, dev)
        Qb, Db = Q.bfloat16(), D.bfloat16()
        flops = 2.0 * Bq * nq * 128 * tok
        for path, label in ((1, "warp-MMA (mma.sync)"), (2, "wgmma (compact + TMA/wgmma pipeline)")):
            L.flmr_debug_set_argmax_path(path)
            ms = timed(lambda: maxsim_argmax(Qb, Db, mask, return_rowmax=True))
            print("| %s | arg-max forward, %s | %.3f | %.0f |" % (name, label, ms, flops / ms / 1e9))
        L.flmr_debug_set_argmax_path(0)
    # the pieces of one rank's step and the step itself
    Q, D, mask, tok = make(B, B * nway, nq, nd, 0, dev)
    Qb, Db = Q.bfloat16(), D.bfloat16()
    arg, rowmax = maxsim_argmax(Qb, Db, mask, return_rowmax=True)
    _, _, ds = ib_loss_head(rowmax, nway)
    t_f = timed(lambda: maxsim_argmax(Qb, Db, mask, return_rowmax=True))
    t_l = timed(lambda: ib_loss_head(rowmax, nway))
    t_b = timed(lambda: maxsim_backward(Qb, Db, arg, ds))
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    m3 = mask.unsqueeze(-1)

    def step():
        Qg.grad = Dg.grad = None
        R.in_batch_negatives_loss(Qg, Dg, m3, nway).backward()

    def ref():
        Qg.grad = Dg.grad = None
        ref_loss(Qg, Dg, m3, nway).backward()
    t_s = timed(step)
    t_r = timed(ref, reps=5)
    # the same step with forward and backward captured as CUDA graphs (autograd-aware: make_graphed_callables) ...
    graphed = R.graphed_in_batch_negatives_loss(Qg, Dg, m3, nway)

    def step_graphed():
        Qg.grad = Dg.grad = None
        graphed(Qg, Dg, m3).backward()
    t_g = timed(step_graphed)
    # ... and as ONE graph of forward + backward over static buffers (what a fully captured training step replays)
    Qs, Ds = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            Qs.grad = Ds.grad = None
            R.in_batch_negatives_loss(Qs, Ds, m3, nway).backward()
    torch.cuda.current_stream().wait_stream(side)
    whole = torch.cuda.CUDAGraph()
    Qs.grad = Ds.grad = None
    with torch.cuda.graph(whole):
        loss_static = R.in_batch_negatives_loss(Qs, Ds, m3, nway)
        loss_static.backward()
    t_w = timed(whole.replay)
    Qg.grad = Dg.grad = None
    eager_loss = R.in_batch_negatives_loss(Qg, Dg, m3, nway)
    eager_loss.backward()
    whole.replay()
    torch.cuda.synchronize()
    same = (torch.equal(eager_loss.detach(), loss_static.detach()) and torch.equal(Qg.grad, Qs.grad)
            and torch.allclose(Dg.grad, Ds.grad, rtol=1e-5, atol=1e-7))
    # where the host time of a step goes (CPU-side cost of each call, launches are asynchronous)
    import time
    from ravqa_b200 import modeling
    def host(fn, reps=50):
        fn(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        dt = (time.perf_counter() - t0) / reps * 1e3
        torch.cuda.synchronize()
        return dt
    h = {
        "casts Q,D -> bf16": host(lambda: (Q.detach().to(torch.bfloat16).contiguous(), D.detach().to(torch.bfloat16).contiguous())),
        "maxsim_argmax (python + C call: cudaMallocAsync, compact, 2 tensor maps, tc kernel, free)": host(lambda: maxsim_argmax(Qb, Db, mask, return_rowmax=True)),
        "ib_loss_head": host(lambda: ib_loss_head(rowmax, nway)),
        "maxsim_backward": host(lambda: maxsim_backward(Qb, Db, arg, ds)),
        "loss.mean + dscores * g": host(lambda: (rowmax[0, 0].mean(), ds * 1.0)),
        "forward only (autograd function)": host(lambda: R.in_batch_negatives_loss(Qg, Dg, m3, nway)),
        "whole step": host(step),
    }
    print("\n| host-side cost per call | ms |\n|---|---:|")
    for k, v in h.items():
        print("| %s | %.3f |" % (k, v))
    print("\n| one rank of the C4 step (8 q x 16 docs) | ms |\n|---|---:|")
    print("| arg-max forward kernel(s) | %.3f |" % t_f)
    print("| loss head kernel (scores, cross-entropy, d loss / d scores) | %.3f |" % t_l)
    print("| backward kernels (dQ gather, dD scatter, memset) | %.3f |" % t_b)
    print("| sum of the kernels | %.3f |" % (t_f + t_l + t_b))
    print("| whole step: in_batch_negatives_loss(...).backward() incl. casts and autograd | %.3f (kernels = %.0f %%) |"
          % (t_s, 100 * (t_f + t_l + t_b) / t_s))
    print("| the same step, forward and backward replayed as CUDA graphs (graphed_in_batch_negatives_loss) | %.3f "
          "(kernels = %.0f %%) |" % (t_g, 100 * (t_f + t_l + t_b) / t_g))
    print("| the same step as ONE captured graph of forward + backward (static buffers; loss and gradients equal "
          "to eager: %s) | %.3f (kernels = %.0f %%) |" % (same, t_w, 100 * (t_f + t_l + t_b) / t_w))
    print("| torch restatement of compute_ib_loss_new (fp32, materialised) | %.3f |" % t_r)


def multi_gpu():
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    dist.init_process_group("nccl", device_id=dev)
    B, nway, nq, nd = 8, 2, 832, 512
    Q, D, mask, _ = make(B, B * nway, nq, nd, 100 + rank, dev)
    Qg, Dg = Q.clone().requires_grad_(True), D.clone().requires_grad_(True)
    m3 = mask.unsqueeze(-1)

    def step(cross):
        Qg.grad = Dg.grad = None
        R.in_batch_negatives_loss(Qg, Dg, m3, nway, cross_rank_negatives=cross).backward()
    out = {}
    for cross in (False, True):
        for _ in range(3):
            step(cross)
        dist.barrier()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            step(cross)
        b.record()
        dist.barrier()
        torch.cuda.synchronize()
        t = torch.tensor([a.elapsed_time(b) / 20], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        out[cross] = t.item()
    if rank == 0:
        print("| C4 loss step on %d ranks (bsz %d = %d per rank, nway 2, Nq 832, Nd 512), max over ranks | ms |\n|---|---:|"
              % (world, B * world, B))
        print("| local in-batch negatives only (the reference's behaviour, colbert.py:69 commented out) | %.3f |" % out[False])
        print("| cross-rank negatives: all-gather of D + [8, %d] matrix per rank + reduce-scatter of dD | %.3f |"
              % (B * nway * world, out[True]))
    dist.destroy_process_group()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--torchrun", action="store_true")
    if ap.parse_args().torchrun:
        multi_gpu()
    else:
        single_gpu()
