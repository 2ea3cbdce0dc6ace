"""Timing probe for the scan kernel (GPU box): q/s and per-launch scan time for a synthetic corpus, each run in a
fresh child process (--modes 0,0,0 repeats it; the label is the FLMR_DEBUG_MODE the child sees, which the scan
kernel ignores).

    python tools/perf_probe.py --passages 200000 --modes 0,0,0
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def one(args):
    import numpy as np
    import torch
    import ravqa_b200 as R
    from ravqa_b200 import _cabi
    n_p, nd, nq, B = args.passages, args.nd, args.nq, args.batch
    g = torch.Generator(device="cuda").manual_seed(0)
    D = torch.empty((n_p * nd, 128), dtype=torch.bfloat16, device="cuda")
    step = 20000
    for c0 in range(0, n_p, step):
        c1 = min(n_p, c0 + step)
        D[c0 * nd:c1 * nd] = torch.nn.functional.normalize(
            torch.randn(((c1 - c0) * nd, 128), device="cuda", generator=g), dim=-1).to(torch.bfloat16)
    Q = torch.nn.functional.normalize(torch.randn((B, nq, 128), device="cuda", generator=g), dim=-1).to(torch.bfloat16)
    corpus = R.FlatCorpus(D, np.full(n_p, nd, dtype=np.int32))
    L = _cabi.lib()
    for _ in range(2):
        R.maxsim_topk(corpus, Q, args.k)
    torch.cuda.synchronize()
    L.flmr_set_profiling(1)
    L.flmr_scan_kernel_stats(None, None, 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        R.maxsim_topk(corpus, Q, args.k)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.iters
    tot, n = C.c_double(), C.c_int64()
    L.flmr_scan_kernel_stats(C.byref(tot), C.byref(n), 1)
    scan_ms = tot.value / max(n.value, 1)
    launches_per_call = n.value / args.iters
    q_per_launch = B / launches_per_call
    flops = 2.0 * q_per_launch * nq * 128 * n_p * nd
    byts = n_p * nd * 256.0
    print("mode=%s passages=%d nq=%d B=%d: %.3f ms/call (%.1f q/s; x%.1f -> %.1f q/s at 1M) | scan launch %.3f ms "
          "(%d/call): %.0f TFLOP/s, %.0f GB/s" %
          (os.environ.get("FLMR_DEBUG_MODE", "0"), n_p, nq, B, ms, B / ms * 1e3, 1e6 / n_p,
           B / ms * 1e3 * n_p / 1e6, scan_ms, launches_per_call, flops / scan_ms / 1e9, byts / scan_ms / 1e6),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=200_000)
    ap.add_argument("--nd", type=int, default=180)
    ap.add_argument("--nq", type=int, default=320)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--modes", default="0")
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        one(args)
        return
    for m in args.modes.split(","):
        env = dict(os.environ, FLMR_DEBUG_MODE=m)
        cmd = [sys.executable, os.path.abspath(__file__), "--child"] + [a for a in sys.argv[1:] if a != "--child"]
        try:
            subprocess.run(cmd, env=env, timeout=300)
        except subprocess.TimeoutExpired:
            print("mode=%s TIMEOUT" % m, flush=True)


if __name__ == "__main__":
    main()
