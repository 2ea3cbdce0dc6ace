"""GPU probe: does a scan launch have a FIXED cost that strong scaling exposes?

    python tools/launch_fixed_cost_probe.py [--block-seconds 1.5] [--rounds 3]

Strong scaling over N GPUs divides the shard (1M passages / N) but not whatever a launch costs independent of its
size (prologue: barrier init, query tiles into shared memory; pipeline fill; tail: the slowest CTA, the
reducers' last tiles, candidate lists; launch gap).  This probe runs the headline call (16 queries of Nq = 320, k = 5:
sixteen passes) against shards of 125k / 250k / 500k / 1M passages x 180 tokens on ONE GPU, interleaved in
blocks of --block-seconds so every size sees the same power-capped regime, and fits
    scan launch ms = a + b * passages          (a = fixed cost per launch, b = streaming cost)
    call ms        = scans + c                 (c = staging + merge launches + gaps per call)
so that the 8-GPU step can be predicted from one GPU: step(1M / 8) vs step(1M) / 8.
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ravqa_b200 as R  # noqa: E402
from ravqa_b200 import _cabi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--block-seconds", type=float, default=1.5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import bench
    L = _cabi.lib()
    dev = torch.device("cuda", 0)
    nd, sizes = 180, [125_000, 250_000, 500_000, 1_000_000]
    D = bench.build_shard(0, sizes[-1], nd, dev)
    corpora = {n: R.FlatCorpus(D[: n * nd], np.full(n, nd, dtype=np.int32)) for n in sizes}
    g = torch.Generator(device=dev).manual_seed(0)
    Q = torch.nn.functional.normalize(torch.randn((16, 320, 128), device=dev, generator=g), dim=-1).bfloat16()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rows = {n: [] for n in sizes}
    # warm the power regime up on the largest shard
    t_end = time.time() + 3.0
    while time.time() < t_end:
        for _ in range(2):
            R.maxsim_topk(corpora[sizes[-1]], Q, 5)
        torch.cuda.synchronize()
    for rnd in range(args.rounds):
        for n in (sizes if rnd % 2 == 0 else sizes[::-1]):
            c = corpora[n]
            R.maxsim_topk(c, Q, 5)
            torch.cuda.synchronize()
            L.flmr_scan_kernel_stats(None, None, 1)
            L.flmr_set_profiling(1)
            per = max(1, int(4 * sizes[-1] / n))
            t_end, calls = time.time() + args.block_seconds, 0
            e0.record()
            while time.time() < t_end:
                for _ in range(per):
                    R.maxsim_topk(c, Q, 5)
                calls += per
                e1.record()
                e1.synchronize()
            tot, cnt = C.c_double(0), C.c_int64(0)
            L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
            L.flmr_set_profiling(0)
            rows[n].append((tot.value / cnt.value, e0.elapsed_time(e1) / calls, cnt.value // calls))
    print("| passages | scan launch ms (per round) | call ms (per round) | launches / call | call - scans (ms) |")
    print("|---:|---|---|---:|---:|")
    xs, ys, cs = [], [], []
    for n in sizes:
        lm = [r[0] for r in rows[n]]
        cm = [r[1] for r in rows[n]]
        k = rows[n][0][2]
        over = float(np.mean(cm) - k * np.mean(lm))
        print("| %d | %s | %s | %d | %.3f |" % (n, " / ".join("%.3f" % v for v in lm), " / ".join("%.3f" % v for v in cm),
                                               k, over))
        xs.append(n)
        ys.append(float(np.mean(lm)))
        cs.append(over)
    b, a = np.polyfit(np.array(xs, dtype=np.float64), np.array(ys), 1)
    print("\nfit: scan launch ms = %.4f + %.4f * (passages / 125k)   -> fixed cost %.1f us per launch = %.2f %% of a "
          "125k-passage launch" % (a, b * 125_000, a * 1e3, 100 * a / ys[0]))
    print("profiling on (events around every scan launch) adds a few us of gap per launch to 'call - scans'")
    print("predicted strong-scaling efficiency at 8 shards from this GPU alone: call(1M) / (8 * call(125k)) = %.4f"
          % (np.mean([r[1] for r in rows[sizes[-1]]]) / (8 * np.mean([r[1] for r in rows[sizes[0]]]))))


if __name__ == "__main__":
    main()
