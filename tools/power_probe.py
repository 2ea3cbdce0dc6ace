"""Sustained-regime probe (GPU box): the scan kernel run back to back for `--seconds` per configuration, with
the SM clock and board power sampled by nvidia-smi during the second half of the run.  Question it answers:
how much of the power-capped (sustained) throughput depends on DATA MOVEMENT — compare a corpus streamed from
HBM (1M passages, 46 GB) with one that stays in L2 (2k passages, 92 MB): same MMA / epilogue work per
token, no HBM traffic.

    python tools/power_probe.py --passages 1000000,2000 --seconds 8
"""
import argparse
import ctypes as C
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", default="1000000,2000")
    ap.add_argument("--nd", type=int, default=180)
    ap.add_argument("--nq", type=int, default=320)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=8.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import ravqa_b200 as R
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    Q = torch.nn.functional.normalize(torch.randn((args.batch, args.nq, 128), device=dev, generator=g), dim=-1).bfloat16()
    for n_p in [int(x) for x in args.passages.split(",")]:
        D = bench.build_shard(0, n_p, args.nd, dev)
        corpus = R.FlatCorpus(D, np.full(n_p, args.nd, dtype=np.int32))
        for _ in range(3):
            R.maxsim_topk(corpus, Q, 5)
        torch.cuda.synchronize()
        # calls per timing block sized to ~0.25 s
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        R.maxsim_topk(corpus, Q, 5)
        e1.record()
        torch.cuda.synchronize()
        per_call = e0.elapsed_time(e1)
        block = max(1, int(250.0 / per_call))
        flops_call = 2.0 * args.batch * args.nq * 128 * n_p * args.nd
        t_end = time.time() + args.seconds
        rates, sampler = [], None
        while time.time() < t_end:
            if sampler is None and time.time() > t_end - args.seconds / 2:
                sampler = bench.ClockSampler(0)
                sampler.start()
            e0.record()
            for _ in range(block):
                R.maxsim_topk(corpus, Q, 5)
            e1.record()
            torch.cuda.synchronize()
            rates.append((time.time(), flops_call * block / (e0.elapsed_time(e1) * 1e-3) / 1e12))
        clk = sampler.stop() if sampler else {}
        half = [r for t, r in rates if t > t_end - args.seconds / 2]
        print("passages=%d (%.2f GB of tokens%s): first block %.0f TFLOP/s, second-half mean %.0f TFLOP/s "
              "(%.1f q/s at this size), sm %.0f MHz, power max %s W, reasons %s" %
              (n_p, n_p * args.nd * 256 / 1e9, ", L2-resident" if n_p * args.nd * 256 < 100e6 else "",
               rates[0][1], sum(half) / len(half), args.batch / (flops_call / (sum(half) / len(half) * 1e12)),
               clk.get("sm_mhz") or -1, clk.get("power_w_max"), clk.get("reasons")), flush=True)
        corpus.close()
        del D
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
