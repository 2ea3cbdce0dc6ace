"""GPU: the scan kernel's variants — flmr_scan_kernel<2> (two consumer warpgroups), <3> (three), flmr_scan_split_kernel
(three, split-tile loop) and CTA-pair passes — bit-identical results of <2>, <3> and the split kernel over a spread of
shapes, then timing of all four.

    python tools/scan_variant_probe.py [--passages 200000]
"""
import argparse
import ctypes as C
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ravqa_b200 as R  # noqa: E402
from ravqa_b200 import _cabi  # noqa: E402
from oracle import maxsim_oracle as O  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=200_000)
    ap.add_argument("--skip-parity", action="store_true")
    ap.add_argument("--repeat", type=int, default=1, help="timed repetitions per shape and variant (median, spread)")
    ap.add_argument("--sustained", type=float, default=0.0, help="seconds per block of the power-capped A/B (0 = skip)")
    args = ap.parse_args()
    L = _cabi.lib()
    dev = torch.device("cuda", 0)
    if not args.skip_parity:
        bad = 0
        for (n, nd, B, nq, ragged, relu, k) in [
                (3000, 60, 1, 32, True, False, 5), (3000, 60, 2, 64, True, True, 7), (2000, 180, 1, 320, False, False, 5),
                (2000, 180, 2, 320, True, False, 100), (1500, 90, 3, 129, True, False, 5), (1500, 90, 4, 128, True, False, 5),
                (1200, 100, 5, 97, True, False, 3), (900, 64, 20, 32, True, False, 5), (700, 50, 3, 832, True, False, 10),
                (5, 7, 2, 320, True, False, 5), (2500, 13, 2, 320, True, False, 5), (800, 200, 16, 320, True, False, 5)]:
            Q, D, dl = O.synth(n, nd, B, nq, seed=n + nq, ragged=ragged)
            corpus = R.FlatCorpus(torch.from_numpy(D).to(torch.bfloat16), dl, device=0)
            Qt = torch.from_numpy(Q)
            L.flmr_debug_set_scan_variant(2)
            s2 = R.maxsim_scores(corpus, Qt, relu=relu)
            t2 = R.maxsim_topk(corpus, Qt, min(k, n), relu=relu)
            ok = True
            for variant in (3, 6, 4):
                L.flmr_debug_set_scan_variant(variant)
                s3 = R.maxsim_scores(corpus, Qt, relu=relu)
                t3 = R.maxsim_topk(corpus, Qt, min(k, n), relu=relu)
                torch.cuda.synchronize()
                if variant != 4:     # same partition, same summation order: bit-identical
                    ok = ok and torch.equal(s2, s3) and torch.equal(t2[0], t3[0]) and torch.equal(t2[1], t3[1])
                else:                # the pair partition moves tile boundaries: a passage that is the 5th+ to end
                    # in its tile is summed lanes-first instead of row-blocks-first -> last-bit differences
                    ok = ok and torch.allclose(s2, s3, rtol=2e-6, atol=0) and torch.equal(t2[1], t3[1])
            ref = O.maxsim_scores(Q, D, dl, relu=relu)
            rel = float(np.max(np.abs(s3.cpu().numpy() - ref) / np.maximum(np.abs(ref), 1e-6)))
            print("n=%d nd=%d B=%d nq=%d ragged=%s relu=%s k=%d: identical=%s max_rel_vs_oracle=%.1e"
                  % (n, nd, B, nq, ragged, relu, k, ok, rel), flush=True)
            bad += (not ok) or rel > 2e-5
            corpus.close()
        print("parity:", "OK" if bad == 0 else "%d FAILED" % bad, flush=True)
        if bad:
            sys.exit(1)
    import bench
    n_p, nd = args.passages, 180
    D = bench.build_shard(0, n_p, nd, dev)
    corpus = R.FlatCorpus(D, np.full(n_p, nd, dtype=np.int32))
    g = torch.Generator(device=dev).manual_seed(0)
    print("| shape | variant | scan launch ms | spread ms | TFLOP/s (algorithmic) | GB/s | q/s at 1M |\n"
          "|---|---|---:|---:|---:|---:|---:|")
    for (B, nq) in [(16, 320), (2, 320), (1, 320), (20, 32), (12, 32), (1, 32), (3, 832), (4, 256), (2, 128)]:
        Q = torch.nn.functional.normalize(torch.randn((B, nq, 128), device=dev, generator=g), dim=-1).bfloat16()
        for variant in (2, 3, 6, 4):
            if variant == 4 and (B % 2 or nq > 384):   # pairs of whole queries that fit one pass
                continue
            L.flmr_debug_set_scan_variant(variant)
            for _ in range(2):
                R.maxsim_topk(corpus, Q, 5)
            torch.cuda.synchronize()
            samples = []   # (ms per call, ms per scan launch, ms of scan per call)
            for _ in range(args.repeat):
                L.flmr_scan_kernel_stats(None, None, 1)
                L.flmr_set_profiling(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                iters = 6
                for _ in range(iters):
                    R.maxsim_topk(corpus, Q, 5)
                e1.record()
                torch.cuda.synchronize()
                tot, cnt = C.c_double(0), C.c_int64(0)
                L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
                L.flmr_set_profiling(0)
                samples.append((e0.elapsed_time(e1) / iters, tot.value / cnt.value, tot.value / iters))
            ms_call, ms_launch, scan_call = (statistics.median(x) for x in zip(*samples))
            spread = max(x[1] for x in samples) - min(x[1] for x in samples)
            flops_call = 2.0 * B * nq * 128 * n_p * nd
            print("| B=%d Nq=%d | %s | %.3f | %.3f | %.0f | %.0f | %.1f |"
                  % (B, nq, {2: "2 WGs", 3: "3 WGs", 6: "3 WGs, split", 4: "CTA pairs (multicast)"}[variant], ms_launch, spread,
                     flops_call / scan_call / 1e9, n_p * nd * 256.0 / ms_launch / 1e6, B / ms_call * 1e3 * n_p / 1e6),
                  flush=True)
    # sustained (power-capped) A/B at the headline shape: alternate the two variants in blocks of ~2 s, three rounds
    if args.sustained:
        import time
        Q = torch.nn.functional.normalize(torch.randn((16, 320, 128), device=dev, generator=g), dim=-1).bfloat16()
        flops_call = 2.0 * 16 * 320 * 128 * n_p * nd
        print("\n| sustained block | variant | TFLOP/s |\n|---|---|---:|")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for rnd in range(3):
            for variant in (2, 4):
                L.flmr_debug_set_scan_variant(variant)
                R.maxsim_topk(corpus, Q, 5)
                torch.cuda.synchronize()
                t_end, calls = time.time() + args.sustained, 0
                e0.record()
                while time.time() < t_end:
                    for _ in range(4):
                        R.maxsim_topk(corpus, Q, 5)
                    calls += 4
                    e1.record()
                    e1.synchronize()
                print("| %d | %s | %.0f |" % (rnd, {2: "2 WGs", 4: "CTA pairs (multicast)"}[variant],
                                            flops_call * calls / (e0.elapsed_time(e1) * 1e-3) / 1e12), flush=True)
        Q1 = Q[:1].contiguous()
        flops1 = 2.0 * 320 * 128 * n_p * nd
        print("\n| sustained block, B=1 Nq=320 | variant | TFLOP/s (algorithmic) |\n|---|---|---:|")
        for rnd in range(3):
            for variant in (2, 3):
                L.flmr_debug_set_scan_variant(variant)
                R.maxsim_topk(corpus, Q1, 5)
                torch.cuda.synchronize()
                t_end, calls = time.time() + args.sustained, 0
                e0.record()
                while time.time() < t_end:
                    for _ in range(8):
                        R.maxsim_topk(corpus, Q1, 5)
                    calls += 8
                    e1.record()
                    e1.synchronize()
                print("| %d | %d WGs | %.0f |" % (rnd, variant, flops1 * calls / (e0.elapsed_time(e1) * 1e-3) / 1e12), flush=True)
    L.flmr_debug_set_scan_variant(0)


if __name__ == "__main__":
    main()
