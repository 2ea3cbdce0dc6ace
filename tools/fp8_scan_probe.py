"""GPU: the e4m3 corpus (storage="fp8") against bf16 over the same 180-token passages, in alternating rounds.

    python tools/fp8_scan_probe.py [--passages 1000000] [--rounds 3] [--json out.json]

Prints the card, its power limit and the median SM clock of the timed window, then:
  * scan launch time, queries/s and TFLOP/s (algorithmic: 2 B Nq 128 N Nd) of 16 x Nq = 320 (one query per pass),
    and GB/s (algorithmic: N Nd 128 bytes per element) of the HBM-bound pass, one Nq = 32 query, and of twelve
    Nq = 32 queries in one pass;
  * the two- and three-warpgroup fp8 kernels by occupied 64-row query blocks (launch_scan's threshold);
  * Searcher end-to-end queries/s (k = 10): fp8 scan + exact re-rank of ndocs / 4 = 256 candidates against bf16;
  * on isotropic random queries: the shortlist depth each query needed to contain its exact top-5 / top-100, the
    largest relative score error of the fp8 scan, and Recall@5 of planted positives (bench.planted_queries).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import ravqa_b200 as R  # noqa: E402
from ravqa_b200 import _cabi  # noqa: E402

ND = 180


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out


def timed_topk(L, corpus, Q, k, reps):
    """(ms per call, ms per scan launch, ms of scan launches per call) of maxsim_topk, after one warm-up call."""
    R.maxsim_topk(corpus, Q, k)
    torch.cuda.synchronize()
    L.flmr_scan_kernel_stats(None, None, 1)
    L.flmr_set_profiling(1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        R.maxsim_topk(corpus, Q, k)
    e1.record()
    torch.cuda.synchronize()
    tot, cnt = C.c_double(0), C.c_int64(0)
    L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
    L.flmr_set_profiling(0)
    return e0.elapsed_time(e1) / reps, tot.value / cnt.value, tot.value / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    L = _cabi.lib()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.passages
    while True:
        D = bench.build_shard(0, n, ND, dev)
        dl = np.full(n, ND, dtype=np.int32)
        c16 = R.FlatCorpus(D, dl)                     # adopts D
        try:
            c8 = R.FlatCorpus(D, dl, storage="fp8")  # e4m3 copy in HBM + pinned bf16 master (n x 46 kB of host RAM)
            break
        except _cabi.FlmrError as e:
            if n <= 100_000:
                raise
            print("fp8 corpus of %d passages failed (%s); halving" % (n, e), flush=True)
            c16.close()
            del D
            torch.cuda.empty_cache()
            n //= 2
    rec = {"card": card(), "passages": n, "nd": ND}
    print("card (name, power limit, max SM clock):", rec["card"], "passages:", n, flush=True)
    rec["hbm_bytes"] = {"bf16": int(c16.info.hbm_bytes), "fp8": int(c8.info.hbm_bytes)}
    print("hbm_bytes bf16 %.2f GB (adopted matrix not counted), fp8 %.2f GB"
          % (c16.info.hbm_bytes / 1e9, c8.info.hbm_bytes / 1e9), flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    corpora = {"bf16": c16, "fp8": c8}

    # ---- scan: flagship and HBM-bound passes, bf16 / fp8 alternating ----
    shapes = {"flagship 16 x Nq=320": (16, 320, 2), "HBM-bound 1 x Nq=32": (1, 32, 10),
              "12 x Nq=32 in one pass": (12, 32, 10)}
    Qs = {name: torch.nn.functional.normalize(torch.randn((B, nq, 128), device=dev, generator=g), dim=-1).bfloat16()
          for name, (B, nq, _) in shapes.items()}
    samples = {(name, st): [] for name in shapes for st in corpora}
    sampler = bench.ClockSampler(0)
    sampler.start()
    for _ in range(args.rounds):
        for name, (B, nq, reps) in shapes.items():
            for st, c in corpora.items():
                samples[(name, st)].append(timed_topk(L, c, Qs[name], 10, reps))
    clocks = sampler.stop()
    rec["scan_clocks"] = clocks
    print("\nmedian SM clock of the scan window: %s MHz (max %s, reasons %s)"
          % (clocks.get("sm_mhz"), clocks.get("sm_max_mhz"), clocks.get("reasons")))
    print("\n| pass | storage | scan launch ms (median, spread) | queries/s | TFLOP/s | GB/s (algorithmic) |\n"
          "|---|---|---:|---:|---:|---:|")
    rec["scan"] = {}
    for name, (B, nq, _) in shapes.items():
        for st in corpora:
            s = samples[(name, st)]
            ms_call, ms_launch, scan_call = (statistics.median(x) for x in zip(*s))
            spread = max(x[1] for x in s) - min(x[1] for x in s)
            tflops = 2.0 * B * nq * 128 * n * ND / scan_call / 1e9
            gbs = n * ND * 128 * (1 if st == "fp8" else 2) / ms_launch / 1e6
            rec["scan"]["%s %s" % (name, st)] = {"launch_ms": ms_launch, "spread_ms": spread, "qps": B / ms_call * 1e3,
                                                 "tflops": tflops, "gbs": gbs}
            print("| %s | %s | %.2f (%.2f) | %.1f | %.0f | %.0f |"
                  % (name, st, ms_launch, spread, B / ms_call * 1e3, tflops, gbs), flush=True)

    # ---- fp8 warpgroup variants by occupied 64-row blocks ----
    print("\n| fp8 pass | blocks | 2 WGs launch ms | 3 WGs launch ms |\n|---|---:|---:|---:|")
    rec["fp8_variants"] = {}
    for (B, nq, blocks) in [(1, 320, 5), (3, 832, 6), (1, 256, 4), (12, 32, 6), (2, 64, 2)]:
        Q = torch.nn.functional.normalize(torch.randn((B, nq, 128), device=dev, generator=g), dim=-1).bfloat16()
        t = {2: [], 3: []}
        for _ in range(3):
            for v in (2, 3):
                L.flmr_debug_set_scan_variant(v)
                t[v].append(timed_topk(L, c8, Q, 5, 2)[1])
        L.flmr_debug_set_scan_variant(0)
        m2, m3 = statistics.median(t[2]), statistics.median(t[3])
        rec["fp8_variants"]["B=%d Nq=%d" % (B, nq)] = {"blocks": blocks, "2": m2, "3": m3}
        print("| B=%d Nq=%d | %d | %.2f | %.2f |" % (B, nq, blocks, m2, m3), flush=True)

    # ---- Searcher end to end (k = 10), planted positives ----
    Qp, targets = bench.planted_queries(16, 320, ND, n, 1, dev)
    Qp = Qp.bfloat16()
    s16, s8 = R.Searcher(index=c16), R.Searcher(index=c8, storage="fp8")
    tms = {"bf16": [], "fp8": []}
    res = {}
    for _ in range(args.rounds):
        for st, s in (("bf16", s16), ("fp8", s8)):
            s._search_tensors(Qp, 10)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res[st] = s._search_tensors(Qp, 10)
            e1.record()
            torch.cuda.synchronize()
            tms[st].append(e0.elapsed_time(e1))
    recall = {st: float(np.mean([targets[b] in res[st][1][b, :5].tolist() for b in range(16)])) for st in res}
    same = bool(torch.equal(res["fp8"][1], res["bf16"][1]))
    rec["searcher"] = {st: {"ms": statistics.median(tms[st]), "qps": 16e3 / statistics.median(tms[st]),
                            "recall@5_planted": recall[st]} for st in tms}
    rec["searcher"]["ids_identical"] = same
    print("\n| Searcher k=10, 16 x Nq=320 | ms per call | queries/s | planted Recall@5 |\n|---|---:|---:|---:|")
    for st in tms:
        r = rec["searcher"][st]
        print("| %s | %.1f | %.1f | %.2f |" % (st, r["ms"], r["qps"], r["recall@5_planted"]))
    print("top-10 ids identical:", same, flush=True)

    # ---- shortlist depth needed, score error (isotropic queries) ----
    Qi = Qs["flagship 16 x Nq=320"]
    e16 = R.maxsim_scores(c16, Qi)
    e8 = R.maxsim_scores(c8, Qi)
    rel = ((e8 - e16).abs() / e16.abs().clamp_min(1e-6)).max().item()
    pid = torch.arange(n, device=dev)
    need = {5: [], 100: []}
    _, top = R.topk_select(e16, 100)
    for b in range(Qi.size(0)):
        ranks = []
        for i in top[b].tolist():
            v = e8[b, i]
            ranks.append(int(((e8[b] > v) | ((e8[b] == v) & (pid < i))).sum().item()))
        need[5].append(max(ranks[:5]) + 1)
        need[100].append(max(ranks) + 1)
    rec["depth_needed"] = {"top5": need[5], "top100": need[100], "ndocs/4": 256}
    rec["max_rel_score_error"] = rel
    print("\nmax relative score error of the fp8 scan (isotropic 16 x Nq=320): %.2e" % rel)
    print("depth needed for the exact top-5:   max %d, median %d (ndocs/4 = 256)"
          % (max(need[5]), statistics.median(need[5])))
    print("depth needed for the exact top-100: max %d, median %d (ndocs/4 = 256; %d of %d queries need more)"
          % (max(need[100]), statistics.median(need[100]), sum(x > 256 for x in need[100]), len(need[100])),
          flush=True)
    c8.close()
    c16.close()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
