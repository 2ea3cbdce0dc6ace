"""GPU: what the per-query allow test costs the scan at the benchmark size (1M passages x 180 tokens), both storages.

    python tools/allowed_scan_probe.py [--passages 1000000] [--rounds 3] [--reps 10] [--storages bf16,fp8]
                                       [--shapes 16xNq320,12xNq32] [--no-searcher] [--json out.json]

Prints the card, its power limit and max SM clock, then per storage and shape the scan launch time (maxsim_topk,
k = 10) of four arms, median and spread over rounds of --reps launches each (the arm order reversed every other
round): unrestricted, one shared bitmap (stride 0, density 50 %), per-query bitmaps of density 50 %, and per-query
bitmaps of density 0.1 %.  Shapes:
the flagship 16 x Nq = 320 (one query per pass: the reducer's warp mode) and 12 x Nq = 32 in one pass (lane mode:
every lane loads its own query's bitmap word at every passage end, the worst case).

Then, per storage, the whole restricted Searcher call (``_search_all_Q``, 16 x Nq = 320, k = 10; host clock around a
call that ends in a device synchronise): unrestricted, and with ``qid_to_pids`` of 1k and of 100k random ids per
query (numpy arrays), plus the time of building those bitmaps alone (``FlatCorpus.allow_bitmaps``).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import ravqa_b200 as R  # noqa: E402
from ravqa_b200 import _cabi  # noqa: E402

ND = 180


def card():
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def scan_ms(L, corpus, Q, allow, reps):
    """Milliseconds per scan launch of maxsim_topk(k = 10), after a warm-up call."""
    R.maxsim_topk(corpus, Q, 10, allow=allow)
    torch.cuda.synchronize()
    L.flmr_scan_kernel_stats(None, None, 1)
    L.flmr_set_profiling(1)
    for _ in range(reps):
        R.maxsim_topk(corpus, Q, 10, allow=allow)
    torch.cuda.synchronize()
    tot, cnt = C.c_double(0), C.c_int64(0)
    L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
    L.flmr_set_profiling(0)
    return tot.value / cnt.value


def random_bitmaps(B, n, density, dev, seed):
    """int32 [B, ceil(n / 32)] with each bit set with probability `density` (drawn on the device)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    words = (n + 31) // 32
    bits = torch.rand((B, words, 32), device=dev, generator=g) < density
    w = (bits.to(torch.int64) << torch.arange(32, device=dev)).sum(-1)
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32)


def timed_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def searcher_ms(c, Q, n, rounds):
    """Median / spread (ms) of whole Searcher calls, unrestricted and restricted, and of the bitmap builds alone."""
    sr = R.Searcher(index=c)
    rng = np.random.default_rng(4)
    lists = {size: {b: rng.integers(0, n, size=size) for b in range(Q.size(0))} for size in (1_000, 100_000)}
    arms = {"unrestricted": lambda: sr._search_all_Q(list(range(Q.size(0))), Q, k=10)}
    for size, q2p in lists.items():
        arms["qid_to_pids %d ids/query" % size] = (
            lambda q2p=q2p: sr._search_all_Q(list(range(Q.size(0))), Q, k=10, qid_to_pids=q2p))
        arms["bitmaps alone, %d ids/query" % size] = lambda q2p=q2p: c.allow_bitmaps(list(q2p.values()))
    for fn in arms.values():
        fn()                                                       # warm-up
    times = {a: [] for a in arms}
    for _ in range(rounds):
        for a, fn in arms.items():
            times[a].append(timed_ms(fn))
    out = {}
    for a, t in times.items():
        out[a] = {"ms": statistics.median(t), "spread_ms": max(t) - min(t), "samples": t}
        print("[%s searcher 16xNq320 k=10] %-32s %.2f ms (spread %.2f)"
              % (c.storage, a, statistics.median(t), max(t) - min(t)), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10, help="scan launches per arm and round")
    ap.add_argument("--storages", default="bf16,fp8")
    ap.add_argument("--shapes", default="16xNq320,12xNq32")
    ap.add_argument("--no-searcher", action="store_true", help="skip the whole-Searcher timings")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    L = _cabi.lib()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.passages
    rec = {"card": card(), "passages": n, "nd": ND}
    print("card (name, power limit, max SM clock):", rec["card"], "passages:", n, flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    shapes = {s: {"16xNq320": (16, 320), "12xNq32": (12, 32)}[s] for s in args.shapes.split(",")}
    Qs = {s: torch.nn.functional.normalize(torch.randn((B, nq, 128), device=dev, generator=g), dim=-1).bfloat16()
          for s, (B, nq) in shapes.items()}
    for storage in args.storages.split(","):
        D = bench.build_shard(0, n, ND, dev)
        c = R.FlatCorpus(D, np.full(n, ND, dtype=np.int32), storage=storage)   # bf16: adopted, no second copy
        del D
        torch.cuda.empty_cache()
        rec[storage] = {}
        for sname, (B, _) in shapes.items():
            arms = {"unrestricted": None,
                    "shared 50%": random_bitmaps(1, n, 0.5, dev, 1)[0],
                    "per-query 50%": random_bitmaps(B, n, 0.5, dev, 2),
                    "per-query 0.1%": random_bitmaps(B, n, 0.001, dev, 3)}
            times = {a: [] for a in arms}
            sampler = bench.ClockSampler(0)
            sampler.start()
            for r in range(args.rounds):
                for a in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                    times[a].append(scan_ms(L, c, Qs[sname], arms[a], args.reps))
            clocks = sampler.stop()
            out = {"clocks": clocks}
            for a, t in times.items():
                out[a] = {"launch_ms": statistics.median(t), "spread_ms": max(t) - min(t), "samples": t}
                print("[%s %s] %-15s scan launch %.3f ms (spread %.3f)"
                      % (storage, sname, a, statistics.median(t), max(t) - min(t)), flush=True)
            rec[storage][sname] = out
        if not args.no_searcher:
            Q = torch.nn.functional.normalize(torch.randn((16, 320, 128), device=dev, generator=g), dim=-1).bfloat16()
            rec[storage]["searcher"] = searcher_ms(c, Q, n, args.rounds)
        c.close()
        del c
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(rec, f, indent=1, default=str)


if __name__ == "__main__":
    main()
