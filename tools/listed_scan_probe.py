"""GPU: what a restricted search costs on the listed scan (maxsim_topk(pids=): the scan over a plan of the listed passages'
rows) against the bitmap scan (maxsim_topk(allow=): the whole shard, the allow test in the reducer) and the
unrestricted scan, at the benchmark size (1M passages x 180 tokens), both storages.

    python tools/listed_scan_probe.py [--passages 1000000] [--rounds 3] [--reps 5] [--storages bf16,fp8]
                                      [--shapes 16xNq320,12xNq32] [--sizes 10,100,1000,10000,100000]
                                      [--no-searcher] [--json out.json]

Prints the card, its power limit and max SM clock (read in the same command as the timings; nothing is set), then per
storage, shape, list size and list kind (random ids, or one contiguous range per query) the time of one maxsim_topk
call (k = 10; CUDA events around --reps calls, after a warm-up) of three arms, median and spread over --rounds rounds,
the arm order reversed every other round: listed (its device planner, the plan-mode scans and the merge), bitmap
(bitmaps built beforehand: the scans and the merge) and unrestricted.  For each shape and kind, the crossover: the
smallest list size at which the listed call is no faster than the bitmap call.

Then, per storage, whole Searcher calls (``_search_all_Q``, 16 x Nq = 320, k = 10, 1k random ids per query; host
clock around a call that ends in a device synchronise) on the listed path, on the bitmap path (the module's threshold
patched either way) and unrestricted.
"""
import argparse
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
import ravqa_b200.searcher as S  # noqa: E402

ND = 180
K = 10


def card():
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def call_ms(fn, reps):
    """Milliseconds per call of fn (CUDA events around `reps` calls), after a warm-up call."""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def make_lists(B, n, size, kind, rng):
    if kind == "random":
        return [rng.choice(n, size=min(size, n), replace=False).astype(np.int64) for _ in range(B)]
    starts = rng.integers(0, n - size + 1, size=B)
    return [np.arange(s, s + size, dtype=np.int64) for s in starts]


def stats(t):
    return {"ms": statistics.median(t), "spread_ms": max(t) - min(t), "samples": t}


def searcher_ms(c, Q, n, rounds):
    sr = R.Searcher(index=c)
    rng = np.random.default_rng(4)
    q2p = {b: rng.choice(n, size=1000, replace=False) for b in range(Q.size(0))}
    keep = S.LISTED_SCAN_MAX_ROW_FRACTION

    def restricted(fraction):
        S.LISTED_SCAN_MAX_ROW_FRACTION = fraction
        try:
            return sr._search_all_Q(list(q2p), Q, k=K, qid_to_pids=q2p)
        finally:
            S.LISTED_SCAN_MAX_ROW_FRACTION = keep

    arms = {"listed path, 1000 ids/query": lambda: restricted(float("inf")),
            "bitmap path, 1000 ids/query": lambda: restricted(-1.0),
            "unrestricted": lambda: sr._search_all_Q(list(q2p), Q, k=K)}
    assert arms["listed path, 1000 ids/query"]().todict() == arms["bitmap path, 1000 ids/query"]().todict()
    times = {a: [] for a in arms}
    for r in range(rounds):
        for a in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            arms[a]()
            torch.cuda.synchronize()
            times[a].append((time.perf_counter() - t0) * 1e3)
    out = {a: stats(t) for a, t in times.items()}
    for a, s in out.items():
        print("[%s searcher 16xNq320 k=%d] %-30s %.2f ms (spread %.2f)" % (c.storage, K, a, s["ms"], s["spread_ms"]),
              flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5, help="calls per arm and round")
    ap.add_argument("--storages", default="bf16,fp8")
    ap.add_argument("--shapes", default="16xNq320,12xNq32")
    ap.add_argument("--sizes", default="10,100,1000,10000,100000")
    ap.add_argument("--no-searcher", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.passages
    rec = {"card": card(), "passages": n, "nd": ND, "k": K}
    print("card (name, power limit, max SM clock):", rec["card"], "passages:", n, flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    shapes = {s: {"16xNq320": (16, 320), "12xNq32": (12, 32)}[s] for s in args.shapes.split(",")}
    Qs = {s: torch.nn.functional.normalize(torch.randn((B, nq, 128), device=dev, generator=g), dim=-1).bfloat16()
          for s, (B, nq) in shapes.items()}
    sizes = [int(x) for x in args.sizes.split(",")]
    for storage in args.storages.split(","):
        D = bench.build_shard(0, n, ND, dev)
        c = R.FlatCorpus(D, np.full(n, ND, dtype=np.int32), storage=storage)
        del D
        torch.cuda.empty_cache()
        rec[storage] = {}
        for sname, (B, _) in shapes.items():
            Q = Qs[sname]
            rec[storage][sname] = out = {"unrestricted": stats([call_ms(lambda: R.maxsim_topk(c, Q, K), args.reps)
                                                                for _ in range(args.rounds)])}
            print("[%s %s] unrestricted %.3f ms" % (storage, sname, out["unrestricted"]["ms"]), flush=True)
            for kind in ("random", "contiguous"):
                crossover = None
                for size in sizes:
                    lists = make_lists(B, n, size, kind, np.random.default_rng(size))
                    allow = c.allow_bitmaps(lists)
                    assert all(torch.equal(x, y) for x, y in zip(R.maxsim_topk(c, Q, K, pids=lists),
                                                                  R.maxsim_topk(c, Q, K, allow=allow)))
                    arms = {"listed": lambda: R.maxsim_topk(c, Q, K, pids=lists),
                            "bitmap": lambda: R.maxsim_topk(c, Q, K, allow=allow)}
                    times = {a: [] for a in arms}
                    for r in range(args.rounds):
                        for a in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                            times[a].append(call_ms(arms[a], args.reps))
                    res = {a: stats(t) for a, t in times.items()}
                    out["%s %d" % (kind, size)] = res
                    if crossover is None and res["listed"]["ms"] >= res["bitmap"]["ms"]:
                        crossover = size
                    print("[%s %s %s %6d ids/query] listed %.3f ms (spread %.3f)  bitmap %.3f ms (spread %.3f)"
                          % (storage, sname, kind, size, res["listed"]["ms"], res["listed"]["spread_ms"],
                             res["bitmap"]["ms"], res["bitmap"]["spread_ms"]), flush=True)
                out["crossover %s" % kind] = crossover
                print("[%s %s %s] listed stops winning at: %s ids/query" % (storage, sname, kind, crossover),
                      flush=True)
        if not args.no_searcher:
            Q = torch.nn.functional.normalize(torch.randn((16, 320, 128), device=dev, generator=g), dim=-1).bfloat16()
            rec[storage]["searcher"] = searcher_ms(c, Q, n, args.rounds)
        c.close()
        del c
        torch.cuda.empty_cache()
    rec["card_after"] = card()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
