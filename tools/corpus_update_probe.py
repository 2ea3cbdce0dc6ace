"""GPU: what updating a resident corpus costs at the benchmark size (1M passages x 180 tokens), for both storages.

    python tools/corpus_update_probe.py [--passages 1000000] [--rounds 3] [--json out.json]

Prints the card, its power limit and the median SM clock of the timed window, then per storage:
  * the scan launch time of the flagship 16 x Nq = 320 top-k (one query per pass) with 0 % and with 10 % of the
    passages deleted (the same handle before and after the delete), median and spread over the rounds (deleted rows
    are still streamed, so the launch is expected to stay the same);
  * the latency of appending 1k and 100k passages (host clock around the synchronous call, device source) and of
    deleting 10k ids;
  * hbm_bytes (and host_bytes of the fp8 master) before and after.
The bf16 corpus is built by appending 50k-passage chunks to a small one, which keeps HBM at one matrix plus a chunk;
the fp8 corpus is created in one go from a device matrix that is freed afterwards.  A step that runs out of memory is
recorded with its error instead of a time.
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
CHUNK = 50_000


def card():
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def scan_ms(L, corpus, Q, reps=2):
    """Milliseconds per scan launch of maxsim_topk(k = 10), after a warm-up call."""
    R.maxsim_topk(corpus, Q, 10)
    torch.cuda.synchronize()
    L.flmr_scan_kernel_stats(None, None, 1)
    L.flmr_set_profiling(1)
    for _ in range(reps):
        R.maxsim_topk(corpus, Q, 10)
    torch.cuda.synchronize()
    tot, cnt = C.c_double(0), C.c_int64(0)
    L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
    L.flmr_set_profiling(0)
    return tot.value / cnt.value


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        fn()
    except _cabi.FlmrError as e:
        return {"error": str(e)}
    return {"ms": (time.perf_counter() - t0) * 1e3}


def memory(corpus):
    host = C.c_int64(0)
    _cabi.check(_cabi.lib().flmr_corpus_storage(corpus.handle, None, C.byref(host)))
    return {"hbm_bytes": int(corpus.info.hbm_bytes), "host_bytes": int(host.value)}


def build(storage, n, dev):
    dl = np.full(CHUNK, ND, dtype=np.int32)
    if storage == "bf16":
        c = R.FlatCorpus(bench.build_shard(0, min(n, CHUNK), ND, dev), dl[:min(n, CHUNK)], adopt=False)
        for p0 in range(CHUNK, n, CHUNK):
            p1 = min(n, p0 + CHUNK)
            c.append(bench.build_shard(p0, p1, ND, dev), dl[:p1 - p0])
        torch.cuda.empty_cache()
        return c
    D = bench.build_shard(0, n, ND, dev)
    c = R.FlatCorpus(D, np.full(n, ND, dtype=np.int32), storage="fp8")
    del D
    torch.cuda.empty_cache()
    return c


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
    rec = {"card": card(), "passages": n, "nd": ND}
    print("card (name, power limit, max SM clock):", rec["card"], "passages:", n, flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    Q = torch.nn.functional.normalize(torch.randn((16, 320, 128), device=dev, generator=g), dim=-1).bfloat16()
    for storage in ("bf16", "fp8"):
        sampler = bench.ClockSampler(0)
        t0 = time.perf_counter()
        c = build(storage, n, dev)
        out = {"build_s": time.perf_counter() - t0, "memory_before": memory(c)}
        print("\n[%s] built in %.1f s; %s" % (storage, out["build_s"], out["memory_before"]), flush=True)
        # flagship scan with 0 % and 10 % deleted: a second 1M-passage handle does not fit, so the same handle is
        # timed before and after deleting 10 %
        rng = np.random.default_rng(1)
        dead = np.sort(rng.choice(n, size=n // 10, replace=False))
        sampler.start()
        clean = [scan_ms(L, c, Q) for _ in range(args.rounds)]
        t_del = timed(lambda: c.delete(dead))
        deleted = [scan_ms(L, c, Q) for _ in range(args.rounds)]
        out["scan_clocks"] = sampler.stop()
        for name, s in (("0% deleted", clean), ("10% deleted", deleted)):
            out["scan " + name] = {"launch_ms": statistics.median(s), "spread_ms": max(s) - min(s), "samples": s}
            print("[%s] flagship 16 x Nq=320 scan launch, %s: %.2f ms (spread %.2f)"
                  % (storage, name, statistics.median(s), max(s) - min(s)), flush=True)
        out["delete 100k ids (first delete, allocates the bitmap)"] = t_del
        more = np.setdiff1d(np.arange(0, n, 7), dead)[:10_000]
        out["delete 10k ids"] = timed(lambda: c.delete(more))
        print("[%s] delete 10k ids: %s" % (storage, out["delete 10k ids"]), flush=True)
        for count in (1_000, 100_000):
            src = bench.build_shard(n, n + count, ND, dev)
            out["append %d" % count] = timed(lambda: c.append(src, np.full(count, ND, dtype=np.int32)))
            del src
            torch.cuda.empty_cache()
            print("[%s] append %d passages: %s" % (storage, count, out["append %d" % count]), flush=True)
        out["memory_after"] = memory(c)
        out["n_passages_after"] = c.n_passages
        out["n_live_after"] = c.n_live
        print("[%s] after: %s, %d passages, %d live" % (storage, out["memory_after"], c.n_passages, c.n_live),
              flush=True)
        rec[storage] = out
        c.close()
        del c
        torch.cuda.empty_cache()
        if args.json:
            os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
            with open(args.json, "w") as f:
                json.dump(rec, f, indent=1, default=str)


if __name__ == "__main__":
    main()
