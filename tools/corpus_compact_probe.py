"""GPU: what compacting a resident corpus costs and gives back at the benchmark size (1M passages x 180 tokens).

    python tools/corpus_compact_probe.py [--passages 1000000] [--rounds 3] [--json out.json]
    python tools/corpus_compact_probe.py --create-ab lib/libflmr_maxsim_base.so [--rounds 3]

Prints the card, its power limit and max SM clock, then per storage (bf16, fp8) and per deleted fraction (10 %, 30 %,
50 %, at random): the compaction's wall time (host clock around the synchronous call, median over --rounds freshly
built corpora for bf16, one for fp8, whose pinned 46 GB master makes a build slow); the scan launch of the flagship
16 x Nq = 320 top-k and of one Nq = 32 query (HBM-bound) before and after; hbm_bytes, mapped_device_bytes and the
stored rows before and after; and whether the top-100 of both query sets is bitwise equal before and after.
--create-ab times creating a 500k x 180 bf16 corpus from a device matrix with this tree's library and with the
given one (e.g. the parent's, built by tools/scan_ab.py --build-base), in alternating fresh processes.
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
FRACTIONS = (0.1, 0.3, 0.5)


def card():
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def scan_ms(L, corpus, Q, reps=3):
    """Milliseconds per scan launch of maxsim_topk(k = 100), after a warm-up call."""
    R.maxsim_topk(corpus, Q, 100)
    torch.cuda.synchronize()
    L.flmr_scan_kernel_stats(None, None, 1)
    L.flmr_set_profiling(1)
    for _ in range(reps):
        R.maxsim_topk(corpus, Q, 100)
    torch.cuda.synchronize()
    tot, cnt = C.c_double(0), C.c_int64(0)
    L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
    L.flmr_set_profiling(0)
    return tot.value / cnt.value


def stored(L, corpus):
    n, mapped = C.c_int64(0), C.c_int64(0)
    _cabi.check(L.flmr_corpus_stored(corpus.handle, C.byref(n), C.byref(mapped)))
    return {"n_stored": int(n.value), "n_rows": int(corpus.info.n_rows), "hbm_bytes": int(corpus.info.hbm_bytes),
            "mapped_device_bytes": int(mapped.value)}


def build(storage, n, dev):
    dl = np.full(CHUNK, ND, dtype=np.int32)
    if storage == "bf16":   # appends of 50k passages: HBM holds one matrix plus a chunk
        c = R.FlatCorpus(bench.build_shard(0, min(n, CHUNK), ND, dev), dl[:min(n, CHUNK)], adopt=False)
        for p0 in range(CHUNK, n, CHUNK):
            p1 = min(n, p0 + CHUNK)
            c.append(bench.build_shard(p0, p1, ND, dev), dl[:p1 - p0])
    else:
        D = bench.build_shard(0, n, ND, dev)
        c = R.FlatCorpus(D, np.full(n, ND, dtype=np.int32), storage="fp8")
        del D
    torch.cuda.empty_cache()
    return c


def one_compaction(L, storage, n, frac, Qs, dev, seed):
    c = build(storage, n, dev)
    dead = np.sort(np.random.default_rng(seed).choice(n, size=int(n * frac), replace=False))
    c.delete(dead)
    rec = {"before": stored(L, c)}
    tops = {name: R.maxsim_topk(c, Q, 100) for name, Q in Qs.items()}
    rec["scan_before_ms"] = {name: statistics.median([scan_ms(L, c, Q) for _ in range(3)]) for name, Q in Qs.items()}
    torch.cuda.synchronize()
    stats = c.compact()
    rec["compact_s"] = stats["seconds"]
    rec["bytes_released"] = stats["bytes_released"]
    rec["after"] = stored(L, c)
    rec["scan_after_ms"] = {name: statistics.median([scan_ms(L, c, Q) for _ in range(3)]) for name, Q in Qs.items()}
    rec["top100_bitwise_equal"] = all(
        torch.equal(tops[name][0].view(torch.int32), R.maxsim_topk(c, Q, 100)[0].view(torch.int32)) and
        torch.equal(tops[name][1], R.maxsim_topk(c, Q, 100)[1]) for name, Q in Qs.items())
    c.close()
    del c
    torch.cuda.empty_cache()
    return rec


def create_once(n):
    """Seconds to create an n x 180 bf16 corpus from a device matrix (median of 3), in this process."""
    dev = torch.device("cuda", 0)
    D = bench.build_shard(0, n, ND, dev)
    dl = np.full(n, ND, dtype=np.int32)
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c = R.FlatCorpus(D, dl, adopt=False)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        c.close()
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--create-ab", default=None, help="library to time corpus creation against")
    ap.add_argument("--create-once", type=int, default=0, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.create_once:
        print(json.dumps({"create_s": create_once(args.create_once)}))
        return
    rec = {"card": card(), "passages": args.passages, "nd": ND}
    print("card (name, power limit, max SM clock):", rec["card"], flush=True)
    if args.create_ab:
        arms = {"this tree": os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200", "lib",
                                          "libflmr_maxsim.so"), "other": os.path.abspath(args.create_ab)}
        res = {name: [] for name in arms}
        for _ in range(args.rounds):
            for name, lib in arms.items():
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--create-once", "500000"],
                                     env=dict(os.environ, FLMR_MAXSIM_LIB=lib), capture_output=True, text=True,
                                     check=True).stdout
                res[name].append(json.loads(out.splitlines()[-1])["create_s"])
        for name, s in res.items():
            print("create 500k x 180 bf16 from device, %s: median %.3f s, samples %s" % (name, statistics.median(s), s))
        rec["create_ab"] = res
    else:
        L = _cabi.lib()
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(0)
        g = torch.Generator(device=dev).manual_seed(0)
        Qs = {"16 x Nq=320": torch.nn.functional.normalize(torch.randn((16, 320, 128), device=dev, generator=g),
                                                           dim=-1).bfloat16(),
              "1 x Nq=32": torch.nn.functional.normalize(torch.randn((1, 32, 128), device=dev, generator=g),
                                                         dim=-1).bfloat16()}
        for storage in ("bf16", "fp8"):
            for frac in FRACTIONS:
                runs = [one_compaction(L, storage, args.passages, frac, Qs, dev, seed=r)
                        for r in range(args.rounds if storage == "bf16" else 1)]
                out = runs[0]
                out["compact_s_samples"] = [r["compact_s"] for r in runs]
                out["compact_s"] = statistics.median(out["compact_s_samples"])
                out["top100_bitwise_equal"] = all(r["top100_bitwise_equal"] for r in runs)
                rec["%s %d%%" % (storage, round(frac * 100))] = out
                print("[%s, %d%% deleted] compact %.3f s (samples %s); scan before %s, after %s; before %s; after %s; "
                      "released %d B; top-100 bitwise equal: %s"
                      % (storage, round(frac * 100), out["compact_s"], out["compact_s_samples"],
                         out["scan_before_ms"], out["scan_after_ms"], out["before"], out["after"],
                         out["bytes_released"], out["top100_bitwise_equal"]), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(rec, f, indent=1, default=str)


if __name__ == "__main__":
    main()
