"""GPU: the MMA ceiling of the three-warpgroup scan loops — each loop with and without its fold, five-block passes.

    python tools/scan_split_probe.py [--passages 200000] [--repeat 5] [--nq 320] [--out DIR]

Builds the library once more with -DFLMR_SCAN_SKELETON into DIR (the three-warpgroup consumer loops then issue their
MMAs and keep every wait and barrier but fold nothing), then times, over passages of 180 tokens, B x Nq = 320 (one
query and five occupied 64-row query blocks per pass; --nq 384: six) with a bf16, an fp16 and an e4m3 corpus:

  * skeleton n96 serial loop   (skeleton library, flmr_scan_kernel<3>, variant 3)
  * skeleton n48 split loop    (skeleton library, flmr_scan_split_kernel, variant 6)
  * full n96 serial loop       (release library, variant 3: the kernel the product ran before the split loop)
  * full n48 split loop        (release library, variant 6)

fp16 has no serial three-warpgroup kernel: its variant-3 rows are n/a.

Each library is driven by a worker process of its own (FLMR_MAXSIM_LIB); inside a worker the variants and storages
alternate, --repeat rounds, median and spread of the scan launch time (CUDA events around every launch).  Prints the
card, its power limit and the median SM clock of each worker's timed window.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200")
ND = 180
ARMS = [("skeleton", 3, "skeleton n96 serial"), ("skeleton", 6, "skeleton n48 split"),
        ("release", 3, "full n96 serial"), ("release", 6, "full n48 split")]
STORAGES = ("bf16", "fp16", "e4m3")


def worker(args):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import bench
    import ravqa_b200 as R
    from ravqa_b200 import _cabi
    L = _cabi.lib()
    dev = torch.device("cuda", 0)
    n = args.passages
    D = bench.build_shard(0, n, ND, dev)
    dl = np.full(n, ND, dtype=np.int32)
    corpora = {"bf16": R.FlatCorpus(D, dl), "fp16": R.FlatCorpus(D.half(), dl, storage="fp16"),
               "e4m3": R.FlatCorpus(D, dl, storage="fp8")}
    g = torch.Generator(device=dev).manual_seed(0)
    Q = torch.nn.functional.normalize(torch.randn((args.batch, args.nq, 128), device=dev, generator=g), dim=-1).bfloat16()
    variants = [int(v) for v in args.variants.split(",")]
    # fp16 has no serial three-warpgroup kernel
    samples = {(st, v): [] for st in corpora for v in variants if not (st == "fp16" and v == 3)}
    sampler = bench.ClockSampler(0)
    sampler.start()
    for _ in range(args.repeat):
        for st, c in corpora.items():
            for v in variants:
                if (st, v) not in samples:
                    continue
                _cabi.check(L.flmr_debug_set_scan_variant(v))
                R.maxsim_topk(c, Q, 5)
                torch.cuda.synchronize()
                L.flmr_scan_kernel_stats(None, None, 1)
                L.flmr_set_profiling(1)
                for _ in range(args.reps):
                    R.maxsim_topk(c, Q, 5)
                torch.cuda.synchronize()
                tot, cnt = C.c_double(0), C.c_int64(0)
                L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
                L.flmr_set_profiling(0)
                samples[(st, v)].append(tot.value / cnt.value)
    clocks = sampler.stop()
    L.flmr_debug_set_scan_variant(0)
    for c in corpora.values():
        c.close()
    print(json.dumps({"clocks": clocks, "launch_ms": {"%s %d" % k: s for k, s in samples.items()}}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=200_000)
    ap.add_argument("--batch", type=int, default=4, help="queries per call (one pass each)")
    ap.add_argument("--nq", type=int, default=320, help="query rows: 320 = five occupied 64-row blocks, 384 = six")
    ap.add_argument("--reps", type=int, default=3, help="timed calls per sample")
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the skeleton library and the raw samples")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--variants", default="3,6", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        worker(args)
        return
    sys.path.insert(0, PKG)
    import build as B
    out = os.path.abspath(args.out or tempfile.mkdtemp(prefix="scan_split_probe_"))
    os.makedirs(out, exist_ok=True)
    libs = {"release": B.build(), "skeleton": os.path.join(out, "libflmr_maxsim_skeleton.so")}
    subprocess.run([B.find_nvcc(), *B.NVCC_FLAGS, "-DFLMR_SCAN_SKELETON", "-o", libs["skeleton"], *B.SOURCES],
                   check=True)
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card (name, power limit, max SM clock):", card or "nvidia-smi unavailable", flush=True)
    res = {}
    for name, lib in libs.items():
        variants = ",".join(str(v) for arm, v, _ in ARMS if arm == name)
        cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--variants", variants, "--passages",
               str(args.passages), "--batch", str(args.batch), "--nq", str(args.nq), "--reps", str(args.reps), "--repeat", str(args.repeat)]
        proc = subprocess.run(cmd, env=dict(os.environ, FLMR_MAXSIM_LIB=lib), capture_output=True, text=True)
        if proc.returncode != 0:
            raise SystemExit("%s worker failed:\n%s" % (name, proc.stderr[-4000:]))
        res[name] = json.loads(proc.stdout.strip().splitlines()[-1])
        print("%s library: median SM clock %s MHz (reasons %s)"
              % (name, res[name]["clocks"].get("sm_mhz"), res[name]["clocks"].get("reasons")), flush=True)
    with open(os.path.join(out, "scan_split_probe.json"), "w") as f:
        json.dump({"card": card, "passages": args.passages, "batch": args.batch, "nq": args.nq, "results": res}, f,
                  indent=1)
    print("\n%d x 180-token passages, %d x Nq = %d (%d 64-row blocks per pass), launch ms median (spread) of %d"
          % (args.passages, args.batch, args.nq, (args.nq + 63) // 64, args.repeat))
    print("| loop | %s |\n|---|%s" % (" | ".join(STORAGES), "---:|" * len(STORAGES)))
    for arm, v, label in ARMS:
        cols = []
        for st in STORAGES:
            s = res[arm]["launch_ms"].get("%s %d" % (st, v))
            cols.append("%.3f (%.3f)" % (statistics.median(s), max(s) - min(s)) if s else "n/a")
        print("| %s | %s |" % (label, " | ".join(cols)))


if __name__ == "__main__":
    main()
