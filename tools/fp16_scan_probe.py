"""GPU: the fp16 corpus (storage="fp16") against bf16 over the same 180-token passages, in alternating rounds.

    python tools/fp16_scan_probe.py [--passages 600000] [--rounds 5] [--json out.json]

Both corpora are resident at once so that the rounds alternate: 600k x 180 tokens is 27.6 GB per storage (1M would
need 92 GB for the two).  The fp16 tokens are the bf16 ones converted with .half() (exact for these unit rows but for
a few entries below fp16's normal range), so the two corpora hold the same passages.  Their top-10 are compared twice:
for fp32 queries, which each storage rounds to its own query type (fp16 keeps 3 more bits), and for queries already
rounded to bf16, which both storages receive exactly.

Prints the card, its power limit and SM clock, then per storage the median and spread (min..max) over the rounds of:
  * the scan launch time of 16 x Nq = 320 queries (one pass each, five occupied 64-row blocks: the split kernel) and
    of one Nq = 32 query (the HBM-bound pass: the two-warpgroup kernel), with TFLOP/s (algorithmic: 2 Nq 128 N Nd
    per launch) and GB/s (N Nd 256 bytes per launch);
  * Searcher end to end (maxsim_topk through Searcher._search_tensors, k = 10) queries/s on 16 x Nq = 320;
and whether the two storages return the same top-10 ids and how far their scores are apart.
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
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def scan_ms(L, corpus, Q, k, reps):
    """ms per scan launch of maxsim_topk (CUDA events around every launch), after one warm-up call."""
    R.maxsim_topk(corpus, Q, k)
    torch.cuda.synchronize()
    L.flmr_scan_kernel_stats(None, None, 1)
    L.flmr_set_profiling(1)
    for _ in range(reps):
        R.maxsim_topk(corpus, Q, k)
    torch.cuda.synchronize()
    tot, cnt = C.c_double(0), C.c_int64(0)
    L.flmr_scan_kernel_stats(C.byref(tot), C.byref(cnt), 1)
    L.flmr_set_profiling(0)
    return tot.value / cnt.value


def searcher_qps(s, Q, reps):
    s._search_tensors(Q, 10)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        s._search_tensors(Q, 10)
    e1.record()
    torch.cuda.synchronize()
    return Q.size(0) * reps / (e0.elapsed_time(e1) / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=600_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("this probe times the GPU; there is no CPU measurement")
    L = _cabi.lib()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.passages
    D = bench.build_shard(0, n, ND, dev)
    dl = np.full(n, ND, dtype=np.int32)
    corpora = {"bf16": R.FlatCorpus(D, dl), "fp16": R.FlatCorpus(D.half(), dl, storage="fp16")}
    searchers = {k: R.Searcher(c) for k, c in corpora.items()}
    g = torch.Generator(device=dev).manual_seed(1)
    Q320 = torch.nn.functional.normalize(torch.randn(16, 320, 128, device=dev, generator=g), dim=-1)
    Q32 = torch.nn.functional.normalize(torch.randn(1, 32, 128, device=dev, generator=g), dim=-1)
    flop320 = 2.0 * 320 * 128 * n * ND             # per launch: one Nq = 320 query per pass
    bytes_scan = float(n) * ND * 128 * 2
    res = {k: {"scan320_ms": [], "scan32_ms": [], "searcher_qps": []} for k in corpora}
    info = {"card": card(), "passages": n, "nd": ND}
    print("[fp16 probe] card: %s" % info["card"], flush=True)
    for r in range(args.rounds):
        for k in (("bf16", "fp16") if r % 2 == 0 else ("fp16", "bf16")):
            res[k]["scan320_ms"].append(scan_ms(L, corpora[k], Q320, 10, 3))
            res[k]["scan32_ms"].append(scan_ms(L, corpora[k], Q32, 10, 10))
            res[k]["searcher_qps"].append(searcher_qps(searchers[k], Q320, 3))
        print("[fp16 probe] round %d: %s" % (r, {k: {m: round(v[-1], 3) for m, v in res[k].items()} for k in res}),
              flush=True)
    info["card_after"] = card()
    summary = {}
    for k in res:
        summary[k] = {}
        for m, v in res[k].items():
            summary[k][m] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
        med = summary[k]["scan320_ms"]["median"]
        summary[k]["scan320_tflops"] = flop320 / (med * 1e-3) / 1e12
        summary[k]["scan32_gbps"] = bytes_scan / (summary[k]["scan32_ms"]["median"] * 1e-3) / 1e9
    for name, Q in (("fp32_queries", Q320), ("bf16_queries", Q320.to(torch.bfloat16).float())):
        s16, p16 = R.maxsim_topk(corpora["fp16"], Q, 10)
        sb, pb = R.maxsim_topk(corpora["bf16"], Q, 10)
        summary[name] = {"topk_ids_equal": bool(torch.equal(p16, pb)),
                         "topk_ids_equal_fraction": float((p16 == pb).float().mean()),
                         "topk_score_max_abs_diff": float((s16 - sb).abs().max())}
    out = {"info": info, "rounds": res, "summary": summary}
    print(json.dumps(summary, indent=1))
    print("[fp16 probe] card after: %s" % info["card_after"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    for c in corpora.values():
        c.close()


if __name__ == "__main__":
    main()
