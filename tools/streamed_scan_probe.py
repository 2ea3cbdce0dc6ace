"""GPU: what a streamed corpus (FlatCorpus(residency="host"): rows in pinned host memory, copied through two HBM windows
per search) costs against the same rows resident in HBM, over a corpus of at least 10 GB.

    python tools/streamed_scan_probe.py [--passages 240000] [--window-mb 1024] [--rounds 3] [--reps 2]
                                        [--trace-dir DIR] [--json out.json]

Prints the card, its power limit and max SM clock (read in the same command as the timings; nothing is set), then:
  * pinned host-to-device bandwidth (one 1 GiB copy, CUDA events, median of 5);
  * per query length (Nq 32 / 320 / 832) and batch B, queries per second of one maxsim_topk call (k = 10; CUDA events
    around --reps calls after a warm-up) on the resident and on the streamed corpus, alternated, the order reversed
    every other round, median and range over --rounds rounds, and their ratio;
  * per Nq, the smallest B at which the streamed corpus reaches 0.9 of the resident rate;
  * the HBM of the windows (device memory around creating the streamed corpus and its workspace);
  * whole ``Searcher._search_all_Q`` calls of more than ``query_batch`` queries (host clock around a call that ends in
    a device synchronise, median and range over --rounds alternated rounds), resident against streamed;
  * a torch.profiler trace of one streamed call (Nq 320, B 16) written to --trace-dir, and from it the share of the
    host-to-device copy time that ran under a scan kernel.

Both corpora hold the same rows: a block of random unit vectors repeated (the rates do not depend on the values),
180-token passages, built on the device; the streamed one is packed into pinned memory by the library's repack kernel.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ravqa_b200 as R  # noqa: E402
from ravqa_b200.maxsim import maxsim_topk  # noqa: E402

ND = 180
K = 10
SHAPES = {32: [1, 2, 4, 8, 16, 32, 64, 128, 256], 320: [1, 2, 4, 8, 16, 32, 64], 832: [1, 2, 4, 8, 16, 32]}


def card():
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def call_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def h2d_gbps():
    src = torch.empty(1 << 29, dtype=torch.int16).pin_memory()
    dst = torch.empty_like(src, device="cuda")
    out = []
    for _ in range(5):
        out.append(call_ms(lambda: dst.copy_(src, non_blocking=True), 1))
    return src.numel() * 2 / (statistics.median(out) / 1e3) / 1e9


def copy_overlap(trace_path):
    """Share of the host-to-device copy time of a chrome trace that overlaps a scan kernel."""
    ev = json.load(open(trace_path))["traceEvents"]
    copies = [(e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("cat") == "gpu_memcpy" and "HtoD" in e.get("name", "")]
    scans = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("cat") == "kernel" and "scan" in e.get("name", ""))
    total = sum(b - a for a, b in copies)
    under = 0.0
    for a, b in copies:
        for s, e in scans:
            under += max(0.0, min(b, e) - max(a, s))
    return {"copies": len(copies), "copy_us": total, "copy_us_under_scans": under,
            "share": under / total if total else 0.0, "scan_kernels": len(scans)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=240_000)
    ap.add_argument("--window-mb", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--trace-dir", default=None)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU; there is no CPU fallback"
    torch.cuda.set_device(0)
    out = {"card": card()}
    print("card (name, power limit, max SM clock):", out["card"])
    out["h2d_gbps"] = h2d_gbps()
    print("pinned H2D: %.1f GB/s" % out["h2d_gbps"])

    n, rows = a.passages, a.passages * ND
    g = torch.Generator(device="cuda").manual_seed(0)
    block = torch.nn.functional.normalize(torch.randn(1 << 16, 128, device="cuda", generator=g), dim=-1)
    tokens = block.to(torch.bfloat16).repeat((rows + (1 << 16) - 1) >> 16, 1)[:rows].contiguous()
    del block
    dl = np.full(n, ND, np.int32)
    out["corpus_gb"] = rows * 256 / 1e9
    print("corpus: %d passages x %d tokens = %.2f GB bf16" % (n, ND, out["corpus_gb"]))
    res = R.FlatCorpus(tokens, dl)                      # adopts the device tensor
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    st = R.FlatCorpus(tokens, dl, residency="host", window_bytes=a.window_mb << 20)
    st.workspace()
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    out["window_hbm_bytes"] = free0 - free1
    out["hbm_bytes_info"] = int(st.info.hbm_bytes)
    res.workspace()
    print("streamed corpus + workspace: device memory %+.1f MB (windows of %d MiB), corpus hbm_bytes %.1f MB"
          % (out["window_hbm_bytes"] / 1e6, a.window_mb, out["hbm_bytes_info"] / 1e6))

    rows_out, cross = [], {}
    for nq, Bs in SHAPES.items():
        for B in Bs:
            Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, device="cuda", generator=g), dim=-1)
            Q = Q.to(torch.bfloat16)
            arms = {"resident": lambda c=res: maxsim_topk(c, Q, K), "streamed": lambda c=st: maxsim_topk(c, Q, K)}
            t = {"resident": [], "streamed": []}
            for r in range(a.rounds):
                for name in (("resident", "streamed") if r % 2 == 0 else ("streamed", "resident")):
                    t[name].append(call_ms(arms[name], a.reps))
            sa, pa = arms["resident"]()
            sb, pb = arms["streamed"]()
            same = bool(torch.equal(sa, sb) and torch.equal(pa, pb))
            ms = {k: statistics.median(v) for k, v in t.items()}
            rec = {"nq": nq, "B": B, "resident_ms": ms["resident"], "streamed_ms": ms["streamed"],
                   "resident_qps": B / ms["resident"] * 1e3, "streamed_qps": B / ms["streamed"] * 1e3,
                   "ratio": ms["resident"] / ms["streamed"], "spread": {k: [min(v), max(v)] for k, v in t.items()},
                   "bitwise": same}
            rows_out.append(rec)
            print("Nq %4d B %4d: resident %9.2f ms [%.2f-%.2f] (%8.1f q/s)  streamed %9.2f ms [%.2f-%.2f] (%8.1f q/s)"
                  "  ratio %.3f  bitwise %s"
                  % (nq, B, rec["resident_ms"], *rec["spread"]["resident"], rec["resident_qps"], rec["streamed_ms"],
                     *rec["spread"]["streamed"], rec["streamed_qps"], rec["ratio"], same))
            if nq not in cross and rec["ratio"] >= 0.9:
                cross[nq] = B
    out["rows"] = rows_out
    out["crossover_B_at_0.9"] = {str(k): cross.get(k) for k in SHAPES}
    print("smallest B at which streamed reaches 0.9 of resident:", out["crossover_B_at_0.9"])

    import time
    cfg = R.ColBERTConfig(total_visible_gpus=1)
    searchers = {"resident": R.Searcher(index=res, config=cfg), "streamed": R.Searcher(index=st, config=cfg)}
    out["searcher"] = []
    for nq, B in ((32, 512), (320, 128), (832, 64)):
        Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, device="cuda", generator=g), dim=-1).cpu()
        t = {"resident": [], "streamed": []}
        for name in t:
            searchers[name]._search_all_Q(None, Q, k=K)               # warm-up
        for r in range(a.rounds):
            for name in (("resident", "streamed") if r % 2 == 0 else ("streamed", "resident")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                searchers[name]._search_all_Q(None, Q, k=K)
                torch.cuda.synchronize()
                t[name].append(1e3 * (time.perf_counter() - t0))
        ms = {k: statistics.median(v) for k, v in t.items()}
        rec = {"nq": nq, "B": B, "resident_ms": ms["resident"], "streamed_ms": ms["streamed"],
               "ratio": ms["resident"] / ms["streamed"], "spread": {k: [min(v), max(v)] for k, v in t.items()}}
        out["searcher"].append(rec)
        print("Searcher._search_all_Q Nq %4d B %4d (query_batch %d): resident %9.1f ms [%.1f-%.1f]  streamed %9.1f ms "
              "[%.1f-%.1f]  ratio %.3f" % (nq, B, searchers["streamed"].query_batch, rec["resident_ms"],
                                           *rec["spread"]["resident"], rec["streamed_ms"], *rec["spread"]["streamed"],
                                           rec["ratio"]))
    del searchers

    if a.trace_dir:
        os.makedirs(a.trace_dir, exist_ok=True)
        Q = torch.nn.functional.normalize(torch.randn(16, 320, 128, device="cuda", generator=g), dim=-1)
        Q = Q.to(torch.bfloat16)
        maxsim_topk(st, Q, K)
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            maxsim_topk(st, Q, K)
            torch.cuda.synchronize()
        path = os.path.join(a.trace_dir, "streamed_nq320_b16.json")
        prof.export_chrome_trace(path)
        out["trace"] = dict(copy_overlap(path), path=path)
        print("trace %s: %d H2D copies, %.1f ms of copies, %.1f%% of it under %d scan kernels"
              % (path, out["trace"]["copies"], out["trace"]["copy_us"] / 1e3, 100 * out["trace"]["share"],
                 out["trace"]["scan_kernels"]))
    res.close()
    st.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
