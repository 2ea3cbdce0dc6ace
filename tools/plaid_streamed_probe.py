"""GPU: what a PLAID-coded streamed corpus (FlatCorpus.from_plaid(residency="host", compressed=True): codes and residuals
in pinned host memory, each window copied and decoded on the GPU before the scan) costs against the same decoded rows
resident in HBM and streamed as bf16 rows, at the size of tools/streamed_scan_probe.py (240k passages x 180 tokens,
1 GiB windows).

    python tools/plaid_streamed_probe.py [--passages 240000] [--window-mb 1024] [--nbits 2 4] [--rounds 3] [--reps 2]
                                         [--json out.json]

Prints the card, its power limit and max SM clock (read in the same command as the timings; nothing is set), then:
  * pinned host-to-device bandwidth (one 1 GiB copy, CUDA events, median of 5);
  * per nbits: pinned host bytes, hbm_bytes and the device memory a workspace adds, for the compressed corpus and
    (nbits 2) for the bf16-streamed corpus of the same rows;
  * the window decode kernel's time per window (torch.profiler, one call) and its rate, from the bytes it reads
    (codes and residuals) and writes (bf16 rows), computed from shapes;
  * per query length (Nq 32 / 320 / 832) and batch B, the time of one maxsim_topk call (k = 10; CUDA events around
    --reps calls after a warm-up) on the resident, bf16-streamed (nbits 2 only) and compressed corpora, alternated,
    median over --rounds rounds, and whether every compressed result is torch.equal to the resident one;
  * per Nq, the smallest B at which each streamed arm reaches 0.9 of the resident rate;
  * whole Searcher._search_all_Q calls, resident against compressed.

The corpus is synthetic: seeded random codes and residuals over 2^16 normalised centroids, with bucket weights shaped
like the reference's, built on the device (the rates do not depend on the values).  The resident corpus holds the rows
flmr_plaid_decode decodes from them, as FlatCorpus.from_plaid does.
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
import ravqa_b200 as R  # noqa: E402
from ravqa_b200 import _cabi  # noqa: E402
from ravqa_b200.maxsim import maxsim_topk  # noqa: E402
from ravqa_b200.plaid import decode_chunk  # noqa: E402

ND = 180
K = 10
N_CENTROIDS = 1 << 16
SHAPES = {32: [1, 4, 16, 64, 256], 320: [1, 4, 16, 64], 832: [1, 4, 16, 32]}


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
    out = [call_ms(lambda: dst.copy_(src, non_blocking=True), 1) for _ in range(5)]
    return src.numel() * 2 / (statistics.median(out) / 1e3) / 1e9


def workspace_bytes(c):
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    c.workspace()
    torch.cuda.synchronize()
    return free0 - torch.cuda.mem_get_info()[0]


def build(n, nbits, window_bytes, g):
    """(resident corpus, compressed corpus, decoded tokens) of n passages of ND tokens."""
    rows = n * ND
    centroids = torch.nn.functional.normalize(torch.randn(N_CENTROIDS, 128, device="cuda", generator=g), dim=-1)
    weights = torch.sort(0.1 * torch.randn(1 << nbits, device="cuda", generator=g)).values
    codes = torch.randint(0, N_CENTROIDS, (rows,), device="cuda", generator=g, dtype=torch.int32)
    residuals = torch.randint(0, 256, (rows, 16 * nbits), device="cuda", generator=g, dtype=torch.uint8)
    tokens = torch.empty((rows, 128), dtype=torch.bfloat16, device="cuda")
    decode_chunk(codes, residuals, centroids, weights, nbits, tokens)
    dl = np.full(n, ND, np.int32)
    res = R.FlatCorpus(tokens, dl)                                  # adopts the decoded rows, as from_plaid does
    hc, hr = codes.cpu(), residuals.cpu()

    def feed(L, b):
        step = 1 << 22
        for a in range(0, rows, step):
            e = min(rows, a + step)
            _cabi.check(L.flmr_corpus_builder_append_plaid(b, C.c_void_p(hc[a:].data_ptr()),
                                                           C.c_void_p(hr[a:].data_ptr()), e - a))
    cmp = R.FlatCorpus._build(dl, res.device, 0, 0, "host", window_bytes, feed,
                              codec=(nbits, centroids.cpu(), weights.cpu()))[0]
    return res, cmp, tokens


def decode_rate(cmp, nbits, reps=3):
    """(ms per window decode, GB/s read + written) of the window decode kernel, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    Q = torch.nn.functional.normalize(torch.randn(1, 32, 128, device="cuda"), dim=-1).to(torch.bfloat16)
    maxsim_topk(cmp, Q, K)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            maxsim_topk(cmp, Q, K)
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if "plaid_window_decode" in e.name]
    us = [e.device_time for e in ks] if ks and hasattr(ks[0], "device_time") else [e.cuda_time for e in ks]
    total_rows = cmp.info.n_rows * reps
    moved = total_rows * (4 + 16 * nbits + 256)
    return {"launches": len(ks), "ms_per_window": statistics.median(us) / 1e3,
            "gbps": moved / (sum(us) / 1e6) / 1e9, "windows_per_call": len(ks) // reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=240_000)
    ap.add_argument("--window-mb", type=int, default=1024)
    ap.add_argument("--nbits", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU; there is no CPU fallback"
    torch.cuda.set_device(0)
    out = {"card": card(), "runs": []}
    print("card (name, power limit, max SM clock):", out["card"])
    out["h2d_gbps"] = h2d_gbps()
    print("pinned H2D: %.1f GB/s" % out["h2d_gbps"])
    g = torch.Generator(device="cuda").manual_seed(0)
    wb = a.window_mb << 20
    for nbits in a.nbits:
        res, cmp, tokens = build(a.passages, nbits, wb, g)
        run = {"nbits": nbits, "rows": int(cmp.info.n_rows), "corpus_gb": cmp.info.n_rows * 256 / 1e9}
        arms = {"resident": res, "compressed": cmp}
        if nbits == a.nbits[0]:
            arms["bf16_streamed"] = R.FlatCorpus(tokens, np.full(a.passages, ND, np.int32), residency="host",
                                                 window_bytes=wb)
        del tokens
        run["memory"] = {}
        for name, c in arms.items():
            run["memory"][name] = {"host_bytes": c.residency_info()["host_bytes"], "hbm_bytes": int(c.info.hbm_bytes),
                                   "workspace_device_bytes": workspace_bytes(c)}
            print("nbits %d %-13s host %.2f GB  hbm_bytes %.1f MB  workspace %+.1f MB" % (
                nbits, name, run["memory"][name]["host_bytes"] / 1e9, run["memory"][name]["hbm_bytes"] / 1e6,
                run["memory"][name]["workspace_device_bytes"] / 1e6))
        run["decode"] = decode_rate(cmp, nbits)
        print("nbits %d window decode: %.2f ms per window, %.0f GB/s read+written (%d windows per call)" % (
            nbits, run["decode"]["ms_per_window"], run["decode"]["gbps"], run["decode"]["windows_per_call"]))
        run["rows_out"], cross = [], {}
        all_equal = True
        for nq, Bs in SHAPES.items():
            for B in Bs:
                Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, device="cuda", generator=g), dim=-1)
                Q = Q.to(torch.bfloat16)
                t = {name: [] for name in arms}
                order = list(arms)
                for r in range(a.rounds):
                    for name in (order if r % 2 == 0 else order[::-1]):
                        t[name].append(call_ms(lambda c=arms[name]: maxsim_topk(c, Q, K), a.reps))
                sa, pa = maxsim_topk(res, Q, K)
                sb, pb = maxsim_topk(cmp, Q, K)
                same = bool(torch.equal(sa, sb) and torch.equal(pa, pb))
                all_equal &= same
                ms = {k: statistics.median(v) for k, v in t.items()}
                rec = {"nq": nq, "B": B, "ms": ms, "spread": {k: [min(v), max(v)] for k, v in t.items()},
                       "ratio": {k: ms["resident"] / ms[k] for k in ms if k != "resident"}, "bitwise": same}
                run["rows_out"].append(rec)
                print("nbits %d Nq %4d B %4d: " % (nbits, nq, B) + "  ".join(
                    "%s %8.2f ms" % (k, v) for k, v in ms.items()) + "  ratio " + " ".join(
                    "%s %.3f" % kv for kv in rec["ratio"].items()) + "  bitwise %s" % same)
                for k, v in rec["ratio"].items():
                    if v >= 0.9 and (k, nq) not in cross:
                        cross[(k, nq)] = B
        run["crossover_B_at_0.9"] = {"%s/%d" % k: v for k, v in cross.items()}
        run["all_compressed_results_equal"] = all_equal
        print("nbits %d smallest B at 0.9 of resident:" % nbits, run["crossover_B_at_0.9"], "all equal:", all_equal)
        cfg = R.ColBERTConfig(total_visible_gpus=1)
        searchers = {"resident": R.Searcher(index=res, config=cfg), "compressed": R.Searcher(index=cmp, config=cfg)}
        run["searcher"] = []
        for nq, B in ((32, 512), (320, 128)):
            Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, device="cuda", generator=g), dim=-1).cpu()
            t = {name: [] for name in searchers}
            for name in t:
                searchers[name]._search_all_Q(None, Q, k=K)
            for r in range(a.rounds):
                for name in (("resident", "compressed") if r % 2 == 0 else ("compressed", "resident")):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    searchers[name]._search_all_Q(None, Q, k=K)
                    torch.cuda.synchronize()
                    t[name].append(1e3 * (time.perf_counter() - t0))
            ms = {k: statistics.median(v) for k, v in t.items()}
            run["searcher"].append({"nq": nq, "B": B, "ms": ms, "ratio": ms["resident"] / ms["compressed"]})
            print("nbits %d Searcher._search_all_Q Nq %d B %d: resident %.1f ms  compressed %.1f ms  ratio %.3f" % (
                nbits, nq, B, ms["resident"], ms["compressed"], ms["resident"] / ms["compressed"]))
        del searchers
        for c in arms.values():
            c.close()
        out["runs"].append(run)
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
