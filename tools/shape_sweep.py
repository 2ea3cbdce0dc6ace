"""GPU probe: the scan path across the workload shapes BASELINE.json / SURVEY.md §8 name (not only the
headline C3 shape): queries/s, per-launch scan time and the two roofline figures of each.

    python tools/shape_sweep.py > shape_sweep.md
"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ravqa_b200 as R  # noqa: E402
from ravqa_b200 import _cabi  # noqa: E402

# name, passages, (nd_lo, nd_hi), nq, batch, k, iters
CASES = [
    ("C1 (16 q x 1k passages, Nq=32, Nd=64)", 1_000, (64, 64), 32, 16, 5, 50),
    ("C2 text-only (112k passages, ragged Nd 40-220, Nq=32)", 112_000, (40, 220), 32, 64, 5, 20),
    ("C2 FLMR (112k passages, ragged Nd 40-220, Nq=832 = 512 text + 320 vision)", 112_000, (40, 220), 832, 16, 5, 5),
    ("C3 B=1 (400k of 1M passages, Nd=180, Nq=320)", 400_000, (180, 180), 320, 1, 5, 5),
    ("C3 B=16", 400_000, (180, 180), 320, 16, 5, 3),
    ("C3 B=64", 400_000, (180, 180), 320, 64, 5, 2),
    ("C3 B=16, k=100", 400_000, (180, 180), 320, 16, 100, 3),
    ("C3 ragged (400k passages, Nd 90-180, Nq=320), B=16", 400_000, (90, 180), 320, 16, 5, 3),
]


def run(name, n_p, nd_rng, nq, B, k, iters):
    g = torch.Generator(device="cuda").manual_seed(0)
    gc = torch.Generator().manual_seed(0)
    if nd_rng[0] == nd_rng[1]:
        doclens = np.full(n_p, nd_rng[0], dtype=np.int32)
    else:
        doclens = torch.randint(nd_rng[0], nd_rng[1] + 1, (n_p,), generator=gc).numpy().astype(np.int32)
    n_tok = int(doclens.sum())
    D = torch.empty((n_tok, 128), dtype=torch.bfloat16, device="cuda")
    for a in range(0, n_tok, 1 << 22):
        b = min(n_tok, a + (1 << 22))
        D[a:b] = torch.nn.functional.normalize(torch.randn((b - a, 128), device="cuda", generator=g), dim=-1).bfloat16()
    Q = torch.nn.functional.normalize(torch.randn((B, nq, 128), device="cuda", generator=g), dim=-1).bfloat16()
    corpus = R.FlatCorpus(D, doclens)
    del D
    L = _cabi.lib()
    for _ in range(2):
        R.maxsim_topk(corpus, Q, k)
    torch.cuda.synchronize()
    L.flmr_set_profiling(1)
    L.flmr_scan_kernel_stats(None, None, 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        R.maxsim_topk(corpus, Q, k)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    tot, n = C.c_double(), C.c_int64()
    L.flmr_scan_kernel_stats(C.byref(tot), C.byref(n), 1)
    L.flmr_set_profiling(0)
    launches = n.value / iters
    scan_ms = tot.value / max(n.value, 1)
    info = corpus.info
    flops_call = 2.0 * B * nq * 128 * float(n_tok)               # algorithmic: real tokens, real query rows
    bytes_launch = float(info.n_rows) * 256.0                      # stored rows (incl. group padding) per pass
    tf = flops_call / (tot.value / iters) / 1e9 if tot.value else 0.0
    gbs = bytes_launch / scan_ms / 1e6 if scan_ms else 0.0
    print("| %s | %d | %d | %.3f | %.1f | %.0f | %.3f | %.0f | %.0f | %.0f%% |" % (
        name, B, k, ms, B / ms * 1e3, launches, scan_ms, tf, gbs, 100.0 * tot.value / iters / ms), flush=True)
    corpus.close()
    torch.cuda.empty_cache()


def main():
    print("# Shape sweep of the scan path\n")
    print("`python tools/shape_sweep.py` on one GPU; synthetic unit-norm bf16 embeddings; CUDA-event timing of "
          "`maxsim_topk` calls (queries resident on the device); scan columns from per-launch events "
          "(`flmr_set_profiling`).  TFLOP/s counts real tokens x real query rows only (padding is overhead); GB/s "
          "counts the stored token rows one launch streams.  Corpora below 1M passages: q/s scale ~1/N.\n")
    print("| workload | batch | k | ms / call | queries/s | scan launches / call | ms / scan launch | "
          "scan TFLOP/s | scan GB/s | scan share of call |")
    print("|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|")
    for case in CASES:
        run(*case)


if __name__ == "__main__":
    main()
