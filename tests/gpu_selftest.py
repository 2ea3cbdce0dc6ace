"""Diagnostic GPU self-test (not collected by pytest): runs each case in its own subprocess with a
timeout, so a trapped or hung launch cannot take the whole gpurun call down, and prints enough to
debug descriptor / layout mistakes from one run.

    python tests/gpu_selftest.py            # all cases
    python tests/gpu_selftest.py --case c1  # one case, in-process
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _mk(n_passages, nd, n_queries, nq, seed=0, ragged=False):
    import numpy as np
    import torch
    from oracle import maxsim_oracle as O
    Q, D, doclens = O.synth(n_passages, nd, n_queries, nq, seed=seed, ragged=ragged)
    return Q, D, doclens


def _report(name, got, ref):
    import numpy as np
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref)
    rel = err / np.maximum(np.abs(ref), 1e-6)
    print("  %-28s max_abs=%.3e max_rel=%.3e  (ref range %.3f..%.3f)" %
          (name, err.max(), rel.max(), ref.min(), ref.max()), flush=True)
    return rel.max()


def case_structured():
    """One-hot operands: exposes K-slicing / swizzle / row-mapping mistakes as readable patterns."""
    import numpy as np
    import torch
    import ravqa_b200 as R
    nq, n_p = 32, 128
    Q = np.zeros((1, nq, 128), dtype=np.float32)
    for i in range(nq):
        Q[0, i, 4 * i] = 1.0            # query row i looks at dim 4i
    D = np.zeros((n_p * 4, 128), dtype=np.float32)
    for p in range(n_p):
        D[4 * p:4 * p + 4, p] = 1.0 + p / 256.0   # passage p lives on dim p with a unique value
    doclens = np.full(n_p, 4, dtype=np.int32)
    corpus = R.FlatCorpus(torch.from_numpy(D), doclens)
    print("  corpus:", corpus, flush=True)
    s = R.maxsim_scores(corpus, torch.from_numpy(Q)).cpu().numpy()[0]
    exp = np.array([(1.0 + p / 256.0) if p % 4 == 0 else 0.0 for p in range(n_p)], dtype=np.float32)
    print("  got[:16] =", np.round(s[:16], 3))
    print("  exp[:16] =", np.round(exp[:16], 3))
    bad = np.nonzero(np.abs(s - exp) > 1e-3)[0]
    print("  mismatches: %d %s" % (len(bad), bad[:20]))
    if len(bad):
        print("  got full =", np.round(s, 3).tolist())
    return len(bad) == 0


def _run_parity(n_passages, nd, n_queries, nq, k, ragged=False, relu=False, simt=True, tol=1e-3):
    import numpy as np
    import torch
    import ravqa_b200 as R
    from oracle import maxsim_oracle as O
    Q, D, doclens = _mk(n_passages, nd, n_queries, nq, ragged=ragged)
    corpus = R.FlatCorpus(torch.from_numpy(D).to(torch.bfloat16), doclens)
    print("  corpus:", corpus, flush=True)
    t0 = time.time()
    ref = O.maxsim_scores(Q, D, doclens, relu=relu)
    print("  oracle %.2fs" % (time.time() - t0), flush=True)
    Qt = torch.from_numpy(Q)
    ok = True
    if simt:
        s_simt = R.debug_scores_simt(corpus, Qt, relu=relu).cpu().numpy()
        ok &= _report("simt vs oracle", s_simt, ref) < tol
    s_tc = R.maxsim_scores(corpus, Qt, relu=relu)
    torch.cuda.synchronize()
    s_tc = s_tc.cpu().numpy()
    r = _report("wgmma scores vs oracle", s_tc, ref)
    ok &= r < tol
    if r >= tol:
        bad = np.argwhere(np.abs(s_tc - ref) / np.maximum(np.abs(ref), 1e-6) > tol)
        print("  first mismatches (b,p):", bad[:10].tolist())
        for b, p in bad[:5]:
            print("    b=%d p=%d got=%.5f ref=%.5f" % (b, p, s_tc[b, p], ref[b, p]))
    ts, tp = R.maxsim_topk(corpus, Qt, k, relu=relu)
    torch.cuda.synchronize()
    ts, tp = ts.cpu().numpy(), tp.cpu().numpy()
    rs, rp = O.topk(ref, k)
    ids_ok = bool((tp == rp).all())
    print("  topk ids identical: %s" % ids_ok)
    if not ids_ok:
        print("   got", tp[:2].tolist(), "\n   ref", rp[:2].tolist())
    if n_passages >= k:
        ok &= _report("topk scores vs oracle", ts, rs) < tol
    ok &= ids_ok
    corpus.close()
    return ok


def case_tiny():
    return _run_parity(8, 64, 1, 32, k=5)


def case_c1():
    return _run_parity(1000, 64, 16, 32, k=5)


def case_c1_ragged():
    return _run_parity(1000, 64, 16, 32, k=10, ragged=True)


def case_c1_relu():
    return _run_parity(500, 12, 4, 32, k=5, ragged=True, relu=True)


def case_nq320():
    return _run_parity(4000, 180, 2, 320, k=5)


def case_nq832():
    return _run_parity(1500, 150, 1, 832, k=100, ragged=True)


def case_perf():
    """First throughput number: 200k passages x 180 tokens (9.2 GB), Nq=320."""
    import torch
    import ravqa_b200 as R
    n_p, nd, nq = 200_000, 180, 320
    g = torch.Generator(device="cuda").manual_seed(0)
    D = torch.randn((n_p * nd, 128), device="cuda", generator=g, dtype=torch.float32)
    D = torch.nn.functional.normalize(D, dim=-1).to(torch.bfloat16)
    Q = torch.nn.functional.normalize(torch.randn((4, nq, 128), device="cuda", generator=g), dim=-1)
    corpus = R.FlatCorpus(D, torch.full((n_p,), nd, dtype=torch.int32))
    print("  corpus:", corpus, flush=True)
    for B in (1, 4):
        for _ in range(2):
            R.maxsim_topk(corpus, Q[:B], 5)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 5
        e0.record()
        for _ in range(iters):
            s, p = R.maxsim_topk(corpus, Q[:B], 5)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        bytes_pass = n_p * nd * 256
        flops = 2.0 * B * nq * 128 * n_p * nd
        print("  B=%d: %.3f ms/call  %.1f q/s  | corpus pass BW %.0f GB/s (x%d passes)  %.1f TFLOP/s "
              "| extrapolated to 1M passages: %.1f q/s"
              % (B, ms, B / ms * 1e3, bytes_pass * B / ms / 1e6, B, flops / ms / 1e9,
                 B / (ms * 5) * 1e3), flush=True)
    # cross-check against the SIMT kernel on a slice of queries
    s_all = R.maxsim_scores(corpus, Q[:1])
    s_simt = R.debug_scores_simt(corpus, Q[:1])
    torch.cuda.synchronize()
    rel = ((s_all - s_simt).abs() / s_simt.abs().clamp_min(1e-6)).max().item()
    print("  full-size wgmma vs simt max_rel = %.3e" % rel)
    ts, tp = R.maxsim_topk(corpus, Q[:1], 5)
    rs, rp = torch.topk(s_all, 5, dim=1)
    print("  fused topk ids == topk(all scores): %s" % bool((tp == rp).all().item()))
    return rel < 1e-3 and bool((tp == rp).all().item())


CASES = {
    "structured": case_structured, "tiny": case_tiny, "c1": case_c1, "c1_ragged": case_c1_ragged,
    "c1_relu": case_c1_relu, "nq320": case_nq320, "nq832": case_nq832, "perf": case_perf,
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    ap.add_argument("--timeout", type=int, default=300)
    args = ap.parse_args()
    if args.case:
        ok = CASES[args.case]()
        print("CASE %s: %s" % (args.case, "PASS" if ok else "FAIL"), flush=True)
        sys.exit(0 if ok else 1)
    results = {}
    for name in CASES:
        print("=== %s ===" % name, flush=True)
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", name],
                               timeout=args.timeout)
            results[name] = "PASS" if r.returncode == 0 else "FAIL(rc=%d)" % r.returncode
        except subprocess.TimeoutExpired:
            results[name] = "TIMEOUT"
    print("SUMMARY:", results, flush=True)
    sys.exit(0 if all(v == "PASS" for v in results.values()) else 1)


if __name__ == "__main__":
    main()
