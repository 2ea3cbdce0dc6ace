"""GPU: the stages of a PLAID index build (Indexer(index_format="plaid")) and the encode kernel's rate.

    python tools/plaid_build_probe.py [--passages 240000] [--doclen 180] [--K 65536] [--nbits 2]
                                      [--encode-tokens 1048576] [--reps 3] [--json out.json]

Prints the card, its power limit and max SM clock (read in the same command as the timings; nothing is set), then:
  * the build stages on synthetic clustered embeddings (4096 topic directions plus noise, made on the device; the
    encoder is out of scope), sized as the reference sizes them for --passages x --doclen tokens: the sample
    (16 sqrt(120 n) passages), k-means (--K centroids, 4 iterations), the bucket quantiles of the held-out 5 %, the
    encode of --encode-tokens chunk tokens (codes and residuals, with the device-to-host copy), and the IVF of the
    codes; each stage timed with a device synchronise around it;
  * the encode kernel (flmr_plaid_encode, residuals on) and its assignment-only mode: CUDA events over --reps calls,
    TFLOP/s from 2 n K 128 operations, against 989 dense fp16 (data sheet);
  * the reference's composition on the same rows: (C @ X.T).max(0) in batches of (1 << 29) // K tokens, then the
    fp16 subtraction, torch.bucketize and the bit packing of ResidualCodec.binarize (restated with torch ops);
  * flmr_maxsim_argmax_fp16 for assignment only: the rows as one query batch against one "document" of K rows;
  * the extrapolated encode time of all --passages x --doclen tokens at the measured kernel rate.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ravqa_b200 import plaid  # noqa: E402
from ravqa_b200.maxsim import maxsim_argmax  # noqa: E402

PEAK_FP16 = 989e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


def rows(n, topics, g):
    t = topics[torch.randint(0, topics.size(0), (n,), device="cuda", generator=g)]
    return torch.nn.functional.normalize(t + 0.6 * torch.randn(n, 128, device="cuda", generator=g) / 128 ** 0.5,
                                         dim=-1).half()


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def reference_composition(x, c, cutoffs, nbits):
    """ResidualCodec.compress_into_codes + compress + binarize (residual.py:169-222), GPU branch, on the same rows."""
    K = c.size(0)
    codes = torch.cat([(c @ b.T).max(dim=0).indices for b in x.split((1 << 29) // K)])
    r = x - c[codes]
    bk = torch.bucketize(r.float(), cutoffs).to(torch.uint8)
    bits = (bk.unsqueeze(-1) >> torch.arange(nbits, device=x.device, dtype=torch.uint8)) & 1
    bits = bits.reshape(x.size(0), -1, 8)
    packed = (bits << torch.arange(7, -1, -1, device=x.device, dtype=torch.uint8)).sum(-1, dtype=torch.uint8)
    return codes, packed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=240000)
    ap.add_argument("--doclen", type=int, default=180)
    ap.add_argument("--K", type=int, default=65536)
    ap.add_argument("--nbits", type=int, default=2)
    ap.add_argument("--encode-tokens", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this probe measures the GPU"
    out = {"card": card(), "passages": a.passages, "doclen": a.doclen, "K": a.K, "nbits": a.nbits}
    print("card:", out["card"])
    g = torch.Generator(device="cuda").manual_seed(0)
    topics = torch.nn.functional.normalize(torch.randn(4096, 128, device="cuda", generator=g), dim=-1)
    n_sample_passages = min(1 + int(16 * np.sqrt(120 * a.passages)), a.passages)
    t, sample = timed(lambda: rows(n_sample_passages * a.doclen, topics, g))
    stages = {"sample_rows": int(sample.size(0)), "sample_s (synthetic, no encoder)": t}
    held = int(min(0.05 * sample.size(0), 50_000))
    train, heldout = sample.split([sample.size(0) - held, held])
    t, cents = timed(lambda: plaid.kmeans(train, a.K, niters=4, seed=123))
    stages["kmeans_s"] = t
    t, (cutoffs, weights, _) = timed(lambda: plaid.residual_buckets(cents, heldout, a.nbits))
    stages["buckets_s"] = t
    del sample, train
    x = rows(a.encode_tokens, topics, g)
    cut_d = cutoffs.cuda()
    t, enc = timed(lambda: [v.cpu() for v in plaid.encode(x, cents, cut_d, nbits=a.nbits)])
    stages["encode_s (%d tokens, with copy-out)" % a.encode_tokens] = t
    t, _ = timed(lambda: plaid.build_ivf(enc[0].cuda(), [a.doclen] * (a.encode_tokens // a.doclen)
                                         + ([a.encode_tokens % a.doclen] if a.encode_tokens % a.doclen else []), a.K))
    stages["ivf_s (%d tokens)" % a.encode_tokens] = t
    out["stages"] = stages
    for k, v in stages.items():
        print("  %-44s %s" % (k, ("%.3f" % v) if isinstance(v, float) else v))

    flop = 2.0 * a.encode_tokens * a.K * 128
    rates = {}
    t_enc = events(lambda: plaid.encode(x, cents, cut_d, nbits=a.nbits), a.reps)
    rates["flmr_plaid_encode (codes + residuals)"] = t_enc
    rates["flmr_plaid_encode (assignment only)"] = events(lambda: plaid.encode(x, cents), a.reps)
    try:
        rates["reference composition (matmul + max + bucketize + pack)"] = events(
            lambda: reference_composition(x, cents, cut_d, a.nbits), a.reps)
        rc, rp = reference_composition(x, cents, cut_d, a.nbits)
        kc, kp = plaid.encode(x, cents, cut_d, nbits=a.nbits)
        out["codes_equal_reference_composition"] = float((rc.int() == kc).float().mean())
    except torch.cuda.OutOfMemoryError:
        rates["reference composition (matmul + max + bucketize + pack)"] = None
    try:
        Q = x.unsqueeze(0)
        D = cents.unsqueeze(0)
        mask = torch.ones((1, a.K), dtype=torch.bool, device="cuda")
        rates["flmr_maxsim_argmax_fp16 (assignment only)"] = events(lambda: maxsim_argmax(Q, D, mask), a.reps)
    except Exception as e:                                       # noqa: BLE001  (reported, not hidden)
        print("  flmr_maxsim_argmax_fp16: not measured (%s)" % e)
        rates["flmr_maxsim_argmax_fp16 (assignment only)"] = None
    out["rates"] = {}
    print("encode of %d tokens against K=%d (%.3g FLOP):" % (a.encode_tokens, a.K, flop))
    for k, v in rates.items():
        if v is None:
            print("  %-58s not measured" % k)
            continue
        out["rates"][k] = {"s": v, "tflops": flop / v / 1e12, "of_989": flop / v / PEAK_FP16}
        print("  %-58s %8.3f s  %6.1f TFLOP/s  %.2f of 989" % (k, v, flop / v / 1e12, flop / v / PEAK_FP16))
    total = a.passages * a.doclen
    out["extrapolated_full_encode_s"] = t_enc * total / a.encode_tokens
    print("extrapolated encode of all %d tokens at that rate: %.0f s" % (total, out["extrapolated_full_encode_s"]))
    if "codes_equal_reference_composition" in out:
        print("codes equal to the reference composition's: %.6f of rows" % out["codes_equal_reference_composition"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=2)


if __name__ == "__main__":
    main()
