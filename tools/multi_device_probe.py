"""GPU: what a corpus split across the devices of one process (``Searcher(devices=...)``) costs per search, against the
same corpus on one device, and what the merge kernel of ``flmr_topk_merge_devices`` costs by itself.

    python tools/multi_device_probe.py [--passages 1000000] [--devices 1 2 4 8] [--reps 20] [--out PATH]

Writes ``profiles/r13_multi_device_probe.md`` (or ``--out``) with:
  * every visible card's name, power limit and max SM clock, read in the same command as the timings (nothing is set),
    and whether each pair of the devices used can read the other's memory (``torch.cuda.can_device_access_peer``);
  * per device count n (those of ``--devices`` the node has): the time of one ``maxsim_topk``-shaped search (k = 10;
    CUDA events around ``--reps`` calls after a warm-up, on the home device's stream, which the merge orders after every
    shard's stream) at Nq = 32 and Nq = 320, B = 1 and 16, over ``--passages`` passages of 180 tokens split into n
    token-balanced shards on devices 0 .. n-1, and whether every result is torch.equal to the n = 1 result;
  * the merge kernel's own time per call (CUDA events around ``--reps`` merges of n lists of [B, k] already on their
    devices, k = 10 and 128), home device 0.

The shards are built on their devices from seeded random rows (the rates do not depend on the values); each shard's
search is ``maxsim_topk`` on it, the per-shard call of an unrestricted Searcher search, and the split and merge are the
Searcher's own (``sharded.DeviceShardedSearcher``).
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ravqa_b200 as R  # noqa: E402
from ravqa_b200.maxsim import maxsim_topk  # noqa: E402
from ravqa_b200.sharded import DeviceShardedSearcher, merge_device_lists  # noqa: E402

ND = 180
K = 10
SHAPES = [(32, 1), (32, 16), (320, 1), (320, 16)]


def cards():
    return subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()


def events_ms(fn, reps, device):
    fn()
    torch.cuda.synchronize(device)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(torch.cuda.current_stream(device))
    for _ in range(reps):
        fn()
    b.record(torch.cuda.current_stream(device))
    b.synchronize()
    return a.elapsed_time(b) / reps


def build_shards(n_passages, n_dev, seed=0):
    dl = np.full(n_passages, ND, dtype=np.int32)
    shards = []
    for i, (p0, p1) in enumerate(R.shard_ranges(dl, n_dev)):
        g = torch.Generator(device="cuda:%d" % i).manual_seed(seed + i)
        tokens = torch.randn((int(dl[p0:p1].sum()), 128), generator=g, device="cuda:%d" % i, dtype=torch.bfloat16)
        shards.append(R.FlatCorpus(tokens, dl[p0:p1], device=i, pid_base=p0))
    return shards


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=1_000_000)
    ap.add_argument("--devices", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r13_multi_device_probe.md"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_device_probe needs CUDA devices")
    n_vis = torch.cuda.device_count()
    counts = [n for n in a.devices if n <= n_vis]
    g = torch.Generator().manual_seed(1)
    queries = {(nq, b): torch.nn.functional.normalize(torch.randn(b, nq, 128, generator=g), dim=-1)
               .to(torch.bfloat16).cuda() for nq, b in SHAPES}
    peer = [(i, j, torch.cuda.can_device_access_peer(i, j)) for i in range(max(counts)) for j in range(max(counts))
            if i != j]
    lines = ["# Multi-device search in one process (`Searcher(devices=...)`)", "",
             "Command: `python tools/multi_device_probe.py --passages %d --devices %s --reps %d`"
             % (a.passages, " ".join(map(str, a.devices)), a.reps), "", "Cards (index, name, power limit, max SM clock),"
             " read in the same run:", ""] + ["    " + c for c in cards()] + [""]
    if peer:
        lines += ["Peer access among the devices used: " + ", ".join("%d->%d %s" % (i, j, "yes" if ok else "no")
                                                                      for i, j, ok in peer), ""]
    lines += ["%d visible device(s); device counts measured: %s; %s not measured here."
              % (n_vis, counts, [n for n in a.devices if n not in counts] or "none"), "",
              "## One search: %d passages x %d tokens, k = %d, ms per call (CUDA events, %d calls)" % (a.passages, ND, K,
                                                                                                       a.reps), "",
              "| devices | " + " | ".join("Nq %d, B %d" % s for s in SHAPES) + " | equal to 1 device |",
              "|---|" + "---|" * len(SHAPES) + "---|"]
    merge_rows = []
    ref = {}
    for n in counts:
        shards = build_shards(a.passages, n)
        ds = DeviceShardedSearcher([c.device.index for c in shards], lambda i, Q, k: maxsim_topk(shards[i], Q, k))
        times, equal = [], True
        for s in SHAPES:
            Q = queries[s]
            with torch.cuda.device(0):
                times.append(events_ms(lambda: ds.search(Q, K), a.reps, 0))
                out = ds.search(Q, K)
            torch.cuda.synchronize()
            if n == counts[0]:
                ref[s] = out
            else:
                equal &= torch.equal(out[0].cpu(), ref[s][0].cpu()) and torch.equal(out[1].cpu(), ref[s][1].cpu())
        lines.append("| %d | " % n + " | ".join("%.3f" % t for t in times) + " | %s |" % ("reference" if n == counts[0]
                                                                                         else equal))
        for B in (1, 16):
            for k in (K, 128):
                lists = [(torch.randn(B, k, device=c.device), torch.randint(0, a.passages, (B, k), device=c.device))
                         for c in shards]
                torch.cuda.synchronize()
                with torch.cuda.device(0):
                    ms = events_ms(lambda: merge_device_lists(lists, ds.streams, k, ds.home), a.reps * 10, 0)
                merge_rows.append("| %d | %d | %d | %.4f |" % (n, B, k, ms))
        del ds, shards
        torch.cuda.empty_cache()
    lines += ["", "## The merge kernel alone: `flmr_topk_merge_devices` on device 0, ms per call (CUDA events, %d calls)"
              % (a.reps * 10), "", "| lists (devices) | B | k | ms |", "|---|---|---|---|"] + merge_rows
    lines += ["", "Rows with more than one device need a multi-GPU node; where this file lists none, the scaling across "
              "devices and the cost of peer reads are not measured."]
    text = "\n".join(lines) + "\n"
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()
