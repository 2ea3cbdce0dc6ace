"""Turn an `ncu --metrics gpu__time_duration.sum --csv --log-file X.csv` launch list into the markdown
summary (per-kernel launches, total time, share; this library's kernels apart).

    python tools/launch_list_md.py launches.csv "<command that produced it>" > launches.md
"""
import csv
import sys
from collections import OrderedDict


def main():
    path, command = sys.argv[1], sys.argv[2]
    rows = []
    with open(path, newline="") as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    reader = csv.DictReader(lines)
    for r in reader:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        val = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "ns")
        ms = val * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(unit, 1e-6)
        rows.append((r["Kernel Name"], ms))
    agg = OrderedDict()
    for name, ms in rows:
        short = name.split("(")[0].replace("at::", "")[:70]
        n, t = agg.get(short, (0, 0.0))
        agg[short] = (n + 1, t + ms)
    total = sum(t for _, t in agg.values())
    print("# ncu launch list\n")
    print("Command (1 GPU): `%s`\n" % command)
    print("Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes. Includes corpus "
          "generation (torch randn/normalize), the bench's HBM-regime leg, its self-check and the library-GPU "
          "baseline leg (torch/cuBLAS kernels) when enabled.\n")
    print("| kernel | launches | total ms | share |\n|---|---:|---:|---:|")
    for name, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("| `%s` | %d | %.3f | %.1f%% |" % (name, n, t, 100.0 * t / total))
    ours = {k: v for k, v in agg.items() if "flmr_" in k}
    tot_o = sum(t for _, t in ours.values())
    print("\nAmong this library's own kernels (the hot path proper):\n")
    print("| kernel | launches | total ms | share of flmr_* time |\n|---|---:|---:|---:|")
    for name, (n, t) in sorted(ours.items(), key=lambda kv: -kv[1][1]):
        print("| `%s` | %d | %.3f | %.2f%% |" % (name, n, t, 100.0 * t / tot_o))


if __name__ == "__main__":
    main()
