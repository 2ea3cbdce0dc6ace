"""A/B of two builds of libflmr_maxsim.so on the flagship benchmark, in alternating rounds.

    python tools/scan_ab.py --build-base REV          # CPU: compile revision REV's library into lib/ (needs git, nvcc)
    python tools/scan_ab.py [--rounds 3] [--out DIR]  # GPU: bench.py against lib/libflmr_maxsim_base.so, then
                                                      #      against lib/libflmr_maxsim.so, alternately

Each round runs the unmodified bench.py (``--steps 10 --warmup 3 --no-cpu-baseline``; the CPU and PLAID legs do
not touch the scan) in a fresh process with FLMR_MAXSIM_LIB naming the arm's library.  Both libraries share the C
ABI of include/flmr_maxsim.h, so one Python package drives both.  Prints per round: value, the scan launch time,
the median SM clock, the C2 record's value and the HBM-bound regime's launch time; per arm the median and spread
(max - min); the card name and power limit; and whether the arms' --dump-outputs top-k files are bitwise equal.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "retrieval-augmented-visual-question-answering_b200")
LIB_DIR = os.path.join(PKG, "lib")
BASE_LIB = os.path.join(LIB_DIR, "libflmr_maxsim_base.so")
NEW_LIB = os.path.join(LIB_DIR, "libflmr_maxsim.so")


def build_base(rev):
    """Compiles revision `rev`'s sources (from git) with the package's nvcc flags into lib/libflmr_maxsim_base.so."""
    sys.path.insert(0, PKG)
    import build as B
    rel_pkg = os.path.relpath(PKG, ROOT)
    with tempfile.TemporaryDirectory() as tmp:
        arch = subprocess.run(["git", "-C", ROOT, "archive", rev, os.path.join(rel_pkg, "csrc"), "include"],
                              check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=arch, check=True)
        os.makedirs(LIB_DIR, exist_ok=True)
        src = os.path.join(tmp, rel_pkg, "csrc", "flmr_maxsim.cu")
        subprocess.run([B.find_nvcc(), *B.NVCC_FLAGS, "-o", BASE_LIB, src], check=True)
    print("built %s from %s" % (BASE_LIB, rev))


def run_bench(lib, dump_dir, steps, warmup):
    env = dict(os.environ, FLMR_MAXSIM_LIB=lib)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
           str(warmup), "--no-cpu-baseline", "--dump-outputs", dump_dir]
    proc = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=tempfile.gettempdir())
    if proc.returncode != 0:
        raise SystemExit("bench.py failed with %s:\n%s" % (lib, proc.stderr[-4000:]))
    return json.loads([l for l in proc.stdout.splitlines() if l.startswith("{")][-1])


def summary(rec):
    rl = rec["roofline"]
    return {"value": rec["value"], "launch_ms": rl["launch_ms"], "sm_mhz": (rec.get("clocks") or {}).get("sm_mhz"),
            "c2_value": (rec.get("c2") or {}).get("value"),
            "c2_recall_at_1": (rec.get("c2") or {}).get("recall_at_1"),
            "c2_recall_at_100": (rec.get("c2") or {}).get("recall_at_100"),
            "hbm_launch_ms": (rl.get("hbm_bound_regime") or {}).get("launch_ms")}


def same_files(a, b):
    names = sorted(os.listdir(a))
    if names != sorted(os.listdir(b)) or not names:
        return False
    for n in names:
        with open(os.path.join(a, n), "rb") as fa, open(os.path.join(b, n), "rb") as fb:
            if fa.read() != fb.read():
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-base", metavar="REV", help="compile REV's library into lib/ and exit (CPU, needs git)")
    ap.add_argument("--base-lib", default=BASE_LIB)
    ap.add_argument("--new-lib", default=NEW_LIB)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the raw bench lines and dumped outputs")
    args = ap.parse_args()
    if args.build_base:
        build_base(args.build_base)
        return
    if os.path.abspath(args.new_lib) == os.path.abspath(NEW_LIB):
        # the package's own library: rebuilt here if it is older than the sources, so the new arm is what they say
        sys.path.insert(0, PKG)
        import build as B
        B.build()
    for lib in (args.base_lib, args.new_lib):
        if not os.path.exists(lib):
            raise SystemExit("missing %s (build it first)" % lib)
    out = os.path.abspath(args.out or tempfile.mkdtemp(prefix="scan_ab_"))
    os.makedirs(out, exist_ok=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card:", smi.stdout.strip() or "nvidia-smi unavailable", flush=True)
    arms = {"base": args.base_lib, "new": args.new_lib}
    rows = {a: [] for a in arms}
    with open(os.path.join(out, "bench_lines.jsonl"), "w") as raw:
        for r in range(args.rounds):
            for arm, lib in arms.items():
                rec = run_bench(lib, os.path.join(out, "%s_r%d" % (arm, r)), args.steps, args.warmup)
                raw.write(json.dumps({"arm": arm, "round": r, "bench": rec}) + "\n")
                raw.flush()
                s = summary(rec)
                rows[arm].append(s)
                print("round %d %-4s value %.3f q/s | launch %.2f ms | SM %s MHz | c2 %.1f q/s (R@1 %s, R@100 %s) | "
                      "hbm-bound launch %.3f ms" % (r, arm, s["value"], s["launch_ms"], s["sm_mhz"], s["c2_value"],
                                                    s["c2_recall_at_1"], s["c2_recall_at_100"], s["hbm_launch_ms"]),
                      flush=True)
    print("\n| arm | value q/s median (spread) | launch ms | SM MHz | c2 q/s | hbm-bound launch ms |")
    print("|---|---|---|---|---|---|")
    med = {}
    for arm in arms:
        cols = []
        for key in ("value", "launch_ms", "sm_mhz", "c2_value", "hbm_launch_ms"):
            v = [x[key] for x in rows[arm] if x[key] is not None]
            cols.append("%.3f (%.3f)" % (statistics.median(v), max(v) - min(v)) if v else "n/a")
            med[(arm, key)] = statistics.median(v) if v else None
        print("| %s | %s |" % (arm, " | ".join(cols)))
    if med[("base", "value")]:
        print("\nspeed-up of value (medians): %.3fx" % (med[("new", "value")] / med[("base", "value")]))
    equal = all(same_files(os.path.join(out, "base_r%d" % r), os.path.join(out, "new_r%d" % r))
                for r in range(args.rounds))
    print("dumped top-k scores / pids bitwise equal between arms in every round:", equal)
    c2_same = all((a["c2_recall_at_1"], a["c2_recall_at_100"]) == (b["c2_recall_at_1"], b["c2_recall_at_100"])
                  for a, b in zip(rows["base"], rows["new"]))
    print("c2 recall@1 / recall@100 equal between arms:", c2_same)
    if not equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
