"""Times the training / re-scoring path on bf16 and fp16 operands of the same values, in alternating rounds.

    python tools/fp16_train_probe.py [--rounds 5] [--out results/fp16_train_probe.json]

Per round and type:
  * the C4 step of bench.py's c4_record (8 queries x 16 documents, Nq 832, Nd 512 ragged): in_batch_negatives_loss
    forward + backward, eager and CUDA-graphed (the documents' dtype picks the kernels: bf16 or fp16 ones);
  * the arg-max forward alone on each kernel (forced warp-MMA and wgmma), with its TFLOP/s (2 * B * n * Nq * Nd * 128
    flops over the padded tokens);
  * Searcher.retrieve_and_rescore at B = 16, n_docs = 5 on a bf16 and an fp16 corpus of the same rows.
The fp16 documents are the bf16 ones converted, so both arms score the same values.  Prints medians and spreads (max -
min) per arm, with the card name, its power limit and the median SM clock while timing."""
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


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + query, "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out.splitlines()[0] if out else "not measured"
    except Exception:
        return "not measured"


def timed(fn, reps=20, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import ravqa_b200 as R
    from ravqa_b200 import _cabi
    from ravqa_b200.maxsim import maxsim_argmax
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = _cabi.lib()
    B, nway, nq, nd = 8, 2, 832, 512
    g = torch.Generator().manual_seed(1000)
    Q = torch.nn.functional.normalize(torch.randn(B, nq, 128, generator=g), dim=-1).to(dev)
    D32 = torch.nn.functional.normalize(torch.randn(B * nway, nd, 128, generator=g), dim=-1)
    lens = torch.randint(nd // 2, nd + 1, (B * nway,), generator=g)
    mask = (torch.arange(nd)[None, :] < lens[:, None]).unsqueeze(-1).to(dev)
    # the same values in both arms: bf16 documents, and those converted to fp16 (exact); the fp32 query is rounded by
    # each route to its own type
    docs = {"bf16": D32.to(torch.bfloat16).to(dev)}
    docs["fp16"] = docs["bf16"].to(torch.float16)
    Qd = {"bf16": Q.to(torch.bfloat16), "fp16": Q.to(torch.bfloat16).to(torch.float16)}
    flops = 2.0 * B * (B * nway) * nq * nd * 128
    # RAG block: one corpus per type of the same rows
    gr = torch.Generator().manual_seed(7)
    dl = torch.randint(20, 181, (20000,), generator=gr).numpy().astype(np.int32)
    rows = torch.nn.functional.normalize(torch.randn(int(dl.sum()), 128, generator=gr), dim=-1).to(torch.bfloat16)
    searchers = {"bf16": R.Searcher(index=R.FlatCorpus(rows, dl, device=0)),
                 "fp16": R.Searcher(index=R.FlatCorpus(rows.to(torch.float16), dl, device=0, storage="fp16"))}
    Qr = torch.nn.functional.normalize(torch.randn(16, 32, 128, generator=gr), dim=-1).to(torch.bfloat16).to(dev)
    results = {k: {} for k in docs}
    clocks = []

    def add(arm, key, v):
        results[arm].setdefault(key, []).append(v)

    for rnd in range(args.rounds):
        for arm in (("bf16", "fp16") if rnd % 2 == 0 else ("fp16", "bf16")):
            Dg = docs[arm].clone().requires_grad_(True)
            Qg = Q.clone().requires_grad_(True)

            def step():
                Qg.grad = Dg.grad = None
                R.in_batch_negatives_loss(Qg, Dg, mask, nway).backward()
            add(arm, "c4_eager_ms", timed(step))
            graphed = R.graphed_in_batch_negatives_loss(Qg, Dg, mask, nway)

            def gstep():
                Qg.grad = Dg.grad = None
                graphed(Qg, Dg, mask).backward()
            add(arm, "c4_graphed_ms", timed(gstep))
            m2 = mask.view(B * nway, nd)
            for path, name in ((1, "argmax_mma"), (2, "argmax_wgmma")):
                _cabi.check(L.flmr_debug_set_argmax_path(path))
                ms = timed(lambda: maxsim_argmax(Qd[arm], docs[arm], m2, return_rowmax=True))
                add(arm, name + "_ms", ms)
                add(arm, name + "_tflops", flops / (ms * 1e-3) / 1e12)
            _cabi.check(L.flmr_debug_set_argmax_path(0))
            Qrg = Qr.float().clone().requires_grad_(True)

            def rag():
                Qrg.grad = None
                out = searchers[arm].retrieve_and_rescore(Qrg, 5, generator=torch.Generator().manual_seed(0))
                out["doc_scores"].sum().backward()
            add(arm, "rag_b16_ndocs5_ms", timed(rag, reps=10))
            clocks.append(smi("clocks.sm"))
    summary = {"card": smi("name"), "power_limit_w": smi("power.limit"),
               "sm_clock_mhz_median": statistics.median(float(c) for c in clocks if c != "not measured")
               if any(c != "not measured" for c in clocks) else "not measured",
               "rounds": args.rounds, "arms": {}}
    for arm, d in results.items():
        summary["arms"][arm] = {k: {"median": statistics.median(v), "spread": max(v) - min(v), "all": v}
                                for k, v in d.items()}
    print(json.dumps(summary, indent=1))
    for k in results["bf16"]:
        a, b = summary["arms"]["bf16"][k], summary["arms"]["fp16"][k]
        print("%-24s bf16 %9.4f (spread %.4f)   fp16 %9.4f (spread %.4f)   fp16/bf16 %.3f"
              % (k, a["median"], a["spread"], b["median"], b["spread"], b["median"] / a["median"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)
    for s in searchers.values():
        s.corpus.close()


if __name__ == "__main__":
    main()
