"""Recall@5 of the REFERENCE's PLAID CPU search vs exhaustive MaxSim (build container only, CPU).

    python tools/plaid_recall_probe.py [--passages 5000] [--queries 40]

What RA-VQA actually runs at evaluation time under DDP is ColBERT's PLAID pipeline on CPU
(src/executors/FLMR_executor.py:778-792 -> colbert/searcher.py:91-132 -> IndexScorer.rank): centroid
candidate generation, centroid-only pruning (filter_pids.cpp), residual decompression, exact MaxSim on
<= ndocs/4 survivors.  This script builds a PLAID index over a synthetic clustered corpus with the
reference's own ResidualCodec / optimize_ivf (k-means by seeded torch Lloyd iterations: faiss is not
installed), runs the reference's IndexScorer.rank per query, and compares its top-5 with exhaustive
scoring of (a) the same decompressed embeddings and (b) the original embeddings — the ranking the
H100 scan returns (tests/test_plaid.py and tests/test_gpu_parity.py pin the CUDA path to the oracle
used here).  Queries are noisy token subsets of a planted passage, so a known positive exists.
Prints the tables as markdown.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden import import_reference  # noqa: E402
from oracle import maxsim_oracle as O  # noqa: E402


def kmeans(x, k, iters, g):
    c = x[torch.randperm(x.size(0), generator=g)[:k]].clone()
    for _ in range(iters):
        assign = torch.cat([(xb @ c.T).argmax(dim=1) for xb in x.split(1 << 15)])
        sums = torch.zeros_like(c).index_add_(0, assign, x)
        cnt = torch.bincount(assign, minlength=k).clamp_min(1).unsqueeze(1)
        c = torch.nn.functional.normalize(sums / cnt, dim=-1)
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=5000)
    ap.add_argument("--nd", type=int, default=64)
    ap.add_argument("--queries", type=int, default=40)
    ap.add_argument("--nq", type=int, default=32)
    ap.add_argument("--nbits", type=int, default=2)
    args = ap.parse_args()
    ColBERTConfig = import_reference()[0]
    md = ["# Recall@5: reference PLAID search vs exhaustive MaxSim (round 1, CPU probe)", "",
          "Command (build container, CPU): `python tools/plaid_recall_probe.py --passages %d --queries %d --nbits %d`"
          % (args.passages, args.queries, args.nbits), "",
          "PLAID is an approximate search: how much it loses against exhaustive scoring depends on how well the "
          "centroids summarise the token embeddings.  Two synthetic regimes bracket that: (A) clustered tokens with "
          "residual norms in the range real ColBERT indexes show, (B) nearly isotropic tokens, where centroid "
          "scores carry almost no information.  Real collections sit much closer to (A).", ""]
    for tag, noise, qnoise, topics, ndocs in (("A: clustered", 0.06, 0.04, 200, 128),
                                              ("B: near-isotropic (stress)", 0.6, 0.35, 200, 1024)):
        md += run_regime(args, ColBERTConfig, tag, noise, qnoise, topics, ndocs) + [""]
    md += ["The CUDA path returns exactly the exhaustive ranking (parity tests pin it to the oracle used here): its "
           "Recall@5 equals the exhaustive rows, whatever the regime; the first row of each table is the reference's "
           "pruned search.  Latencies are for this container's %d CPU threads." % torch.get_num_threads()]
    print("\n".join(md))


def run_regime(args, ColBERTConfig, tag, noise, qnoise, n_topics, ndocs):
    from colbert.indexing.codecs.residual import ResidualCodec
    from colbert.indexing.utils import optimize_ivf
    from colbert.search.index_storage import IndexScorer

    g = torch.Generator().manual_seed(0)
    n, nd = args.passages, args.nd
    # clustered corpus: each passage mixes 3 topic directions; tokens = topic direction + per-dimension noise
    # (noise 0.06 -> |noise| ~ 0.68, token/topic cosine ~ 0.83: residual norms in the range real ColBERT indexes show)
    topics = torch.nn.functional.normalize(torch.randn(n_topics, 128, generator=g), dim=-1)
    ptop = torch.randint(0, n_topics, (n, 3), generator=g)
    tok_topic = ptop[torch.arange(n).repeat_interleave(nd), torch.randint(0, 3, (n * nd,), generator=g)]
    D = torch.nn.functional.normalize(topics[tok_topic] + noise * torch.randn(n * nd, 128, generator=g), dim=-1)
    D = D.bfloat16().float()
    doclens = torch.full((n,), nd, dtype=torch.long)
    # queries: 32 noisy tokens of a planted passage
    targets = torch.randint(0, n, (args.queries,), generator=g)
    Q = []
    for t in targets.tolist():
        rows = D[t * nd:(t + 1) * nd][torch.randperm(nd, generator=g)[:args.nq]]
        Q.append(torch.nn.functional.normalize(rows + qnoise * torch.randn(args.nq, 128, generator=g), dim=-1))
    Q = torch.stack(Q).bfloat16().float()

    # ---- PLAID index with the reference's codec ----
    n_emb = n * nd
    K = int(2 ** np.floor(np.log2(16 * np.sqrt(n_emb))))          # collection_indexer.py:93
    t0 = time.time()
    centroids = kmeans(D[torch.randperm(n_emb, generator=g)[: min(n_emb, 200_000)]], K, 4, g).half().float()
    print("k-means K=%d: %.1fs" % (K, time.time() - t0), flush=True)
    index_path = tempfile.mkdtemp(prefix="plaid_probe_")
    cfg = ColBERTConfig(nbits=args.nbits, dim=128, total_visible_gpus=0, index_path=index_path)
    c0 = ResidualCodec(config=cfg, centroids=centroids, avg_residual=None)
    held = D[torch.randperm(n_emb, generator=g)[:50_000]]
    res = held - c0.lookup_centroids(c0.compress_into_codes(held, out_device="cpu"), out_device="cpu")
    num_options = 2 ** args.nbits
    quant = torch.arange(0, num_options) * (1 / num_options)
    codec = ResidualCodec(config=cfg, centroids=centroids, avg_residual=torch.abs(res).mean(dim=0).mean(),
                          bucket_cutoffs=res.float().quantile(quant[1:]),
                          bucket_weights=res.float().quantile(quant + 0.5 / num_options))
    comp = codec.compress(D)
    codec.save(index_path)
    comp.save(os.path.join(index_path, "0"))
    json.dump(doclens.tolist(), open(os.path.join(index_path, "doclens.0.json"), "w"))
    json.dump({"passage_offset": 0, "num_passages": n, "num_embeddings": n_emb, "embedding_offset": 0},
              open(os.path.join(index_path, "0.metadata.json"), "w"))
    exported = cfg.export()
    exported.pop("collection", None)
    json.dump({"config": exported, "num_chunks": 1, "num_partitions": K, "num_embeddings": n_emb,
               "avg_doclen": nd}, open(os.path.join(index_path, "metadata.json"), "w"))
    codes_sorted = comp.codes.long().sort()
    optimize_ivf(codes_sorted.indices, torch.bincount(codes_sorted.values, minlength=K), index_path)

    # ---- reference PLAID search (CPU), defaults of Searcher.dense_search for k <= 10 ----
    scorer = IndexScorer(index_path, use_gpu=False)
    search_cfg = ColBERTConfig(ncells=2, centroid_score_threshold=0.45, ndocs=ndocs, total_visible_gpus=0,
                               query_maxlen=args.nq)
    plaid_top, n_cands, t_plaid = [], [], 0.0
    for i in range(args.queries):
        qi = Q[i:i + 1]
        cand_pids, _ = scorer.retrieve(search_cfg, qi)
        n_cands.append(int(cand_pids.numel()))
        t0 = time.time()
        pids, scores = scorer.rank(search_cfg, qi)
        t_plaid += time.time() - t0
        plaid_top.append(list(pids[:5]))
    # ---- exhaustive rankings ----
    D_dec = codec.decompress(comp).numpy()
    exact_dec = O.topk(O.maxsim_scores(Q.numpy(), D_dec, doclens.numpy()), 5)[1]
    exact_orig = O.topk(O.maxsim_scores(Q.numpy(), D.numpy(), doclens.numpy()), 5)[1]

    def overlap(a, b):
        return float(np.mean([len(set(x) & set(y)) / 5.0 for x, y in zip(a, b)]))

    def hit(tops):
        return float(np.mean([int(t) in set(map(int, top)) for t, top in zip(targets.tolist(), tops)]))

    rows = [
        ("reference PLAID CPU search (ncells=2, thr=0.45, ndocs=%d)" % ndocs, hit(plaid_top),
         overlap(plaid_top, exact_dec), overlap(plaid_top, exact_orig)),
        ("exhaustive MaxSim over the decompressed index (this repo on a PLAID index)", hit(exact_dec), 1.0,
         overlap(exact_dec, exact_orig)),
        ("exhaustive MaxSim over the original bf16 embeddings (this repo, flat index)", hit(exact_orig),
         overlap(exact_orig, exact_dec), 1.0),
    ]
    min_c = min(n_cands)
    md = ["## Regime %s" % tag, "",
          "%d passages x %d tokens (%d topic directions, 3 per passage, per-dimension noise %.2f; query noise %.2f), "
          "K = %d centroids (seeded torch k-means, faiss absent), nbits = %d; %d queries = %d noisy tokens of a "
          "planted passage." % (n, nd, n_topics, noise, qnoise, K, args.nbits, args.queries, args.nq), "",
          "| ranking | planted passage in top-5 | top-5 overlap with exact (decompressed) | top-5 overlap with exact (original) |",
          "|---|---:|---:|---:|"]
    for name, h, o1, o2 in rows:
        md.append("| %s | %.3f | %.3f | %.3f |" % (name, h, o1, o2))
    min_c = min(n_cands)
    md += ["", "PLAID candidates per query: min %d / median %d (ndocs = %d%s); reference PLAID latency %.1f ms/query." % (
        min_c, int(np.median(n_cands)), ndocs,
        "; fewer than ndocs -> filter_pids.cpp pops an empty queue (SURVEY hazard 2)" if min_c < ndocs else "",
        1e3 * t_plaid / args.queries)]
    shutil.rmtree(index_path, ignore_errors=True)
    return md


if __name__ == "__main__":
    main()
