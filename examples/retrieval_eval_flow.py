"""End-to-end drop-in flow, mirroring what FLMRExecutor does at validation/test time
(src/executors/FLMR_executor.py: prepare_item_embeddings :515-719, evaluate_outputs :722-1018):

    1. encode the passage collection           (PyTorch encoder - here a stand-in)   -> Indexer.index
    2. encode the queries                       (PyTorch encoder - here a stand-in)   -> Q [n, Nq, 128]
    3. searcher._search_all_Q(queries, Q, k)    (the H100 scan: exhaustive, batched)  -> Ranking
    4. Recall@K over the ranking                (as compute_DPR_scores, metrics_processors.py:481-542)

    python examples/retrieval_eval_flow.py [--passages 20000] [--queries 64]

The stand-in encoders produce clustered unit vectors so that every query has a known relevant passage;
swap them for `model.doc(...)` / `model.query(...)` of an FLMR checkpoint in real use.
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ravqa_b200 as R  # noqa: E402


def make_standin_encoders(n_topics=500, seed=0):
    g = torch.Generator().manual_seed(seed)
    topics = torch.nn.functional.normalize(torch.randn(n_topics, 128, generator=g), dim=-1)

    def passage_tokens(pid: int, n: int):
        gp = torch.Generator().manual_seed(10_000 + pid)
        t = torch.randint(0, n_topics, (3,), generator=gp)
        rows = topics[t[torch.randint(0, 3, (n,), generator=gp)]] + 0.5 * torch.randn(n, 128, generator=gp)
        return torch.nn.functional.normalize(rows, dim=-1)

    def encode_docs(passages):                       # CollectionEncoder.encode_passages contract
        embs, doclens = [], []
        for text in passages:
            pid = int(text.split()[1])
            n = 40 + pid % 90
            embs.append(passage_tokens(pid, n))
            doclens.append(n)
        return torch.cat(embs), doclens

    def encode_query(pid: int, nq: int = 64):        # a noisy view of passage `pid` (its "question")
        gp = torch.Generator().manual_seed(77 + pid)
        rows = passage_tokens(pid, 40 + pid % 90)
        rows = rows[torch.randint(0, rows.size(0), (nq,), generator=gp)] + 0.3 * torch.randn(nq, 128, generator=gp)
        return torch.nn.functional.normalize(rows, dim=-1)

    return encode_docs, encode_query


def run(n_passages=20_000, n_queries=64, ks=(1, 5, 10, 20, 50, 100), index_root=None, verbose=True):
    encode_docs, encode_query = make_standin_encoders()
    collection = ["passage %d" % i for i in range(n_passages)]
    index_root = index_root or tempfile.mkdtemp(prefix="flmr_flat_")
    path = R.Indexer(encode_fn=encode_docs, index_root=index_root, chunksize=5000).index(
        "temp_index.nbits=8", collection, overwrite=True)
    searcher = R.Searcher(index=path)
    gq = torch.Generator().manual_seed(1)
    gold = torch.randint(0, n_passages, (n_queries,), generator=gq).tolist()
    queries = {"q%d" % i: "question about passage %d" % p for i, p in enumerate(gold)}
    Q = torch.stack([encode_query(p) for p in gold])                       # [n, Nq, 128] on the CPU, as the executor has it
    ranking = searcher._search_all_Q(queries, Q, k=max(ks), progress=False).todict()
    recall = {}
    for k in ks:
        hits = sum(gold[i] in [pid for pid, _, _ in ranking["q%d" % i][:k]] for i in range(n_queries))
        recall["Recall@%d" % k] = hits / n_queries
    if verbose:
        print("index:", path, "| passages:", n_passages, "| queries:", n_queries)
        print(recall)
    return recall, ranking, (path, Q, gold)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=20_000)
    ap.add_argument("--queries", type=int, default=64)
    a = ap.parse_args()
    run(a.passages, a.queries)
