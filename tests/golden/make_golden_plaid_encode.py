"""Generate the encode fixture of flmr_plaid_encode with the REFERENCE's own codec (build container only).

    python tests/golden/make_golden_plaid_encode.py

For nbits in {1, 2, 4, 8}: fp16-valued unit rows and centroids, bucket cutoffs as CollectionIndexer.
_compute_avg_residual takes them (quantiles of held-out residuals, collection_indexer.py:290-314), and what
ResidualCodec.compress (CPU branch, colbert/indexing/codecs/residual.py:169-222) writes for them: codes and packed
residuals.  The CPU branch keeps the residual in fp32 where the kernel rounds it to fp16 first, as the reference's
GPU branch does; ``straddle_<nbits>`` marks the rows where the two fall on different sides of a cutoff.
Output: tests/golden/plaid_encode.npz.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import import_reference  # noqa: E402  (same import shims)
import plaid_encode_oracle as E           # noqa: E402


def main():
    ColBERTConfig = import_reference()[0]
    from colbert.indexing.codecs.residual import ResidualCodec
    out = {}
    for nbits in (1, 2, 4, 8):
        g = torch.Generator().manual_seed(700 + nbits)
        n, K = 600, 300
        x = torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1).half()
        cents = torch.nn.functional.normalize(torch.randn(K, 128, generator=g), dim=-1).half()
        cfg = ColBERTConfig(nbits=nbits, dim=128, total_visible_gpus=0)
        c0 = ResidualCodec(config=cfg, centroids=cents.float(), avg_residual=None)
        heldout = x[torch.randperm(n, generator=g)[:500]].float()
        res = heldout - c0.lookup_centroids(c0.compress_into_codes(heldout, out_device="cpu"), out_device="cpu")
        q = torch.arange(0, 1 << nbits) * (1 / (1 << nbits))
        cutoffs = res.float().quantile(q[1:])
        weights = res.float().quantile(q + 0.5 / (1 << nbits))
        codec = ResidualCodec(config=cfg, centroids=cents.float(), avg_residual=0.0, bucket_cutoffs=cutoffs,
                              bucket_weights=weights)
        comp = codec.compress(x.float())
        codes = comp.codes.numpy().astype(np.int32)
        out.update({"x_%d" % nbits: x.numpy(), "centroids_%d" % nbits: cents.numpy(),
                    "cutoffs_%d" % nbits: cutoffs.numpy(), "codes_%d" % nbits: codes,
                    "residuals_%d" % nbits: comp.residuals.numpy(),
                    "straddle_%d" % nbits: E.straddle_rows(x.numpy(), cents.numpy(), codes, cutoffs.numpy())})
        print("nbits=%d: %d of %d rows straddle a cutoff" % (nbits, out["straddle_%d" % nbits].sum(), n))
    np.savez_compressed(os.path.join(HERE, "plaid_encode.npz"), **out)


if __name__ == "__main__":
    main()
