"""Switch a process that runs the reference (RA-VQA + its vendored ``colbert`` package) onto this path with
ONE call, before the executors are imported or after — every module global that IS one of the reference's
objects is rebound, so ``from colbert import Searcher`` made earlier is covered too:

    import ravqa_b200.integration as flmr_b200
    flmr_b200.patch_colbert()

What is replaced (reference -> here):

    colbert.Searcher / colbert.searcher.Searcher                         -> ravqa_b200.Searcher
        (third_party/ColBERT/colbert/searcher.py:22; callers src/executors/FLMR_executor.py:774-792,
         src/models/rag/rag_model_blip.py:297-301, 397)
    colbert.modeling.colbert.colbert_score                               -> modeling.colbert_score
        (colbert.py:268-286; reached through ColBERT.score, colbert.py:217-224, i.e. FLMR*.score:
         FLMR_executor.py:828-833, rag_model_blip.py:430-435, colbert.py:71-73)
    colbert.modeling.colbert.colbert_score_packed                        -> integration.colbert_score_packed
        (colbert.py:289-311; callers IndexScorer.score_pids, index_storage.py:176-182)
    ColBERT.compute_ib_loss_new                                          -> integration.compute_ib_loss_new
        (colbert.py:82-113: materialises [B, B*nway, Nd, Nq]; here one fused all-pairs launch)

    colbert.Indexer (opt-in: ``patch_colbert(indexer=True)``)            -> ravqa_b200.Indexer
        (indexer.py:16-84, caller FLMR_executor.py:601-617: flat bf16 store instead of the PLAID build)
    colbert.Indexer (opt-in: ``patch_colbert(indexer="plaid")``)         -> ravqa_b200.indexer.PlaidIndexer
        (the same call lines write a PLAID directory, built on the GPU: k-means, codes, residuals and IVF)

Nothing of the reference is modified on disk; ``unpatch_colbert()`` restores the originals.  Encoders, data
pipeline, executors and (unless opted out of as above) the PLAID index *build* stay the reference's own.
"""
from __future__ import annotations

import sys
from typing import Dict, List, Tuple

import torch

from .modeling import all_pairs_maxsim, colbert_score, in_batch_negatives_loss
from .searcher import Searcher

_undo: List[Tuple[object, str, object]] = []


def colbert_score_packed(Q, D_packed, D_lengths, config=None):
    """colbert.modeling.colbert.colbert_score_packed (colbert.py:289-311): ONE query ``Q [1, Nq, d]`` against
    ``D_packed [sum(D_lengths), d]``.  Returns ``[n]`` fp32 scores on the GPU.  The reference's CPU branch
    clamps every row maximum at 0 (segmented_maxsim.cpp:58-59) while its GPU branch takes the true maximum;
    ``config.total_visible_gpus == 0`` selects the clamped variant here too, so either branch is reproduced."""
    from .corpus import FlatCorpus
    from .maxsim import maxsim_scores
    if Q.dim() == 3:
        assert Q.size(0) == 1, Q.size()
        Q = Q.squeeze(0)
    assert Q.dim() == 2, Q.size()
    assert D_packed.dim() == 2, D_packed.size()
    if config is not None and getattr(config, "interaction", "colbert") == "flipr":
        # colbert.py:306-309: the 'flipr' reduction always takes the padded route; here: pad, then the arg-max
        # launch + selection of modeling.colbert_score
        lengths = torch.as_tensor(D_lengths).long().to(D_packed.device)
        n, nd = int(lengths.numel()), int(lengths.max())
        mask = torch.arange(nd, device=D_packed.device)[None, :] < lengths[:, None]
        D_padded = D_packed.new_zeros((n, nd, D_packed.size(1)))
        D_padded[mask] = D_packed[: int(lengths.sum())]
        return colbert_score(Q.unsqueeze(0), D_padded, mask.unsqueeze(-1), config=config)
    relu = config is not None and getattr(config, "total_visible_gpus", 1) == 0
    dev = torch.device("cuda", torch.cuda.current_device())
    corpus = FlatCorpus(D_packed.to(dev), torch.as_tensor(D_lengths).cpu(), device=dev)
    try:
        scores = maxsim_scores(corpus, Q.unsqueeze(0), relu=relu)[0].clone()
        torch.cuda.current_stream(dev).synchronize()
    finally:
        corpus.close()
    return scores


def compute_ib_loss_new(self, Q, D, D_mask):
    """ColBERT.compute_ib_loss_new (colbert.py:82-113) as a method replacement: in-batch scores
    ``[B, B*nway]`` from one fused all-pairs launch, positives at column ``i * nway`` (:103-108), the model's
    own ``loss_fn`` (cross-entropy, colbert.py:31)."""
    step = D.shape[0] // Q.shape[0]
    lf = getattr(self, "loss_fn", None)
    plain_ce = (isinstance(lf, torch.nn.CrossEntropyLoss) and lf.reduction == "mean" and lf.weight is None
                and lf.ignore_index == -100 and getattr(lf, "label_smoothing", 0.0) == 0.0)
    if plain_ce and Q.is_cuda and D.shape[0] == Q.shape[0] * step:
        return in_batch_negatives_loss(Q, D, D_mask, step)        # arg-max kernel + fused loss head
    scores = all_pairs_maxsim(Q, D, D_mask)
    labels = torch.arange(Q.shape[0], device=scores.device) * step
    return self.loss_fn(scores, labels)


def _rebind_everywhere(old, new) -> int:
    """Rebind every module-level name that currently refers to ``old``."""
    n = 0
    for mod in list(sys.modules.values()):
        d = getattr(mod, "__dict__", None)
        if not isinstance(d, dict):
            continue
        for name, val in list(d.items()):
            if val is old and val is not new:
                _undo.append((mod, name, old))
                setattr(mod, name, new)
                n += 1
    return n


def patch_colbert(searcher: bool = True, scoring: bool = True, ib_loss: bool = True, indexer=False
                  ) -> Dict[str, int]:
    """Install the replacements listed in the module docstring into the loaded ``colbert`` package (imports it
    if needed: ``third_party/ColBERT`` must be on ``sys.path`` as the reference arranges).  Returns how many
    module globals were rebound per replaced object.

    ``indexer=True`` (opt-in) also replaces ``colbert.Indexer`` (indexer.py:16, called at FLMR_executor.py:601-617)
    by ``ravqa_b200.Indexer``: same constructor and ``index(name, collection, overwrite)``, the reference's own
    ``Checkpoint`` as document encoder, but the embeddings are stored flat in bf16 — no k-means, residual codec or
    IVF — where the reference would put its PLAID directory; ``Searcher`` opens either kind.  ``indexer="plaid"``
    replaces it by ``indexer.PlaidIndexer`` instead, which writes the PLAID directory itself (``nbits`` from the
    config the executor passes), built on the GPU."""
    import colbert                                      # noqa: F401  (the reference's vendored package)
    import colbert.modeling.colbert as M
    import colbert.searcher as S
    done: Dict[str, int] = {}
    if indexer not in (False, True, "plaid"):
        raise ValueError("patch_colbert(indexer=...) takes False, True (flat store) or 'plaid', got %r" % (indexer,))
    if indexer:
        import colbert.indexer as IX
        from .indexer import Indexer, PlaidIndexer
        ours = PlaidIndexer if indexer == "plaid" else Indexer
        if IX.Indexer is not ours:
            done["Indexer"] = _rebind_everywhere(IX.Indexer, ours)
    if searcher and S.Searcher is not Searcher:
        done["Searcher"] = _rebind_everywhere(S.Searcher, Searcher)
    if scoring:
        if M.colbert_score is not colbert_score:
            done["colbert_score"] = _rebind_everywhere(M.colbert_score, colbert_score)
        if M.colbert_score_packed is not colbert_score_packed:
            done["colbert_score_packed"] = _rebind_everywhere(M.colbert_score_packed, colbert_score_packed)
    if ib_loss and M.ColBERT.compute_ib_loss_new is not compute_ib_loss_new:
        _undo.append((M.ColBERT, "compute_ib_loss_new", M.ColBERT.__dict__["compute_ib_loss_new"]))
        M.ColBERT.compute_ib_loss_new = compute_ib_loss_new
        done["ColBERT.compute_ib_loss_new"] = 1
    return done


def unpatch_colbert() -> None:
    while _undo:
        owner, name, old = _undo.pop()
        setattr(owner, name, old)
