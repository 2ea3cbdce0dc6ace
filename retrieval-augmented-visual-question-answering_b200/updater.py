"""``IndexUpdater``: add passages to and remove passages from the index behind a live ``Searcher``, with the surface of
the updater later ColBERT releases ship (``IndexUpdater(config, searcher, checkpoint)`` with ``add`` / ``remove`` /
``persist_to_disk``; the ColBERT release the reference vendors has no update path).

    updater = IndexUpdater(config=config, searcher=searcher, checkpoint=checkpoint)   # or encode_fn=...
    new_pids = updater.add(["a new passage", ...])       # searchable as soon as add returns
    updater.remove([17, 42])                             # never returned again
    updater.persist_to_disk()                            # the flat index on disk catches up

The resident corpus grows in place (``FlatCorpus.append``) and deletions are tombstones tested inside the scan
(``FlatCorpus.delete``): no rebuild, no reload.  ``compact`` drops the deleted passages' rows from HBM and from the
scan.  Ids are stable: an added passage gets the next id, a removed one keeps its id and is never reused, compaction
moves rows but renumbers nothing; only a fresh ``Indexer`` build renumbers.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from .index_io import persist_updates, read_metadata

# passages gathered per step when persist_to_disk reads appended rows back out of the corpus
_PERSIST_BATCH = 4096


class IndexUpdater:
    def __init__(self, config=None, searcher=None, checkpoint=None, encode_fn: Optional[Callable] = None):
        if searcher is None:
            raise ValueError("IndexUpdater needs searcher=...: it updates the corpus that Searcher holds")
        if searcher._sharded is not None:
            raise NotImplementedError("updating a corpus sharded across ranks is not supported; update an unsharded "
                                      "Searcher and persist it, then load the index sharded")
        if searcher._devices is not None:
            raise NotImplementedError("updating a corpus sharded across devices (Searcher(devices=...)) is not "
                                      "supported; update a one-device Searcher and persist it, then load it sharded")
        if searcher.corpus is None:
            raise ValueError("the searcher holds no corpus")
        self.searcher = searcher
        self.config = config if config is not None else searcher.config
        self.checkpoint = checkpoint
        self.encode_fn = encode_fn

    @property
    def corpus(self):
        return self.searcher.corpus

    def _encoder(self) -> Callable:
        """``encode_fn`` if given, else the reference's document encoder, built by ``Indexer`` on first use."""
        if self.encode_fn is None:
            from .indexer import Indexer
            ckpt = self.checkpoint or self.searcher.checkpoint or getattr(self.searcher.index_config, "checkpoint", None)
            self.encode_fn = Indexer(checkpoint=ckpt, config=self.config)._reference_encode_fn()
        return self.encode_fn

    def add(self, passages: Sequence[str]) -> List[int]:
        """Encode ``passages`` and append them; returns their new ids.  A list ``searcher.collection`` is extended
        with them, so that id -> text keeps working."""
        passages = list(passages)
        if not passages:
            return []
        embs, doclens = self._encoder()(passages)
        pids = self.add_embeddings(torch.as_tensor(embs), doclens)
        if isinstance(self.searcher.collection, list):
            self.searcher.collection.extend(passages)
        return pids

    def add_embeddings(self, tokens: torch.Tensor, doclens) -> List[int]:
        """Append already encoded passages; returns their new ids.  ``tokens`` is either packed ``[sum(doclens), d]``
        (``docFromText(..., keep_dims='flatten')``) or padded ``[n, Nd, d]`` as ``ColBERT.doc`` returns it, passage
        i's tokens being its first ``doclens[i]`` rows."""
        doclens = np.asarray(doclens.detach().cpu() if isinstance(doclens, torch.Tensor) else doclens,
                             dtype=np.int32).reshape(-1)
        if tokens.dim() == 3:
            if tokens.size(0) != doclens.shape[0] or int(doclens.max(initial=0)) > tokens.size(1):
                raise ValueError("padded tokens [n, Nd, d] need n doclens of at most Nd")
            real = torch.arange(tokens.size(1), device=tokens.device)[None, :] < \
                torch.as_tensor(doclens, device=tokens.device)[:, None]
            tokens = tokens[real]
        return self.corpus.append(tokens, doclens).tolist()

    def remove(self, pids) -> None:
        """Delete passages by id: no search returns them again.  Every id must exist."""
        self.corpus.delete(pids)

    def compact(self) -> dict:
        """Remove the removed passages' rows from the resident corpus (``FlatCorpus.compact``): memory and scan time
        shrink, ids and search results stay as they are.  The index on disk is not rewritten: ``persist_to_disk``
        writes what it would have written without compaction."""
        return self.corpus.compact()

    def persist_to_disk(self) -> dict:
        """Write the updates to the flat index the searcher was opened on: appended passages as new chunks, the
        deleted ids as ``deleted.npy`` (format "flmr-flat-v2"), metadata.json last.  A passage that was added and
        removed again is written with zero rows of its length, so that every later id stays where it is."""
        s = self.searcher
        if s.index is None:
            raise ValueError("the searcher was given a resident corpus, not an index path: there is nothing to persist to")
        if s.index_kind != "flat":
            raise NotImplementedError("persisting updates to a %s index is not supported; the updates live in memory "
                                      "only (rebuild with Indexer to write a flat index)" % s.index_kind)
        corpus = self.corpus
        n_disk = int(read_metadata(s.index)["n_passages"])
        if corpus.n_passages < n_disk:
            raise ValueError("the index on disk holds %d passages, the corpus only %d" % (n_disk, corpus.n_passages))
        new_doclens = np.asarray(corpus.doclens[n_disk:], dtype=np.int32)
        parts = []
        for a in range(0, new_doclens.shape[0], _PERSIST_BATCH):
            dl = new_doclens[a:a + _PERSIST_BATCH]
            pids = torch.arange(n_disk + a, n_disk + a + dl.shape[0], dtype=torch.int64) + corpus.pid_base
            D, _ = corpus.gather_padded(pids, int(dl.max()))
            real = torch.arange(D.size(1), device=D.device)[None, :] < torch.as_tensor(dl, device=D.device)[:, None]
            parts.append(D[real].cpu())
        new_tokens = torch.cat(parts) if parts else None
        return persist_updates(s.index, new_tokens, new_doclens, corpus.deleted_pids() - corpus.pid_base)
