"""H100-native (sm_90a) FLMR / ColBERT late-interaction MaxSim + top-k (the one hot path of RA-VQA this
repository accelerates).  Import name: ``ravqa_b200`` (the directory name carries hyphens)."""
from . import _cabi  # noqa: F401
from .corpus import FlatCorpus, allow_bitmaps  # noqa: F401
from .maxsim import maxsim_scores, maxsim_scores_listed, maxsim_topk, topk_merge, topk_select, debug_scores_simt  # noqa: F401

__all__ = ["FlatCorpus", "allow_bitmaps", "maxsim_scores", "maxsim_scores_listed", "maxsim_topk", "topk_merge", "topk_select",
           "debug_scores_simt"]
from .searcher import Searcher, Ranking  # noqa: F401,E402
from .sharded import ShardedSearcher, shard_ranges  # noqa: F401,E402
from .index_io import save_flat_index, load_flat_index  # noqa: F401,E402
from .indexer import Indexer  # noqa: F401,E402
from .updater import IndexUpdater  # noqa: F401,E402
from .modeling import (FLMRModelForRetrieval, all_pairs_maxsim, colbert_score, grouped_maxsim,  # noqa: F401,E402
                       graphed_in_batch_negatives_loss, in_batch_negatives_loss)
from .infra import ColBERTConfig, Queries, Run, RunConfig, resolve_index_path  # noqa: F401,E402

__all__ += ["Searcher", "Ranking", "ShardedSearcher", "shard_ranges", "save_flat_index", "load_flat_index", "Indexer", "IndexUpdater",
            "FLMRModelForRetrieval", "all_pairs_maxsim", "colbert_score", "grouped_maxsim",
            "in_batch_negatives_loss", "graphed_in_batch_negatives_loss", "ColBERTConfig", "Queries", "Run", "RunConfig", "resolve_index_path"]
