/*
 * flmr_maxsim.h — C ABI of the H100-native FLMR / ColBERT late-interaction MaxSim + top-k path.
 *
 * This is the drop-in boundary for the ONE hot path this repository accelerates
 * (SURVEY.md §8b).  The reference has no FFI registry for this path: it binds four pybind11
 * torch extensions and calls Python scoring functions.  Each entry point below names the
 * reference interface it replaces (paths relative to the reference checkout, `CB/` =
 * third_party/ColBERT/colbert/):
 *
 *   flmr_corpus_create / _destroy / _info
 *       replaces the PLAID index residency built by IndexScorer.__init__ / IndexLoader
 *       (CB/search/index_storage.py:21-66, CB/search/index_loader.py:13-86) and the packed
 *       `D_packed [sum(doclens), dim]` + `D_lengths` operand pair of colbert_score_packed
 *       (CB/modeling/colbert.py:289-311).
 *   flmr_maxsim_scores
 *       replaces colbert_score / colbert_score_reduce / colbert_score_packed
 *       (CB/modeling/colbert.py:235-311) and the native segmented_maxsim_cpp
 *       (CB/modeling/segmented_maxsim.cpp:49-93): all-passage MaxSim scores of each query.
 *   flmr_maxsim_topk
 *       replaces IndexScorer.rank (CB/search/index_storage.py:86-98: retrieve -> score_pids ->
 *       sort) as called per query from Searcher.dense_search (CB/searcher.py:91-132); exhaustive
 *       instead of PLAID-pruned, batched over queries, top-k fused into the scoring kernel.
 *   flmr_topk_merge
 *       the only exchange step of the sharded path (SURVEY.md §8e): merges per-shard top-k lists
 *       (gathered by the host with one NCCL all-gather) into the global top-k.
 *   flmr_topk_merge_devices
 *       the same exchange for shards one process holds on several devices: the merge kernel reads every shard's
 *       lists on the home device, through peer access, with no collective and no host synchronisation.
 *   FLMR_CORPUS_FP8, flmr_corpus_storage
 *       an e4m3 corpus: the scan reads half the bytes per token and runs fp8 MMAs, so its scores are
 *       APPROXIMATE; the exact bf16 rows stay in pinned host memory for flmr_corpus_gather.  The first stage of
 *       a two-stage search whose exact second stage re-scores a shortlist (the Python Searcher does both), as
 *       PLAID scores its ndocs/4 survivors exactly (CB/search/index_storage.py:160-177).
 *   FLMR_CORPUS_FP16, flmr_plaid_decode_fp16, flmr_maxsim_argmax_fp16 / _backward_fp16 (and _grouped_fp16)
 *       an fp16 corpus: the precision the reference keeps and scores its embeddings in (ColBERT.doc returns
 *       D.half(), colbert_score multiplies in D's dtype, CB/modeling/colbert.py:205-206, 284; the residual codec
 *       decodes to fp16, CB/indexing/codecs/residual.py:273), scanned with fp16 MMAs instead of being rounded to bf16;
 *       and the training / re-scoring calls on fp16 documents, with the query converted to fp16 as colbert_score does.
 *   flmr_corpus_append / _delete / _deleted
 *       the add / remove of ColBERT's later IndexUpdater (the vendored release has no update path): passages are
 *       appended to a resident shard in place and deleted ones are tombstoned, tested in the scan's reducer.
 *   flmr_corpus_compact / _stored
 *       drops the rows of deleted passages from HBM and from every later scan, keeping every id (a fresh index
 *       build is the reference's only way to shrink an index, and it renumbers the passages).
 *   flmr_maxsim_scores_allowed / flmr_maxsim_topk_allowed / flmr_maxsim_topk_sharded_allowed
 *       the pids= / qid_to_pids= restriction of later ColBERT Searchers: a per-query allow bitmap tested in the
 *       scan's reducer (the vendored release filters scores with filter_fn, CB/searcher.py:61-132).
 *   flmr_maxsim_topk_listed / flmr_maxsim_scores_listed
 *       the same restriction given as id lists, at the cost of the listed passages: the scan runs over a per-call
 *       plan of their rows (the reference's pipeline likewise scores only its candidates, CB/search/index_storage.py).
 *   flmr_corpus_create_streamed / flmr_corpus_builder_create_streamed / flmr_corpus_residency
 *       a corpus kept in pinned host memory and streamed through two HBM windows per search, for a shard that does not
 *       fit beside what the GPU already holds (the reference builds its validation Searcher inside the training
 *       process, src/executors/FLMR_executor.py:774-792).
 *   flmr_corpus_builder_create_plaid / flmr_corpus_builder_append_plaid / flmr_corpus_codec
 *       a streamed corpus kept in a PLAID index's compressed form (centroid codes and packed residuals) and decoded
 *       window by window on the GPU before the scan: 20 to 132 B of pinned host memory and PCIe traffic per token
 *       instead of 256.
 *   flmr_plaid_encode
 *       writes a PLAID index's codes and packed residuals: replaces ResidualCodec.compress_into_codes and compress
 *       (CB/indexing/codecs/residual.py:169-222), which materialise a [K, batch] score matrix and an [n, dim]
 *       residual matrix in HBM, by one wgmma kernel that keeps both in registers; its assignment-only mode is the
 *       assignment step of the k-means the Python Indexer runs instead of faiss.
 *   flmr_debug_maxsim_scores_simt
 *       test infrastructure: an independent plain-SIMT fp32 device kernel used by tests to
 *       cross-check the tensor-core kernel at sizes where the CPU oracle is too slow.
 *
 * Conventions (cf. SURVEY.md §8b "ownership / errors / threading"):
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary;
 *   - every function returns an int status (0 = FLMR_OK); no exceptions, aborts or asserts
 *     cross the boundary; flmr_last_error() returns a thread-local message for the last failure;
 *   - the caller owns every input and output buffer; "d_" parameters are DEVICE pointers on the
 *     corpus' device, "h_" parameters are HOST pointers;
 *   - compute entry points are asynchronous on the supplied CUDA stream (passed as void* so the
 *     header needs no CUDA include; NULL = default stream);
 *   - CUDA graph capture: flmr_maxsim_scores, flmr_maxsim_topk and their _allowed forms (every storage, compacted
 *     corpora included), flmr_topk_select, flmr_topk_merge, flmr_corpus_gather, flmr_maxsim_argmax /
 *     flmr_maxsim_backward with their _grouped and _fp16 forms (either arg-max kernel) and flmr_ib_loss and flmr_plaid_encode may be captured
 *     on the stream they are given and replayed with new contents in the same buffers, once a call of the same shape
 *     has run outside the capture on the same workspace (it sizes the workspace's buffers), and while the corpus does
 *     not change.  The _listed calls are not capturable: their host offsets size the plan when the call is made, and
 *     their host tables are copied then.  flmr_plaid_decode synchronises its stream and is not capturable either;
 *   - a corpus changes only through flmr_corpus_append, flmr_corpus_delete and flmr_corpus_compact.  Between
 *     those calls a handle may be shared by threads; concurrent searches on one handle must use distinct
 *     flmr_workspace handles.  The three mutating calls must not run concurrently with any other call on the
 *     handle or on its workspaces; they wait for the device themselves, so work already enqueued on any stream
 *     sees the corpus as it was.
 *   - ID EXTENT and SLOTS: a shard's ids are pid_base .. pid_base + n_passages, and n_passages (the id extent)
 *     never shrinks.  Every id-indexed argument and output (allow bitmaps and their stride, the score rows of
 *     flmr_maxsim_scores, deleted lists) is sized by the id extent.  The slots are the passages that still have
 *     rows: all of them until the first flmr_corpus_compact, afterwards the ones that were live when it ran plus
 *     those appended since.  The scan, its partition and the token matrices are indexed by slot.
 *   - a DELETED passage keeps its id (ids are never reused) and, until the next flmr_corpus_compact, its rows
 *     (they are still scanned); it yields -inf from flmr_maxsim_scores and flmr_debug_maxsim_scores_simt, never
 *     appears in the lists of flmr_maxsim_topk / flmr_maxsim_topk_sharded (short lists are filled with -1 / -inf),
 *     and flmr_corpus_gather returns an all-masked zero row for it, as for an id outside the shard.  A
 *     compacted-away id is a deleted id in every one of these respects.
 */
#ifndef FLMR_MAXSIM_H_
#define FLMR_MAXSIM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FLMR_ABI_VERSION 2

/* status codes */
#define FLMR_OK 0
#define FLMR_ERR_INVALID_ARG 1
#define FLMR_ERR_CUDA 2
#define FLMR_ERR_UNSUPPORTED 3
#define FLMR_ERR_OOM 4
#define FLMR_ERR_KERNEL 5 /* device-side watchdog / self-check tripped */

/* flags for flmr_maxsim_scores / flmr_maxsim_topk */
#define FLMR_FLAG_RELU 1u /* reproduce the reference CPU packed path: sum_i max(0, max_j s_ij)   \
                             (CB/modeling/segmented_maxsim.cpp:58-59 zero-initialises the max) */

/* flags for flmr_corpus_create */
#define FLMR_CORPUS_COPY 0u  /* always copy the token matrix into library-owned HBM            */
#define FLMR_CORPUS_ADOPT 1u /* tokens is a device pointer; keep it (zero-copy) when every     \
                                doclen is a multiple of FLMR_TOKEN_GROUP, else copy+repack     */
#define FLMR_CORPUS_FP8 2u   /* HBM holds the tokens as e4m3 (round to nearest even, saturated;  \
                                half the bytes); the library keeps a pinned host copy of the      \
                                exact bf16 rows.  Not combinable with FLMR_CORPUS_ADOPT.         */
#define FLMR_CORPUS_FP16 4u  /* HBM holds the tokens as fp16 (same bytes and layout as bf16; the  \
                                scan runs fp16 MMAs).  Combines with FLMR_CORPUS_ADOPT; not with  \
                                FLMR_CORPUS_FP8 (FLMR_ERR_INVALID_ARG).                          */

/*
 * INPUT ELEMENT TYPE (one rule for every call below): token rows and query rows arrive in the corpus' element
 * type.  An FLMR_CORPUS_FP16 corpus takes fp16 rows — the tokens of flmr_corpus_create, flmr_corpus_append,
 * flmr_corpus_builder_append(_file) and the d_q of every search call — and flmr_corpus_gather writes fp16 rows
 * from it.  A bf16 corpus and an FLMR_CORPUS_FP8 corpus take (and gather) bf16 rows.  The training calls
 * (flmr_maxsim_argmax, flmr_maxsim_backward and their _grouped forms) take no corpus: their name gives the type.
 * The plain names take bf16 d_q and d_docs, the _fp16 names fp16 ones; outputs are fp32 either way.  Where a comment
 * below says "bf16" for such an operand, it means this type.
 */

#define FLMR_DIM 128        /* embedding dim of FLMR / ColBERT (CB/infra/config/settings.py:101) */
#define FLMR_TOKEN_GROUP 4  /* passages are stored padded to a multiple of this many tokens     */
#define FLMR_MAX_K 128      /* largest k of the fused top-k                                     */
#define FLMR_TILE_TOKENS 96 /* passage tokens per streamed tile of the scan kernel              */

typedef struct flmr_corpus flmr_corpus_t;       /* resident passage-token shard            */
typedef struct flmr_workspace flmr_workspace_t; /* per-caller scratch (candidates, Q pad)  */
typedef struct flmr_comm flmr_comm_t;           /* this rank's end of the shard exchange   */
typedef struct flmr_corpus_builder flmr_corpus_builder_t; /* streaming index load          */

/* After flmr_corpus_compact n_passages and pid_base are unchanged (the id extent); n_tokens, n_rows, n_tiles and
 * hbm_bytes describe the stored corpus (the slots), and n_ctas = min(SMs, slots). */
typedef struct flmr_corpus_info {
  int64_t n_passages;     /* id extent: passages of this shard, deleted and compacted ones included */
  int64_t n_tokens;       /* real tokens (sum of doclens) of the stored passages              */
  int64_t n_rows;         /* stored rows (tokens incl. group padding)                         */
  int64_t pid_base;       /* global id of passage 0 of this shard                             */
  int32_t dim;            /* = FLMR_DIM                                                       */
  int32_t device;         /* CUDA device ordinal                                              */
  int32_t n_ctas;         /* persistent CTAs the scan kernel launches (= min(SMs, stored passages)) */
  int32_t adopted;        /* 1 if the token matrix is the caller's buffer (zero-copy)         */
  int64_t n_tiles;        /* passage-token tiles streamed per corpus pass                     */
  int64_t hbm_bytes;      /* bytes of HBM held by the handle (excluding an adopted matrix)    */
} flmr_corpus_info_t;

/* Thread-local description of the last error returned on this thread ("" if none). */
const char* flmr_last_error(void);

/* ABI version of the loaded library (== FLMR_ABI_VERSION it was built with). */
int flmr_abi_version(void);

/*
 * Create a resident corpus shard from a packed token matrix.
 *   tokens      bf16 [sum(h_doclens), dim] row-major, passage after passage.  Host or device
 *               pointer (detected); with FLMR_CORPUS_ADOPT it must be a device pointer on `device`
 *               that outlives the handle.
 *   h_doclens   int32 [n_passages], every entry >= 1 (a zero-length passage has no defined score
 *               on the reference's two paths, SURVEY.md §8a, and is rejected).
 *   pid_base    added to local passage indices in every returned id (shard offset, §8e).
 */
int flmr_corpus_create(const void* tokens, const int32_t* h_doclens, int64_t n_passages, int dim,
                       int device, int64_t pid_base, unsigned flags, flmr_corpus_t** out);
int flmr_corpus_destroy(flmr_corpus_t* corpus);
int flmr_corpus_info(const flmr_corpus_t* corpus, flmr_corpus_info_t* out);

/*
 * How the corpus stores its tokens: *storage = 0 (bf16 in HBM), 1 (FLMR_CORPUS_FP8: e4m3 in HBM, counted in
 * hbm_bytes, plus the bf16 master in pinned host memory, *host_bytes bytes; 0 for the other storages) or 2
 * (FLMR_CORPUS_FP16: fp16 in HBM).  Either output may be NULL.
 *
 * On an e4m3 corpus flmr_maxsim_scores, flmr_maxsim_topk and flmr_maxsim_topk_sharded compute MaxSim of e4m3(Q)
 * against e4m3(D) with fp32 accumulation (Q rounded to nearest even, no scale): APPROXIMATE scores (up to about 6e-3
 * relative on normalised embeddings), fit to shortlist candidates, not to rank them.  flmr_corpus_gather reads the
 * exact bf16 rows of the master, and flmr_debug_maxsim_scores_simt computes the e4m3 semantics.
 */
int flmr_corpus_storage(const flmr_corpus_t* corpus, int* storage, int64_t* host_bytes);

/*
 * Updating a resident corpus (replaces rebuilding and reloading it: the surface of ColBERT's IndexUpdater add /
 * remove).  Both calls are synchronous: they wait for the device before they free or swap anything and return when
 * the change is complete.  See the conventions above for what may run alongside them.
 *
 * flmr_corpus_append   passages behind the stored ones, of either storage.  tokens: packed bf16 rows
 *                      [sum(h_doclens), dim], host or device pointer (detected as in flmr_corpus_create); every
 *                      doclen >= 1.  The new passages get the ids pid_base + (old n_passages ...); *first_pid (may
 *                      be NULL) receives the first.  A library-owned matrix lives in a reserved virtual address
 *                      range and grows in place (no copy, no second matrix).  An adopted matrix is copied into
 *                      library memory by the first append, which then no longer references the caller's buffer.
 *                      The bf16 master of an FLMR_CORPUS_FP8 corpus is pinned host memory and is reallocated:
 *                      old and new master are held together for the copy.  A shard is limited to 2^31 passages
 *                      and 2^31 stored rows.
 * flmr_corpus_delete   tombstones the GLOBAL ids h_pids[0..n).  The whole list is checked first: an id outside the
 *                      shard gives FLMR_ERR_INVALID_ARG and nothing changes.  Deleting a deleted id does nothing.
 *                      The first delete allocates the shard's bitmap (1 bit per passage, counted in hbm_bytes).
 * flmr_corpus_deleted  *n_deleted = how many ids are deleted; if h_pids is not NULL it receives them (global,
 *                      ascending), capacity >= *n_deleted entries.
 * flmr_corpus_compact  removes the rows of every deleted passage from HBM and from every later scan.  No id changes
 *                      and no result changes: every call on the corpus returns bitwise what it returned before
 *                      (a passage's score does not depend on where it is stored, and the kept passages keep their
 *                      order, so ties still go to the lower id); only memory, time and the storage figures of
 *                      flmr_corpus_info change.  Each run of kept passages moves down by the rows removed before
 *                      it, in chunks of at most 256 MiB of rows, through a staging buffer of at most 256 MiB where a
 *                      chunk overlaps its own source: HBM never holds a second matrix.  Every whole piece of
 *                      physical memory (a matrix is mapped in pieces of at most 1 GiB) behind the new end is
 *                      unmapped and released; *bytes_released (may be NULL) counts those bytes, *n_removed (may be
 *                      NULL) the passages removed.  An adopted matrix is never written: its live rows are copied
 *                      into a library-owned matrix, and the caller's buffer is no longer referenced.  The pinned
 *                      bf16 master of an FLMR_CORPUS_FP8 corpus is compacted in place and keeps its allocation until
 *                      the next append reallocates it.  A later append continues the ids from the id extent; a later
 *                      delete of a compacted-away id does nothing.  With no deleted rows stored the call does
 *                      nothing; when every stored passage is deleted it returns FLMR_ERR_INVALID_ARG and changes
 *                      nothing.  Synchronous, like append and delete.
 * flmr_corpus_stored   *n_stored_passages = the slots (passages with rows); *mapped_device_bytes = physical device
 *                      memory mapped behind the library-owned token matrices (0 for an adopted one).  Either output
 *                      may be NULL.
 */
int flmr_corpus_append(flmr_corpus_t* corpus, const void* tokens, const int32_t* h_doclens, int64_t n_passages,
                       int64_t* first_pid);
int flmr_corpus_delete(flmr_corpus_t* corpus, const int64_t* h_pids, int64_t n);
int flmr_corpus_deleted(const flmr_corpus_t* corpus, int64_t* n_deleted, int64_t* h_pids, int64_t capacity);
int flmr_corpus_compact(flmr_corpus_t* corpus, int64_t* n_removed, int64_t* bytes_released);
int flmr_corpus_stored(const flmr_corpus_t* corpus, int64_t* n_stored_passages, int64_t* mapped_device_bytes);

/*
 * Streaming construction of a corpus shard — the index LOAD path (replaces IndexLoader / ResidualEmbeddings.load_chunks,
 * CB/search/index_loader.py:24-62, CB/indexing/codecs/residual_embeddings.py:24-69): the padded token matrix is
 * allocated once from the doclens, then packed bf16 rows arrive IN ORDER, in chunks of any size, from host memory
 * or straight from a file, through two pinned staging buffers (the host fill of one overlaps the DMA of the
 * other; the file variant preads into pinned memory with 8 threads — no intermediate host copy).  If every
 * doclen is a multiple of FLMR_TOKEN_GROUP the rows are copied straight into place, else a scatter kernel puts
 * them into the padded layout.  finish() synchronises, builds the partition metadata and hands over the corpus
 * (the builder is destroyed); *host_fill_seconds (may be NULL) = host time spent reading / copying into the
 * staging buffers.  destroy() abandons a build.
 */
int flmr_corpus_builder_create(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                               int64_t pid_base, flmr_corpus_builder_t** out);
/* The same with corpus flags: FLMR_CORPUS_FP8 builds an e4m3 corpus (the staged rows fill the bf16 master and
 * HBM receives e4m3); FLMR_CORPUS_FP16 an fp16 corpus (the rows appended are fp16); 0 is
 * flmr_corpus_builder_create. */
int flmr_corpus_builder_create_ex(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                  int64_t pid_base, unsigned flags, flmr_corpus_builder_t** out);
int flmr_corpus_builder_append(flmr_corpus_builder_t* b, const void* h_tokens_bf16, int64_t n_rows);
int flmr_corpus_builder_append_file(flmr_corpus_builder_t* b, const char* path, int64_t byte_offset, int64_t n_rows);
int flmr_corpus_builder_finish(flmr_corpus_builder_t* b, flmr_corpus_t** out, double* host_fill_seconds);
int flmr_corpus_builder_destroy(flmr_corpus_builder_t* b);

/*
 * A STREAMED corpus: the padded token rows live in a library-owned pinned host matrix (cudaHostAllocMapped |
 * cudaHostAllocPortable) instead of HBM, so a shard may be larger than the memory a GPU has free — a corpus searched
 * beside a training run, or one larger than the card.  At creation the slots are cut into WINDOWS: contiguous slot
 * ranges whose stored rows fit window_bytes, each with its own CTA partition (row starts relative to the window,
 * slots and ids absolute).  Each workspace holds two window buffers of the largest window's rows (one when the plan
 * has one window) and a copy stream of
 * its own; a search streams the corpus ONCE: window w is copied into buffer w % 2 while the scans of window w - 1 run,
 * the scans of window w wait for its copy, and the copy of window w + 2 waits for the scans of window w.  Every call
 * chunk is scanned over each window in turn and its running top-k merged with the window's per-CTA lists.  Everything
 * is asynchronous on the caller's stream, with no host synchronisation.  The scan kernels, their fold and reducer are
 * the resident corpus's, so every result is bitwise the one a resident corpus of the same rows returns.
 *
 * flmr_corpus_create_streamed   as flmr_corpus_create (tokens host or device, bf16, or fp16 with FLMR_CORPUS_FP16),
 *                               plus window_bytes (>= one row).  FLMR_CORPUS_FP8, FLMR_CORPUS_ADOPT and a window
 *                               smaller than the longest passage's stored rows give FLMR_ERR_UNSUPPORTED.
 * flmr_corpus_builder_create_streamed   the index-load builder of a streamed corpus: flmr_corpus_builder_append(_file)
 *                               read rows straight into the pinned matrix (through one pinned staging buffer when
 *                               passages need padding), with no device copy; finish plans the windows.
 * flmr_corpus_residency         *streamed = 1 for a streamed corpus (0 otherwise), *window_bytes its window_bytes and
 *                               *host_bytes its pinned matrix (0 and 0 for a resident corpus).  Any output may be NULL.
 *
 * On a streamed corpus flmr_maxsim_scores, flmr_maxsim_topk, their _allowed forms, flmr_maxsim_topk_sharded(_allowed),
 * flmr_corpus_delete / _deleted, flmr_corpus_gather and flmr_debug_maxsim_scores_simt work as on a resident one (the
 * gather and the SIMT kernel read the mapped host rows); flmr_corpus_info's hbm_bytes counts no token rows.
 * flmr_corpus_append, flmr_corpus_compact, the _listed calls and flmr_debug_listed_plan return FLMR_ERR_UNSUPPORTED and
 * change nothing.  Searches on a streamed corpus are not capturable in a CUDA graph.
 */
int flmr_corpus_create_streamed(const void* tokens, const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                int64_t pid_base, unsigned flags, int64_t window_bytes, flmr_corpus_t** out);
int flmr_corpus_builder_create_streamed(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                        int64_t pid_base, unsigned flags, int64_t window_bytes,
                                        flmr_corpus_builder_t** out);
int flmr_corpus_residency(const flmr_corpus_t* corpus, int* streamed, int64_t* window_bytes, int64_t* host_bytes);

/*
 * A PLAID-CODED streamed corpus: a streamed corpus that keeps a PLAID index's compressed form in pinned host memory,
 * a 4-byte centroid code and 16 * nbits bytes of packed residual per stored row, instead of 256-byte rows.  Each search
 * copies a window's codes and residuals and decodes them on the GPU into one HBM window buffer, which the unchanged
 * scan kernels read.  Decoding does exactly what flmr_plaid_decode (normalize = 1), or flmr_plaid_decode_fp16 with
 * FLMR_CORPUS_FP16, does to each row, so every result is bitwise that of a resident corpus of those decoded rows.
 *
 * flmr_corpus_builder_create_plaid   as flmr_corpus_builder_create_streamed, plus the codec: nbits (1, 2, 4 or 8),
 *                               the fp32 centroids [n_centroids, 128] and the fp32 bucket weights [2^nbits] (host
 *                               pointers, copied).  window_bytes bounds a window's DECODED rows (256 B each).  Refusals,
 *                               in this order: window_bytes < one row (FLMR_ERR_INVALID_ARG), flags other than
 *                               FLMR_CORPUS_FP16 (FLMR_ERR_UNSUPPORTED), dim != 128 (FLMR_ERR_UNSUPPORTED), no passage
 *                               or null doclens, nbits outside {1, 2, 4, 8}, null tables or n_centroids < 1
 *                               (FLMR_ERR_INVALID_ARG), a passage longer than a window (FLMR_ERR_UNSUPPORTED).
 * flmr_corpus_builder_append_plaid   the next n_rows packed token rows, in order and in any split: codes int32 [n_rows]
 *                               and residuals uint8 [n_rows, 16 * nbits], as an index's chunks hold them.  The library
 *                               stores them in the padded row layout (each passage's last row repeated up to a multiple
 *                               of 4 rows).  A code outside [0, n_centroids) gives FLMR_ERR_INVALID_ARG and stores
 *                               nothing.  flmr_corpus_builder_append(_file) refuse this builder, and this call any other
 *                               (FLMR_ERR_INVALID_ARG).  flmr_corpus_builder_finish copies the tables to HBM (counted in
 *                               hbm_bytes) and plans the windows; flmr_corpus_builder_destroy abandons the build.
 * flmr_corpus_codec             *nbits = the codec's bits of a PLAID-coded corpus, 0 for any other corpus.
 *
 * Each workspace holds one decoded window buffer and two staging buffers of compressed rows (one of each for a
 * one-window plan).  A search copies window w's compressed rows into staging buffer w % 2 on the workspace's copy stream;
 * the caller's stream waits for that copy and decodes the window, and the copy of window w + 2 waits for that decode.
 * On this corpus flmr_corpus_residency gives *streamed = 1 and *host_bytes = its compressed arrays; the calls that work
 * on a streamed corpus work, flmr_corpus_gather decodes the requested rows from the mapped host arrays (and stays
 * capturable), and flmr_debug_maxsim_scores_simt returns FLMR_ERR_UNSUPPORTED, as do the calls a streamed corpus refuses.
 */
int flmr_corpus_builder_create_plaid(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                     int64_t pid_base, unsigned flags, int64_t window_bytes, int nbits,
                                     const float* h_centroids, int64_t n_centroids, const float* h_bucket_weights,
                                     flmr_corpus_builder_t** out);
int flmr_corpus_builder_append_plaid(flmr_corpus_builder_t* b, const int32_t* h_codes, const uint8_t* h_residuals,
                                     int64_t n_rows);
int flmr_corpus_codec(const flmr_corpus_t* corpus, int* nbits);

/* Scratch for searches on `corpus`.  max_queries (>= 1) sizes the per-CTA candidate buffer: a call with more
 * queries is processed in chunks of max_queries (each chunk: its scan passes + ONE merge launch).  max_nq
 * (>= 1) is the longest query expected: if it exceeds the 384 rows one pass holds, the partial-score rows of
 * row-sliced queries are allocated here instead of inside the first such search (longer queries still work,
 * the buffer then grows on demand). */
int flmr_workspace_create(const flmr_corpus_t* corpus, int max_queries, int max_nq,
                          flmr_workspace_t** out);
int flmr_workspace_destroy(flmr_workspace_t* ws);
/* Device-side watchdog code of the last scan on this workspace (0 = none; 101 producer, 102 MMA
 * issuer, 103 epilogue starved).  Readable even after the launch trapped. */
int flmr_workspace_status(const flmr_workspace_t* ws, int* out);

/*
 * MaxSim scores of every passage for each of n_queries queries.
 *   d_q          bf16 [n_queries, nq, dim] (rows L2-normalised by the encoder; all-zero rows allowed
 *                and contribute exactly 0, as in the reference)
 *   d_out_scores fp32 [n_queries, n_passages]:  out[b][p] = sum_i max_{j<len_p} <Q_b,i , D_p,j>
 */
int flmr_maxsim_scores(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q,
                       int n_queries, int nq, unsigned flags, float* d_out_scores, void* stream);

/*
 * Fused MaxSim + top-k: the k best passages of each query, sorted by descending score
 * (ties: ascending id).  No score matrix is written to HBM when nq fits one resident query tile.
 *   d_out_scores fp32  [n_queries, k]
 *   d_out_pids   int64 [n_queries, k]  (pid_base + local index; -1 / -inf fill if n_passages < k)
 */
int flmr_maxsim_topk(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q,
                     int n_queries, int nq, int k, unsigned flags, float* d_out_scores,
                     int64_t* d_out_pids, void* stream);

/*
 * Restricted search: each query is scored against its own set of passages (the pids= / qid_to_pids= of later
 * ColBERT Searchers: re-ranking a first stage's candidates, one entity's or tenant's passages, a training query
 * without its positives).  The restriction is tested inside the scan's reducer, so no score matrix is written.  The
 * _allowed calls take bitmaps and stream the whole shard: they cost what an unrestricted search does.  The _listed
 * calls (below) take id lists and stream only the listed passages' rows.
 *   d_allow             uint32 device bitmaps, one per query: bit p & 31 of word p >> 5 set <=> query b may return
 *                       LOCAL passage p (global id pid_base + p).  Query b's bitmap starts at
 *                       d_allow + b * allow_stride_words.  Bits at or beyond n_passages are ignored.
 *   allow_stride_words  0 (every query uses the one bitmap at d_allow) or >= ceil(n_passages / 32); any other value
 *                       gives FLMR_ERR_INVALID_ARG.  d_allow == NULL is the unrestricted call.
 * A bitmap describes the shard as it is at call time: after flmr_corpus_append a bitmap must be rebuilt (with the
 * new stride) to reach the new passages.  A disallowed pair behaves like a deleted passage for that query only: -inf
 * from flmr_maxsim_scores_allowed; never in the lists of the two top-k calls, which are filled with (-inf, -1) when
 * fewer than k passages are allowed and live.  Allowed scores are bitwise those of the unrestricted call.
 * flmr_maxsim_topk_sharded_allowed (see below) takes each rank's bitmaps of its own shard.
 */
int flmr_maxsim_scores_allowed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries,
                               int nq, unsigned flags, const uint32_t* d_allow, int64_t allow_stride_words,
                               float* d_out_scores, void* stream);
int flmr_maxsim_topk_allowed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries,
                             int nq, int k, unsigned flags, const uint32_t* d_allow, int64_t allow_stride_words,
                             float* d_out_scores, int64_t* d_out_pids, void* stream);

/*
 * Restricted search over id lists, at the cost of the listed passages: the same scan kernel runs over a per-call plan
 * of the listed passages' rows only, re-balanced over the persistent CTAs (the planner runs on the device, in stream
 * order, without a host synchronisation).  The fold and the reducer are those of every other scan, so results are
 * bitwise those of the _allowed calls for bitmaps of the same sets.  The host tables of a call (h_list_offsets and the
 * pass plan of each call chunk) are copied when the call is made, so h_list_offsets may be reused as soon as the call
 * returns.  The first call whose plan outgrows the workspace's plan buffer waits for the device (the buffer is
 * reallocated).  These calls cannot be captured in a CUDA graph.
 *   h_list_offsets  HOST int64 [n_queries + 1], non-decreasing: query b's list is
 *                   d_list_pids[h_list_offsets[b] .. h_list_offsets[b + 1])
 *   d_list_pids     DEVICE int64 GLOBAL ids (pid_base + local id), in any order, duplicates allowed.  Ids outside this
 *                   shard are ignored (every rank of a sharded search may pass the same lists); deleted and
 *                   compacted-away ids are never returned.
 * flmr_maxsim_topk_listed    = flmr_maxsim_topk_allowed for bitmaps of the same sets: the same (score, id) lists, ties
 *                              to the lower id, (-inf, -1) fill when fewer than k listed passages are live.
 * flmr_maxsim_scores_listed  d_out_scores fp32 [h_list_offsets[n_queries]], aligned with d_list_pids (entry i at
 *                              index i): the flmr_maxsim_scores_allowed score of the pair; -inf for an id outside the
 *                              shard, deleted or compacted away.
 * Scan variants 3 and 4 have no plan-mode kernel (FLMR_ERR_UNSUPPORTED).
 */
int flmr_maxsim_topk_listed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries, int nq,
                            int k, unsigned flags, const int64_t* h_list_offsets, const int64_t* d_list_pids,
                            float* d_out_scores, int64_t* d_out_pids, void* stream);
int flmr_maxsim_scores_listed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries,
                              int nq, unsigned flags, const int64_t* h_list_offsets, const int64_t* d_list_pids,
                              float* d_out_scores, void* stream);

/*
 * Merge n_lists candidate lists per query into one top-k (the post-all-gather step of the
 * sharded path).  Entries with pid < 0 are ignored.
 *   d_in_scores fp32  [n_lists, n_queries, k_in]     d_in_pids int64 [n_lists, n_queries, k_in]
 *   d_out_*           [n_queries, k_out], k_out <= FLMR_MAX_K, n_lists * k_in <= 20480
 */
int flmr_topk_merge(const float* d_in_scores, const int64_t* d_in_pids, int n_lists, int n_queries,
                    int k_in, int k_out, float* d_out_scores, int64_t* d_out_pids, int device,
                    void* stream);

/*
 * The exchange of shards held by ONE process on several devices: merge lists that live on different devices into
 * one top-k on the device of `stream` (the home device), in flmr_topk_merge's order (score descending, then the lower
 * pid on exact ties; pid < 0 marks an empty entry; short results end in (-inf, -1)).
 *   d_scores[i] fp32 / d_pids[i] int64 [n_queries, k_in]: list i, on device devices[i], written by work on
 *   src_streams[i] (a cudaStream_t of devices[i]; NULL = that device's default stream)
 *   d_out_*  [n_queries, k_out] on the home device; k_out <= FLMR_MAX_K, k_out <= n_lists * k_in,
 *   n_lists * k_in <= 20480, n_lists <= 128 (FLMR_ERR_UNSUPPORTED above either)
 * Asynchronous: an event recorded on each source stream is waited for on `stream`, and the host never waits.  One
 * kernel on the home device reads each list where it lives: in place on the home device, through peer access where
 * cudaDeviceCanAccessPeer allows it (enabled by the first call for each device pair), else after a
 * cudaMemcpyPeerAsync into a stream-ordered staging buffer on the home device.  A device may hold several lists.
 * Argument errors (null arrays or lists, the shapes above) are refused before any CUDA call.
 */
int flmr_topk_merge_devices(const float* const* d_scores, const int64_t* const* d_pids, const int* devices,
                            void* const* src_streams, int n_lists, int n_queries, int k_in, int k_out,
                            float* d_out_scores, int64_t* d_out_pids, void* stream);

/*
 * The sharded search at the C boundary (SURVEY.md 8e; the reference has no counterpart: under DDP every rank
 * repeats the whole CPU search, src/executors/FLMR_executor.py:778-781).  Each rank holds a contiguous passage
 * shard (flmr_corpus_create with its pid_base); ONE exchange step — an NCCL all-gather of every rank's [B, k]
 * (score, pid) lists — then the merge kernel, all asynchronous on `stream`, no host synchronisation, so a
 * non-Python host can run the multi-GPU path.  NCCL is dlopen'ed at run time (the process's own copy if it has
 * loaded one); without it these calls return FLMR_ERR_UNSUPPORTED.
 *
 *   flmr_comm_unique_id   rank 0 obtains the 128-byte NCCL id and hands it to the other ranks (any host channel)
 *   flmr_comm_create      collective: ncclCommInitRank on `device`
 *   flmr_comm_adopt       wrap an existing ncclComm_t (not destroyed with the handle)
 *   flmr_topk_exchange    all-gather + merge of lists the caller already has (d_scores / d_pids [n_queries, k_in],
 *                         entries with pid < 0 ignored) -> [n_queries, k_out] on EVERY rank
 *   flmr_maxsim_topk_sharded   flmr_maxsim_topk on this rank's shard + flmr_topk_exchange, one call
 *   flmr_maxsim_topk_sharded_allowed   the same with flmr_maxsim_topk_allowed: every rank passes the bitmaps of its
 *                         own shard (indexed by local passage)
 */
int flmr_comm_unique_id(void* out_id_128_bytes);
int flmr_comm_create(const void* id_128_bytes, int rank, int world_size, int device, flmr_comm_t** out);
int flmr_comm_adopt(void* nccl_comm, int device, flmr_comm_t** out);
int flmr_comm_destroy(flmr_comm_t* comm);
int flmr_comm_info(const flmr_comm_t* comm, int* rank, int* world_size);
int flmr_topk_exchange(flmr_comm_t* comm, const float* d_scores, const int64_t* d_pids, int n_queries, int k_in,
                       int k_out, float* d_out_scores, int64_t* d_out_pids, void* stream);
int flmr_maxsim_topk_sharded(const flmr_corpus_t* corpus, flmr_workspace_t* ws, flmr_comm_t* comm, const void* d_q,
                             int n_queries, int nq, int k, unsigned flags, float* d_out_scores,
                             int64_t* d_out_pids, void* stream);
int flmr_maxsim_topk_sharded_allowed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, flmr_comm_t* comm,
                                     const void* d_q, int n_queries, int nq, int k, unsigned flags,
                                     const uint32_t* d_allow, int64_t allow_stride_words, float* d_out_scores,
                                     int64_t* d_out_pids, void* stream);

/*
 * Top-k of dense score rows for k beyond FLMR_MAX_K (Searcher.dense_search accepts any k,
 * CB/searcher.py:91-132; replaces the `scores.sort(descending=True)[:k]` of IndexScorer.rank):
 * radix select + order-preserving compaction + bitonic sort, one block per query.
 *   d_scores fp32 [n_queries, n] (e.g. from flmr_maxsim_scores), k <= 2048, ties -> lower id first;
 *   outputs as flmr_maxsim_topk (pid = pid_base + column; -inf / -1 fill when n < k).
 */
int flmr_topk_select(const float* d_scores, int n_queries, int64_t n, int k, int64_t pid_base,
                     float* d_out_scores, int64_t* d_out_pids, int device, void* stream);

/*
 * Decode a chunk of a PLAID (ColBERTv2 residual-compressed) index into bf16 token embeddings,
 * so existing reference indexes can be scanned without re-encoding.  Replaces
 * decompress_residuals_cpp (CB/search/decompress_residuals.cpp:80-155), its CUDA twin
 * (CB/indexing/codecs/decompress_residuals.cu:8-75) and the F.normalize that follows
 * (CB/search/index_storage.py:173).  Synchronous on `stream` (validates the centroid codes).
 *   d_codes      int32 [n_tokens]            nearest-centroid id per token   (<c>.codes.pt)
 *   d_residuals  uint8 [n_tokens, dim*nbits/8] packed bucket indices         (<c>.residuals.pt)
 *   d_centroids  fp32  [n_centroids, dim]    (centroids.pt, upcast)
 *   d_bucket_weights fp32 [2^nbits]          (buckets.pt[1])
 *   d_out_bf16   bf16  [n_tokens, dim]       = normalize(centroids[code] + weights[idx]) if normalize
 */
int flmr_plaid_decode(const int32_t* d_codes, const uint8_t* d_residuals, int64_t n_tokens,
                      const float* d_centroids, int64_t n_centroids, const float* d_bucket_weights,
                      int nbits, int dim, int normalize, void* d_out_bf16, int device, void* stream);
/* The same decode into fp16 (d_out_fp16 fp16 [n_tokens, dim]): computed in fp32, normalised, rounded once to fp16
 * (nearest even), as the bf16 output is rounded to bf16 — the rows an FLMR_CORPUS_FP16 corpus takes. */
int flmr_plaid_decode_fp16(const int32_t* d_codes, const uint8_t* d_residuals, int64_t n_tokens,
                           const float* d_centroids, int64_t n_centroids, const float* d_bucket_weights,
                           int nbits, int dim, int normalize, void* d_out_fp16, int device, void* stream);

/*
 * Encode token embeddings against PLAID centroids: what ResidualCodec.compress computes (CB/indexing/codecs/
 * residual.py:169-222), with neither its score matrix nor its residual matrix ever written.  Asynchronous on `stream`,
 * no host synchronisation, capturable in a CUDA graph.
 *   d_x          fp16  [n, 128]              token embeddings (16-byte aligned)
 *   d_centroids  fp16  [K, 128]              (centroids.pt; 16-byte aligned)
 *   d_cutoffs    fp32  [2^nbits - 1]         non-decreasing bucket cutoffs (buckets.pt[0]); NULL when d_residuals is
 *   d_codes      int32 [n]                   argmax_c <x_t, C_c>, fp32 accumulation, the lowest c on exact ties
 *   d_residuals  uint8 [n, 16 * nbits]       or NULL (assignment only; 4-byte aligned): with r = fp16(float(x_t) -
 *                                            float(C_code)) per dim and bucket = #{j : cutoffs[j] < float(r)}, bit j
 *                                            of dim d's bucket is element d * nbits + j of the row's bit string,
 *                                            packed MSB-first (np.packbits): flmr_plaid_decode (normalize = 0) of
 *                                            the output is C_code + bucket_weights[bucket] exactly
 *   d_best       fp32  [n]                   the winning score, or NULL
 * Refused before any CUDA call: a null d_x / d_centroids / d_codes, or d_residuals without d_cutoffs, nbits not in
 * {1, 2, 4, 8}, K < 1, n < 0 and misaligned pointers (FLMR_ERR_INVALID_ARG); n >= 2^31 - 256 (FLMR_ERR_UNSUPPORTED).
 * n == 0 does nothing.
 */
int flmr_plaid_encode(const void* d_x, int64_t n, const void* d_centroids, int K, const float* d_cutoffs, int nbits,
                      int32_t* d_codes, uint8_t* d_residuals, float* d_best, int device, void* stream);

/*
 * Gather retrieved passages out of the resident corpus into a padded batch — the operand of the RAG
 * re-score (src/models/rag/rag_model_blip.py:414-435 looks the embeddings up in a host dictionary, stacks
 * them and copies them to the device for every query; here they never leave HBM).
 *   d_pids   int64 [n_pids] GLOBAL passage ids (pid_base-relative ids are derived inside); ids outside
 *            this shard (e.g. the -1 fill of a short result list) produce an all-masked, zero row.
 *   d_out    bf16  [n_pids, nd_max, FLMR_DIM]  tokens, zero-padded; passages longer than nd_max are cut
 *   d_mask   uint8 [n_pids, nd_max]            1 for real tokens (may be NULL)
 * Asynchronous on `stream`.
 */
int flmr_corpus_gather(const flmr_corpus_t* corpus, const int64_t* d_pids, int64_t n_pids, int nd_max,
                       void* d_out_bf16, uint8_t* d_mask, void* stream);

/*
 * Backward of the all-pairs MaxSim used in training and RAG re-scoring (SURVEY.md 8f-2).  The
 * reference differentiates colbert_score through torch autograd (CB/modeling/colbert.py:235-286,
 * callers colbert.py:64-113 and src/models/rag/rag_model_blip.py:430-437), keeping the [n, Nd, Nq]
 * score tensor alive; here nothing is kept by the forward and the winners are recomputed:
 *
 * flmr_maxsim_argmax:   d_argmax[b, p, i] = argmax_{j : d_mask[p, j] != 0} <Q[b, i], D[p, j]>
 *                       (index into the PADDED document, lowest j on ties, -1 if p is fully masked);
 *                       d_rowmax (optional, fp32, same shape) receives the maximum itself: summed over i it
 *                       is score[b, p], so for a training-sized batch this one launch is the forward AND
 *                       saves what the backward needs (4 B per pair instead of the Nd scores).
 *                       Two kernels behind it: a warp-MMA one for small batches (a RAG re-score of 5 passages) and,
 *                       from 16M (query row, token) pairs up, a wgmma one (documents compacted to their unmasked
 *                       tokens, then a TMA / wgmma pipeline with the query tile stationary).
 * flmr_maxsim_backward: given d_grad[b, p] = dLoss/dScore[b, p],
 *                         d_dq[b, i, :]                  = sum_p grad[b, p] * D[p, argmax[b, p, i], :]
 *                         d_dd[p, argmax[b, p, i], :]   += grad[b, p] * Q[b, i, :]      (d_dd zeroed first)
 *                       either output may be NULL.  d_dd is accumulated with fp32 atomics.
 *   d_q     bf16 [n_queries, nq, FLMR_DIM]        d_docs bf16 [n_docs, nd, FLMR_DIM] (padded, contiguous)
 *   d_mask  uint8 [n_docs, nd] (any pattern, e.g. the punctuation mask of ColBERT.doc)
 *   d_argmax int32 [n_queries, n_docs, nq]        d_dq fp32 [n_queries, nq, FLMR_DIM]
 *   d_dd    fp32 [n_docs, nd, FLMR_DIM]
 * Asynchronous on `stream`; all pointers are device pointers on `device`.
 */
int flmr_maxsim_argmax(const void* d_q, int n_queries, int nq, const void* d_docs,
                       const uint8_t* d_mask, int n_docs, int nd, int32_t* d_argmax, float* d_rowmax,
                       int device, void* stream);
int flmr_maxsim_backward(const void* d_q, int n_queries, int nq, const void* d_docs, int n_docs, int nd,
                         const int32_t* d_argmax, const float* d_grad, float* d_dq, float* d_dd,
                         int device, void* stream);
/* The same two calls on fp16 d_q and d_docs (the reference's fp16 documents, CB/modeling/colbert.py:205-206, with the
 * query converted to their type, :284): fp16 MMAs and loads, fp32 accumulation and outputs, the same kernels'
 * structure, arguments and errors. */
int flmr_maxsim_argmax_fp16(const void* d_q, int n_queries, int nq, const void* d_docs,
                            const uint8_t* d_mask, int n_docs, int nd, int32_t* d_argmax, float* d_rowmax,
                            int device, void* stream);
int flmr_maxsim_backward_fp16(const void* d_q, int n_queries, int nq, const void* d_docs, int n_docs, int nd,
                              const int32_t* d_argmax, const float* d_grad, float* d_dq, float* d_dd,
                              int device, void* stream);

/*
 * The loss head of ColBERT.compute_ib_loss_new (CB/modeling/colbert.py:82-113) on top of flmr_maxsim_argmax's
 * d_rowmax: scores[b, p] = sum_i rowmax[b, p, i]; cross-entropy of row b against the positive at column
 * label0 + b * nway (colbert.py:103-111; label0 = rank * B * nway with cross-rank negatives); and its gradient,
 * one launch instead of torch's sum + log_softmax + nll_loss and their backward kernels:
 *   d_scores fp32 [n_queries, n_docs]     d_loss_per_query fp32 [n_queries] (the loss is their mean)
 *   d_dscores fp32 [n_queries, n_docs] = d mean-loss / d scores — the d_grad operand of flmr_maxsim_backward
 */
int flmr_ib_loss(const float* d_rowmax, int n_queries, int n_docs, int nq, int nway, int label0,
                 float* d_scores, float* d_loss_per_query, float* d_dscores, int device, void* stream);

/*
 * Block-diagonal ("aligned") form of the two calls above: query b meets only ITS docs_per_query documents,
 * d_docs[b * docs_per_query .. (b + 1) * docs_per_query).  This is ColBERT.score(Q.repeat_interleave(nway), D,
 * D_mask) (CB/modeling/colbert.py:71-73, 217-224; src/models/rag/rag_model_blip.py:430-435;
 * src/executors/FLMR_executor.py:828-833) without materialising the repeated queries and without scoring the
 * off-diagonal pairs.
 *   d_docs  bf16 [n_queries * docs_per_query, nd, FLMR_DIM]    d_mask uint8 [n_queries * docs_per_query, nd]
 *   d_argmax / d_rowmax [n_queries, docs_per_query, nq]        d_grad fp32 [n_queries, docs_per_query]
 *   d_dq fp32 [n_queries, nq, FLMR_DIM]                        d_dd fp32 [n_queries * docs_per_query, nd, FLMR_DIM]
 */
int flmr_maxsim_argmax_grouped(const void* d_q, int n_queries, int nq, const void* d_docs,
                               const uint8_t* d_mask, int docs_per_query, int nd, int32_t* d_argmax,
                               float* d_rowmax, int device, void* stream);
int flmr_maxsim_backward_grouped(const void* d_q, int n_queries, int nq, const void* d_docs,
                                 int docs_per_query, int nd, const int32_t* d_argmax, const float* d_grad,
                                 float* d_dq, float* d_dd, int device, void* stream);
/* The grouped calls on fp16 d_q and d_docs (see flmr_maxsim_argmax_fp16). */
int flmr_maxsim_argmax_grouped_fp16(const void* d_q, int n_queries, int nq, const void* d_docs,
                                    const uint8_t* d_mask, int docs_per_query, int nd, int32_t* d_argmax,
                                    float* d_rowmax, int device, void* stream);
int flmr_maxsim_backward_grouped_fp16(const void* d_q, int n_queries, int nq, const void* d_docs,
                                      int docs_per_query, int nd, const int32_t* d_argmax, const float* d_grad,
                                      float* d_dq, float* d_dd, int device, void* stream);

/* Test infrastructure: plain SIMT fp32 MaxSim of every passage (same contract as
 * flmr_maxsim_scores, e4m3 semantics on an e4m3 corpus, fp16 operands on an fp16 corpus), independent of the
 * tensor-core kernel. */
int flmr_debug_maxsim_scores_simt(const flmr_corpus_t* corpus, const void* d_q, int n_queries,
                                  int nq, unsigned flags, float* d_out_scores, void* stream);

/* Test infrastructure: which scan kernel searches on the calling thread launch — 0 = chosen per call and pass (the
 * product behaviour: normal passes, those with three resident query tiles on the three-warpgroup kernel),
 * 2 = flmr_scan_kernel<2> (two consumer warpgroups), normal passes only, 3 = flmr_scan_kernel<3> (three
 * warpgroups), normal passes only, 4 = CTA-pair passes (clusters of two CTAs stream one token
 * range, each D tile fetched once and TMA-multicast to both) whenever a call has enough queries, on any bf16 shard
 * (a search on an e4m3 corpus returns FLMR_ERR_UNSUPPORTED), 6 = flmr_scan_split_kernel (three warpgroups,
 * split-tile loop with warp-uniform MMA descriptors; listed searches run its listed form) — so the parity suite can run
 * against any of them at any shape.  Any other variant, 5 and 7 included, returns FLMR_ERR_INVALID_ARG.  An
 * FLMR_CORPUS_FP16 corpus has fp16 forms of variants 2 and 6 only: a search on it under variant 3 or 4 returns
 * FLMR_ERR_UNSUPPORTED. */
int flmr_debug_set_scan_variant(int variant);

/* Test infrastructure: which kernel flmr_maxsim_argmax(_grouped)(_fp16) runs on the calling thread — 0 = chosen by
 * size (the product behaviour), 1 = the warp-MMA kernel, 2 = the wgmma kernel, for bf16 and fp16 operands alike — so
 * tests can hold either against the other and the oracle at any shape. */
int flmr_debug_set_argmax_path(int path);

/* Test infrastructure: how flmr_topk_merge_devices reads its lists on the calling thread — 0 = in place or through
 * peer access where the devices allow it (the product behaviour), 1 = every list copied into the home staging buffer
 * first, those on the home device included — so tests reach the staged copy on a node whose devices all read each
 * other. */
int flmr_debug_set_merge_path(int path);

/* Test infrastructure, host-only (no GPU needed): the token-balanced CTA partition + per-tile
 * passage-end metadata the scan kernel consumes, for `n_ctas` persistent CTAs and
 * FLMR_TILE_TOKENS-token tiles (bit g of a tile's mask: a passage ends with 4-token group g).
 * cta_row_begin / cta_tile_base hold min(n_ctas, n_passages) + 1 entries; tile arrays may be NULL
 * to query *n_tiles_out only. */
int flmr_debug_build_partition(const int32_t* h_doclens, int64_t n_passages, int n_ctas,
                               int32_t* cta_row_begin, int64_t* cta_tile_base,
                               uint32_t* tile_end_mask, int32_t* tile_first_pid,
                               int64_t tile_capacity, int64_t* n_tiles_out);

/* Test infrastructure, host-only: the windows of a streamed corpus of these doclens (see flmr_corpus_create_streamed)
 * for `n_ctas` SMs.  out_windows (may be NULL to query *n_windows_out) receives 6 int64 per window: first slot, end slot
 * (exclusive), first stored row, stored rows, CTAs (min(n_ctas, slots of the window)), tiles.  The four partition
 * arrays (all four or none) receive each window's flmr_debug_build_partition of its own passages, concatenated in
 * window order, with cta_row_begin relative to the window and tile_first_pid ABSOLUTE slots; each holds up to
 * tile_capacity entries (cta_row_begin / cta_tile_base take CTAs + 1 per window).  *n_tiles_out (may be NULL) = all
 * windows' tiles.  A passage longer than a window gives FLMR_ERR_UNSUPPORTED. */
int flmr_debug_window_plan(const int32_t* h_doclens, int64_t n_passages, int64_t window_bytes, int n_ctas,
                           int64_t* out_windows, int64_t capacity, int64_t* n_windows_out, int32_t* cta_row_begin,
                           int64_t* cta_tile_base, uint32_t* tile_end_mask, int32_t* tile_first_pid,
                           int64_t tile_capacity, int64_t* n_tiles_out);

/* Test infrastructure, host-only: the corpus passes flmr_maxsim_scores / flmr_maxsim_topk run for a batch of
 * `n_queries` queries of `nq` tokens (a pass = one scan-kernel launch with up to 384 query rows resident per CTA);
 * allow_pair != 0 plans CTA-pair passes (clusters of two CTAs share a token range, each with its own queries) for
 * the query prefix that fills them, as the library does on shards that span every SM.
 * out_plan (may be NULL to query *n_passes_out) receives 8 int32 per pass: first query, queries resident PER CTA (a
 * pair pass covers twice as many: CTA r the r-th half), first row, rows, 32-row blocks per query, 128-row tiles per
 * CTA, flags (1 = adds earlier partial scores, 2 = stores partial scores, 4 = final: scores complete, top-k taken,
 * 8 = pair pass), row of the pass's first query in the partial-score buffer. */
int flmr_debug_plan_passes(int n_queries, int nq, int allow_pair, int32_t* out_plan, int capacity, int* n_passes_out);

/* Test infrastructure, host-only: the row moves flmr_corpus_compact makes on a corpus of these doclens when the LOCAL
 * passages h_deleted[0..n_deleted) are removed, in execution order.  out_moves (may be NULL to query *n_moves_out)
 * receives 5 int64 per move: source row, destination row, rows, 1 if the move goes through the staging buffer, chunk.
 * The moves of one chunk run together: a staged chunk reads all of its source rows before it writes any.
 * chunk_rows bounds the rows of a chunk (0: the library's bound, 256 MiB of bf16 rows). */
int flmr_debug_compact_plan(const int32_t* h_doclens, int64_t n_passages, const int64_t* h_deleted, int64_t n_deleted,
                            int64_t chunk_rows, int64_t* out_moves, int64_t capacity, int64_t* n_moves_out);

/* Test infrastructure: the plans a listed search of these lists (n_queries <= the workspace's max_queries) would scan,
 * computed on the device as flmr_maxsim_topk_listed computes them and copied back (synchronous, default stream).
 * h_out (may be NULL to query *n_out) receives int64: the number of passes, then per pass q_first, n_q, n_ctas, the
 * union size U, the tile count T and the tile bound the buffers hold, the union's slots (U, sorted), cta_tile_base
 * (n_ctas + 1: CTA c scans tiles [base[c], base[c + 1])), each tile's first stored row (T), end mask (T: bit g = a
 * listed passage ends with 4-token group g, bit 31 = the tile starts a run of consecutive slots or a CTA's share of
 * one) and first slot ending in it (T; 0x7fffffff when none does). */
int flmr_debug_listed_plan(const flmr_corpus_t* corpus, flmr_workspace_t* ws, int n_queries, int nq,
                           const int64_t* h_list_offsets, const int64_t* d_list_pids, int64_t* h_out,
                           int64_t capacity, int64_t* n_out);

/* Kernels launched by this library on the calling thread since the last reset (bench evidence). */
int64_t flmr_launch_count(int reset);

/* Average device time (ms) of the scan kernel launches recorded since the last reset, measured
 * with CUDA events on the launching stream; requires flmr_set_profiling(1). */
int flmr_set_profiling(int enable);
int flmr_scan_kernel_stats(double* total_ms, int64_t* launches, int reset);

#ifdef __cplusplus
}
#endif
#endif /* FLMR_MAXSIM_H_ */
