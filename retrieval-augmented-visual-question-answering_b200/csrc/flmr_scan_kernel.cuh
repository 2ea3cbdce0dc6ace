// flmr_scan_kernel.cuh — the fused late-interaction scan:
//
//   for every passage p of this GPU's shard and every resident query b:
//       score[b][p] = sum_i max_{j < len_p} <Q[b][i], D[p][j]>          (SURVEY.md §8a)
//   + per-CTA running top-k of those scores, so no score matrix reaches HBM.
//
// Replaces, in one kernel, the reference's `D_packed @ Q.T` GEMM, the StridedTensor padding +
// colbert_score_reduce masked max/sum (CB/modeling/colbert.py:235-311), the CPU
// segmented_maxsim.cpp reduction (CB/modeling/segmented_maxsim.cpp:22-93) and the per-query
// `scores.sort()` of IndexScorer.rank (CB/search/index_storage.py:95).
//
// Structure (one persistent CTA per SM, kWgs consumer warpgroups + 2 warps, warp-specialised):
//   consumer warpgroups : the pass's query rows are STATIONARY IN SHARED MEMORY (up to kMtMax x 128 rows,
//                         128B-swizzled, the wgmma A operand).  Warpgroup w owns the 64-row query blocks
//                         j = w, w + kWgs, ...; per D tile and block it issues 8 wgmma.m64n96k16 (K = 8 x 16),
//                         acc[64 x 96] = Qblock . Dtile^T in registers, then folds the accumulator into the
//                         passage maxima.  A thread holds two rows and 24 columns per row; the max over a
//                         passage's tokens is a per-thread max over its columns of the passage's 4-token groups
//                         plus two shuffles inside the lane quad.  At a passage end (bit in the tile's end mask)
//                         the per-row maxima (first kFastSlots ends of a tile) or the 16-row sums (later ends)
//                         go to shared memory for the reducer.  The running max of the passage straddling two
//                         D tiles stays in a register: a query block never changes warpgroup.
//   warp 4 kWgs         : reducer.  Per D tile (mbarrier-fed, double-buffered partials): per (query, passage
//                         ending in the tile) sums the row partials in one fixed order (chunk_sum16: the same for
//                         every passage end, so a score does not depend on where the passage is stored), optionally
//                         accumulates / stores scores to HBM, and maintains the per-CTA top-k.  A passage marked
//                         in the corpus' tombstone bitmap (ScanParams::dead) is skipped: -inf score, no top-k offer.
//                         A (query, passage) pair whose bit is clear in the query's allow bitmap (ScanParams::allow)
//                         is treated the same way for that query only.
//   warp 4 kWgs + 1     : TMA producer.  Streams the CTA's contiguous range of passage tokens through a
//                         kDStages-deep ring of D stages (96 tokens x 128 dims bf16, 128B-swizzled, 2 boxes;
//                         e4m3 corpora: one box of 96 x 128 bytes).
//
// Layout contracts (see DESIGN.md "Data layout"):
//   * passages are stored back to back, each padded to a multiple of 4 tokens by repeating its last
//     token (duplicates cannot change a max), so passage boundaries fall on 4-column groups and one
//     mask per tile marks the groups that end a passage;
//   * each query is padded to a multiple of 32 rows with zero rows (contribute exactly 0, like the
//     reference's masked query tokens).
#pragma once
#include "../../include/flmr_maxsim.h"
#include "flmr_device.cuh"

#include <type_traits>

namespace flmr {

constexpr int kDim = 128;
constexpr int kTileM = 128;               // query rows per staged query tile
constexpr int kTileN = FLMR_TILE_TOKENS;  // passage tokens per streamed tile (wgmma N)
constexpr int kMtMax = 3;                 // resident 128-row query tiles per pass (96 KB of shared memory)
constexpr int kRbMax = kMtMax * 4;        // resident 32-row blocks
constexpr int kNqMax = kRbMax;            // queries per pass (each has >= 1 row block)
constexpr int kHbMax = 2 * kRbMax;        // resident 16-row blocks (one per consumer warp and 64-row block)
constexpr int kMaxK = 128;                // fused top-k capacity (== FLMR_MAX_K)
constexpr int kGroup = 4;                 // token padding granularity (== FLMR_TOKEN_GROUP)
constexpr int kSlots = kTileN / kGroup;   // passage ends per tile, at most (24 <= 32 lanes)
constexpr int kNb = kTileN / 8;           // 8-column blocks of an accumulator
constexpr int kFastSlots = 4;             // passage ends per tile whose per-row maxima are left to the reducer
constexpr int kLaneStride = 33;           // padded row of 32 row values (conflict-free transposed reads)
constexpr int kDStages = 4;
constexpr int kDTileBytes = kTileN * kDim * 2;   // 24 KiB: [2 k-blocks][96 rows][64 bf16]; the D stage stride
constexpr int kDKBlockBytes = kTileN * 128;      // 12 KiB; also a whole e4m3 tile: [1 k-block][96 rows][128 e4m3]
constexpr int kQKBlockBytes = kMtMax * kTileM * 128;   // one 64-dim half of the resident bf16 queries (all of e4m3)
// bytes one D tile brings into its stage: two 128-B k-blocks of a 16-bit type, or one of e4m3
template <Elem kE>
__host__ __device__ constexpr int d_tile_bytes() { return kE == Elem::kE4M3 ? kDKBlockBytes : kDTileBytes; }
constexpr int kRedWarps = 1;

static_assert(kTileN == 96, "the wgmma shape and accumulator fragment are written for 96-token tiles");
static_assert(kDKBlockBytes % 1024 == 0, "swizzle atoms need 1024-B aligned k-blocks");

__host__ __device__ constexpr int scan_threads(int wgs) { return (wgs * 4 + 2) * 32; }
// 64-row query blocks that hold resident rows: the MMAs of a pass stop at its last occupied block (the staged tiles
// are zero-padded to 128 rows, but nobody reads the sums of rows past nq_pass * rbq * 32)
__host__ __device__ constexpr int scan_blocks(int nq_pass, int rbq) { return (nq_pass * rbq * 32 + 63) / 64; }

struct ScanParams {
  // corpus partition (built once per corpus, see build_partition() in flmr_maxsim.cu)
  const int32_t* cta_row_begin;    // [n_ctas + 1] first stored row of each CTA's passage range
  const int64_t* cta_tile_base;    // [n_ctas + 1] index of each CTA's first tile in tile_* arrays
  const uint32_t* tile_end_mask;   // [n_tiles] bit g set <=> a passage ends with 4-token group g
  const int32_t* tile_first_pid;   // [n_tiles] local id of the first passage ending in the tile
  // resident queries of this pass
  const uint4* q_pad;              // bf16 (e4m3 kernel: e4m3) [n_mtiles * 128][128], zero-padded (stage_queries kernel)
  int32_t n_mtiles;                // 128-row query tiles (1..kMtMax)
  int32_t nq_pass;                 // queries resident in this pass (1..kNqMax)
  int32_t rbq;                     // 32-row blocks per query in this pass
  int32_t lane_mode_max_rbq;       // reducer: lane-per-query summation when rbq <= this, else warp-per-item
  float init_val;                  // -inf (true max) or 0 (reference CPU "ReLU" variant)
  // score plumbing
  const float* acc_in;             // [nq_pass][n_passages] partial scores of earlier row slices, or null
  float* acc_out;                  // [nq_pass][n_passages] scores (or partial scores) out, or null
  int64_t n_passages;
  const uint32_t* dead;            // [ceil(n_passages / 32)] tombstones (bit p & 31 of word p >> 5), or null: none
  // per-query allow bitmaps (layout of `dead`): the pass's query b may return passage p only if bit p of
  // allow[(q_off + b) * allow_stride ...] is set (q_off: the CTA-pair offset); null: every passage allowed
  const uint32_t* allow;
  int64_t allow_stride;            // words between consecutive queries' bitmaps; 0 = one bitmap for all
  // fused top-k
  int32_t k;                       // 0 = disabled
  uint64_t* cand_keys;             // [n_ctas][cand_q_stride][k]  (ordered score << 32 | ~local pid)
  int32_t cand_q_stride;           // queries of the whole call chunk (one merge launch serves them all)
  int32_t cand_q_first;            // index of this pass's first query inside the chunk
  int* status;                     // mapped pinned host word: watchdog code of a trapped launch
  // plan mode (the listed kernels): the tile arrays above are a per-call plan over the listed passages' rows only, and
  // tile i starts at stored row tile_row[i] instead of cta_row_begin + 96 t (null for the partition kernels)
  const int32_t* tile_row;
};

// Plan mode: bit 31 of a tile's end mask marks a tile that starts a run of listed passages or a CTA's share of one.
// The passage open at such a tile's start is a new one, whatever the CTA's previous tile folded, so the consumers
// reset their running maxima there; the end groups proper stay in bits 0 .. kSlots - 1.
constexpr uint32_t kTileRunStart = 1u << 31;

struct ScanSmem {
  static constexpr int kOffQ = 0;                                     // [2 k-blocks][kMtMax * 128 rows][128 B]
  static constexpr int kOffD = kOffQ + 2 * kQKBlockBytes;
  static constexpr int kOffPartial = kOffD + kDStages * kDTileBytes;  // float[2][kHbMax][kSlots]
  static constexpr int kPartialBytes = 2 * kHbMax * kSlots * 4;
  // per-row passage maxima of the first kFastSlots passage ends of a tile: [2][kFastSlots][kRbMax][33]
  static constexpr int kOffLanePart = kOffPartial + kPartialBytes;
  static constexpr int kLanePartBytes = 2 * kFastSlots * kRbMax * kLaneStride * 4;
  static constexpr int kOffKeys = kOffLanePart + kLanePartBytes;
  static constexpr int kKeysBytes = kNqMax * kMaxK * 8;
  static constexpr int kOffMinKey = kOffKeys + kKeysBytes;           // u64[kNqMax]
  static constexpr int kOffMinPos = kOffMinKey + kNqMax * 8;         // int[kNqMax]
  static constexpr int kOffBars = (kOffMinPos + kNqMax * 4 + 7) / 8 * 8;
  static constexpr int kNumBars = 2 * kDStages + 4;
  static constexpr int kBytes = kOffBars + kNumBars * 8 + 1024;   // + slack for 1024-B alignment
  static_assert(kBytes <= 232448, "exceeds 227 KiB of shared memory per CTA");
};

// Shared-memory addresses of the kernel's mbarriers.
struct ScanBars {
  uint32_t base;   // smem address of ScanSmem::kOffBars
  __device__ uint32_t d_full(int s) const { return base + 8u * s; }                      // D stage s loaded
  __device__ uint32_t d_empty(int s) const { return base + 8u * (kDStages + s); }        // ... and released
  __device__ uint32_t p_full(int b) const { return base + 8u * (2 * kDStages + b); }     // partials of buffer b written
  __device__ uint32_t p_empty(int b) const { return base + 8u * (2 * kDStages + 2 + b); }  // ... and consumed
};

// ---- epilogue helpers ---------------------------------------------------------------------------
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
  const uint32_t lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v), src);
  const uint32_t hi = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), src);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

// Replace the current minimum of an unsorted k-entry list by `cand`, then recompute the minimum.
__device__ __noinline__ void topk_replace_min(uint64_t* keys, int k, uint64_t cand,
                                              uint64_t& minkey, int& minpos, int lane) {
  if (lane == 0) keys[minpos] = cand;
  __syncwarp();
  uint64_t mk = ~0ull;
  int mp = 0x7fffffff;
  for (int i = lane; i < k; i += 32) {
    const uint64_t x = keys[i];
    if (x < mk) {
      mk = x;
      mp = i;
    }
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const uint64_t ok = shfl64(mk, lane ^ off);
    const int op = __shfl_xor_sync(0xffffffffu, mp, off);
    if (ok < mk || (ok == mk && op < mp)) {
      mk = ok;
      mp = op;
    }
  }
  minkey = mk;
  minpos = mp;
  __syncwarp();
}

// -inf into column `out` of the nq rows (stride n) of a score output: a deleted passage.  Out of line: the reducer's
// cold path, kept from adding to the kernel's register allocation.
__device__ __noinline__ void store_dead_scores(float* out, int64_t n, int nq, int lane) {
  for (int b = lane; b < nq; b += 32) out[b * n] = -INFINITY;
}

// May query qb of the pass (its index in the per-query arrays, CTA-pair offset included) return local passage pid?
__device__ __forceinline__ bool pair_allowed(const ScanParams& p, int qb, int64_t pid) {
  return p.allow == nullptr ||
         ((__ldg(p.allow + static_cast<int64_t>(qb) * p.allow_stride + (pid >> 5)) >> (pid & 31)) & 1u);
}

// THE summation order of a passage's score, whichever path computes it (so the score depends on the query and the
// passage's tokens only, not on where the passage is stored).  The rows of a pass are cut into 16-row chunks; chunk c
// is summed as ((v0 + v1) + (v2 + v3)) + ((v4 + v5) + (v6 + v7)) with v_q = r[16 c + q] + r[16 c + q + 8], and a query's
// chunks are then added in row order starting from 0.f (acc_in of earlier row slices last).  A passage that is the
// 5th or later to end in its tile is chunk-summed by the consumer warp that holds the rows (fold_accumulator's
// shuffle tree), the first kFastSlots by the reducer from the parked row maxima (chunk_sum16).
// chunk_sum16: the sum of one chunk whose 16 row values are x[0..15], in that order.
__device__ __forceinline__ float chunk_sum16(const float* x) {
  float v[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) v[q] = x[q] + x[q + 8];
  return ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
}

// Max of a thread's values x over the quad's four lanes (they hold the same rows, different columns).
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}

// Fold one 64 x 96 accumulator (rows of query block j, the D tile's 96 tokens) into the passage maxima.
// `m[h]` is the running max of row half h of the passage that is open at the tile start; on return, of the one
// open at its end.  Every lane of a quad holds the same m (the quad's columns are combined by shuffles).
// Max is exact, so the order of the maxima is free: each thread first reduces its own columns of a passage, and
// the quad is combined once per passage end instead of once per 8-column block.  A thread's two columns of
// 8-column block i in row half h are acc[4 i + 2 h] and acc[4 i + 2 h + 1]; lanes with the same hi (lane, lane ^ 1)
// together cover the 4-token group 2 i + hi.  The accumulator is read in place: no per-block maxima are kept,
// which leaves the registers for the second accumulator of the pipelined consumer loop.
// kPart = 0 folds a whole tile (kCb = kNb).  The split loop folds a tile as two halves of kCb = kNb / 2 blocks (its
// m64n48 accumulators: 4-token groups 12 hf .. 12 hf + 11, `mask` shifted down to them), kPart = 1 and 2.  `slot` is
// the tile's passage-end count before these columns (0, or half 0's ends for half 1) and the count after them is
// returned, so the halves park their ends in the slots a whole-tile fold gives them.  Half 0 leaves the maxima of the
// passage open at its end in `pend`, per thread (not yet combined over the quad), and half 1 starts from them: the
// quad is combined once per passage end and once per tile, as in the whole-tile fold.  `pend` is unused for kPart = 0.
template <int kCb = kNb, int kPart = 0>
__device__ __forceinline__ int fold_accumulator(const float (&acc)[4 * kCb], uint32_t mask, float (&m)[2],
                                                float (&pend)[2], float init, float* lane_part_buf,
                                                float* partial_buf, int j, int wq, int lane, int slot = 0) {
  static_assert(kPart == 0 ? kCb == kNb : kCb == kNb / 2, "a whole tile or one of its halves");
  const int hi = (lane >> 1) & 1;
  float carry[2];   // this thread's max over the open passage's columns before these ones (half 1 only)
#pragma unroll
  for (int h = 0; h < 2; ++h) carry[h] = kPart == 2 ? pend[h] : -INFINITY;
  if (mask == 0) {   // warp-uniform: no passage ends in these columns (about half the tiles at Nd = 180)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float c[4];   // four independent max chains over the thread's columns
#pragma unroll
      for (int i = 0; i < 4; ++i) c[i] = fmaxf(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
#pragma unroll
      for (int i = 4; i < kCb; ++i) c[i & 3] = fmax3(c[i & 3], acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
      const float x = fmaxf(fmaxf(c[0], c[1]), fmaxf(c[2], c[3]));
      if constexpr (kPart == 1)
        pend[h] = x;
      else if constexpr (kPart == 2)
        m[h] = fmaxf(m[h], quad_max(fmaxf(carry[h], x)));
      else
        m[h] = fmaxf(m[h], quad_max(x));
    }
    return slot;
  }
  const int row0 = j * 64 + wq * 16 + (lane >> 2);   // row of h = 0 inside the pass; h = 1 is row0 + 8
  uint32_t live = (1u << (2 * kCb)) - 1u;            // groups not yet consumed by a finished passage
  uint32_t bits = mask;
#pragma unroll 1
  while (bits) {   // warp-uniform: one iteration per passage ending in this tile
    const uint32_t upto = bits ^ (bits - 1u);   // groups 0..(lowest set bit)
    const uint32_t seg = (upto & live) >> hi;
    float s[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float x = carry[h];
#pragma unroll
      for (int i = 0; i < kCb; ++i)
        if ((seg >> (2 * i)) & 1u) x = fmax3(x, acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
      s[h] = fmaxf(quad_max(x), m[h]);
      m[h] = init;
      carry[h] = -INFINITY;
    }
    if (slot < kFastSlots) {
      // common case: one lane per quad parks its two rows' maxima, the reducer sums them later
      if ((lane & 3) == 0) {
        float* lp = lane_part_buf + slot * (kRbMax * kLaneStride);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = row0 + 8 * h;
          lp[(r >> 5) * kLaneStride + (r & 31)] = s[h];
        }
      }
    } else {
      // this warp's 16 rows summed in chunk_sum16's order (the lanes of a quad hold equal values; lane group g holds
      // rows g and g + 8, and the xor-4 / 8 / 16 shuffles pair g with g ^ 1, g ^ 2, g ^ 4)
      float v = s[0] + s[1];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (lane == 0) partial_buf[(j * 4 + wq) * kSlots + slot] = v;
    }
    ++slot;
    live &= ~upto;
    bits &= bits - 1u;
  }
  const uint32_t rest = live >> hi;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float x = carry[h];
#pragma unroll
    for (int i = 0; i < kCb; ++i)
      if ((rest >> (2 * i)) & 1u) x = fmax3(x, acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
    if constexpr (kPart == 1)
      pend[h] = x;
    else
      m[h] = fmaxf(m[h], quad_max(x));
  }
  return slot;
}

// acc = (64-row query block at q_block) . (D tile at d_stage)^T over K = 128, one commit group: bf16 or fp16, 8 x
// wgmma.m64n96k16 over two 128-byte k-blocks; e4m3, 4 x wgmma.m64n96k32 over one.  Either way a k-step is 32
// bytes along the row, and the accumulator fragment is the same.
template <Elem kE>
__device__ __forceinline__ void issue_block_mma(float (&acc)[4 * kNb], uint32_t q_block, uint32_t d_stage) {
  // the query block's descriptors are loop-invariant: hidden from the compiler so that they are rebuilt here (a
  // few integer adds) rather than hoisted out of the tile loop into 16 registers per block
  asm volatile("" : "+r"(q_block));
  wgmma_fence();
  if constexpr (kE == Elem::kE4M3) {
#pragma unroll
    for (int k = 0; k < kDim / 32; ++k) {
      const uint64_t a_desc = make_kmajor_sw128_desc(q_block + k * 32u);   // 32 elements along the 128-byte row
      const uint64_t b_desc = make_kmajor_sw128_desc(d_stage + k * 32u);
      wgmma_m64n96k32_e4m3(acc, a_desc, b_desc, k > 0 ? 1u : 0u);
    }
  } else {
#pragma unroll
    for (int k = 0; k < kDim / 16; ++k) {
      const uint32_t koff = (k & 3) * 32u;   // 16 elements along the 128-byte row
      const uint64_t a_desc = make_kmajor_sw128_desc(q_block + (k >> 2) * kQKBlockBytes + koff);
      const uint64_t b_desc = make_kmajor_sw128_desc(d_stage + (k >> 2) * kDKBlockBytes + koff);
      if constexpr (kE == Elem::kF16)
        wgmma_m64n96k16_f16(acc, a_desc, b_desc, k > 0 ? 1u : 0u);
      else
        wgmma_m64n96k16(acc, a_desc, b_desc, k > 0 ? 1u : 0u);
    }
  }
  wgmma_commit();
}

// The m64n48 MMAs of one half tile (issue_block_mma's k-steps, in its order) from the low words of its two descriptors,
// `a_lo` for the 64-row query block and `b_lo` for the half tile (sw128_desc_lo).  A k-step moves a start address by 32
// bytes, 2 in the descriptor's address field, and a k-block by a constant; the field never carries into the word's
// LBO bits (shared addresses are below 2^18), so each k-step is one 32-bit add per operand and the high word is the
// constant kSw128DescHi.  With warp-uniform bases the adds run on the uniform datapath and every descriptor stays in
// uniform registers, where the HGMMA reads it, instead of being rebuilt from regular registers for each MMA.
template <Elem kE>
__device__ __forceinline__ void issue_half_mma_udesc(float (&acc)[2 * kNb], uint32_t a_lo, uint32_t b_lo) {
  auto desc = [](uint32_t lo) { return (static_cast<uint64_t>(kSw128DescHi) << 32) | lo; };
  wgmma_fence();
  if constexpr (kE == Elem::kE4M3) {
#pragma unroll
    for (int k = 0; k < kDim / 32; ++k)
      wgmma_m64n48k32_e4m3(acc, desc(a_lo + 2u * k), desc(b_lo + 2u * k), k > 0 ? 1u : 0u);
  } else {
#pragma unroll
    for (int k = 0; k < kDim / 16; ++k) {
      const uint32_t a = a_lo + (k >> 2) * (kQKBlockBytes >> 4) + 2u * (k & 3);
      const uint32_t b = b_lo + (k >> 2) * (kDKBlockBytes >> 4) + 2u * (k & 3);
      if constexpr (kE == Elem::kF16)
        wgmma_m64n48k16_f16(acc, desc(a), desc(b), k > 0 ? 1u : 0u);
      else
        wgmma_m64n48k16(acc, desc(a), desc(b), k > 0 ? 1u : 0u);
    }
  }
  wgmma_commit();
}

// One consumer warpgroup that owns NB of the pass's 64-row query blocks (j = wg + u kWgs, u < NB), over all tiles.
// Software-pipelined over the sequence of (tile, block) pairs with two accumulators: the MMAs of the next pair are
// issued before the accumulator of the current one is folded (wait_group 1), so the tensor pipe works while the
// warpgroup folds.  Pair q = t NB + u uses accumulator q & 1; tiles are walked two at a time so that the index is
// a compile-time constant for every NB.  The next pair of the last block of tile t is the first block of tile t + 1,
// which reads the next D stage: after the wait, every MMA that read stage t has completed and the stage is released.
// ptxas tracks which accumulator is in flight only along compile-time structure: every join of the control flow
// has the same group in flight (acc[0] at the loop head, none at the end), so the last one or two tiles, whose
// last pair has no successor, are peeled out of the loop.
// kOverlap = false is the serial form with one accumulator (next MMAs issued after the fold, wait_group 0), for
// instantiations without the registers for two; the arithmetic and its order are the same.
//
// -DFLMR_SCAN_SKELETON (a timing build of tools/scan_split_probe.py, never the library's): the three-warpgroup
// consumer loops, serial and split, issue their MMAs and keep every wait and barrier but fold nothing, so they time
// the MMA pipe and the loop's synchronisation alone.  Their scores are meaningless.
#ifdef FLMR_SCAN_SKELETON
constexpr bool kScanSkeleton = true;
#else
constexpr bool kScanSkeleton = false;
#endif

//
// kPlan (the listed kernels): a tile whose mask has kTileRunStart set starts from init maxima (see kTileRunStart).
template <int NB, int kWgs, bool kPair, bool kOverlap, Elem kE, bool kPlan = false>
__device__ __forceinline__ void scan_consumer(const ScanParams& p, uint8_t* smem, uint32_t smem_base, ScanBars bars,
                                              int n_tiles, int64_t tile_base, int wg, int wq, int lane) {
  using S = ScanSmem;
  const float init = p.init_val;
  float m[NB][2];   // running passage maxima of block u's two rows of this thread
#pragma unroll
  for (int u = 0; u < NB; ++u) m[u][0] = m[u][1] = init;
  float* const lane_part = reinterpret_cast<float*>(smem + S::kOffLanePart);
  float* const partial = reinterpret_cast<float*>(smem + S::kOffPartial);
  const uint32_t q_smem = smem_base + S::kOffQ;
  auto q_block = [&](int u) { return q_smem + (wg + u * kWgs) * 64 * 128; };
  auto d_stage = [&](int t) { return smem_base + S::kOffD + (t % kDStages) * kDTileBytes; };
  float acc[kOverlap ? 2 : 1][4 * kNb];
  uint32_t mask_next = 0;

  // tile t, entered with the MMAs of (t, 0) in flight in acc[(kH * NB) & 1]; kNext: a tile t + 1 follows
  auto tile = [&](int t, auto kh, auto knext) {
    constexpr int kH = decltype(kh)::value;
    constexpr bool kNext = decltype(knext)::value;
    uint32_t mask = mask_next;
    if constexpr (kPlan) {
      if (mask & kTileRunStart) {
#pragma unroll
        for (int u = 0; u < NB; ++u) m[u][0] = m[u][1] = init;
      }
      mask &= ~kTileRunStart;
    }
    const int buf = t & 1;
    float* lane_part_buf = lane_part + buf * (kFastSlots * kRbMax * kLaneStride);
    float* partial_buf = partial + buf * (kHbMax * kSlots);
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      const int a = kOverlap ? (kH * NB + u) & 1 : 0;   // accumulator of (t, u); the other one takes the next pair
      const bool last = u + 1 == NB;
      auto issue_next = [&](float (&acc_next)[4 * kNb]) {
        if (!last) {
          issue_block_mma<kE>(acc_next, q_block(u + 1), d_stage(t));
        } else if (kNext) {
          mbar_wait_inline(bars.d_full((t + 1) % kDStages), ((t + 1) / kDStages) & 1u, p.status, kDevTimeoutMma);
          mask_next = __ldg(p.tile_end_mask + tile_base + t + 1);
          issue_block_mma<kE>(acc_next, q_block(0), d_stage(t + 1));
        }
      };
      if (kOverlap && (!last || kNext)) {
        issue_next(acc[a ^ 1]);
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      wgmma_fence_operands(acc[a]);
      if (last) {
        // every wgmma reading D stage t has completed (the one in flight reads stage t + 1) -> release it
        __syncwarp();
        if (wq == 0 && lane == 0) {
          if constexpr (kPair) {
            mbar_arrive_cluster(bars.d_empty(t % kDStages), 0);
            mbar_arrive_cluster(bars.d_empty(t % kDStages), 1);
          } else {
            mbar_arrive(bars.d_empty(t % kDStages));
          }
        }
      }
      // the reducer must have consumed the partial sums of tile t-2 before this buffer is reused
      if (u == 0)
        mbar_wait_inline(bars.p_empty(buf), ((static_cast<uint32_t>(t) >> 1) & 1u) ^ 1u, p.status,
                         kDevTimeoutEpilogue);
      float unused[2];
      if (!(kScanSkeleton && kWgs == 3))
        fold_accumulator(acc[a], mask, m[u], unused, init, lane_part_buf, partial_buf, wg + u * kWgs, wq, lane);
      if (!kOverlap) issue_next(acc[0]);
    }
    // this warp's row maxima / partial sums of tile t are written: order every lane's stores
    // before lane 0's arrive (release); the reducer's wait is the matching acquire
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.p_full(buf));
  };
  using H0 = std::integral_constant<int, 0>;
  using H1 = std::integral_constant<int, 1>;
  using Next = std::true_type;
  using Final = std::false_type;

  if (n_tiles <= 0) return;
  mbar_wait(bars.d_full(0), 0u, p.status, kDevTimeoutMma);
  mask_next = __ldg(p.tile_end_mask + tile_base);
  issue_block_mma<kE>(acc[0], q_block(0), d_stage(0));
  int t = 0;
  for (; t + 2 < n_tiles; t += 2) {
    tile(t, H0{}, Next{});
    tile(t + 1, H1{}, Next{});
  }
  if (t + 2 == n_tiles) {
    tile(t, H0{}, Next{});
    tile(t + 1, H1{}, Final{});
  } else {
    tile(t, H0{}, Final{});
  }
}

// The consumer loop of flmr_scan_split_kernel: one of three warpgroups, NB (1 or 2) query blocks, with the registers of
// the serial loop (two 24-register half accumulators) but its fold overlapped with its own MMAs.  Each (tile, block)
// pair is split along N into two commit groups of m64n48 MMAs: half 0 = tokens 0..47 (4-token groups 0..11) in
// acc[0], half 1 = tokens 48..95 (groups 12..23) in acc[1].  The sequence of (tile, block, half) triples is
// software-pipelined: the next triple is issued, wait_group 1, the current one is folded — half 0 under the MMAs of
// half 1, half 1 under those of half 0 of the next block (or of the first block of the next tile).  The half index is
// the accumulator index, so every tile is entered with half 0 of its first block in flight in acc[0] and only the
// last tile is peeled.  The fold carries the open passage's maxima and the passage-end slot from half 0 to half 1 in
// the same thread: a passage's row maxima and chunk sums are the values, in the order, of the whole-tile fold (max is
// exact, whatever order it is taken in), and the scores bitwise those of flmr_scan_kernel.
// The MMAs take their descriptors from warp-uniform bases (issue_half_mma_udesc): the query blocks' once per
// warpgroup, the half tile's once per tile.
// kPlan: as scan_consumer's (the reset happens before half 0 of the tile is folded).
template <int NB, Elem kE, bool kPlan = false>
__device__ __forceinline__ void scan_split_consumer(const ScanParams& p, uint8_t* smem, uint32_t smem_base,
                                                    ScanBars bars, int n_tiles, int64_t tile_base, int wg, int wq,
                                                    int lane) {
  using S = ScanSmem;
  constexpr int kWgs = 3;
  constexpr int kHalfGroups = kSlots / 2;                  // 4-token groups of a half tile
  constexpr uint32_t kHalfBytes = (kTileN / 2) * 128;      // 48 rows of a k-block: the B offset of half 1
  static_assert(kHalfBytes % 1024 == 0, "half 1 must start on a swizzle atom");
  const float init = p.init_val;
  float m[NB][2];   // running passage maxima of block u's two rows of this thread
#pragma unroll
  for (int u = 0; u < NB; ++u) m[u][0] = m[u][1] = init;
  float* const lane_part = reinterpret_cast<float*>(smem + S::kOffLanePart);
  float* const partial = reinterpret_cast<float*>(smem + S::kOffPartial);
  // Descriptor low words.  The shuffles from lane 0 tell ptxas that the warpgroup, the shared-memory base and the tile
  // count (hence every base below, and the tile index the D stage follows) are the same in all lanes, so it can keep
  // them in uniform registers.
  n_tiles = __shfl_sync(0xffffffffu, n_tiles, 0);
  const int wg_u = __shfl_sync(0xffffffffu, wg, 0);
  const uint32_t base_u = __shfl_sync(0xffffffffu, smem_base, 0);
  uint32_t q_lo[NB];
#pragma unroll
  for (int u = 0; u < NB; ++u) q_lo[u] = sw128_desc_lo(base_u + S::kOffQ + (wg_u + u * kWgs) * 64 * 128);
  const uint32_t d_lo = sw128_desc_lo(base_u + S::kOffD);
  // acc (+)= the MMAs of block u and half hf of tile t, one commit group
  auto issue = [&](float (&a)[2 * kNb], int u, int t, int hf) {
    issue_half_mma_udesc<kE>(a, q_lo[u], d_lo + (t % kDStages) * (kDTileBytes >> 4) + hf * (kHalfBytes >> 4));
  };
  float acc[2][2 * kNb];
  uint32_t mask_next = 0;

  // tile t, entered with the MMAs of (t, 0, half 0) in flight in acc[0]; kNext: a tile t + 1 follows
  auto tile = [&](int t, auto knext) {
    constexpr bool kNext = decltype(knext)::value;
    uint32_t mask = mask_next;
    if constexpr (kPlan) {
      if (mask & kTileRunStart) {
#pragma unroll
        for (int u = 0; u < NB; ++u) m[u][0] = m[u][1] = init;
      }
      mask &= ~kTileRunStart;
    }
    const int buf = t & 1;
    float* lane_part_buf = lane_part + buf * (kFastSlots * kRbMax * kLaneStride);
    float* partial_buf = partial + buf * (kHbMax * kSlots);
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      const bool last = u + 1 == NB;
      const int j = wg + u * kWgs;
      issue(acc[1], u, t, 1);
      wgmma_wait<1>();
      wgmma_fence_operands(acc[0]);
      // the reducer must have consumed the partial sums of tile t-2 before this buffer is reused
      if (u == 0)
        mbar_wait_inline(bars.p_empty(buf), ((static_cast<uint32_t>(t) >> 1) & 1u) ^ 1u, p.status,
                         kDevTimeoutEpilogue);
      int slot = 0;
      float pend[2];   // half 0's per-thread maxima of the passage open at its end, for half 1
      if (!kScanSkeleton)
        slot = fold_accumulator<kNb / 2, 1>(acc[0], mask & ((1u << kHalfGroups) - 1u), m[u], pend, init,
                                            lane_part_buf, partial_buf, j, wq, lane);
      if (!last) {
        issue(acc[0], u + 1, t, 0);
        wgmma_wait<1>();
      } else if (kNext) {
        mbar_wait_inline(bars.d_full((t + 1) % kDStages), ((t + 1) / kDStages) & 1u, p.status, kDevTimeoutMma);
        mask_next = __ldg(p.tile_end_mask + tile_base + t + 1);
        issue(acc[0], 0, t + 1, 0);
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      wgmma_fence_operands(acc[1]);
      if (last) {
        // every wgmma reading D stage t has completed (the one in flight reads stage t + 1) -> release it
        __syncwarp();
        if (wq == 0 && lane == 0) mbar_arrive(bars.d_empty(t % kDStages));
      }
      if (!kScanSkeleton)
        fold_accumulator<kNb / 2, 2>(acc[1], mask >> kHalfGroups, m[u], pend, init, lane_part_buf, partial_buf, j,
                                     wq, lane, slot);
    }
    // this warp's row maxima / partial sums of tile t are written: order every lane's stores
    // before lane 0's arrive (release); the reducer's wait is the matching acquire
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.p_full(buf));
  };

  if (n_tiles <= 0) return;
  mbar_wait(bars.d_full(0), 0u, p.status, kDevTimeoutMma);
  mask_next = __ldg(p.tile_end_mask + tile_base);
  issue(acc[0], 0, 0, 0);
  int t = 0;
  for (; t + 1 < n_tiles; ++t) tile(t, std::true_type{});
  tile(t, std::false_type{});
}

// ---- the kernel -------------------------------------------------------------------------------
// kWgs = consumer warpgroups (2 or 3): the 64-row query blocks are dealt to them round-robin, so with three
// resident 128-row tiles (six blocks) three warpgroups take two blocks each.  The per-row arithmetic and its
// order do not depend on kWgs: every instantiation returns bit-identical scores.
//
// kPair = true is the CTA-PAIR pass (launched as clusters of two CTAs): both CTAs of a pair stream the SAME
// token range, each with its own resident queries (twice the queries per corpus pass); every D tile is fetched
// from L2 / HBM once — CTA r loads rows [48 r, 48 r + 48) of the tile and TMA-multicasts them into both CTAs'
// shared memory — and a D stage is recycled when the consumers of BOTH CTAs have released it (remote arrive).
//
// kE = Elem::kE4M3 is the e4m3 corpus (FLMR_CORPUS_FP8): the staged queries and the D tiles hold one 128-byte e4m3
// k-block per row (a D tile is one 96-row TMA box of 12 KiB) and the MMAs are wgmma.m64n96k32 e4m3.  Tiles, masks,
// the shared-memory layout (each stage and the query area keep their bf16 size, half used), the fold, the reducer and
// the top-k are those of the bf16 kernel.  kE = Elem::kF16 (FLMR_CORPUS_FP16) differs from bf16 only in the MMA
// instruction.  There is no CTA-pair kernel for either.
//
// kSplit = true (flmr_scan_split_kernel, three warpgroups) runs scan_split_consumer instead of scan_consumer; the
// producer, the reducer, the barriers and the shared-memory layout are the same code.
//
// kPlan = true (the listed kernels) scans a per-call plan instead of the corpus partition: CTA c's tiles are
// cta_tile_base[c] .. cta_tile_base[c + 1] of the plan's arrays, tile i is loaded from stored row tile_row[i], and a
// tile with kTileRunStart set resets the consumers' running maxima.  The fold, the reducer (its tombstone and allow
// tests drop whatever the plan's tiles cover besides the listed passages) and the top-k are the same code, so every
// score is bitwise the one the partition kernels compute.  A CTA without tiles publishes its empty top-k lists and
// waits on no barrier.
template <int kWgs, bool kPair, Elem kE, bool kSplit, bool kPlan = false>
__device__ __forceinline__ void scan_kernel_body(const CUtensorMap& tmap_d, const ScanParams& p) {
  static_assert(!(kPair && kE != Elem::kBF16), "the CTA-pair kernel is bf16 only");
  static_assert(!(kPair && kPlan), "plan mode has no CTA-pair kernel");
  constexpr bool kFp8 = kE == Elem::kE4M3;
  static_assert(!kSplit || (kWgs == 3 && !kPair), "the split consumer loop is written for three single-CTA warpgroups");
  using S = ScanSmem;
  constexpr int kConsumerWarps = kWgs * 4;
  constexpr int kWarpRed0 = kConsumerWarps;
  constexpr int kWarpProducer = kConsumerWarps + kRedWarps;
  constexpr int kBlocksPerWg = (2 * kMtMax + kWgs - 1) / kWgs;   // 64-row query blocks per warpgroup, at most
  // Two accumulators per consumer thread (the overlapped loop): ptxas allocates that loop with 166 registers and
  // fails outright (C7600) below 168.  A sub-partition's 16K registers serve one warp of every warpgroup, so two
  // consumer warpgroups (10 warps) get 168; three (14 warps, 4 on a sub-partition) get 128, and moving registers
  // with setmaxnreg cannot help: 3 x 168 leaves the producer / reducer warps less than setmaxnreg's minimum of 24.
  // Three warpgroups therefore run the serial loop.
  constexpr bool kOverlap = kWgs == 2;
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment by pointer arithmetic on the __shared__ array (keeps the shared address space
  // visible to the compiler: LDS/STS instead of generic loads/stores)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t smem_base = smem_u32(smem);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int cta = kPair ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);   // partition / list index
  const uint32_t pair_rank = kPair ? cluster_ctarank() : 0u;

  const ScanBars bars{smem_base + S::kOffBars};

  const int32_t row_begin = kPlan ? 0 : p.cta_row_begin[cta];
  const int64_t tile_base = p.cta_tile_base[cta];
  const int n_tiles = static_cast<int>(p.cta_tile_base[cta + 1] - tile_base);
  const int n_mtiles = p.n_mtiles;
  const int n_blocks = scan_blocks(p.nq_pass, p.rbq);   // 64-row query blocks with resident rows
  // warpgroups that own at least one 64-row query block (three warpgroups, one block: one); only these read the
  // D stages, release them and deliver partial sums; the others have nothing to do
  const int n_busy_wgs = min(kWgs, n_blocks);

  // ---- one-time setup --------------------------------------------------------------------------
  if (warp == kWarpProducer && lane == 0) {
    tma_prefetch_desc(&tmap_d);
    for (int s = 0; s < kDStages; ++s) {
      mbar_init(bars.d_full(s), 1);
      mbar_init(bars.d_empty(s), (kPair ? 2 : 1) * n_busy_wgs);   // pair: the consumers of both CTAs
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(bars.p_full(b), 4 * n_busy_wgs);   // partial sums of a D tile complete (every busy consumer warp)
      mbar_init(bars.p_empty(b), kRedWarps);       // ... and consumed by the reducer warp
    }
    mbar_fence_init();
  }
  {
    // top-k lists start empty (key 0 sorts below every real candidate)
    uint64_t* keys = reinterpret_cast<uint64_t*>(smem + S::kOffKeys);
    for (int i = threadIdx.x; i < kNqMax * kMaxK; i += blockDim.x) keys[i] = 0ull;
    if (threadIdx.x < kNqMax) {
      reinterpret_cast<uint64_t*>(smem + S::kOffMinKey)[threadIdx.x] = 0ull;
      reinterpret_cast<int*>(smem + S::kOffMinPos)[threadIdx.x] = 0;
    }
    // stage the resident queries in the 128B-swizzled K-major layout the wgmma descriptors describe:
    // row r, 16-byte chunk c of dims [64 kb, 64 kb + 64) at kb * kQKBlockBytes + r * 128 + ((c ^ (r & 7)) * 16)
    // (e4m3: 8 chunks per row, all in k-block 0)
    constexpr int kChunkBits = kFp8 ? 3 : 4;   // log2 of the 16-byte chunks of a staged row
    const uint4* src = p.q_pad + static_cast<int64_t>(pair_rank) * (kMtMax * kTileM * 16);   // pair: CTA r's slot
    const int n_chunks = n_mtiles * kTileM << kChunkBits;
    for (int i = threadIdx.x; i < n_chunks; i += blockDim.x) {
      const int r = i >> kChunkBits, c = i & ((1 << kChunkBits) - 1), kb = c >> 3;
      *reinterpret_cast<uint4*>(smem + S::kOffQ + kb * kQKBlockBytes + r * 128 + (((c & 7) ^ (r & 7)) << 4)) =
          __ldg(src + i);
    }
    fence_proxy_async_smem();
  }
  __syncthreads();
  if constexpr (kPair) cluster_sync_all();   // the peer's barriers exist before anything is multicast to them

  if (warp >= kConsumerWarps) {
    if (warp == kWarpProducer) {
      // ===================== TMA producer =====================
      // The whole warp runs the loop (warp-uniform control flow keeps addresses in uniform
      // registers); one elected lane issues the bulk copies.
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t % kDStages;
        const uint32_t ph = (t / kDStages) & 1;
        mbar_wait(bars.d_empty(s), ph ^ 1u, p.status, kDevTimeoutProducer);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(bars.d_full(s), d_tile_bytes<kE>());   // (pair: 12 KB from this CTA's loads + 12 KB from the peer's)
          const uint32_t dst = smem_base + S::kOffD + s * kDTileBytes;
          const int32_t row = kPlan ? __ldg(p.tile_row + tile_base + t) : row_begin + t * kTileN;
          if constexpr (kPair) {   // tmap_d has a (kTileN / 2)-row box here
            const uint32_t half = pair_rank * (kTileN / 2);
            tma_load_2d_multicast(dst + half * 128, &tmap_d, bars.d_full(s), 0, row + half, 3, kPolicyEvictFirst);
            tma_load_2d_multicast(dst + kDKBlockBytes + half * 128, &tmap_d, bars.d_full(s), 64, row + half, 3,
                                  kPolicyEvictFirst);
          } else if constexpr (kFp8) {   // tmap_d: e4m3 rows, one 128-column box
            tma_load_2d(dst, &tmap_d, bars.d_full(s), 0, row, kPolicyEvictFirst);
          } else {
            tma_load_2d(dst, &tmap_d, bars.d_full(s), 0, row, kPolicyEvictFirst);
            tma_load_2d(dst + kDKBlockBytes, &tmap_d, bars.d_full(s), 64, row, kPolicyEvictFirst);
          }
        }
        __syncwarp();
      }
    } else if (warp == kWarpRed0) {
      // ===================== reducer: score finalisation + per-CTA top-k =====================
      // Per D tile and per (query, passage ending in the tile): sum the row partials in fixed
      // order (deterministic), add/store partial scores if requested, offer to the top-k list.
      const int rw = warp - kWarpRed0;  // reducer 0..kRedWarps-1 owns queries b = rw (mod kRedWarps)
      const int q_off = static_cast<int>(pair_rank) * p.nq_pass;   // pair: CTA r's queries follow CTA 0's in every per-query array
      const float* partial = reinterpret_cast<const float*>(smem + S::kOffPartial);
      uint64_t* keys = reinterpret_cast<uint64_t*>(smem + S::kOffKeys);
      uint64_t* minkey_s = reinterpret_cast<uint64_t*>(smem + S::kOffMinKey);
      int* minpos_s = reinterpret_cast<int*>(smem + S::kOffMinPos);
      const int n_tiles_red = n_tiles;
      uint32_t mask_next = 0;
      int32_t fpid_next = 0;
      if (n_tiles_red > 0) {
        mask_next = __ldg(p.tile_end_mask + tile_base);
        fpid_next = __ldg(p.tile_first_pid + tile_base);
      }
      for (int t = 0; t < n_tiles_red; ++t) {
        const uint32_t mask = kPlan ? mask_next & ~kTileRunStart : mask_next;
        const int32_t first_pid = fpid_next;
        if (t + 1 < n_tiles_red) {
          mask_next = __ldg(p.tile_end_mask + tile_base + t + 1);
          fpid_next = __ldg(p.tile_first_pid + tile_base + t + 1);
        }
        const int buf = t & 1;
        mbar_wait(bars.p_full(buf), (static_cast<uint32_t>(t) >> 1) & 1u, p.status, kDevTimeoutEpilogue);
        const int n_slots = __popc(mask);
        const float* lane_part0 = reinterpret_cast<const float*>(smem + S::kOffLanePart);
  #pragma unroll 1
        for (int slot = 0; slot < n_slots; ++slot) {
          const int64_t pid = static_cast<int64_t>(first_pid) + slot;
          const float* lp_slot = lane_part0 + ((buf * kFastSlots + slot) * kRbMax) * kLaneStride;
          // a deleted passage (warp-uniform test, once per slot): never offered to the top-k, -inf in the score
          // output.  Its rows were still streamed and folded; only its partial sums are left unread.
          if (p.dead != nullptr && ((__ldg(p.dead + (pid >> 5)) >> (pid & 31)) & 1u)) {
            if (p.acc_out) store_dead_scores(p.acc_out + static_cast<int64_t>(q_off) * p.n_passages + pid,
                                             p.n_passages, p.nq_pass, lane);
            continue;
          }
          if (slot < kFastSlots && p.rbq <= p.lane_mode_max_rbq) {
            // many short queries per pass: lane = query, each lane sums its query's 2 * rbq row chunks in order
            // (transposed read of the stride-33 layout: conflict-free for rbq = 1)
  #pragma unroll 1
            for (int b0 = 0; b0 < p.nq_pass; b0 += 32) {
              const int b = b0 + lane;
              const bool valid = b < p.nq_pass;
              // this lane's query may return the passage (a disallowed lane stores -inf and makes no offer)
              const bool allowed = valid && pair_allowed(p, q_off + b, pid);
              float sc = 0.f;
              uint64_t key = 0ull;
              if (valid) {
                const float* lp = lp_slot + (b * p.rbq) * kLaneStride;
                for (int r = 0; r < p.rbq; ++r) {
                  sc += chunk_sum16(lp + r * kLaneStride);
                  sc += chunk_sum16(lp + r * kLaneStride + 16);
                }
                const int64_t gi = static_cast<int64_t>(q_off + b) * p.n_passages + pid;
                if (p.acc_in) sc += __ldg(p.acc_in + gi);
                if (!allowed) sc = -INFINITY;
                if (p.acc_out) p.acc_out[gi] = sc;
                key = (static_cast<uint64_t>(float_to_ordered(sc)) << 32) |
                      static_cast<uint64_t>(0xFFFFFFFFu - static_cast<uint32_t>(pid));
              }
              if (p.k > 0) {
                uint32_t hits = __ballot_sync(0xffffffffu, allowed && key > minkey_s[valid ? b : 0]);
                while (hits) {  // rare after warm-up: one list update at a time
                  const int src = __ffs(hits) - 1;
                  hits &= hits - 1;
                  const uint64_t cand = shfl64(key, src);
                  const int cb = b0 + src;
                  uint64_t minkey = minkey_s[cb];
                  int minpos = minpos_s[cb];
                  if (cand > minkey) {
                    topk_replace_min(keys + cb * kMaxK, p.k, cand, minkey, minpos, lane);
                    if (lane == 0) {
                      minkey_s[cb] = minkey;
                      minpos_s[cb] = minpos;
                    }
                    __syncwarp();
                  }
                }
              }
            }
          } else {
  #pragma unroll 1
            for (int b = 0; b < p.nq_pass; ++b) {
              // a pair the query's allow bitmap excludes (warp-uniform test): -inf in the score output, no offer
              if (!pair_allowed(p, q_off + b, pid)) {
                if (p.acc_out)
                  store_dead_scores(p.acc_out + static_cast<int64_t>(q_off + b) * p.n_passages + pid, p.n_passages, 1,
                                    lane);
                continue;
              }
              // score of (query b, passage pid): the whole warp adds the query's row chunks in row order
              float sc = 0.f;
              if (slot < kFastSlots) {
                // lane c < 2 rbq <= 24 sums chunk c (rows of lane c at bank (c >> 1) + 16 (c & 1) + q: conflict-free),
                // then every lane adds the chunks in order
                const int n_chunks = 2 * p.rbq;
                float ch = 0.f;
                if (lane < n_chunks)
                  ch = chunk_sum16(lp_slot + (b * p.rbq + (lane >> 1)) * kLaneStride + (lane & 1) * 16);
  #pragma unroll 4
                for (int c = 0; c < n_chunks; ++c) sc += __shfl_sync(0xffffffffu, ch, c);
              } else {
                const float* pr = partial + (buf * kHbMax + 2 * b * p.rbq) * kSlots + slot;
  #pragma unroll 2
                for (int r = 0; r < 2 * p.rbq; ++r) sc += pr[r * kSlots];
              }
              const int64_t gi = static_cast<int64_t>(q_off + b) * p.n_passages + pid;
              if (p.acc_in) sc += __ldg(p.acc_in + gi);
              if (p.acc_out && lane == 0) p.acc_out[gi] = sc;
              if (p.k > 0) {
                const uint64_t key = (static_cast<uint64_t>(float_to_ordered(sc)) << 32) |
                                     static_cast<uint64_t>(0xFFFFFFFFu - static_cast<uint32_t>(pid));
                uint64_t minkey = minkey_s[b];
                if (key > minkey) {  // warp-uniform; rare after warm-up
                  int minpos = minpos_s[b];
                  topk_replace_min(keys + b * kMaxK, p.k, key, minkey, minpos, lane);
                  if (lane == 0) {
                    minkey_s[b] = minkey;
                    minpos_s[b] = minpos;
                  }
                  __syncwarp();
                }
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bars.p_empty(buf));
      }
      // ---- publish this CTA's candidates ----
      if (p.k > 0) {
        __syncwarp();
        for (int b = rw; b < p.nq_pass; b += kRedWarps) {
          uint64_t* dst = p.cand_keys + (static_cast<int64_t>(cta) * p.cand_q_stride + p.cand_q_first + q_off + b) * p.k;
          for (int i = lane; i < p.k; i += 32) dst[i] = keys[b * kMaxK + i];
        }
      }
    }
  } else {
    // ===================== consumers: wgmma + passage maxima =====================
    const int wg = warp >> 2;
    const int wq = warp & 3;           // warp inside the warpgroup: accumulator rows 16 wq .. 16 wq + 15
    // warp-uniform block count of this warpgroup, dispatched to a loop that knows it at compile time (with a
    // run-time count ptxas serialises the wgmma of the two accumulators)
    const int nb = wg < n_blocks ? (n_blocks - wg + kWgs - 1) / kWgs : 0;
    if constexpr (kSplit) {
      if (nb == 1) {
        scan_split_consumer<1, kE, kPlan>(p, smem, smem_base, bars, n_tiles, tile_base, wg, wq, lane);
      } else if (nb == 2) {
        scan_split_consumer<2, kE, kPlan>(p, smem, smem_base, bars, n_tiles, tile_base, wg, wq, lane);
      }
    } else if (nb == 1) {
      scan_consumer<1, kWgs, kPair, kOverlap, kE, kPlan>(p, smem, smem_base, bars, n_tiles, tile_base, wg, wq, lane);
    } else if (nb == 2) {
      scan_consumer<2, kWgs, kPair, kOverlap, kE, kPlan>(p, smem, smem_base, bars, n_tiles, tile_base, wg, wq, lane);
    } else if constexpr (kBlocksPerWg >= 3) {
      if (nb == 3)
        scan_consumer<3, kWgs, kPair, kOverlap, kE, kPlan>(p, smem, smem_base, bars, n_tiles, tile_base, wg, wq, lane);
    }
  }

  // ---- teardown -----------------------------------------------------------------------------------
  if constexpr (kPair) cluster_sync_all();   // no CTA leaves while its peer may still signal its barriers
}

// Every scan kernel is instantiated per storage type kE; there is no CTA-pair kernel for fp16 or e4m3, and no
// three-warpgroup serial kernel for fp16 (launch_scan refuses a forced variant without an instantiation).
template <int kWgs, Elem kE, bool kPair = false>
__global__ void __launch_bounds__(scan_threads(kWgs), 1)
flmr_scan_kernel(const __grid_constant__ CUtensorMap tmap_d, const ScanParams p) {
  scan_kernel_body<kWgs, kPair, kE, false>(tmap_d, p);
}

// Three consumer warpgroups whose loop folds one half of each tile while the MMAs of the other half run
// (scan_split_consumer); bit-identical to flmr_scan_kernel<kWgs, kE>.
template <Elem kE>
__global__ void __launch_bounds__(scan_threads(3), 1)
flmr_scan_split_kernel(const __grid_constant__ CUtensorMap tmap_d, const ScanParams p) {
  scan_kernel_body<3, false, kE, true>(tmap_d, p);
}

// Plan mode (flmr_maxsim_topk_listed / flmr_maxsim_scores_listed): the two- and three-warpgroup loops over a plan of
// the listed passages' rows (see scan_kernel_body's kPlan).
template <Elem kE>
__global__ void __launch_bounds__(scan_threads(2), 1)
flmr_scan_listed_kernel(const __grid_constant__ CUtensorMap tmap_d, const ScanParams p) {
  scan_kernel_body<2, false, kE, false, true>(tmap_d, p);
}
template <Elem kE>
__global__ void __launch_bounds__(scan_threads(3), 1)
flmr_scan_listed_split_kernel(const __grid_constant__ CUtensorMap tmap_d, const ScanParams p) {
  scan_kernel_body<3, false, kE, true, true>(tmap_d, p);
}

}  // namespace flmr
