// flmr_train_tc_kernel.cuh — the training / re-scoring forward on the Hopper tensor cores (wgmma):
//
//   arg[b, p, i]    = argmax_{j : mask[p, j]} <Q[b, i, :], D[p, j, :]>        (lowest j on ties, -1 if none)
//   rowmax[b, p, i] = that maximum;   sum_i rowmax = MaxSim score[b, p]
//
// Same contract as flmr_argmax_mma_kernel (flmr_train_kernels.cuh), which stays the path for small batches;
// this one is for batches whose contraction is worth a TMA/wgmma pipeline — the global in-batch-negatives matrix
// of a training step with cross-rank negatives (CB/modeling/colbert.py:64-113, 115-163: 8 queries x 832 rows
// against 128 documents x 512 tokens per rank) or an exhaustive evaluation through ColBERT.score
// (src/executors/FLMR_executor.py:826-833).
//
// Two launches:
//   1. flmr_compact_docs_kernel: every document's unmasked tokens (ColBERT.doc masks padding AND punctuation,
//      colbert.py:199-210: holes anywhere) are packed to the front of a 128-token-aligned slot, the slot's tail
//      filled with copies of the last unmasked token (a duplicate cannot change a max and never wins the
//      lowest-index tie-break); `idx_map` remembers each packed token's position in the padded document.
//      After this no mask exists any more: the epilogue below has no per-element mask logic.
//   2. flmr_argmax_tc_kernel: CTA = (query b, 128-row tile of its tokens, a range of documents).  The query tile
//      is the stationary A operand (TMA -> shared memory once); the CTA streams its documents in chunks of 128
//      tokens through a kTcStages-deep ring of 32 KB shared-memory stages:
//        warp 8 (producer): TMA, two 128B-swizzled boxes per chunk
//        warps 0-7        : two consumer warpgroups; warpgroup g owns query rows [64 g, 64 g + 64) of the tile and
//                           issues 8 x wgmma.m64n128k16 per chunk into registers, then releases the stage.  A
//                           thread holds two rows and 32 columns per row: a compare-select TREE over its columns
//                           (strict '>' keeps the lower index on ties), two shuffles inside the lane quad, one
//                           compare against the row's running best; one store per output at the document's end.
#pragma once
#include "flmr_device.cuh"

namespace flmr {

constexpr int kTcTile = 128;                 // query rows per CTA and document tokens per chunk
constexpr int kTcStages = 4;                 // shared-memory chunks of the document ring
constexpr int kTcChunkBytes = kTcTile * 128 * 2;   // 32 KiB: [2 k-blocks][128 rows][64 bf16 or fp16]
constexpr int kTcKBlockBytes = kTcTile * 128;      // 16 KiB
constexpr int kTcWgs = 2;                    // consumer warpgroups, 64 query rows each
constexpr int kTcWarpProducer = kTcWgs * 4;
constexpr int kTcThreads = (kTcWarpProducer + 1) * 32;
constexpr int kTcSmemBytes = (1 + kTcStages) * kTcChunkBytes + 512 + 1024;   // A tile + ring + barriers, lengths + align

// grid = total documents; one 256-thread block packs one document.
__global__ void __launch_bounds__(256)
flmr_compact_docs_kernel(const uint4* __restrict__ d, const uint8_t* __restrict__ mask, int nd, int nd_c,
                         uint4* __restrict__ dc, int32_t* __restrict__ idx_map, int32_t* __restrict__ len_out) {
  __shared__ int s_cnt[256];
  __shared__ int s_last;
  const int p = blockIdx.x, tid = threadIdx.x;
  const uint8_t* mp = mask + static_cast<int64_t>(p) * nd;
  // each thread owns a contiguous slice of the document's tokens: exclusive scan of the per-slice counts
  const int per = (nd + 255) / 256;
  const int j0 = tid * per, j1 = min(nd, j0 + per);
  int cnt = 0;
  for (int j = j0; j < j1; ++j) cnt += mp[j] != 0;
  s_cnt[tid] = cnt;
  __syncthreads();
  for (int off = 1; off < 256; off <<= 1) {
    const int v = tid >= off ? s_cnt[tid - off] : 0;
    __syncthreads();
    s_cnt[tid] += v;
    __syncthreads();
  }
  const int len = s_cnt[255];
  int c = s_cnt[tid] - cnt;
  int32_t* im = idx_map + static_cast<int64_t>(p) * nd_c;
  for (int j = j0; j < j1; ++j)
    if (mp[j]) im[c++] = j;
  if (tid == 0) len_out[p] = len;
  __syncthreads();
  // copy rows: 16 threads per row (16 B each), packed position -> source token through idx_map
  const int len_pad = (len + kTcTile - 1) / kTcTile * kTcTile;
  const uint4* src = d + static_cast<int64_t>(p) * nd * 16;
  uint4* dst = dc + static_cast<int64_t>(p) * nd_c * 16;
  if (tid == 0) s_last = len > 0 ? im[len - 1] : 0;
  __syncthreads();
  for (int r = tid >> 4; r < len_pad; r += 16) {
    const int t = r < len ? im[r] : s_last;
    dst[r * 16 + (tid & 15)] = src[static_cast<int64_t>(t) * 16 + (tid & 15)];
  }
}

struct ArgmaxTcParams {
  const int32_t* doc_len;      // [n_docs_total] unmasked tokens per document
  const int32_t* idx_map;      // [n_docs_total][nd_c] packed position -> token index in the padded document
  int32_t* arg;                // [B][n_per][nq]
  float* rowmax;               // same shape, or null
  int32_t nq, nd_c, n_per, stride_b, docs_per_cta;
  int* status;                 // watchdog word (may be null)
};

// (value, column) pair that wins: the larger value, the lower column on equal values.
__device__ __forceinline__ void argmax_take(float& v, int& c, float v2, int c2) {
  if (v2 > v || (v2 == v && c2 < c)) {
    v = v2;
    c = c2;
  }
}

#define FLMR_TC_KERNEL flmr_argmax_tc_kernel
#define FLMR_TC_WGMMA wgmma_m64n128k16
#include "flmr_argmax_tc_body.cuh"
#undef FLMR_TC_KERNEL
#undef FLMR_TC_WGMMA

// fp16 operands (tensor maps encoded as FLOAT16): the same ring, descriptors, tree and epilogue, wgmma .f16.
#define FLMR_TC_KERNEL flmr_argmax_tc_f16_kernel
#define FLMR_TC_WGMMA wgmma_m64n128k16_f16
#include "flmr_argmax_tc_body.cuh"
#undef FLMR_TC_KERNEL
#undef FLMR_TC_WGMMA

}  // namespace flmr
