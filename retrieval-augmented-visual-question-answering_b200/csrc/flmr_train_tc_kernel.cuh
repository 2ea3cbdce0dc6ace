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
constexpr int kTcChunkBytes = kTcTile * 128 * 2;   // 32 KiB: [2 k-blocks][128 rows][64 bf16]
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

__global__ void __launch_bounds__(kTcThreads, 1)
flmr_argmax_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
                      const ArgmaxTcParams p) {
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t a_smem = smem_base;                                   // query tile
  const uint32_t d_smem0 = smem_base + kTcChunkBytes;                  // ring of document chunks
  const uint32_t bar_base = smem_base + (1 + kTcStages) * kTcChunkBytes;
  const uint32_t bar_q = bar_base;
  auto bar_full = [&](int s) { return bar_base + 8u * (1 + s); };
  auto bar_free = [&](int s) { return bar_base + 8u * (1 + kTcStages + s); };          // consumers -> producer
  // lengths of this CTA's documents, read from global memory ONCE (every role walks the same document list)
  int32_t* s_len = reinterpret_cast<int32_t*>(smem + (1 + kTcStages) * kTcChunkBytes + 8 * (1 + 2 * kTcStages));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.z, mt = blockIdx.y;
  const int p_begin = blockIdx.x * p.docs_per_cta;
  const int p_end = min(p.n_per, p_begin + p.docs_per_cta);

  if (warp == kTcWarpProducer && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_d);
    mbar_init(bar_q, 1);
    for (int s = 0; s < kTcStages; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_free(s), kTcWgs);
    }
    mbar_fence_init();
  }
  if (warp == 0 && p_begin + lane < p_end)
    s_len[lane] = __ldg(p.doc_len + static_cast<int64_t>(b) * p.stride_b + p_begin + lane);   // docs_per_cta <= 32
  __syncthreads();

  if (warp == kTcWarpProducer) {
    // ===================== TMA producer =====================
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(bar_q, kTcChunkBytes);
      const int32_t row = b * p.nq + mt * kTcTile;
      tma_load_2d(a_smem, &tmap_q, bar_q, 0, row, kPolicyEvictNormal);
      tma_load_2d(a_smem + kTcKBlockBytes, &tmap_q, bar_q, 64, row, kPolicyEvictNormal);
    }
    __syncwarp();
    uint32_t n = 0;                                 // chunks issued so far
    for (int pl = p_begin; pl < p_end; ++pl) {
      const int64_t pg = static_cast<int64_t>(b) * p.stride_b + pl;
      const int nch = (s_len[pl - p_begin] + kTcTile - 1) / kTcTile;
      for (int c = 0; c < nch; ++c, ++n) {
        const int s = n % kTcStages;
        const uint32_t use = n / kTcStages;         // how often this stage was used before
        if (use > 0) mbar_wait(bar_free(s), (use - 1) & 1u, p.status, kDevTimeoutProducer);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(bar_full(s), kTcChunkBytes);
          const uint32_t dst = d_smem0 + s * kTcChunkBytes;
          const int32_t row = static_cast<int32_t>(pg * p.nd_c + c * kTcTile);
          tma_load_2d(dst, &tmap_d, bar_full(s), 0, row, kPolicyEvictNormal);
          tma_load_2d(dst + kTcKBlockBytes, &tmap_d, bar_full(s), 64, row, kPolicyEvictNormal);
        }
        __syncwarp();
      }
    }
  } else {
    // ===================== consumers: wgmma + running (max, index) per query row =====================
    const int wg = warp >> 2, wq = warp & 3;
    const int i0 = mt * kTcTile + wg * 64 + wq * 16 + (lane >> 2);   // this thread's query rows: i0 and i0 + 8
    const int cq = 2 * (lane & 3);                                   // its first column inside an 8-column block
    mbar_wait(bar_q, 0, p.status, kDevTimeoutMma);
    float acc[64];
    uint32_t n = 0;
    for (int pl = p_begin; pl < p_end; ++pl) {
      const int64_t pg = static_cast<int64_t>(b) * p.stride_b + pl;
      const int nch = (s_len[pl - p_begin] + kTcTile - 1) / kTcTile;
      float best[2] = {-INFINITY, -INFINITY};
      int barg[2] = {-1, -1};
      for (int c = 0; c < nch; ++c, ++n) {
        const int s = n % kTcStages;
        mbar_wait(bar_full(s), (n / kTcStages) & 1u, p.status, kDevTimeoutMma);
        const uint32_t d_smem = d_smem0 + s * kTcChunkBytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t koff = (k >> 2) * kTcKBlockBytes + (k & 3) * 32;
          wgmma_m64n128k16(acc, make_kmajor_sw128_desc(a_smem + wg * 64 * 128 + koff),
                           make_kmajor_sw128_desc(d_smem + koff), k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_operands(acc);
        __syncwarp();
        if (wq == 0 && lane == 0) mbar_arrive(bar_free(s));         // every wgmma of this warpgroup read the chunk
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // compare-select tree over this thread's 32 columns of row h (leaves in column order, so the
          // left operand always has the lower column and strict '>' keeps it on ties)
          float tv[16];
          int ti[16];
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            const float x0 = acc[4 * e + 2 * h], x1 = acc[4 * e + 2 * h + 1];
            const bool g1 = x1 > x0;
            tv[e] = g1 ? x1 : x0;
            ti[e] = 8 * e + cq + (g1 ? 1 : 0);
          }
#pragma unroll
          for (int w = 8; w >= 1; w >>= 1) {
#pragma unroll
            for (int e = 0; e < w; ++e) {
              const bool g1 = tv[2 * e + 1] > tv[2 * e];
              tv[e] = g1 ? tv[2 * e + 1] : tv[2 * e];
              ti[e] = g1 ? ti[2 * e + 1] : ti[2 * e];
            }
          }
          float v = tv[0];
          int col = ti[0];
#pragma unroll
          for (int off = 1; off <= 2; off <<= 1)
            argmax_take(v, col, __shfl_xor_sync(0xffffffffu, v, off), __shfl_xor_sync(0xffffffffu, col, off));
          if (v > best[h]) {                                     // strict: earlier chunks keep ties
            best[h] = v;
            barg[h] = c * kTcTile + col;
          }
        }
      }
      if ((lane & 3) == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = i0 + 8 * h;
          if (i < p.nq) {
            const int64_t o = (static_cast<int64_t>(b) * p.n_per + pl) * p.nq + i;
            p.arg[o] = barg[h] >= 0 ? __ldg(p.idx_map + pg * p.nd_c + barg[h]) : -1;
            if (p.rowmax) p.rowmax[o] = best[h];
          }
        }
      }
    }
  }
}

}  // namespace flmr
