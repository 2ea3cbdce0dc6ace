// flmr_plaid_encode_kernel.cuh — PLAID encode on the Hopper tensor cores (flmr_plaid_encode):
//
//   code[t]     = argmax_c <x_t, C_c>            fp16 operands, fp32 accumulation, the lowest c on exact ties
//   best[t]     = that maximum
//   residual[t] = the token's bucket indices, nbits per dim, packed MSB-first (what ResidualCodec.binarize writes):
//                 r_d = fp16(float(x_t,d) - float(C_code,d)),  bucket_d = #{j : cutoffs[j] < float(r_d)}
//
// Neither the [K, n] score matrix nor the [n, 128] residual matrix exists anywhere: scores live in registers and
// each residual is bucketed and packed by the warp that computes it.
//
// One persistent CTA per SM walks token tiles of kEncRows rows (tile = blockIdx.x, blockIdx.x + gridDim.x, ...).
// The tile is the stationary A operand: TMA -> shared memory once per tile, as four 128-B swizzled boxes.  Centroids
// stream in tiles of kEncTileC rows through a kEncStages-deep ring of 32 KiB stages:
//   warp 8 (producer): TMA, the token tile, then every centroid tile of it; the ring runs on across token tiles (the
//                      rest of its warpgroup leaves at once; the warpgroup gives its registers to the consumers)
//   warps 0-7        : two consumer warpgroups; warpgroup g owns token rows [128 g, 128 g + 128) of the tile, as two
//                      64-row halves with one m64n128 accumulator each.  Per centroid tile it issues half 0, then
//                      half 1, and folds each half while the other half's MMAs run: the tensor pipe always has one
//                      commit group queued while the warpgroup compares.
// Fold: a max tree over a thread's 32 columns of a row, then one strict compare against the thread's running best,
// which only ever sees higher columns later; the column is looked up (the lowest one equal to the maximum) only when
// the best changes.  The lane quad is combined once per token tile (argmax_take, as flmr_argmax_tc_body.cuh: the
// lower column on equal values), so the result is the lowest column among the exact maxima.
// Columns past K in the last centroid tile (TMA fills them with zeros) are masked to -inf in that tile only.
//
// Epilogue (d_residuals != NULL): the warpgroup's codes go through shared memory; each warp then takes 32 of its
// rows, one row per step, lane = 4 dims: the token values from the swizzled A tile, the centroid row from global
// memory (L2), the residual rounded once to fp16, bucketed by a binary search over the cutoffs in shared memory
// (non-decreasing, as torch.bucketize requires), and written as the row's 16 nbits bytes.
//
// L2 traffic: every token tile reads all K * 256 bytes of centroids, i.e. kEncRows FLOP per byte.  256 rows per CTA
// (rather than the arg-max kernel's 128) halve that traffic at the same accumulator registers.
#pragma once
#include <cuda_fp16.h>

#include <type_traits>

#include "flmr_device.cuh"
#include "flmr_scan_kernel.cuh"        // kDim
#include "flmr_train_tc_kernel.cuh"    // argmax_take

namespace flmr {

constexpr int kEncRows = 256;                          // token rows per tile
constexpr int kEncHalfBytes = 128 * 128 * 2;           // one warpgroup's 128 rows: [2 k-blocks][128 rows][128 B]
constexpr int kEncKBlockBytes = 128 * 128;             // 16 KiB
constexpr int kEncTileC = 128;                         // centroids per stage
constexpr int kEncStageBytes = kEncTileC * 128 * 2;    // 32 KiB
constexpr int kEncStages = 4;
constexpr int kEncWgs = 2;
constexpr int kEncWarpProducer = kEncWgs * 4;
constexpr int kEncThreads = (kEncWgs + 1) * 128;       // the producer is a whole warpgroup (setmaxnreg works on those)
// registers per thread after setmaxnreg: 128 x 40 + 256 x 232 <= 64 K; the consumers hold two 64-float accumulators
constexpr int kEncProducerRegs = 40;
constexpr int kEncConsumerRegs = 232;
constexpr int kEncABytes = kEncWgs * kEncHalfBytes;    // 64 KiB
// A tile + ring + barriers (a_full, a_free, full[s], free[s]) + codes [256] + cutoffs [256] + alignment slack
constexpr int kEncSmemBytes = kEncABytes + kEncStages * kEncStageBytes + 8 * (2 + 2 * kEncStages) + 4 * 256 +
                              4 * 256 + 1024;

template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

struct PlaidEncodeParams {
  const __half* centroids;     // [K, 128]
  const float* cutoffs;        // [2^nbits - 1], non-decreasing; read only with residuals
  int32_t* codes;              // [n]
  uint8_t* residuals;          // [n, 16 nbits] or null: assignment only
  float* best;                 // [n] or null
  int64_t n;
  int32_t K, nbits, n_tiles;
  int* status;                 // watchdog word (may be null)
};

// The fold of row h (0: the thread's row r, 1: row r + 8) of one 64-row accumulator of centroid tile
// `col0 / kEncTileC` into the thread's running (max, column) of that row.  kMask: columns at or past `lim` (relative to col0) are not centroids.  The tile maximum of a row's 32
// columns is a max tree; only when it beats the running best (strict '>': an earlier tile keeps a tie), which for
// most tiles of a large K it does not, is the lowest column holding it looked up.
template <bool kMask, int h>
__device__ __forceinline__ void enc_fold_row(const float (&acc)[64], int col0, int lim, int cq, float& best, int& arg) {
  float tv[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) {
    float x0 = acc[4 * e + 2 * h], x1 = acc[4 * e + 2 * h + 1];
    if (kMask) {
      x0 = 8 * e + cq < lim ? x0 : -INFINITY;
      x1 = 8 * e + cq + 1 < lim ? x1 : -INFINITY;
    }
    tv[e] = fmaxf(x0, x1);
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) tv[e] = fmaxf(tv[2 * e], tv[2 * e + 1]);
#pragma unroll
  for (int e = 0; e < 4; ++e) tv[e] = fmaxf(tv[2 * e], tv[2 * e + 1]);
  tv[0] = fmaxf(fmaxf(tv[0], tv[1]), fmaxf(tv[2], tv[3]));
  if (tv[0] > best) {
    // the lowest column equal to the maximum (a column past K is never lower than a real one)
    int col = 0;
#pragma unroll
    for (int e = 15; e >= 0; --e) {
      col = acc[4 * e + 2 * h + 1] == tv[0] ? 8 * e + cq + 1 : col;
      col = acc[4 * e + 2 * h] == tv[0] ? 8 * e + cq : col;
    }
    best = tv[0];
    arg = col0 + col;
  }
}

// 8 x m64n128k16 over the full 128-dim contraction: rows at a_row0 (one 64-row half), centroids of stage c_stage.
__device__ __forceinline__ void enc_issue(float (&acc)[64], uint32_t a_row0, uint32_t c_stage) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t koff = (k >> 2) * kEncKBlockBytes + (k & 3) * 32;
    wgmma_m64n128k16_f16(acc, make_kmajor_sw128_desc(a_row0 + koff), make_kmajor_sw128_desc(c_stage + koff),
                         k > 0 ? 1u : 0u);
  }
  wgmma_commit();
}

__global__ void __launch_bounds__(kEncThreads, 1)
flmr_plaid_encode_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_c,
                         const PlaidEncodeParams p) {
  extern __shared__ uint8_t enc_smem_raw[];
  uint8_t* smem = enc_smem_raw + ((1024u - (smem_u32(enc_smem_raw) & 1023u)) & 1023u);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t a_smem = smem_base;
  const uint32_t c_smem0 = smem_base + kEncABytes;
  const uint32_t bar_base = c_smem0 + kEncStages * kEncStageBytes;
  const uint32_t bar_a_full = bar_base, bar_a_free = bar_base + 8;
  auto bar_full = [&](int s) { return bar_base + 8u * (2 + s); };
  auto bar_free = [&](int s) { return bar_base + 8u * (2 + kEncStages + s); };
  int32_t* s_code = reinterpret_cast<int32_t*>(smem + kEncABytes + kEncStages * kEncStageBytes + 8 * (2 + 2 * kEncStages));
  float* s_cut = reinterpret_cast<float*>(s_code + kEncRows);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nct = (p.K + kEncTileC - 1) / kEncTileC;
  if (warp == kEncWarpProducer && lane == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_c);
    mbar_init(bar_a_full, 1);
    mbar_init(bar_a_free, kEncWgs);
    for (int s = 0; s < kEncStages; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_free(s), kEncWgs);
    }
    mbar_fence_init();
  }
  if (p.residuals)
    for (int i = threadIdx.x; i < (1 << p.nbits) - 1; i += blockDim.x) s_cut[i] = p.cutoffs[i];
  __syncthreads();

  if (warp >= kEncWarpProducer) {
    // ===================== TMA producer: one warp of the last warpgroup =====================
    setmaxnreg_dec<kEncProducerRegs>();
    if (warp != kEncWarpProducer) return;
    uint32_t n = 0;                                   // centroid tiles issued so far (the ring's running count)
    int it = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x, ++it) {
      if (it > 0) mbar_wait(bar_a_free, (it - 1) & 1u, p.status, kDevTimeoutProducer);
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(bar_a_full, kEncABytes);
#pragma unroll
        for (int h = 0; h < kEncWgs; ++h)
#pragma unroll
          for (int kb = 0; kb < 2; ++kb)
            tma_load_2d(a_smem + h * kEncHalfBytes + kb * kEncKBlockBytes, &tmap_x, bar_a_full, 64 * kb,
                        tile * kEncRows + h * 128, kPolicyEvictFirst);
      }
      __syncwarp();
      for (int j = 0; j < nct; ++j, ++n) {
        const int s = n % kEncStages;
        const uint32_t use = n / kEncStages;
        if (use > 0) mbar_wait(bar_free(s), (use - 1) & 1u, p.status, kDevTimeoutProducer);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(bar_full(s), kEncStageBytes);
          const uint32_t dst = c_smem0 + s * kEncStageBytes;
          tma_load_2d(dst, &tmap_c, bar_full(s), 0, j * kEncTileC, kPolicyEvictLast);
          tma_load_2d(dst + kEncKBlockBytes, &tmap_c, bar_full(s), 64, j * kEncTileC, kPolicyEvictLast);
        }
        __syncwarp();
      }
    }
  } else {
    // ===================== consumers =====================
    setmaxnreg_inc<kEncConsumerRegs>();
    const int wg = warp >> 2, wq = warp & 3;
    const int cq = 2 * (lane & 3);
    const uint32_t a_half = a_smem + wg * kEncHalfBytes;
    const uint32_t a_r0 = a_half, a_r1 = a_half + 64 * 128;   // the warpgroup's two 64-row halves
    const int lim_last = p.K - (nct - 1) * kEncTileC;          // centroids in the last tile
    float acc0[64], acc1[64];
    uint32_t n = 0;                                            // centroid tiles consumed so far
    // the running (max, column) of the thread's four rows: half 0's rows r and r + 8, then half 1's
    float best0 = -INFINITY, best1 = -INFINITY, best2 = -INFINITY, best3 = -INFINITY;
    int arg0 = -1, arg1 = -1, arg2 = -1, arg3 = -1;
    // centroid tile j (ring slot n), entered with half 0's MMAs in flight in acc0; kNext: a tile j + 1 follows.
    // Only the last tile can hold columns past K.
    auto step = [&](int j, auto knext) {
      constexpr bool kNext = decltype(knext)::value;
      const uint32_t c_stage = c_smem0 + (n % kEncStages) * kEncStageBytes;
      const int lim = kNext ? kEncTileC : lim_last;
      // half 1 of tile j behind half 0's group; then fold half 0 under it
      enc_issue(acc1, a_r1, c_stage);
      wgmma_wait<1>();
      wgmma_fence_operands(acc0);
      enc_fold_row<!kNext, 0>(acc0, j * kEncTileC, lim, cq, best0, arg0);
      enc_fold_row<!kNext, 1>(acc0, j * kEncTileC, lim, cq, best1, arg1);
      // half 0 of tile j + 1 behind half 1's group; then fold half 1 under it
      if constexpr (kNext) {
        const uint32_t n1 = n + 1;
        mbar_wait_inline(bar_full(n1 % kEncStages), (n1 / kEncStages) & 1u, p.status, kDevTimeoutMma);
        enc_issue(acc0, a_r0, c_smem0 + (n1 % kEncStages) * kEncStageBytes);
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      wgmma_fence_operands(acc1);
      __syncwarp();
      if (wq == 0 && lane == 0) mbar_arrive(bar_free(n % kEncStages));   // both halves read the stage
      enc_fold_row<!kNext, 0>(acc1, j * kEncTileC, lim, cq, best2, arg2);
      enc_fold_row<!kNext, 1>(acc1, j * kEncTileC, lim, cq, best3, arg3);
      ++n;
    };
    int it = 0;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x, ++it) {
      best0 = best1 = best2 = best3 = -INFINITY;
      arg0 = arg1 = arg2 = arg3 = -1;
      // inline waits: the accumulators stay live across token tiles, and a call would have to save them
      mbar_wait_inline(bar_a_full, it & 1u, p.status, kDevTimeoutMma);
      mbar_wait_inline(bar_full(n % kEncStages), (n / kEncStages) & 1u, p.status, kDevTimeoutMma);
      enc_issue(acc0, a_r0, c_smem0 + (n % kEncStages) * kEncStageBytes);
      int j = 0;
      for (; j + 1 < nct; ++j) step(j, std::true_type{});
      step(j, std::false_type{});
      float best[4] = {best0, best1, best2, best3};
      int arg[4] = {arg0, arg1, arg2, arg3};
      // combine the lane quad: the larger value, the lower column on equal values
#pragma unroll
      for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1)
          argmax_take(best[r], arg[r], __shfl_xor_sync(0xffffffffu, best[r], off),
                      __shfl_xor_sync(0xffffffffu, arg[r], off));
      }
      const int64_t row0 = static_cast<int64_t>(tile) * kEncRows + wg * 128;   // the warpgroup's first token
      if ((lane & 3) == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int local = (r >> 1) * 64 + wq * 16 + (lane >> 2) + 8 * (r & 1);   // row within the warpgroup
          const int code = arg[r] < 0 ? 0 : arg[r];                             // no finite score at all: code 0
          s_code[wg * 128 + local] = code;
          if (row0 + local < p.n) {
            p.codes[row0 + local] = code;
            if (p.best) p.best[row0 + local] = best[r];
          }
        }
      }
      if (p.residuals) {
        named_bar_sync(1 + wg, 128);                           // the warpgroup's codes are in shared memory
        const int nbits = p.nbits;
        const int pbytes = 16 * nbits;                         // packed bytes per token
        // this lane's 4 dims (4 lane .. 4 lane + 3) inside a swizzled 128-B row: k-block, 16-B chunk, offset
        const int kb = lane >> 4, chunk = (lane & 15) >> 1, sub = 8 * (lane & 1);
        for (int rr = 0; rr < 32; ++rr) {
          const int local = wq * 32 + rr;
          const int64_t t = row0 + local;
          if (t >= p.n) break;
          const int code = s_code[wg * 128 + local];
          const uint2 xv = *reinterpret_cast<const uint2*>(
              smem + wg * kEncHalfBytes + kb * kEncKBlockBytes + local * 128 + ((chunk ^ (local & 7)) << 4) + sub);
          const uint2 cv = __ldg(reinterpret_cast<const uint2*>(p.centroids + static_cast<int64_t>(code) * kDim) + lane);
          const float2 x01 = __half22float2(*reinterpret_cast<const __half2*>(&xv.x));
          const float2 x23 = __half22float2(*reinterpret_cast<const __half2*>(&xv.y));
          const float2 c01 = __half22float2(*reinterpret_cast<const __half2*>(&cv.x));
          const float2 c23 = __half22float2(*reinterpret_cast<const __half2*>(&cv.y));
          const float diff[4] = {x01.x - c01.x, x01.y - c01.y, x23.x - c23.x, x23.y - c23.y};
          uint32_t val = 0;
#pragma unroll
          for (int dd = 0; dd < 4; ++dd) {
            const float r = __half2float(__float2half_rn(diff[dd]));
            uint32_t b = 0;                                    // #{j : cutoffs[j] < r}, cutoffs non-decreasing
            for (int step = 1 << (nbits - 1); step > 0; step >>= 1)
              if (s_cut[b + step - 1] < r) b += step;
            val = (val << nbits) | (__brev(b) >> (32 - nbits));   // bit j of the bucket at the j-th position
          }
          uint8_t* out = p.residuals + t * pbytes;
          if (nbits == 8) {
            reinterpret_cast<uint32_t*>(out)[lane] = __byte_perm(val, 0, 0x0123);
          } else if (nbits == 4) {
            reinterpret_cast<uint16_t*>(out)[lane] = static_cast<uint16_t>(__byte_perm(val, 0, 0x0001));
          } else if (nbits == 2) {
            out[lane] = static_cast<uint8_t>(val);
          } else {
            const uint32_t odd = __shfl_down_sync(0xffffffffu, val, 1);
            if ((lane & 1) == 0) out[lane >> 1] = static_cast<uint8_t>((val << 4) | odd);
          }
        }
      }
      named_bar_sync(1 + wg, 128);                             // every warp is done with the A tile and the codes
      if (wq == 0 && lane == 0) mbar_arrive(bar_a_free);
    }
  }
}

}  // namespace flmr
