// flmr_train_kernels.cuh — backward of the all-pairs MaxSim used by training / RAG re-scoring
// (SURVEY.md 8f-2).  The reference differentiates colbert_score through torch autograd
// (third_party/ColBERT/colbert/modeling/colbert.py:235-286: matmul -> masked max -> sum), which keeps
// the [n, Nd, Nq] score tensor alive for the backward pass.  Here the forward keeps nothing: the
// backward recomputes, per (query, document) pair, WHICH document token wins each query token
// (flmr_argmax_kernel, 4 bytes per (b, p, i) instead of Nd*4), then routes the gradient:
//     dQ[b, i, :]            = sum_p g[b, p] * D[p, arg[b, p, i], :]      (gather,  flmr_bwd_dq_kernel)
//     dD[p, arg[b, p, i], :] += g[b, p] * Q[b, i, :]                       (scatter, flmr_bwd_dd_kernel)
// Shapes are training-sized (tens of documents, hundreds of tokens): a register-tiled SIMT fp32
// contraction over bf16 operands is within a few percent of what these sizes allow, so the kernels
// stay simple; the corpus-sized forward is the wgmma scan kernel.
//
// Every kernel has an fp16 twin under its own name (flmr_*_f16_kernel) for fp16 documents, the precision the
// reference's ColBERT.doc returns on the GPU (colbert.py:205-206): the same body (a template on the element kind),
// fp16 loads and fp16 MMAs, fp32 outputs.  The bf16 kernels keep their symbols and code.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "flmr_device.cuh"

namespace flmr {

constexpr int kArgTile = 64;        // query rows and document tokens per shared-memory tile
constexpr int kArgThreads = 256;    // 16 x 16 threads, 4 x 4 outputs each
constexpr int kArgStride = 132;     // bf16 per staged row: 264 B = 66 words -> conflict-free column reads

// Storage type of a training operand of element kind kE (bf16 or fp16).
template <Elem kE>
struct TrainElem {
  using T = __nv_bfloat16;
};
template <>
struct TrainElem<Elem::kF16> {
  using T = __half;
};
template <Elem kE>
using train_t = typename TrainElem<kE>::T;

__device__ __forceinline__ void bf16x4_to_float(uint2 v, float* f) {
  const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&v.x);
  const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&v.y);
  const float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
  f[0] = fa.x;
  f[1] = fa.y;
  f[2] = fb.x;
  f[3] = fb.y;
}

__device__ __forceinline__ void f16x4_to_float(uint2 v, float* f) {
  const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
  const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
  f[0] = fa.x;
  f[1] = fa.y;
  f[2] = fb.x;
  f[3] = fb.y;
}

// Four consecutive elements of kind kE, widened (exactly) to fp32.
template <Elem kE>
__device__ __forceinline__ void x4_to_float(uint2 v, float* f) {
  if constexpr (kE == Elem::kF16)
    f16x4_to_float(v, f);
  else
    bf16x4_to_float(v, f);
}

// arg[b, p, i] = argmax_{j : mask[p, j]} <Q[b, i, :], D[p, j, :]>   (lowest j on ties; -1 if p has no
// unmasked token); rowmax[b, p, i] = that maximum (optional: summed over i it is the MaxSim score, which
// makes this kernel the whole forward of a training-sized batch).  grid = (ceil(Nq / 64), n, B), block = 256.
// Query b meets the n documents [b * stride_b, b * stride_b + n): stride_b = 0 is the all-pairs form
// (every query against the same n documents), stride_b = n the block-diagonal one (query b against ITS n
// documents: the aligned `score(Q.repeat_interleave(n), D)` of colbert.py:71 / rag_model_blip.py:433 /
// FLMR_executor.py:828 without scoring the off-diagonal pairs).
template <Elem kE>
__device__ __forceinline__ void argmax_simt_body(const train_t<kE>* __restrict__ q, const train_t<kE>* __restrict__ d,
                                                 const uint8_t* __restrict__ mask, int nq, int nd, int n,
                                                 int stride_b, int32_t* __restrict__ arg, float* __restrict__ rowmax) {
  using T = train_t<kE>;
  __shared__ __align__(16) T qs[kArgTile * kArgStride];
  __shared__ __align__(16) T ds[kArgTile * kArgStride];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int i0 = blockIdx.x * kArgTile, p = blockIdx.y, b = blockIdx.z;
  const int64_t pg = static_cast<int64_t>(b) * stride_b + p;   // document row (stride_b = 0: all pairs)
  const T* qb = q + (static_cast<int64_t>(b) * nq + i0) * 128;
  const T* db = d + pg * nd * 128;
  const uint8_t* mp = mask + pg * nd;

  // stage the query tile once (rows past Nq read as zero; their results are never stored)
  for (int t = tid; t < kArgTile * 32; t += kArgThreads) {
    const int r = t >> 5, c = t & 31;   // 32 uint2 (4 bf16) per row
    uint2 v = make_uint2(0u, 0u);
    if (i0 + r < nq) v = *reinterpret_cast<const uint2*>(qb + static_cast<int64_t>(r) * 128 + c * 4);
    *reinterpret_cast<uint2*>(qs + r * kArgStride + c * 4) = v;
  }
  float best[4];
  int barg[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    best[r] = -INFINITY;
    barg[r] = -1;
  }
  for (int j0 = 0; j0 < nd; j0 += kArgTile) {
    __syncthreads();   // previous chunk fully consumed (and the query tile visible on the first trip)
    for (int t = tid; t < kArgTile * 32; t += kArgThreads) {
      const int r = t >> 5, c = t & 31;
      uint2 v = make_uint2(0u, 0u);
      if (j0 + r < nd) v = *reinterpret_cast<const uint2*>(db + static_cast<int64_t>(j0 + r) * 128 + c * 4);
      *reinterpret_cast<uint2*>(ds + r * kArgStride + c * 4) = v;
    }
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
#pragma unroll 4
    for (int k = 0; k < 128; k += 4) {
      float qf[4][4], df[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
        x4_to_float<kE>(*reinterpret_cast<const uint2*>(qs + (ty * 4 + r) * kArgStride + k), qf[r]);
#pragma unroll
      for (int c = 0; c < 4; ++c)
        x4_to_float<kE>(*reinterpret_cast<const uint2*>(ds + (tx + 16 * c) * kArgStride + k), df[c]);
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[r][c] = fmaf(qf[r][e], df[c][e], acc[r][c]);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {       // this thread's columns ascend with c and j0: '>' keeps the first
      const int j = j0 + tx + 16 * c;
      if (j < nd && mp[j]) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (acc[r][c] > best[r]) {
            best[r] = acc[r][c];
            barg[r] = j;
          }
      }
    }
  }
  // combine the 16 column owners of a row (one half-warp); ties -> lower token index
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best[r], off);
      const int oa = __shfl_xor_sync(0xffffffffu, barg[r], off);
      const bool take = oa >= 0 && (barg[r] < 0 || ob > best[r] || (ob == best[r] && oa < barg[r]));
      if (take) {
        best[r] = ob;
        barg[r] = oa;
      }
    }
    const int i = i0 + ty * 4 + r;
    if (tx == 0 && i < nq) {
      const int64_t o = (static_cast<int64_t>(b) * n + p) * nq + i;
      arg[o] = barg[r];
      if (rowmax) rowmax[o] = best[r];
    }
  }
}

__global__ void __launch_bounds__(kArgThreads)
flmr_argmax_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ d,
                   const uint8_t* __restrict__ mask, int nq, int nd, int n, int stride_b,
                   int32_t* __restrict__ arg, float* __restrict__ rowmax) {
  argmax_simt_body<Elem::kBF16>(q, d, mask, nq, nd, n, stride_b, arg, rowmax);
}
__global__ void __launch_bounds__(kArgThreads)
flmr_argmax_f16_kernel(const __half* __restrict__ q, const __half* __restrict__ d,
                       const uint8_t* __restrict__ mask, int nq, int nd, int n, int stride_b,
                       int32_t* __restrict__ arg, float* __restrict__ rowmax) {
  argmax_simt_body<Elem::kF16>(q, d, mask, nq, nd, n, stride_b, arg, rowmax);
}

// ---- the same contract on the warp-level tensor-core path (mma.sync m16n8k16, bf16 or fp16 -> fp32) -----------
// Training shapes are far too small to amortise the machinery of the scan kernel (mbarrier ring, TMA
// descriptors, a persistent grid), but the legacy warp MMA is still several times the SIMT FMA rate.
// CTA = 4 warps x 16 query rows; the query tile's A fragments are loaded once (ldmatrix) and stay in
// registers for every 64-token chunk of the document.
constexpr int kMmaThreads = 128;
constexpr int kMmaStride = 136;     // bf16 per staged row: 272 B, 16-B aligned rows, conflict-free ldmatrix

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_ptr) {
  const uint32_t addr = static_cast<uint32_t>(__cvta_generic_to_shared(smem_ptr));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

template <Elem kE>
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (kE == Elem::kF16)
    mma_f16_16816(c, a, b0, b1);
  else
    mma_bf16_16816(c, a, b0, b1);
}

template <Elem kE>
__device__ __forceinline__ void argmax_mma_body(const train_t<kE>* __restrict__ q, const train_t<kE>* __restrict__ d,
                                                const uint8_t* __restrict__ mask, int nq, int nd, int n,
                                                int stride_b, int32_t* __restrict__ arg, float* __restrict__ rowmax) {
  using T = train_t<kE>;
  __shared__ __align__(16) T qs[kArgTile * kMmaStride];
  __shared__ __align__(16) T ds[kArgTile * kMmaStride];
  __shared__ uint8_t ms[kArgTile];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int i0 = blockIdx.x * kArgTile, p = blockIdx.y, b = blockIdx.z;
  const int64_t pg = static_cast<int64_t>(b) * stride_b + p;   // document row (stride_b = 0: all pairs)
  const T* qb = q + (static_cast<int64_t>(b) * nq + i0) * 128;
  const T* db = d + pg * nd * 128;
  const uint8_t* mp = mask + pg * nd;

  for (int t = tid; t < kArgTile * 16; t += kMmaThreads) {     // 16 uint4 (8 bf16) per row
    const int r = t >> 4, c = t & 15;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (i0 + r < nq) v = *reinterpret_cast<const uint4*>(qb + static_cast<int64_t>(r) * 128 + c * 8);
    *reinterpret_cast<uint4*>(qs + r * kMmaStride + c * 8) = v;
  }
  __syncthreads();
  uint32_t a[8][4];                                            // this warp's 16 rows x K = 128
  {
    const int row = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int kc = (lane >> 4) * 8;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) ldmatrix_x4(a[ks], qs + row * kMmaStride + ks * 16 + kc);
  }
  float best[2] = {-INFINITY, -INFINITY};                      // rows g and g + 8 of the warp's 16
  int barg[2] = {-1, -1};
  for (int j0 = 0; j0 < nd; j0 += kArgTile) {
    __syncthreads();                                           // previous chunk fully consumed
    for (int t = tid; t < kArgTile * 16; t += kMmaThreads) {
      const int r = t >> 4, c = t & 15;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (j0 + r < nd) v = *reinterpret_cast<const uint4*>(db + static_cast<int64_t>(j0 + r) * 128 + c * 8);
      *reinterpret_cast<uint4*>(ds + r * kMmaStride + c * 8) = v;
    }
    if (tid < kArgTile) ms[tid] = (j0 + tid < nd) ? mp[j0 + tid] : 0;
    __syncthreads();
    float acc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {                         // two 8-token tiles per ldmatrix.x4
        uint32_t bf[4];
        const int tok = np * 16 + (lane & 7) + ((lane >> 4) & 1) * 8;
        const int kc = ks * 16 + ((lane >> 3) & 1) * 8;
        ldmatrix_x4(bf, ds + tok * kMmaStride + kc);
        mma_16816<kE>(acc[2 * np], a[ks], bf[0], bf[1]);
        mma_16816<kE>(acc[2 * np + 1], a[ks], bf[2], bf[3]);
      }
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)                             // this thread's columns ascend: '>' keeps the first
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int jl = nt * 8 + 2 * (lane & 3) + e;
        if (ms[jl]) {
          if (acc[nt][e] > best[0]) {
            best[0] = acc[nt][e];
            barg[0] = j0 + jl;
          }
          if (acc[nt][2 + e] > best[1]) {
            best[1] = acc[nt][2 + e];
            barg[1] = j0 + jl;
          }
        }
      }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {                                // combine the 4 column owners of a row
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best[r], off);
      const int oa = __shfl_xor_sync(0xffffffffu, barg[r], off);
      const bool take = oa >= 0 && (barg[r] < 0 || ob > best[r] || (ob == best[r] && oa < barg[r]));
      if (take) {
        best[r] = ob;
        barg[r] = oa;
      }
    }
    const int i = i0 + warp * 16 + (lane >> 2) + r * 8;
    if ((lane & 3) == 0 && i < nq) {
      const int64_t o = (static_cast<int64_t>(b) * n + p) * nq + i;
      arg[o] = barg[r];
      if (rowmax) rowmax[o] = best[r];
    }
  }
}

__global__ void __launch_bounds__(kMmaThreads)
flmr_argmax_mma_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ d,
                       const uint8_t* __restrict__ mask, int nq, int nd, int n, int stride_b,
                       int32_t* __restrict__ arg, float* __restrict__ rowmax) {
  argmax_mma_body<Elem::kBF16>(q, d, mask, nq, nd, n, stride_b, arg, rowmax);
}
__global__ void __launch_bounds__(kMmaThreads)
flmr_argmax_mma_f16_kernel(const __half* __restrict__ q, const __half* __restrict__ d,
                           const uint8_t* __restrict__ mask, int nq, int nd, int n, int stride_b,
                           int32_t* __restrict__ arg, float* __restrict__ rowmax) {
  argmax_mma_body<Elem::kF16>(q, d, mask, nq, nd, n, stride_b, arg, rowmax);
}

// dQ[b, i, :] = sum_p g[b, p] * D[p, arg[b, p, i], :].  One warp per (b, i), 4 dims per lane.
template <Elem kE>
__device__ __forceinline__ void bwd_dq_body(const train_t<kE>* __restrict__ d, const int32_t* __restrict__ arg,
                                            const float* __restrict__ g, int B, int nq, int n, int nd,
                                            int stride_b, float* __restrict__ dq) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= static_cast<int64_t>(B) * nq) return;
  const int b = static_cast<int>(w / nq), i = static_cast<int>(w % nq);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int p = 0; p < n; ++p) {
    const int j = arg[(static_cast<int64_t>(b) * n + p) * nq + i];
    const float gp = g[static_cast<int64_t>(b) * n + p];
    if (j < 0) continue;
    float f[4];
    x4_to_float<kE>(*reinterpret_cast<const uint2*>(
                        d + ((static_cast<int64_t>(b) * stride_b + p) * nd + j) * 128 + lane * 4), f);
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[e] = fmaf(gp, f[e], acc[e]);
  }
  *reinterpret_cast<float4*>(dq + w * 128 + lane * 4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
}
__global__ void flmr_bwd_dq_kernel(const __nv_bfloat16* __restrict__ d, const int32_t* __restrict__ arg,
                                   const float* __restrict__ g, int B, int nq, int n, int nd,
                                   int stride_b, float* __restrict__ dq) {
  bwd_dq_body<Elem::kBF16>(d, arg, g, B, nq, n, nd, stride_b, dq);
}
// launch bounds of 256 threads x 8 blocks: the register budget (32) of the bf16 kernel, which fp16 widening needs no
// more than (without them ptxas takes 40)
__global__ void __launch_bounds__(256, 8) flmr_bwd_dq_f16_kernel(const __half* __restrict__ d, const int32_t* __restrict__ arg,
                                       const float* __restrict__ g, int B, int nq, int n, int nd,
                                       int stride_b, float* __restrict__ dq) {
  bwd_dq_body<Elem::kF16>(d, arg, g, B, nq, n, nd, stride_b, dq);
}

// dD[p, arg[b, p, i], :] += g[b, p] * Q[b, i, :].  One warp per (b, p, i); fp32 atomics (the order of
// the additions, hence the last bits of dD, varies from run to run — as torch's index_add_ on CUDA).
template <Elem kE>
__device__ __forceinline__ void bwd_dd_body(const train_t<kE>* __restrict__ q, const int32_t* __restrict__ arg,
                                            const float* __restrict__ g, int B, int nq, int n, int nd,
                                            int stride_b, float* __restrict__ dd) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= static_cast<int64_t>(B) * n * nq) return;
  const int i = static_cast<int>(w % nq);
  const int64_t bp = w / nq;
  const int p = static_cast<int>(bp % n), b = static_cast<int>(bp / n);
  const int j = arg[w];
  const float gp = g[bp];
  if (j < 0 || gp == 0.f) return;
  float f[4];
  x4_to_float<kE>(*reinterpret_cast<const uint2*>(q + (static_cast<int64_t>(b) * nq + i) * 128 + lane * 4), f);
  float* dst = dd + ((static_cast<int64_t>(b) * stride_b + p) * nd + j) * 128 + lane * 4;
#pragma unroll
  for (int e = 0; e < 4; ++e) atomicAdd(dst + e, gp * f[e]);
}
__global__ void flmr_bwd_dd_kernel(const __nv_bfloat16* __restrict__ q, const int32_t* __restrict__ arg,
                                   const float* __restrict__ g, int B, int nq, int n, int nd,
                                   int stride_b, float* __restrict__ dd) {
  bwd_dd_body<Elem::kBF16>(q, arg, g, B, nq, n, nd, stride_b, dd);
}
__global__ void flmr_bwd_dd_f16_kernel(const __half* __restrict__ q, const int32_t* __restrict__ arg,
                                       const float* __restrict__ g, int B, int nq, int n, int nd,
                                       int stride_b, float* __restrict__ dd) {
  bwd_dd_body<Elem::kF16>(q, arg, g, B, nq, n, nd, stride_b, dd);
}

// In-batch-negatives loss head (compute_ib_loss_new, CB/modeling/colbert.py:82-113, after the MaxSim matrix):
// one block per query b.  scores[b, p] = sum_i rowmax[b, p, i] (fixed order: deterministic), then the
// cross-entropy against the positive at column label0 + b * nway and its gradient
//     loss_b = logsumexp_p scores[b, p] - scores[b, label_b],   dscores[b, p] = (softmax_p - [p == label_b]) / B
// — what torch would run as sum + log_softmax + nll_loss forward and their three backward kernels.
constexpr int kIbThreads = 256;
__global__ void __launch_bounds__(kIbThreads)
flmr_ib_loss_kernel(const float* __restrict__ rowmax, int B, int n, int nq, int nway, int label0,
                    float* __restrict__ scores, float* __restrict__ loss_q, float* __restrict__ dscores) {
  extern __shared__ float s_sc[];            // [n]
  __shared__ float s_red[kIbThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int p = warp; p < n; p += kIbThreads / 32) {
    const float* r = rowmax + (static_cast<int64_t>(b) * n + p) * nq;
    float acc = 0.f;
    for (int i = lane; i < nq; i += 32) acc += r[i];
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) {
      s_sc[p] = acc;
      scores[static_cast<int64_t>(b) * n + p] = acc;
    }
  }
  __syncthreads();
  float m = -INFINITY;
  for (int p = tid; p < n; p += kIbThreads) m = fmaxf(m, s_sc[p]);
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  m = s_red[0];
#pragma unroll
  for (int w = 1; w < kIbThreads / 32; ++w) m = fmaxf(m, s_red[w]);
  __syncthreads();
  float se = 0.f;
  for (int p = tid; p < n; p += kIbThreads) se += expf(s_sc[p] - m);
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) se += __shfl_xor_sync(0xffffffffu, se, off);
  if (lane == 0) s_red[warp] = se;
  __syncthreads();
  se = 0.f;
#pragma unroll
  for (int w = 0; w < kIbThreads / 32; ++w) se += s_red[w];
  const int label = label0 + b * nway;
  const float lse = m + logf(se);
  if (tid == 0) loss_q[b] = lse - s_sc[label];
  const float inv_b = 1.0f / static_cast<float>(B);
  for (int p = tid; p < n; p += kIbThreads)
    dscores[static_cast<int64_t>(b) * n + p] = (expf(s_sc[p] - lse) - (p == label ? 1.f : 0.f)) * inv_b;
}

// Padded batch of retrieved passages out of the resident corpus.  One warp per (slot, token row).  A deleted passage
// (bit set in `dead`, which may be null) gives the all-masked zero row of an id outside the shard.
__global__ void flmr_gather_kernel(const uint2* __restrict__ tokens, const int64_t* __restrict__ poff,
                                   const int32_t* __restrict__ doclen, const uint32_t* __restrict__ dead,
                                   const int64_t* __restrict__ pids,
                                   int64_t n_pids, int nd_max, int64_t n_passages, int64_t pid_base,
                                   uint2* __restrict__ out, uint8_t* __restrict__ mask) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n_pids * nd_max) return;
  const int64_t slot = w / nd_max;
  const int j = static_cast<int>(w % nd_max);
  const int64_t p = pids[slot] - pid_base;
  uint2 v = make_uint2(0u, 0u);
  bool real = false;
  if (p >= 0 && p < n_passages && j < doclen[p] && !(dead && ((dead[p >> 5] >> (p & 31)) & 1u))) {
    v = tokens[(poff[p] + j) * 32 + lane];
    real = true;
  }
  out[w * 32 + lane] = v;
  if (mask && lane == 0) mask[w] = real ? 1 : 0;
}

}  // namespace flmr
