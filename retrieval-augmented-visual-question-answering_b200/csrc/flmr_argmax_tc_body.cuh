// flmr_argmax_tc_body.cuh — the body of the wgmma arg-max kernel (see flmr_train_tc_kernel.cuh, which includes this
// file once per operand type with FLMR_TC_KERNEL = the kernel's name and FLMR_TC_WGMMA = its m64n128k16 MMA defined).
//
// A macro-parameterised kernel rather than a __device__ template called by two kernels: nvcc simplifies such a
// template on its own before inlining it, which reorders the index arithmetic of the compare-select tree, so the bf16
// kernel would no longer compile to the code it had before the fp16 form existed.  Included this way, the bf16
// kernel's source is the kernel's own body, as it was.
// No include guard: meant to be included more than once.

__global__ void __launch_bounds__(kTcThreads, 1)
FLMR_TC_KERNEL(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
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
          FLMR_TC_WGMMA(acc, make_kmajor_sw128_desc(a_smem + wg * 64 * 128 + koff),
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
