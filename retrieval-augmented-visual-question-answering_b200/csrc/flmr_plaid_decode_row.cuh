// flmr_plaid_decode_row.cuh — the per-token arithmetic of the PLAID decode, included inside the token loop of every
// kernel that decodes PLAID rows (flmr_plaid_decode_kernel, flmr_plaid_window_decode_kernel, flmr_plaid_gather_kernel),
// so that all of them produce the same bits: the same fp32 additions, the same sum-of-squares shuffle order and one
// rounding to bf16 or (kF16) fp16.
//
// In scope where it is included: the template flag kF16; lane; nbits, keys (bucket indices per packed byte) and mask
// ((1 << nbits) - 1); s_w (the bucket weights in shared memory); normalize; c (the lane's 4 centroid values, a float4)
// and row (the token's packed residual bytes).  The whole warp runs it for one token (the shuffle needs every lane).
// It declares v and leaves the lane's 4 output values, packed, in `uint2 w`.
//
// A fragment rather than a __device__ function: a function inlined into flmr_plaid_decode_kernel allocates its
// registers differently, so that kernel would no longer compile to the code it had before the other two existed.
// No include guard: meant to be included more than once.
    float v[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) {
      const int i = 4 * lane + dd;
      const uint32_t byte = __ldg(row + i / keys);
      const uint32_t field = (byte >> (8 - nbits * (i % keys + 1))) & mask;
      v[dd] += s_w[__brev(field) >> (32 - nbits)];
    }
    if (normalize) {
      float ss = v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
      const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);   // torch.nn.functional.normalize eps
#pragma unroll
      for (int dd = 0; dd < 4; ++dd) v[dd] *= inv;
    }
    uint2 w;
    if constexpr (kF16) {
      __half2 lo = __floats2half2_rn(v[0], v[1]);
      __half2 hi = __floats2half2_rn(v[2], v[3]);
      w.x = *reinterpret_cast<uint32_t*>(&lo);
      w.y = *reinterpret_cast<uint32_t*>(&hi);
    } else {
      __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]);
      __nv_bfloat162 hi = __floats2bfloat162_rn(v[2], v[3]);
      w.x = *reinterpret_cast<uint32_t*>(&lo);
      w.y = *reinterpret_cast<uint32_t*>(&hi);
    }
