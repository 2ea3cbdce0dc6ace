// flmr_device.cuh — thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor, cluster multicast), thread-block clusters and wgmma.
// Hand-written for this repository; sm_90a only.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace flmr {

// Element type of a corpus' tokens and staged queries, and of the training kernels' operands.  bf16 and fp16 share
// everything but the MMA instruction (two bytes per element, two 128-B k-blocks per row); e4m3 has one byte per
// element, one k-block per row.
enum class Elem : int { kBF16 = 0, kF16 = 1, kE4M3 = 2 };

// ---- error codes written to ScanParams::status by the device-side watchdog -------------------
enum : int {
  kDevOk = 0,
  kDevTimeoutProducer = 101,
  kDevTimeoutMma = 102,
  kDevTimeoutEpilogue = 103,
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// One lane of the (fully converged) warp, the same lane every time.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes or the
// hint expires, instead of returning (and re-issuing the polling loop) after the short default limit.
// Without the hint ~20 % of all executed warp instructions of the scan kernel were polling iterations.
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(0x989680u)   // up to 10 ms per attempt
      : "memory");
  return ok != 0;
}

// Bounded wait: a protocol bug must surface as a trapped launch, never as a hung GPU box.
// `status` receives `code` before the trap so the host can say which role starved.
//
// The polling loop is written in PTX so that one iteration is the try_wait itself plus four instructions (a C++
// loop compiles to about 15), which keeps fine-grained waits cheap in issue slots.  The watchdog reads the timer
// once per kSpinBlock failed polls.
constexpr uint32_t kSpinBlock = 4096;
__device__ __forceinline__ uint32_t mbar_poll_block(uint32_t bar, uint32_t parity) {
  uint32_t n;
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 c;\n\t"
      "mov.u32 c, 0;\n"
      "FLMR_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "@p bra FLMR_DONE;\n\t"
      "add.u32 c, c, 1;\n\t"
      "setp.lt.u32 p, c, %4;\n\t"
      "@p bra FLMR_WAIT;\n"
      "FLMR_DONE:\n\t"
      "mov.u32 %0, c;\n\t}"
      : "=r"(n)
      : "r"(bar), "r"(parity), "r"(0x989680u), "r"(kSpinBlock)
      : "memory");
  return n;   // < kSpinBlock: the phase completed
}
// 20 s of polling = a protocol bug, not a slow wait (time slicing, a sanitizer or a debugger can stretch a
// legitimate wait to seconds; the longest real wait of a scan is one tile, microseconds)
// The same bounded wait with no function call, for waits while wgmma groups are in flight: ptxas cannot see what a
// call does with the accumulator registers, so it retires the in-flight wgmma before it (warning C7518).
__device__ __forceinline__ void mbar_wait_inline(uint32_t bar, uint32_t parity, int* status, int code) {
  constexpr uint64_t timeout_ns = 20000000000ull;
  uint64_t t0 = 0;
  while (mbar_poll_block(bar, parity) >= kSpinBlock) {
    const uint64_t now = global_timer_ns();
    if (t0 == 0) {
      t0 = now;
    } else if (now - t0 > timeout_ns) {
      if (status) *reinterpret_cast<volatile int*>(status) = code;
      __threadfence_system();
      __trap();
    }
  }
}
__device__ __noinline__ void mbar_wait_slow(uint32_t bar, uint32_t parity, int* status, int code) {
  mbar_wait_inline(bar, parity, status, code);
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* status, int code) {
  if (mbar_try_wait(bar, parity)) return;
  mbar_wait_slow(bar, parity, status, code);
}

// ---- TMA ----------------------------------------------------------------------------------------
constexpr uint64_t kPolicyEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kPolicyEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kPolicyEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// 2-D tiled load global -> shared, completion on an mbarrier (complete_tx::bytes).
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* map, uint32_t bar,
                                            int32_t c0, int32_t c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1),
      "l"(policy)
      : "memory");
}

// Same, delivered to the same shared-memory offset (and signalled on the same barrier offset) of EVERY CTA of the
// cluster whose bit is set in `cta_mask`.
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst_smem, const CUtensorMap* map, uint32_t bar,
                                                      int32_t c0, int32_t c1, uint16_t cta_mask, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask),
      "l"(policy)
      : "memory");
}

// ---- thread-block cluster ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Arrive once on the mbarrier at shared-memory offset `bar` of cluster CTA `cta` (this CTA included), with
// release semantics at cluster scope: the peer's waiter then sees every shared-memory read this thread ordered
// before the arrive as complete.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 r;\n\t"
      "mapa.shared::cluster.u32 r, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [r];\n\t}"
      ::"r"(bar), "r"(cta)
      : "memory");
}

// Generic-proxy writes to shared memory (st.shared) made visible to the async proxy (wgmma operand reads).
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- wgmma --------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (sm_90), K-major operand, 128-byte swizzle, rows of 128 B (64 bf16),
// 8-row groups 1024 B apart.  Field layout: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) |
// layout type [62,64) (1 = SWIZZLE_128B).  A K step of 16 elements inside the 128-byte row advances the
// start address by 32 bytes; the hardware applies the swizzle to the final address.
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;             // LBO (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;     // SBO: 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;             // SWIZZLE_128B
  return d;
}
// The two 32-bit words of make_kmajor_sw128_desc(smem_addr): the low word (start address and LBO) and the high word
// (SBO and layout type), which is the same for every address.
__device__ __forceinline__ uint32_t sw128_desc_lo(uint32_t smem_addr) { return ((smem_addr & 0x3FFFFu) >> 4) | (1u << 16); }
constexpr uint32_t kSw128DescHi = (1024 >> 4) | (1u << 30);

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Wait until at most N committed wgmma groups of this warpgroup are still in flight.
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Pins the accumulator registers in place across the asynchronous MMA: without it the compiler may read or
// move them between the issue and the wait.
template <int N>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Accumulator fragment of m64nNk16 (per warp of the warpgroup, 16 rows): d[4 i + 2 h + e] is row
// 16 * (warp % 4) + lane / 4 + 8 h, column 8 i + 2 * (lane % 4) + e.
// 8 accumulator operands of the wgmma wrappers below.
#define FLMR_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                   "+f"(d[i + 6]), "+f"(d[i + 7])
// D (+)= A[smem] * B[smem]^T, m64n96k16, bf16 in / fp32 accumulate; d[48] per thread.
__device__ __forceinline__ void wgmma_m64n96k16(float (&d)[48], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
      "}, %48, %49, p, 1, 1, 0, 0;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16), FLMR_F8(24), FLMR_F8(32), FLMR_F8(40)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D (+)= A[smem] * B[smem]^T, m64n96k16, fp16 in / fp32 accumulate; operands, layout and fragment of the bf16 form.
__device__ __forceinline__ void wgmma_m64n96k16_f16(float (&d)[48], uint64_t a_desc, uint64_t b_desc,
                                                    uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
      "}, %48, %49, p, 1, 1, 0, 0;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16), FLMR_F8(24), FLMR_F8(32), FLMR_F8(40)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D (+)= A[smem] * B[smem]^T, m64n96k32, e4m3 in / fp32 accumulate; d[48] per thread, the same fragment as
// m64n96k16.  fp8 operands are K-major only and take no transpose immediates.
__device__ __forceinline__ void wgmma_m64n96k32_e4m3(float (&d)[48], uint64_t a_desc, uint64_t b_desc,
                                                     uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k32.f32.e4m3.e4m3 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
      "}, %48, %49, p, 1, 1;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16), FLMR_F8(24), FLMR_F8(32), FLMR_F8(40)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D (+)= A[smem] * B[smem]^T, m64n48k16, bf16 in / fp32 accumulate; d[24] per thread (the fragment of m64n96k16
// restricted to its first six 8-column blocks).
__device__ __forceinline__ void wgmma_m64n48k16(float (&d)[24], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23"
      "}, %24, %25, p, 1, 1, 0, 0;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D (+)= A[smem] * B[smem]^T, m64n48k16, fp16 in / fp32 accumulate; operands, layout and fragment of the bf16 form.
__device__ __forceinline__ void wgmma_m64n48k16_f16(float (&d)[24], uint64_t a_desc, uint64_t b_desc,
                                                    uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23"
      "}, %24, %25, p, 1, 1, 0, 0;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D (+)= A[smem] * B[smem]^T, m64n48k32, e4m3 in / fp32 accumulate; d[24] per thread, the fragment of m64n48k16.
__device__ __forceinline__ void wgmma_m64n48k32_e4m3(float (&d)[24], uint64_t a_desc, uint64_t b_desc,
                                                     uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k32.f32.e4m3.e4m3 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23"
      "}, %24, %25, p, 1, 1;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D (+)= A[smem] * B[smem]^T, m64n128k16, bf16 in / fp32 accumulate; d[64] per thread.
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16), FLMR_F8(24), FLMR_F8(32), FLMR_F8(40), FLMR_F8(48), FLMR_F8(56)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D (+)= A[smem] * B[smem]^T, m64n128k16, fp16 in / fp32 accumulate; operands, layout and fragment of the bf16 form.
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t a_desc, uint64_t b_desc,
                                                     uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : FLMR_F8(0), FLMR_F8(8), FLMR_F8(16), FLMR_F8(24), FLMR_F8(32), FLMR_F8(40), FLMR_F8(48), FLMR_F8(56)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// ---- warp-level MMA (mma.sync m16n8k16, row.col, fp32 accumulate) ------------------------------------------------
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// The same with fp16 operands: fragments, layout and accumulation of the bf16 form.
__device__ __forceinline__ void mma_f16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Order-preserving map float -> uint32 (larger float <-> larger uint).
__host__ __device__ __forceinline__ uint32_t float_to_ordered(float f) {
#ifdef __CUDA_ARCH__
  uint32_t u = __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ordered_to_float(uint32_t u) {
  u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}

}  // namespace flmr
