// flmr_maxsim.cu — C-ABI implementation (include/flmr_maxsim.h) of the H100-native FLMR/ColBERT
// MaxSim + top-k path.  Host logic: corpus residency + partition metadata, query staging, pass
// planning, launches.  Device code: the fused scan kernel (flmr_scan_kernel.cuh) plus four small
// helper kernels (query staging, candidate merge, corpus repack, SIMT cross-check).
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared -Xcompiler -fPIC
// No libcuda link dependency: cuTensorMapEncodeTiled is resolved through the runtime's
// cudaGetDriverEntryPoint, so the library loads (and its symbols can be checked) without a GPU.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <mutex>
#include <new>
#include <cerrno>
#include <ctime>
#include <string>
#include <thread>
#include <vector>

#include "../../include/flmr_maxsim.h"
#include "flmr_scan_kernel.cuh"
#include "flmr_train_kernels.cuh"
#include "flmr_train_tc_kernel.cuh"
#include "flmr_plaid_encode_kernel.cuh"

namespace {

using namespace flmr;

static_assert(kMaxK == FLMR_MAX_K, "header / kernel top-k capacity mismatch");
static_assert(kGroup == FLMR_TOKEN_GROUP, "header / kernel token group mismatch");
static_assert(kDim == FLMR_DIM, "header / kernel dim mismatch");

// ---- error plumbing -----------------------------------------------------------------------------
thread_local std::string g_last_error;
thread_local int64_t g_launches = 0;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define FLMR_CUDA(expr)                                                                     \
  do {                                                                                      \
    cudaError_t e__ = (expr);                                                               \
    if (e__ != cudaSuccess)                                                                 \
      return fail(e__ == cudaErrorMemoryAllocation ? FLMR_ERR_OOM : FLMR_ERR_CUDA,          \
                  "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  bool ok = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) return;
    ok = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// ---- TMA descriptor encoding through the runtime-resolved driver entry point ------------------------
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int get_encode_fn(EncodeTiledFn* out) {
  static EncodeTiledFn fn = nullptr;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    FLMR_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || !p)
      return fail(FLMR_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  *out = fn;
  return FLMR_OK;
}

// ---- growable device matrices: driver virtual memory management, resolved like cuTensorMapEncodeTiled -------------
// A library-owned token matrix lives in a virtual address range reserved once, as large as the device's memory, and
// backed by physical allocations mapped behind its end as it grows.  An append therefore never copies the matrix and
// never needs room for two of it, and the matrix stays one contiguous 2-D tensor for the scan's TMA descriptor.
struct VmmApi {
  CUresult (*AddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*AddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*Create)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*Release)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*Map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*Unmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*SetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*Granularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
};

int get_vmm_api(const VmmApi** out) {
  static VmmApi api;
  static bool ok = false;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if (!ok) {
    VmmApi a;
    const std::pair<const char*, void**> names[] = {
        {"cuMemAddressReserve", reinterpret_cast<void**>(&a.AddressReserve)},
        {"cuMemAddressFree", reinterpret_cast<void**>(&a.AddressFree)},
        {"cuMemCreate", reinterpret_cast<void**>(&a.Create)},
        {"cuMemRelease", reinterpret_cast<void**>(&a.Release)},
        {"cuMemMap", reinterpret_cast<void**>(&a.Map)},
        {"cuMemUnmap", reinterpret_cast<void**>(&a.Unmap)},
        {"cuMemSetAccess", reinterpret_cast<void**>(&a.SetAccess)},
        {"cuMemGetAllocationGranularity", reinterpret_cast<void**>(&a.Granularity)}};
    for (const auto& n : names) {
      cudaDriverEntryPointQueryResult qres;
      FLMR_CUDA(cudaGetDriverEntryPoint(n.first, n.second, cudaEnableDefault, &qres));
      if (qres != cudaDriverEntryPointSuccess || !*n.second)
        return fail(FLMR_ERR_CUDA, "%s not available from the driver", n.first);
    }
    api = a;
    ok = true;
  }
  *out = &api;
  return FLMR_OK;
}

struct GrowableMatrix {
  CUdeviceptr base = 0;         // start of the reserved range (0: none)
  size_t reserved = 0;          // bytes of address space
  size_t mapped = 0;            // bytes backed by physical memory, from base
  size_t gran = 0;              // allocation granularity
  std::vector<std::pair<CUmemGenericAllocationHandle, size_t>> chunks;   // (allocation, bytes) in address order
};

#define FLMR_CU(expr)                                                                                   \
  do {                                                                                                  \
    CUresult r__ = (expr);                                                                              \
    if (r__ != CUDA_SUCCESS)                                                                            \
      return fail(r__ == CUDA_ERROR_OUT_OF_MEMORY ? FLMR_ERR_OOM : FLMR_ERR_CUDA, "%s failed (CUresult %d)", \
                  #expr, (int)r__);                                                                     \
  } while (0)

void gm_free(GrowableMatrix* g) {
  const VmmApi* api = nullptr;
  if (!g->base || get_vmm_api(&api)) return;
  size_t off = 0;
  for (auto& ch : g->chunks) {
    api->Unmap(g->base + off, ch.second);
    api->Release(ch.first);
    off += ch.second;
  }
  api->AddressFree(g->base, g->reserved);
  *g = GrowableMatrix();
}

// Largest physical allocation behind a growable matrix.  A growth is mapped as pieces of at most this size, so that a
// compaction (flmr_corpus_compact) can release every piece that lies wholly behind the matrix's new end; at most one
// piece per matrix then stays partly used.
constexpr size_t kGmPieceBytes = 1ull << 30;

// Back at least `bytes` of g with physical memory on `device` (reserving the range first if g has none).  Only the
// new tail is mapped, in pieces of at most kGmPieceBytes (the last one rounded up to the granularity): rows already
// there stay where they are.  On failure the pieces this call mapped are released again.
int gm_grow(GrowableMatrix* g, int device, size_t bytes) {
  const VmmApi* api = nullptr;
  if (int rc = get_vmm_api(&api)) return rc;
  CUmemAllocationProp prop{};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  if (!g->base) {
    FLMR_CUDA(cudaFree(nullptr));   // the device's primary context is current for the driver calls
    size_t free_b = 0, total_b = 0;
    FLMR_CUDA(cudaMemGetInfo(&free_b, &total_b));
    FLMR_CU(api->Granularity(&g->gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    const size_t reserve = (total_b + g->gran - 1) / g->gran * g->gran;
    FLMR_CU(api->AddressReserve(&g->base, reserve, g->gran, 0, 0));
    g->reserved = reserve;
  }
  if (bytes <= g->mapped) return FLMR_OK;
  const size_t add = (bytes - g->mapped + g->gran - 1) / g->gran * g->gran;
  if (g->mapped + add > g->reserved)
    return fail(FLMR_ERR_OOM, "a token matrix of %zu bytes exceeds the device's %zu bytes", bytes, g->reserved);
  const size_t piece_max = std::max(g->gran, kGmPieceBytes / g->gran * g->gran);
  const size_t mapped0 = g->mapped, chunks0 = g->chunks.size();
  CUmemAccessDesc acc{};
  acc.location = prop.location;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  CUresult r = CUDA_SUCCESS;
  while (g->mapped < mapped0 + add) {
    const size_t piece = std::min(piece_max, mapped0 + add - g->mapped);
    CUmemGenericAllocationHandle h;
    r = api->Create(&h, piece, &prop, 0);
    if (r != CUDA_SUCCESS) break;
    r = api->Map(g->base + g->mapped, piece, 0, h, 0);
    if (r == CUDA_SUCCESS) {
      r = api->SetAccess(g->base + g->mapped, piece, &acc, 1);
      if (r != CUDA_SUCCESS) api->Unmap(g->base + g->mapped, piece);
    }
    if (r != CUDA_SUCCESS) {
      api->Release(h);
      break;
    }
    g->chunks.emplace_back(h, piece);
    g->mapped += piece;
  }
  if (r != CUDA_SUCCESS) {
    while (g->chunks.size() > chunks0) {   // give back what this call mapped: the matrix is as it was
      const auto ch = g->chunks.back();
      g->mapped -= ch.second;
      api->Unmap(g->base + g->mapped, ch.second);
      api->Release(ch.first);
      g->chunks.pop_back();
    }
    return fail(r == CUDA_ERROR_OUT_OF_MEMORY ? FLMR_ERR_OOM : FLMR_ERR_CUDA,
                "mapping %zu bytes behind the token matrix failed (CUresult %d)", add, (int)r);
  }
  return FLMR_OK;
}

// Unmap and release every piece of g that lies wholly at or behind byte `bytes`; returns the bytes released.  The
// rows in front stay mapped where they are, and a later gm_grow maps behind the new end.
size_t gm_shrink(GrowableMatrix* g, size_t bytes) {
  const VmmApi* api = nullptr;
  if (!g->base || get_vmm_api(&api)) return 0;
  size_t released = 0;
  while (!g->chunks.empty() && g->mapped - g->chunks.back().second >= bytes) {
    const auto ch = g->chunks.back();
    g->mapped -= ch.second;
    api->Unmap(g->base + g->mapped, ch.second);
    api->Release(ch.first);
    g->chunks.pop_back();
    released += ch.second;
  }
  return released;
}

// bf16 (or fp16) [rows, 128] row-major matrix, box = 64 columns (128 B, one swizzle span) x box_rows rows; e4m3: a
// [rows, 128] matrix (as bytes), box = 128 columns (128 B) x box_rows rows.
int encode_rows_map(CUtensorMap* map, const void* base, uint64_t rows, uint32_t box_rows, Elem elem = Elem::kBF16) {
  const bool fp8 = elem == Elem::kE4M3;
  EncodeTiledFn enc = nullptr;
  int rc = get_encode_fn(&enc);
  if (rc) return rc;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(kDim), static_cast<cuuint64_t>(rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(kDim) * (fp8 ? 1 : 2)};
  const cuuint32_t box[2] = {fp8 ? 128u : 64u, box_rows};
  const cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(map,
                   fp8                   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                   : elem == Elem::kF16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                         : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                   2,
                   const_cast<void*>(base), gdim, gstride,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(FLMR_ERR_CUDA, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
  return FLMR_OK;
}

// ---- helper kernels --------------------------------------------------------------------------------

// Eight bf16 (16 bytes) -> eight e4m3 (8 bytes): bf16 -> f32 is exact, f32 -> e4m3 rounds to nearest even and
// saturates at +-448 (cvt.rn.satfinite.e4m3x2.f32).  No scale: a zero stays exactly zero.
__device__ __forceinline__ uint32_t bf16x4_to_e4m3x4(uint32_t a, uint32_t b) {
  const float2 fa = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&a));
  const float2 fb = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&b));
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(fa, __NV_SATFINITE, __NV_E4M3);   // element 0 in the low byte
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(fb, __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
__device__ __forceinline__ uint2 bf16x8_to_e4m3x8(uint4 v) {
  return make_uint2(bf16x4_to_e4m3x4(v.x, v.y), bf16x4_to_e4m3x4(v.z, v.w));
}

// Stage the resident queries of EVERY pass of a call in one launch (blockIdx.y = pass): each query padded
// with zero rows to rbq*32 rows, the pass's block padded with zero rows to n_mtiles*128 rows, pass i at
// qpad + i * kMtMax*128 rows.  One thread per 16 bytes of output.  kFp8: the rows are written as e4m3 (128 B per
// row, the slots keep their bf16 stride).
constexpr int kStageMaxPasses = 64;
struct StagePass {
  int32_t q_first, n_q, row0, rows, rbq, n_rows_pad;
};
struct StageParams {
  StagePass pass[kStageMaxPasses];
};
template <bool kFp8>
__global__ void flmr_stage_queries_kernel(const uint4* __restrict__ q, uint4* __restrict__ qpad,
                                          int nq_total_rows, const __grid_constant__ StageParams sp) {
  constexpr int kChunkBits = kFp8 ? 3 : 4;   // log2 of the 16-byte output chunks per row
  const StagePass& ps = sp.pass[blockIdx.y];
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = idx >> kChunkBits, c = idx & ((1 << kChunkBits) - 1);
  if (r >= ps.n_rows_pad) return;
  const int rows_q = ps.rbq * 32;
  const int b = r / rows_q, i = r % rows_q;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (b < ps.n_q && i < ps.rows) {
    const uint4* row = q + (static_cast<int64_t>(ps.q_first + b) * nq_total_rows + ps.row0 + i) * 16;
    if constexpr (kFp8) {
      const uint2 lo = bf16x8_to_e4m3x8(row[2 * c]), hi = bf16x8_to_e4m3x8(row[2 * c + 1]);
      v = make_uint4(lo.x, lo.y, hi.x, hi.y);
    } else {
      v = row[c];
    }
  }
  qpad[static_cast<int64_t>(blockIdx.y) * (kMtMax * kTileM * 16) + idx] = v;
}

// Copy passages into the padded layout: passage p occupies rows [poff[p], poff[p+1]) of dst, its
// last token repeated over the padding rows.  One warp per passage, 2 rows per iteration.  dst8 (an e4m3 corpus,
// may be null): the same rows converted to e4m3, in the same layout with 128-byte rows.
__global__ void flmr_repack_kernel(const uint4* __restrict__ src, const int64_t* __restrict__ soff,
                                   const int64_t* __restrict__ poff, uint4* __restrict__ dst,
                                   uint2* __restrict__ dst8, int64_t p_begin, int64_t p_count,
                                   int64_t src_row_base) {
  const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= p_count) return;
  const int64_t p = p_begin + w;
  const int64_t s0 = soff[p], len = soff[p + 1] - s0;
  const int64_t d0 = poff[p], plen = poff[p + 1] - d0;
  const int half = lane >> 4, c = lane & 15;
  for (int64_t j = half; j < plen; j += 2) {
    const int64_t sj = j < len ? j : len - 1;
    const uint4 v = src[(s0 - src_row_base + sj) * 16 + c];
    dst[(d0 + j) * 16 + c] = v;
    if (dst8) dst8[(d0 + j) * 16 + c] = bf16x8_to_e4m3x8(v);
  }
}

// Streamed corpus load: rows [s0, s0 + n) of the PACKED source order (staged at `src`) go to their place in the
// padded layout; the last token of a passage is also copied over its padding rows.  Chunks need not start or end
// on passage boundaries.  One half-warp per row; the passage of a row is found by binary search in `soff`.
// dst8 (may be null): the rows also go to an e4m3 matrix of the same layout, as in flmr_repack_kernel.
__global__ void flmr_scatter_rows_kernel(const uint4* __restrict__ src, const int64_t* __restrict__ soff,
                                         const int64_t* __restrict__ poff, uint4* __restrict__ dst,
                                         uint2* __restrict__ dst8, int64_t s0, int64_t n, int64_t n_passages) {
  const int64_t r = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 4;
  const int c = threadIdx.x & 15;
  if (r >= n) return;
  const int64_t srow = s0 + r;
  int64_t lo = 0, hi = n_passages;          // largest p with soff[p] <= srow
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (soff[mid] <= srow) lo = mid; else hi = mid;
  }
  const uint4 v = src[r * 16 + c];
  const uint2 v8 = dst8 ? bf16x8_to_e4m3x8(v) : make_uint2(0u, 0u);
  const int64_t d = poff[lo] + (srow - soff[lo]);
  const int64_t d_end = srow == soff[lo + 1] - 1 ? poff[lo + 1] : d + 1;   // last token: fill the group padding
  for (int64_t j = d; j < d_end; ++j) {
    dst[j * 16 + c] = v;
    if (dst8) dst8[j * 16 + c] = v8;
  }
}

// Rows of bf16 rounded to e4m3 and back (exact: every e4m3 value is a bf16 value), 16 bytes per thread: the queries
// of the SIMT cross-check on an e4m3 corpus.
__global__ void flmr_round_e4m3_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int64_t n_chunks) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_chunks) return;
  const uint2 v8 = bf16x8_to_e4m3x8(src[i]);
  const uint32_t w[2] = {v8.x, v8.y};
  uint32_t out[4];
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w[h >> 1] >> (16 * (h & 1))),
                                                     __NV_E4M3);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
    const __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
    out[h] = *reinterpret_cast<const uint32_t*>(&b);
  }
  dst[i] = make_uint4(out[0], out[1], out[2], out[3]);
}

// ---- compacted corpora: rows stored by slot, ids through the slot -> id map -------------------------------------
// slot_pid[0 .. n_slots) holds the global id of each slot, strictly increasing.  The slot of global id `gid`, or -1
// if it has none.
__device__ __forceinline__ int64_t slot_of(const int64_t* __restrict__ slot_pid, int64_t n_slots, int64_t gid) {
  int64_t lo = 0, hi = n_slots;   // first slot whose id is >= gid
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(slot_pid + mid) < gid) lo = mid + 1; else hi = mid;
  }
  return lo < n_slots && __ldg(slot_pid + lo) == gid ? lo : -1;
}

// Compaction row move: destination rows [d0, d0 + rows) of one chunk, each read from the source row its piece gives.
// The chunk's pieces k0 .. k1 - 1 are sorted by destination (piece k starts at destination row pdst[k] and reads from
// source row psrc[k] on); their destinations are contiguous.  Row r is written at dst + (r - dst_row0) rows: in place
// (dst_row0 = 0) when the chunk's destinations overlap none of its sources, else into the staging buffer
// (dst_row0 = d0).  One thread per 16 bytes, row_vecs of them per row.  src and dst may be the same matrix, so they
// are not declared __restrict__.
__global__ void flmr_move_rows_kernel(const uint4* src, uint4* dst, const int64_t* __restrict__ pdst,
                                      const int64_t* __restrict__ psrc, int64_t k0, int64_t k1, int64_t d0,
                                      int64_t rows, int64_t dst_row0, int row_vecs) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * row_vecs) return;
  const int64_t r = d0 + i / row_vecs;
  const int c = static_cast<int>(i % row_vecs);
  int64_t lo = k0, hi = k1;   // last piece starting at or before r
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(pdst + mid) <= r) lo = mid; else hi = mid;
  }
  const int64_t s = __ldg(psrc + lo) + (r - __ldg(pdst + lo));
  dst[(r - dst_row0) * row_vecs + c] = src[s * row_vecs + c];
}

// Id-indexed allow bitmaps (the caller's, `stride` words apart; 0: one shared bitmap) -> the slot-indexed bitmaps the
// scan of a compacted corpus tests, `words` words apart.  One thread per output word.
__global__ void flmr_slot_allow_kernel(const uint32_t* __restrict__ allow, int64_t stride,
                                       const int64_t* __restrict__ slot_pid, int64_t pid_base, int64_t n_slots,
                                       int64_t words, int64_t n_bitmaps, uint32_t* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_bitmaps * words) return;
  const int64_t b = i / words, w = i % words;
  const uint32_t* row = allow + b * stride;
  uint32_t bits = 0u;
  for (int j = 0; j < 32; ++j) {
    const int64_t s = w * 32 + j;
    if (s >= n_slots) break;
    const int64_t p = __ldg(slot_pid + s) - pid_base;
    bits |= ((__ldg(row + (p >> 5)) >> (p & 31)) & 1u) << j;
  }
  out[i] = bits;
}

// Global ids -> the ids the slot-indexed gather reads: pid_base + slot, or pid_base - 1 (outside the shard) for an id
// without a slot (compacted away, or not in this shard).
__global__ void flmr_slot_ids_kernel(const int64_t* __restrict__ pids, int64_t n, const int64_t* __restrict__ slot_pid,
                                     int64_t n_slots, int64_t pid_base, int64_t* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t s = slot_of(slot_pid, n_slots, pids[i]);
  out[i] = pid_base + (s >= 0 ? s : -1);
}

// Slot-indexed score rows [n_rows, n_slots] -> id-indexed rows [n_rows, n_ids]: an id without a slot scores -inf,
// as a deleted passage does.  One thread per output score.
__global__ void flmr_expand_slot_scores_kernel(const float* __restrict__ src, int64_t n_slots,
                                               const int64_t* __restrict__ slot_pid, int64_t pid_base, int64_t n_ids,
                                               int64_t n_rows, float* __restrict__ dst) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_rows * n_ids) return;
  const int64_t b = i / n_ids, p = i % n_ids;
  const int64_t s = slot_of(slot_pid, n_slots, pid_base + p);
  dst[i] = s >= 0 ? src[b * n_slots + s] : -INFINITY;
}

// ---- listed search: the per-call scan plan over the listed passages' rows (flmr_maxsim_*_listed) ----------------
// Slot of global id `gid`, or -1: outside the shard, or compacted away (slot_pid null: slot = local id).
__device__ __forceinline__ int64_t listed_slot(int64_t gid, const int64_t* __restrict__ slot_pid, int64_t n_slots,
                                               int64_t pid_base, int64_t n_ids) {
  const int64_t local = gid - pid_base;
  if (local < 0 || local >= n_ids) return -1;
  return slot_pid ? slot_of(slot_pid, n_slots, gid) : local;
}

// Query of list entry i: the last b < n_q with off[b] <= i (off: the chunk's CSR offsets, off[0] <= i < off[n_q]).
__device__ __forceinline__ int listed_query(const int64_t* __restrict__ off, int n_q, int64_t i) {
  int lo = 0, hi = n_q;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// Entries [off[0], off[n_q]) of the lists -> the queries' slot bitmaps (`words` words apart, zeroed by the caller): the
// allow test of the plan-mode reducer, and the planner's input.  One thread per entry.
__global__ void flmr_listed_mark_kernel(const int64_t* __restrict__ pids, const int64_t* __restrict__ off, int n_q,
                                        const int64_t* __restrict__ slot_pid, int64_t n_slots, int64_t pid_base,
                                        int64_t n_ids, int64_t words, uint32_t* __restrict__ allow) {
  const int64_t i = __ldg(off) + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= __ldg(off + n_q)) return;
  const int64_t s = listed_slot(__ldg(pids + i), slot_pid, n_slots, pid_base, n_ids);
  if (s < 0) return;
  atomicOr(allow + listed_query(off, n_q, i) * words + (s >> 5), 1u << (s & 31));
}

// Slot-indexed score rows [n_q, n_slots] -> the scores of entries [off[0], off[n_q]), aligned with the lists: -inf for
// an id without a slot.  One thread per entry.
__global__ void flmr_listed_scores_kernel(const int64_t* __restrict__ pids, const int64_t* __restrict__ off, int n_q,
                                          const int64_t* __restrict__ slot_pid, int64_t n_slots, int64_t pid_base,
                                          int64_t n_ids, const float* __restrict__ src, float* __restrict__ out) {
  const int64_t i = __ldg(off) + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= __ldg(off + n_q)) return;
  const int64_t s = listed_slot(__ldg(pids + i), slot_pid, n_slots, pid_base, n_ids);
  out[i] = s >= 0 ? src[listed_query(off, n_q, i) * n_slots + s] : -INFINITY;
}

constexpr int kPlanThreads = 1024;

// Exclusive scan of x over the kPlanThreads threads of the block under `op` (identity `id`); *total = the reduction
// of every thread's x.  `s` is 32 elements of shared memory; every thread must call it.
template <typename T, typename Op>
__device__ __forceinline__ T block_exclusive_scan(T x, T id, Op op, T* s, T* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T incl = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl = op(y, incl);
  }
  if (lane == 31) s[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    T w = s[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w = op(y, w);
    }
    s[lane] = w;
  }
  __syncthreads();
  T excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = id;
  if (warp > 0) excl = op(s[warp - 1], excl);
  *total = s[31];
  __syncthreads();   // s is reused by the next call
  return excl;
}

// One pass of a listed search, as the planner sees it.  Offsets are in elements of the plan's arrays.
struct ListedPass {
  int32_t q_first, n_q;   // queries of the pass (bitmaps allow + (q_first .. q_first + n_q - 1) * words)
  int64_t u_off;          // its union entries: u_slot / u_cum / u_tile [u_off, u_off + union bound)
  int64_t c_off;          // its cta_tile_base [c_off, c_off + n_ctas + 1)
  int64_t t_off;          // its tiles: tile_row / tile_mask / tile_first [t_off, t_off + tile bound)
};

// The planner: one block per pass.
//   1. the union of the pass's queries' slot bitmaps -> its slots, sorted and unique (u_slot);
//   2. their stored rows -> each one's first row inside the union (u_cum) and the union's rows R;
//   3. the union is cut into CTA shares at passage boundaries, as build_partition cuts the corpus (CTA c starts at the
//      first passage at or past row R c / n_ctas), and into runs of consecutive slots inside a share; each run is
//      tiled from its first row in steps of 96 rows (u_tile: the run's first tile).  A tile's end mask marks the ends
//      of the run's passages that fall in it (bit g: 4-token group g, as tile_end_mask), plus kTileRunStart on a
//      run's first tile; tile_first is the first slot ending in the tile;
//   4. cta_tile_base: CTA c's tiles, in the scan kernel's layout.
// meta[2 pass] = union size, meta[2 pass + 1] = tiles.
__global__ void __launch_bounds__(kPlanThreads)
flmr_listed_plan_kernel(const ListedPass* __restrict__ passes, const uint32_t* __restrict__ allow, int64_t words,
                        const int64_t* __restrict__ poff, int n_ctas, int32_t* u_slot_all, int64_t* u_cum_all,
                        int64_t* u_tile_all, int64_t* cta_tile_base_all, int32_t* tile_row_all,
                        uint32_t* tile_mask_all, int32_t* tile_first_all, int64_t* meta) {
  __shared__ long long s_scan[32];
  const ListedPass ps = passes[blockIdx.x];
  int32_t* const u_slot = u_slot_all + ps.u_off;
  int64_t* const u_cum = u_cum_all + ps.u_off;
  int64_t* const u_tile = u_tile_all + ps.u_off;
  int32_t* const tile_row = tile_row_all + ps.t_off;
  uint32_t* const tile_mask = tile_mask_all + ps.t_off;
  int32_t* const tile_first = tile_first_all + ps.t_off;
  const int tid = threadIdx.x;
  auto add = [](long long a, long long b) { return a + b; };
  auto mx = [](long long a, long long b) { return a > b ? a : b; };
  long long tot;
  // 1. union slots, in slot order
  long long n = 0;
  for (int64_t w0 = 0; w0 < words; w0 += kPlanThreads) {
    const int64_t w = w0 + tid;
    uint32_t bits = 0u;
    if (w < words)
      for (int q = 0; q < ps.n_q; ++q) bits |= __ldg(allow + (ps.q_first + q) * words + w);
    long long pos = n + block_exclusive_scan<long long>(__popc(bits), 0ll, add, s_scan, &tot);
    while (bits) {
      u_slot[pos++] = static_cast<int32_t>(w * 32 + __ffs(bits) - 1);
      bits &= bits - 1u;
    }
    n += tot;
  }
  __syncthreads();
  // 2. first row of each inside the union
  long long R = 0;
  for (int64_t i0 = 0; i0 < n; i0 += kPlanThreads) {
    const int64_t i = i0 + tid;
    long long rows = 0;
    if (i < n) rows = __ldg(poff + u_slot[i] + 1) - __ldg(poff + u_slot[i]);
    const long long excl = block_exclusive_scan<long long>(rows, 0ll, add, s_scan, &tot);
    if (i < n) u_cum[i] = R + excl;
    R += tot;
  }
  __syncthreads();
  // 3. shares, runs, tiles
  auto cta_of = [&](long long x) {   // the last c with R c / n_ctas <= x
    return static_cast<int>(min(static_cast<long long>(n_ctas) - 1, (static_cast<long long>(n_ctas) * (x + 1) + R - 1) / R - 1));
  };
  long long run_carry = -1, tile_carry = 0;
  for (int64_t i0 = 0; i0 < n; i0 += kPlanThreads) {
    const int64_t i = i0 + tid;
    const bool ok = i < n;
    long long x = 0, rows = 0;
    int32_t s = 0;
    bool start = false;
    if (ok) {
      s = u_slot[i];
      x = u_cum[i];
      rows = __ldg(poff + s + 1) - __ldg(poff + s);
      start = i == 0 || u_slot[i - 1] != s - 1 || cta_of(u_cum[i - 1]) != cta_of(x);
    }
    // first row of the run holding i: the last run start at or before it (a running max: u_cum increases)
    const long long mine = start ? x : -1ll;
    const long long rs = mx(mx(run_carry, block_exclusive_scan<long long>(mine, -1ll, mx, s_scan, &tot)), mine);
    run_carry = mx(run_carry, tot);
    const long long b = x - rs, e = b + rows;               // the passage's rows inside its run
    const long long t0 = (b + kTileN - 1) / kTileN, t1 = (e + kTileN - 1) / kTileN;   // tiles starting in it
    const long long T = tile_carry + block_exclusive_scan<long long>(ok ? t1 - t0 : 0ll, 0ll, add, s_scan, &tot);
    tile_carry += tot;
    const long long run_tile = T - t0;                      // the run's first tile
    if (ok) {
      u_tile[i] = run_tile;
      for (long long t = t0; t < t1; ++t) {
        tile_row[run_tile + t] = static_cast<int32_t>(__ldg(poff + s) - b + t * kTileN);
        tile_mask[run_tile + t] = t == 0 ? kTileRunStart : 0u;
        tile_first[run_tile + t] = 0x7fffffff;
      }
    }
    __syncthreads();   // a tile is initialised (above, by the passage it starts in) before anyone marks an end in it
    if (ok) {
      const long long g = run_tile + (e - 1) / kTileN;
      atomicOr(tile_mask + g, 1u << (((e - 1) % kTileN) / kGroup));
      atomicMin(tile_first + g, s);
    }
    __syncthreads();
  }
  // 4. CTA c's tiles start at the run of its first passage (the first one at or past row R c / n_ctas)
  for (int c = tid; c <= n_ctas; c += kPlanThreads) {
    int64_t first = n;
    if (c == 0) {
      first = 0;
    } else if (c < n_ctas && R > 0) {
      const long long target = R * c / n_ctas;
      int64_t lo = 0, hi = n;
      while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (u_cum[mid] < target) lo = mid + 1; else hi = mid;
      }
      first = lo;
    }
    cta_tile_base_all[ps.c_off + c] = first < n ? u_tile[first] : tile_carry;
  }
  if (tid == 0) {
    meta[2 * blockIdx.x] = n;
    meta[2 * blockIdx.x + 1] = tile_carry;
  }
}

// Independent plain-SIMT MaxSim (test infrastructure): one block per (passage, query), one thread
// per query token (looping if nq > blockDim), fp32 FMA over bf16 inputs, fixed-order block sum.
// kE4M3: the corpus matrix is e4m3 (the queries come already rounded to e4m3 as bf16, flmr_round_e4m3_kernel).
// kF16: corpus and queries are fp16.  A deleted passage (bit set in `dead`, which may be null) scores -inf.
template <Elem kE>
__device__ __forceinline__ float simt_query_elem(const void* q, int64_t i) {
  if constexpr (kE == Elem::kF16)
    return __half2float(static_cast<const __half*>(q)[i]);
  else
    return __bfloat162float(static_cast<const __nv_bfloat16*>(q)[i]);
}
template <Elem kE>
__global__ void flmr_simt_maxsim_kernel(const void* __restrict__ d_any, const int64_t* poff,
                                        const int32_t* doclen, const uint32_t* __restrict__ dead,
                                        const void* __restrict__ q,
                                        int nq, float init, float* __restrict__ out,
                                        int64_t n_passages) {
  __shared__ float drow[kDim];
  __shared__ float red[256];
  const int64_t p = blockIdx.x;
  const int b = blockIdx.y;
  if (dead && ((dead[p >> 5] >> (p & 31)) & 1u)) {   // block-uniform, before any barrier
    if (threadIdx.x == 0) out[static_cast<int64_t>(b) * n_passages + p] = -INFINITY;
    return;
  }
  const int len = doclen[p];
  const int64_t d0 = poff[p] * kDim;
  float total = 0.f;
  for (int i0 = 0; i0 < nq; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    float m = init;
    const int64_t qi = (static_cast<int64_t>(b) * nq + (i < nq ? i : 0)) * kDim;
    for (int j = 0; j < len; ++j) {
      __syncthreads();
      if (threadIdx.x < kDim) {
        const int64_t e = d0 + j * kDim + threadIdx.x;
        if constexpr (kE == Elem::kE4M3) {
          const __half_raw h = __nv_cvt_fp8_to_halfraw(static_cast<const __nv_fp8_storage_t*>(d_any)[e], __NV_E4M3);
          drow[threadIdx.x] = __half2float(__half(h));
        } else if constexpr (kE == Elem::kF16) {
          drow[threadIdx.x] = __half2float(static_cast<const __half*>(d_any)[e]);
        } else {
          drow[threadIdx.x] = __bfloat162float(static_cast<const __nv_bfloat16*>(d_any)[e]);
        }
      }
      __syncthreads();
      float acc = 0.f;
#pragma unroll 16
      for (int c = 0; c < kDim; ++c) acc = fmaf(simt_query_elem<kE>(q, qi + c), drow[c], acc);
      m = fmaxf(m, acc);
    }
    if (i < nq) total += m;
  }
  red[threadIdx.x] = total;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[static_cast<int64_t>(b) * n_passages + p] = red[0];
}

// PLAID residual decode (SURVEY.md 8f-3): emb[t][i] = centroids[code[t]][i] + bucket_weights[idx(t, i)],
// idx = the nbits-wide field of dim i in the token's packed residual bytes, bit-reversed (the
// reference packs each bucket index LSB-first into big-endian bytes: residual.py:188-204 binarize,
// :51-73 reversed_bit_map, :77-93 lookup table; decode loop decompress_residuals.cpp:27-78), then the
// row is L2-normalised (index_storage.py:173) and stored as bf16 (kF16: fp16, the reference's own decode type,
// residual.py:273), rounded once from fp32.  HBM-bound byte work: one warp per token, lane = 4 dims, centroid rows
// come from L2, bucket weights from shared memory.  The per-token arithmetic is flmr_plaid_decode_row.cuh, which the
// window decode and the gather of a PLAID-coded streamed corpus include too.
template <bool kF16>
__global__ void flmr_plaid_decode_kernel(const int32_t* __restrict__ codes,
                                         const uint8_t* __restrict__ residuals,
                                         const float* __restrict__ centroids,
                                         const float* __restrict__ bucket_weights, int nbits,
                                         int normalize, int64_t n_tokens, int64_t n_centroids,
                                         uint2* __restrict__ out, int* __restrict__ bad_code) {
  __shared__ float s_w[256];
  for (int i = threadIdx.x; i < (1 << nbits); i += blockDim.x) s_w[i] = bucket_weights[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int keys = 8 / nbits;                 // bucket indices per packed byte
  const int packed_dim = kDim * nbits / 8;    // bytes per token
  const uint32_t mask = (1u << nbits) - 1u;
  for (int64_t t = warp0; t < n_tokens; t += n_warps) {
    const int32_t code = codes[t];
    if (code < 0 || code >= n_centroids) {    // corrupt index: flag, never read out of bounds
      if (lane == 0) {
        *reinterpret_cast<volatile int*>(bad_code) = 1;
        __threadfence_system();
      }
      continue;
    }
    const float4 c = __ldg(reinterpret_cast<const float4*>(centroids + static_cast<int64_t>(code) * kDim) + lane);
    const uint8_t* row = residuals + t * packed_dim;
#include "flmr_plaid_decode_row.cuh"
    out[t * 32 + lane] = w;
  }
}

// The window decode of a PLAID-coded streamed corpus: the staged compressed rows of one window (codes [rows], packed
// residuals [rows, 16 nbits], in the padded row layout, so rows is a multiple of kGroup) into the window buffer, in
// bf16 or (kF16) fp16, always L2-normalised as a PLAID index's embeddings are.  The codes were checked when the corpus
// was built.  A warp decodes kGroup consecutive rows per step and issues their code and centroid loads before the
// first row's arithmetic, so it keeps four tokens' loads in flight rather than one.
template <bool kF16>
__global__ void __launch_bounds__(256)
flmr_plaid_window_decode_kernel(const int32_t* __restrict__ codes, const uint8_t* __restrict__ residuals,
                                const float* __restrict__ centroids, const float* __restrict__ bucket_weights,
                                int nbits, int64_t rows, uint2* __restrict__ out) {
  __shared__ float s_w[256];
  for (int i = threadIdx.x; i < (1 << nbits); i += blockDim.x) s_w[i] = bucket_weights[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int keys = 8 / nbits;
  const int packed_dim = kDim * nbits / 8;
  const uint32_t mask = (1u << nbits) - 1u;
  const int normalize = 1;
  for (int64_t t0 = warp0 * kGroup; t0 < rows; t0 += n_warps * kGroup) {
    float4 cg[kGroup];
#pragma unroll
    for (int g = 0; g < kGroup; ++g)
      cg[g] = __ldg(reinterpret_cast<const float4*>(centroids + static_cast<int64_t>(__ldg(codes + t0 + g)) * kDim) +
                    lane);
#pragma unroll
    for (int g = 0; g < kGroup; ++g) {
      const float4 c = cg[g];
      const uint8_t* row = residuals + (t0 + g) * packed_dim;
#include "flmr_plaid_decode_row.cuh"
      out[(t0 + g) * 32 + lane] = w;
    }
  }
}

// The gather of a PLAID-coded streamed corpus: flmr_gather_kernel's batch (one warp per (id, token) of the
// [n_pids, nd_max, 128] output; an all-masked zero row for an id outside the shard, a deleted id and every token past
// the passage's length), each row decoded from the corpus's mapped host arrays as the window decode decodes it.
template <bool kF16>
__global__ void flmr_plaid_gather_kernel(const int32_t* __restrict__ codes, const uint8_t* __restrict__ residuals,
                                         const float* __restrict__ centroids,
                                         const float* __restrict__ bucket_weights, int nbits,
                                         const int64_t* __restrict__ poff, const int32_t* __restrict__ doclen,
                                         const uint32_t* __restrict__ dead, const int64_t* __restrict__ pids,
                                         int64_t n_pids, int nd_max, int64_t n_passages, int64_t pid_base,
                                         uint2* __restrict__ out, uint8_t* __restrict__ mask_out) {
  __shared__ float s_w[256];
  for (int i = threadIdx.x; i < (1 << nbits); i += blockDim.x) s_w[i] = bucket_weights[i];
  __syncthreads();
  const int64_t wi = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wi >= n_pids * nd_max) return;
  const int keys = 8 / nbits;
  const uint32_t mask = (1u << nbits) - 1u;
  const int normalize = 1;
  const int64_t slot = wi / nd_max;
  const int j = static_cast<int>(wi % nd_max);
  const int64_t p = pids[slot] - pid_base;
  uint2 o = make_uint2(0u, 0u);
  bool real = false;
  if (p >= 0 && p < n_passages && j < doclen[p] && !(dead && ((dead[p >> 5] >> (p & 31)) & 1u))) {   // warp-uniform
    const int64_t r = poff[p] + j;
    const float4 c = __ldg(reinterpret_cast<const float4*>(centroids + static_cast<int64_t>(codes[r]) * kDim) + lane);
    const uint8_t* row = residuals + r * (kDim * nbits / 8);
#include "flmr_plaid_decode_row.cuh"
    o = w;
    real = true;
  }
  out[wi * 32 + lane] = o;
  if (mask_out && lane == 0) mask_out[wi] = real ? 1 : 0;
}

// Candidate merge: per query, select the k_out best of n candidates by (score desc, pid asc).
// Candidates come either as packed keys written by the scan kernel (keys != null; slot = ~low32, pid = pid_base +
// slot, or slot_pid[slot] on a compacted corpus) or as (score, pid) arrays laid out [list][query][k_in].  One 1024-thread block per query,
// up to kMergePer candidates per thread in registers, k_out selection rounds.
constexpr int kMergeThreads = 1024;
constexpr int kMergePer = 20;
constexpr int64_t kPidEmpty = 0x7fffffffffffffffll;

struct Cand {
  uint32_t ord;  // ordered score; 0 = empty
  int64_t pid;
};
__device__ __forceinline__ bool cand_better(const Cand& a, const Cand& b) {
  return a.ord > b.ord || (a.ord == b.ord && a.pid < b.pid);
}

__global__ void __launch_bounds__(kMergeThreads)
flmr_merge_kernel(const uint64_t* __restrict__ keys, const float* __restrict__ in_scores,
                  const int64_t* __restrict__ in_pids, int n_lists, int n_queries, int k_in,
                  int k_out, int64_t pid_base, const int64_t* __restrict__ slot_pid, float* __restrict__ out_scores,
                  int64_t* __restrict__ out_pids, int q_offset, bool merge_out = false) {
  __shared__ uint32_t s_ord[32];
  __shared__ int64_t s_pid[32];
  __shared__ uint32_t w_ord;
  __shared__ int64_t w_pid;
  const int b = q_offset + blockIdx.x;   // n_queries = stride of the per-list arrays; blocks cover [q_offset, q_offset + grid)
  // merge_out: the k_out entries already in the output row (a streamed corpus's running top-k of earlier windows) are
  // one more list.  Every thread loads its candidates before the first __syncthreads, and only then is a row written.
  const int n_in = n_lists * k_in;
  const int n = n_in + (merge_out ? k_out : 0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Cand c[kMergePer];
#pragma unroll
  for (int i = 0; i < kMergePer; ++i) {
    const int idx = threadIdx.x + i * kMergeThreads;
    c[i].ord = 0u;
    c[i].pid = kPidEmpty;
    if (idx >= n_in && idx < n) {
      const int64_t g = static_cast<int64_t>(b) * k_out + (idx - n_in);
      const int64_t pid = out_pids[g];
      if (pid >= 0) {
        c[i].ord = float_to_ordered(out_scores[g]);   // written by this kernel from an ordered key: the same key back
        c[i].pid = pid;
      }
    } else if (idx < n) {
      const int l = idx / k_in, j = idx % k_in;
      const int64_t g = (static_cast<int64_t>(l) * n_queries + b) * k_in + j;
      if (keys) {
        const uint64_t key = keys[g];
        if (key != 0ull) {
          c[i].ord = static_cast<uint32_t>(key >> 32);
          const uint32_t slot = 0xFFFFFFFFu - static_cast<uint32_t>(key);
          c[i].pid = slot_pid ? __ldg(slot_pid + slot) : pid_base + slot;   // slots keep the order of their ids
        }
      } else {
        const int64_t pid = in_pids[g];
        if (pid >= 0) {
          c[i].ord = float_to_ordered(in_scores[g] + 0.0f);   // -0 -> +0: equal scores tie on pid (as in select)
          c[i].pid = pid;
        }
      }
    }
  }
  for (int r = 0; r < k_out; ++r) {
    Cand best = c[0];
#pragma unroll
    for (int i = 1; i < kMergePer; ++i)
      if (cand_better(c[i], best)) best = c[i];
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      Cand o;
      o.ord = __shfl_xor_sync(0xffffffffu, best.ord, off);
      o.pid = __shfl_xor_sync(0xffffffffu, best.pid, off);
      if (cand_better(o, best)) best = o;
    }
    if (lane == 0) {
      s_ord[warp] = best.ord;
      s_pid[warp] = best.pid;
    }
    __syncthreads();
    if (warp == 0) {
      Cand x;
      x.ord = s_ord[lane];
      x.pid = s_pid[lane];
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) {
        Cand o;
        o.ord = __shfl_xor_sync(0xffffffffu, x.ord, off);
        o.pid = __shfl_xor_sync(0xffffffffu, x.pid, off);
        if (cand_better(o, x)) x = o;
      }
      if (lane == 0) {
        w_ord = x.ord;
        w_pid = x.pid;
        const bool empty = (x.ord == 0u);
        out_scores[static_cast<int64_t>(b) * k_out + r] =
            empty ? -INFINITY : ordered_to_float(x.ord);
        out_pids[static_cast<int64_t>(b) * k_out + r] = empty ? -1 : x.pid;
      }
    }
    __syncthreads();
    const uint32_t wo = w_ord;
    const int64_t wp = w_pid;
    if (wo != 0u) {
#pragma unroll
      for (int i = 0; i < kMergePer; ++i)
        if (c[i].ord == wo && c[i].pid == wp) {
          c[i].ord = 0u;
          c[i].pid = kPidEmpty;
        }
    }
    // (w_ord/w_pid are rewritten only after the next round's first __syncthreads)
  }
}

// The merge of flmr_topk_merge_devices: list l is its own [n_queries, k_in] array, read where it lives (on this device,
// through peer access, or in the home staging buffer).  The pointer tables are kernel parameters (__grid_constant__), so
// indexing them by list reads the parameter bank with no local copy.  Each candidate is read once: its ordered score
// stays in a register and its pid goes to shared memory, where the selection reads it only to break an exact tie and to
// publish a thread's best; so the selection order is flmr_merge_kernel's (score desc, pid asc), and the kernel holds
// kMergePer candidates per thread without spilling.
constexpr int kMergeMaxLists = 128;
struct MergeLists {
  const float* scores[kMergeMaxLists];
  const int64_t* pids[kMergeMaxLists];
};

__global__ void __launch_bounds__(kMergeThreads)
flmr_merge_lists_kernel(const __grid_constant__ MergeLists lists, int n_lists, int k_in, int k_out,
                        float* __restrict__ out_scores, int64_t* __restrict__ out_pids) {
  extern __shared__ int64_t s_cand_pid[];   // [n_lists * k_in]
  __shared__ uint32_t s_ord[32];
  __shared__ int64_t s_pid[32];
  __shared__ uint32_t w_ord;
  __shared__ int64_t w_pid;
  const int b = blockIdx.x;
  const int n = n_lists * k_in;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t ord[kMergePer];   // candidate threadIdx.x + i * kMergeThreads; 0 = empty
#pragma unroll
  for (int i = 0; i < kMergePer; ++i) {
    const int idx = threadIdx.x + i * kMergeThreads;
    ord[i] = 0u;
    if (idx < n) {
      const int l = idx / k_in;
      const int64_t g = static_cast<int64_t>(b) * k_in + (idx - l * k_in);
      const int64_t pid = lists.pids[l][g];
      s_cand_pid[idx] = pid;
      if (pid >= 0) ord[i] = float_to_ordered(lists.scores[l][g] + 0.0f);   // -0 -> +0, as in flmr_merge_kernel
    }
  }
  __syncthreads();
  for (int r = 0; r < k_out; ++r) {
    Cand best;
    best.ord = 0u;
    best.pid = kPidEmpty;
#pragma unroll
    for (int i = 0; i < kMergePer; ++i) {
      if (ord[i] != 0u && ord[i] >= best.ord) {
        const int64_t pid = s_cand_pid[threadIdx.x + i * kMergeThreads];
        if (ord[i] > best.ord || pid < best.pid) {
          best.ord = ord[i];
          best.pid = pid;
        }
      }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      Cand o;
      o.ord = __shfl_xor_sync(0xffffffffu, best.ord, off);
      o.pid = __shfl_xor_sync(0xffffffffu, best.pid, off);
      if (cand_better(o, best)) best = o;
    }
    if (lane == 0) {
      s_ord[warp] = best.ord;
      s_pid[warp] = best.pid;
    }
    __syncthreads();
    if (warp == 0) {
      Cand x;
      x.ord = s_ord[lane];
      x.pid = s_pid[lane];
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) {
        Cand o;
        o.ord = __shfl_xor_sync(0xffffffffu, x.ord, off);
        o.pid = __shfl_xor_sync(0xffffffffu, x.pid, off);
        if (cand_better(o, x)) x = o;
      }
      if (lane == 0) {
        w_ord = x.ord;
        w_pid = x.pid;
        const bool empty = (x.ord == 0u);
        out_scores[static_cast<int64_t>(b) * k_out + r] = empty ? -INFINITY : ordered_to_float(x.ord);
        out_pids[static_cast<int64_t>(b) * k_out + r] = empty ? -1 : x.pid;
      }
    }
    __syncthreads();
    const uint32_t wo = w_ord;
    const int64_t wp = w_pid;
    if (wo != 0u) {   // every copy of the winner leaves, as in flmr_merge_kernel
#pragma unroll
      for (int i = 0; i < kMergePer; ++i)
        if (ord[i] == wo && s_cand_pid[threadIdx.x + i * kMergeThreads] == wp) ord[i] = 0u;
    }
    // (w_ord/w_pid are rewritten only after the next round's first __syncthreads)
  }
}

// Top-k selection over a dense score row for k beyond the fused capacity (SURVEY 8a a10:
// Searcher.dense_search accepts any k).  One 1024-thread block per query:
//   1. 4-pass MSB radix select (8 bits per pass, 256-bin histogram in shared memory) over the
//      order-preserving uint32 image of the scores -> key T of the k-th best score, and how many keys
//      are strictly better;
//   2. order-preserving compaction: every thread owns a contiguous slice of the row, block-wide
//      exclusive scans place the keys > T, then as many keys == T (ascending pid) as still fit;
//   3. bitonic sort of the k survivors by (score desc, pid asc) in shared memory.
constexpr int kSelectThreads = 1024;
constexpr int kSelectMaxK = 2048;

__global__ void __launch_bounds__(kSelectThreads)
flmr_select_kernel(const float* __restrict__ scores, int64_t n, int k, int64_t pid_base,
                   float* __restrict__ out_scores, int64_t* __restrict__ out_pids) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_prefix, s_need, s_gt_total;
  __shared__ uint32_t scan_gt[kSelectThreads], scan_eq[kSelectThreads];
  __shared__ uint32_t sel_ord[kSelectMaxK];
  __shared__ uint32_t sel_pid[kSelectMaxK];
  const int tid = threadIdx.x;
  const float* row = scores + static_cast<int64_t>(blockIdx.x) * n;
  const int kk = static_cast<int>(n < k ? n : k);
  // ---- 1. radix select of the kk-th largest ordered key ----
  if (tid == 0) {
    s_prefix = 0u;
    s_need = static_cast<uint32_t>(kk);
  }
  uint32_t mask_hi = 0u;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kSelectThreads) hist[i] = 0u;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (int64_t i = tid; i < n; i += kSelectThreads) {
      const uint32_t key = float_to_ordered(row[i] + 0.0f);
      if ((key & mask_hi) == prefix) atomicAdd(&hist[(key >> shift) & 0xFFu], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t need = s_need, bin = 255;
      for (;; --bin) {                       // from the largest digit down
        if (hist[bin] >= need || bin == 0) break;
        need -= hist[bin];
      }
      s_need = need;                         // still to take inside this bin
      s_prefix = prefix | (bin << shift);
    }
    __syncthreads();
    mask_hi |= 0xFFu << shift;
  }
  const uint32_t T = s_prefix;               // key of the kk-th best; s_need of the keys == T are taken
  // ---- 2. order-preserving compaction ----
  const int64_t per = (n + kSelectThreads - 1) / kSelectThreads;
  const int64_t i0 = static_cast<int64_t>(tid) * per, i1 = (i0 + per < n) ? i0 + per : n;
  uint32_t c_gt = 0, c_eq = 0;
  for (int64_t i = i0; i < i1; ++i) {
    const uint32_t key = float_to_ordered(row[i] + 0.0f);
    c_gt += key > T;
    c_eq += key == T;
  }
  scan_gt[tid] = c_gt;
  scan_eq[tid] = c_eq;
  __syncthreads();
  for (int off = 1; off < kSelectThreads; off <<= 1) {   // Hillis-Steele inclusive scans
    const uint32_t a = tid >= off ? scan_gt[tid - off] : 0u, b = tid >= off ? scan_eq[tid - off] : 0u;
    __syncthreads();
    scan_gt[tid] += a;
    scan_eq[tid] += b;
    __syncthreads();
  }
  if (tid == kSelectThreads - 1) s_gt_total = scan_gt[tid];
  __syncthreads();
  const uint32_t gt_total = s_gt_total;
  uint32_t o_gt = scan_gt[tid] - c_gt, o_eq = gt_total + scan_eq[tid] - c_eq;
  for (int64_t i = i0; i < i1; ++i) {
    const uint32_t key = float_to_ordered(row[i] + 0.0f);
    if (key > T) {
      sel_ord[o_gt] = key;
      sel_pid[o_gt++] = static_cast<uint32_t>(i);
    } else if (key == T) {
      if (o_eq < static_cast<uint32_t>(kk)) {
        sel_ord[o_eq] = key;
        sel_pid[o_eq] = static_cast<uint32_t>(i);
      }
      ++o_eq;
    }
  }
  // ---- 3. bitonic sort (descending score, ascending pid) over the next power of two ----
  int m = 1;
  while (m < kk) m <<= 1;
  __syncthreads();
  for (int i = kk + tid; i < m; i += kSelectThreads) {
    sel_ord[i] = 0u;                         // empty entries sort last
    sel_pid[i] = 0xFFFFFFFFu;
  }
  __syncthreads();
  auto before = [&](int a, int b) {          // true if entry a must come before entry b
    return sel_ord[a] > sel_ord[b] || (sel_ord[a] == sel_ord[b] && sel_pid[a] < sel_pid[b]);
  };
  for (int size = 2; size <= m; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < m; i += kSelectThreads) {
        const int j = i ^ stride;
        if (j > i) {
          const bool up = (i & size) == 0;   // ascending position = better entries first
          if (up ? before(j, i) : before(i, j)) {
            const uint32_t to = sel_ord[i], tp = sel_pid[i];
            sel_ord[i] = sel_ord[j];
            sel_pid[i] = sel_pid[j];
            sel_ord[j] = to;
            sel_pid[j] = tp;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < k; i += kSelectThreads) {
    const bool ok = i < kk;
    out_scores[static_cast<int64_t>(blockIdx.x) * k + i] = ok ? ordered_to_float(sel_ord[i]) : -INFINITY;
    out_pids[static_cast<int64_t>(blockIdx.x) * k + i] = ok ? pid_base + sel_pid[i] : -1;
  }
}

// A token-balanced split of the slots into contiguous ranges (one per CTA, or per pair of CTAs) and the per-tile
// metadata the scan reads, on the device.
struct Partition {
  int64_t n_tiles = 0;
  int32_t* row_begin = nullptr;   // [ranges + 1]
  int64_t* tile_base = nullptr;   // [ranges + 1]
  uint32_t* end_mask = nullptr;   // [n_tiles]
  int32_t* first_pid = nullptr;   // [n_tiles]
};

// One window of a corpus: the slots [slot0, slot1), stored rows [row0, row0 + rows), scanned from a buffer that holds
// exactly those rows from its row 0 (a resident corpus: its one window, the token matrix).  Its partition's row starts
// are relative to the window; its tiles' first slots are absolute, so candidate keys, tombstones, allow bitmaps and
// score rows are indexed alike in every window.
struct Window {
  int64_t slot0 = 0, slot1 = 0, row0 = 0, rows = 0;
  int n_ctas = 0;                      // min(SMs, slots of the window)
  Partition cta;
};

// Everything build_layout derives from the stored passages' (the slots') offsets: what the scan, the SIMT kernel and
// the gather read.  An append or a compaction builds a new one and swaps it in whole (free_layout frees one).
struct SlotLayout {
  std::vector<int64_t> h_poff;         // [slots + 1] stored-row offsets
  std::vector<int32_t> h_doclen;       // [slots] real lengths
  int64_t* d_poff = nullptr;           // device copies of the two above
  int32_t* d_doclen = nullptr;
  int64_t max_rows = 0;                // stored rows of the longest slot (bounds a listed search's plan)
  int n_ctas = 0;                      // the most CTAs a window launches (sizes a workspace's candidate lists)
  std::vector<Window> windows;         // a resident corpus has one, over every slot
  int64_t window_rows = 0;             // rows of the largest window (a streamed corpus's window buffers hold this many)
  // resident corpus only: the token matrix's tensor map, and the CTA-pair experiment (flmr_debug_set_scan_variant(4),
  // bf16 only): n_pairs ranges, and a tensor map with a half-tile box
  CUtensorMap tmap_d;
  int n_pairs = 0;
  Partition pair;
  CUtensorMap tmap_half;
  int64_t bytes = 0;                   // HBM the device arrays above take
};

}  // namespace

// ---- handles -----------------------------------------------------------------------------------------
struct flmr_corpus {
  int device = 0;
  int64_t n_passages = 0, n_tokens = 0, n_rows = 0, pid_base = 0;
  bool adopted = false;
  // FLMR_CORPUS_FP16 (kF16): d_tokens holds fp16 rows, and queries arrive as fp16.  FLMR_CORPUS_FP8 (kE4M3): the scan
  // reads an e4m3 copy in HBM; the exact bf16 rows stay in pinned, mapped host memory
  Elem elem = Elem::kBF16;
  __nv_bfloat16* d_tokens = nullptr;   // [n_rows, 128] padded layout (e4m3 corpus: device alias of h_master; fp16
                                       // corpus: the fp16 rows, which every kernel but the scan only moves)
  GrowableMatrix vm_tokens;            // backs d_tokens of a library-owned bf16 (or fp16) corpus
  void* h_master = nullptr;            // bf16 [n_rows, 128] padded layout, pinned + mapped (e4m3 corpus only)
  uint8_t* d_fp8 = nullptr;            // e4m3 [n_rows, 128] padded layout (e4m3 corpus only), backed by vm_fp8
  GrowableMatrix vm_fp8;
  // Ids and slots.  n_passages is the id extent: ids pid_base .. pid_base + n_passages, never shrinking.  A slot is a
  // passage that has rows.  Until the first flmr_corpus_compact every id has the slot of the same index and
  // h_slot_pid / d_slot_pid stay empty / null; after it, slot s holds global id h_slot_pid[s] (strictly increasing).
  // Everything the scan reads (layout, d_dead) is indexed by slot.
  std::vector<int64_t> h_slot_pid;
  int64_t* d_slot_pid = nullptr;
  SlotLayout layout;
  // tombstones: h_dead is indexed by LOCAL ID (bit p & 31 of word p >> 5 set <=> local passage p is deleted, a
  // compacted-away id included); d_dead by SLOT, for the scan's reducer, the gather and the SIMT kernel.  d_dead stays
  // null while no slot is deleted (until the first delete, and again right after a compaction), so a corpus without
  // deletions runs the scan exactly as before
  uint32_t* d_dead = nullptr;
  std::vector<uint32_t> h_dead;
  int64_t n_deleted = 0;
  int sm_total = 0;                    // SMs of the device
  // A streamed corpus (flmr_corpus_create_streamed): the padded rows live in h_stream (pinned, mapped; d_tokens is its
  // device alias, which the gather and the SIMT kernel read) and searches copy them window by window into the
  // workspace's two window buffers.  Its layout has no tensor map of the matrix and no CTA-pair partition.
  bool streamed = false;
  void* h_stream = nullptr;
  int64_t window_bytes = 0;            // as requested at creation
  // A PLAID-coded streamed corpus (flmr_corpus_builder_create_plaid; codec_nbits > 0): no row matrix at all (h_stream
  // and d_tokens stay null).  h_codes [n_rows] and h_residuals [n_rows, 16 nbits] hold each stored row's centroid code
  // and packed residual in the padded row layout, in one pinned, mapped allocation (d_codes / d_residuals: its device
  // aliases, which the gather reads); searches copy a window's compressed rows and decode them on the GPU.
  int codec_nbits = 0;
  int32_t* h_codes = nullptr;
  uint8_t* h_residuals = nullptr;
  const int32_t* d_codes = nullptr;
  const uint8_t* d_residuals = nullptr;
  float* d_centroids = nullptr;        // fp32 [n_centroids, 128], in HBM
  float* d_bucket_weights = nullptr;   // fp32 [2^nbits], in HBM
  int64_t n_centroids = 0;
  int64_t codec_hbm_bytes = 0;         // the two arrays above
};

// Streaming corpus construction (index load): the padded token matrix is allocated once, packed rows arrive in
// order through two pinned staging buffers (host fill of one overlaps the DMA of the other).
struct flmr_corpus_builder {
  flmr_corpus* corpus = nullptr;        // under construction (owned until finish)
  std::vector<int64_t> soff, poff;
  std::vector<int32_t> doclens;
  bool aligned = true;                  // every doclen a multiple of kGroup: rows land in place, no scatter
  int64_t rows_done = 0;
  cudaStream_t stream = nullptr;
  static constexpr int kBufs = 2;
  static constexpr int64_t kBufRows = (64ll << 20) / (kDim * 2);   // 64 MB of rows per staging buffer
  void* h_pin[kBufs] = {nullptr, nullptr};
  uint4* d_stage[kBufs] = {nullptr, nullptr};   // device staging (unaligned corpora only)
  cudaEvent_t free_ev[kBufs] = {nullptr, nullptr};
  int64_t *d_soff = nullptr, *d_poff = nullptr;
  int next = 0;
  double fill_s = 0.0;                  // host time spent filling the pinned buffers (read / memcpy)
  // a PLAID-coded corpus (corpus->codec_nbits > 0): the codec tables, copied to HBM by finish
  std::vector<float> centroids, bucket_weights;
};

struct flmr_workspace {
  const flmr_corpus* corpus = nullptr;
  int device = 0;
  int max_queries = 0, max_nq = 0;
  __nv_bfloat16* d_qpad = nullptr;     // [kStageMaxPasses][kMtMax*128, 128] staged (zero-padded) queries, one slot per pass
  uint64_t* d_cand_keys = nullptr;     // [n_ctas][max_queries][k] candidate keys of one call chunk
  int cand_lists = 0;                  // CTAs d_cand_keys is sized for (grown when an append raises n_ctas)
  float* d_acc = nullptr;              // [group][n_passages] lazily allocated (row-sliced queries)
  int64_t acc_capacity = 0;            // floats allocated at d_acc
  void* d_plan = nullptr;              // a listed search's slot bitmaps and scan plans (one call chunk), grown on demand
  size_t plan_capacity = 0;            // bytes allocated at d_plan
  int* h_status = nullptr;             // pinned + mapped: readable by the host even after a device trap
  int* d_status = nullptr;             // device alias of h_status
  int dbg_lane_rbq = 4;  // -DFLMR_DEBUG builds: FLMR_LANE_RBQ, read once at creation
  // streamed corpus only: two window buffers filled on a copy stream of the workspace's own, and the events that order
  // the copies against the scans (see run_search)
  __nv_bfloat16* d_win[2] = {nullptr, nullptr};
  CUtensorMap tmap_win[2];
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t fork_ev = nullptr;
  cudaEvent_t copied_ev[2] = {nullptr, nullptr};
  cudaEvent_t scanned_ev[2] = {nullptr, nullptr};
  // PLAID-coded streamed corpus only: d_win[0] is the one decoded window buffer; a window's compressed rows are copied
  // into staging buffer w % 2 (codes, then residuals from byte window_rows * 4), and decoded_ev[w % 2] marks the
  // decode that read it
  uint8_t* d_cstage[2] = {nullptr, nullptr};
  cudaEvent_t decoded_ev[2] = {nullptr, nullptr};
};

// NCCL is resolved at RUN time (dlopen): the library has no link dependency on it, loads on a box without
// NCCL, and shares the libnccl the host process already loaded (torch ships its own) when there is one.
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, /* ncclUniqueId by value: 128 bytes */ struct NcclId, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  int (*CommCount)(void*, int*) = nullptr;
  int (*CommUserRank)(void*, int*) = nullptr;
};
struct NcclId {
  char internal[128];
};

struct flmr_comm {
  void* nccl = nullptr;   // ncclComm_t
  int rank = 0, world = 1, device = 0;
  bool owned = false;     // created by flmr_comm_create (destroyed with the handle) vs adopted
  // exchange buffers, grown on demand: this rank's [B, k] lists and everybody's [world, B, k]
  float* d_send_s = nullptr;
  int64_t* d_send_p = nullptr;
  float* d_recv_s = nullptr;
  int64_t* d_recv_p = nullptr;
  int64_t capacity = 0;        // entries (B * k) per rank the receive buffers hold
  int64_t send_capacity = 0;   // entries (B * k) the send buffers hold
};

namespace {

int load_nccl(const NcclApi** out) {
  static NcclApi api;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if (!api.handle) {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);   // the copy the process already uses, if any
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return fail(FLMR_ERR_UNSUPPORTED, "NCCL is not available (dlopen libnccl.so.2: %s)", dlerror());
    NcclApi a;
    a.handle = h;
    a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
    a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
    a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
    a.AllGather = reinterpret_cast<decltype(a.AllGather)>(dlsym(h, "ncclAllGather"));
    a.GroupStart = reinterpret_cast<decltype(a.GroupStart)>(dlsym(h, "ncclGroupStart"));
    a.GroupEnd = reinterpret_cast<decltype(a.GroupEnd)>(dlsym(h, "ncclGroupEnd"));
    a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
    a.CommCount = reinterpret_cast<decltype(a.CommCount)>(dlsym(h, "ncclCommCount"));
    a.CommUserRank = reinterpret_cast<decltype(a.CommUserRank)>(dlsym(h, "ncclCommUserRank"));
    if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.AllGather || !a.GroupStart || !a.GroupEnd ||
        !a.GetErrorString || !a.CommCount || !a.CommUserRank)
      return fail(FLMR_ERR_UNSUPPORTED, "libnccl.so.2 lacks an expected entry point");
    api = a;
  }
  *out = &api;
  return FLMR_OK;
}

#define FLMR_NCCL(api, expr)                                                                          \
  do {                                                                                                \
    int r__ = (expr);                                                                                 \
    if (r__ != 0)                                                                                     \
      return fail(FLMR_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, (api)->GetErrorString(r__), __FILE__, __LINE__); \
  } while (0)

constexpr int kNcclInt64 = 4, kNcclFloat32 = 7;   // ncclDataType_t values (nccl.h: ncclInt64 = 4, ncclFloat32 = 7)

thread_local bool g_profiling = false;
// which scan kernel a search on this thread launches: 0 = chosen per pass (pick_scan), 2 = flmr_scan_kernel<2> (two
// consumer warpgroups), 3 = flmr_scan_kernel<3> (three), 4 = CTA-pair passes forced, 6 = flmr_scan_split_kernel or
// flmr_scan_listed_split_kernel (three, split-tile loop; 5 and 7 stay unassigned); flmr_debug_set_scan_variant
thread_local int g_scan_variant = 0;
struct EventPair {
  cudaEvent_t a, b;
};
thread_local std::vector<EventPair> g_scan_events;

int64_t slots(const flmr_corpus* c) {
  return c->h_slot_pid.empty() ? c->n_passages : static_cast<int64_t>(c->h_slot_pid.size());
}

// Bytes per row of the matrix the scan reads (an e4m3 corpus's bf16 master is host memory).
int64_t hbm_row_bytes(Elem elem) { return elem == Elem::kE4M3 ? kDim : kDim * 2; }

const char* elem_name(Elem elem) { return elem == Elem::kE4M3 ? "e4m3" : elem == Elem::kF16 ? "fp16" : "bf16"; }

// HBM a corpus holds: its matrix (an adopted one is the caller's, a streamed one is host memory), its layout, its
// tombstones by slot and its slot -> id map (and a PLAID-coded corpus's centroids and bucket weights).
int64_t hbm_bytes(const flmr_corpus* c) {
  const int64_t ns = slots(c);
  return (c->adopted || c->streamed ? 0 : c->n_rows * hbm_row_bytes(c->elem)) + c->layout.bytes +
         (c->d_dead ? (ns + 31) / 32 * 4 : 0) + (c->d_slot_pid ? ns * 8 : 0) + c->codec_hbm_bytes;
}

// Bytes per stored row of a PLAID-coded corpus's compressed arrays: a 4-byte code and 16 nbits bytes of residual.
int64_t codec_row_bytes(int nbits) { return 4 + kDim * nbits / 8; }

// The storage a corpus's flags select (FLMR_CORPUS_ADOPT reaches here only from flmr_corpus_create).
int storage_from_flags(unsigned flags, Elem* elem) {
  if ((flags & FLMR_CORPUS_FP8) && (flags & FLMR_CORPUS_ADOPT))
    return fail(FLMR_ERR_INVALID_ARG, "FLMR_CORPUS_FP8 keeps its own copies of the tokens and cannot adopt them");
  if ((flags & FLMR_CORPUS_FP8) && (flags & FLMR_CORPUS_FP16))
    return fail(FLMR_ERR_INVALID_ARG, "FLMR_CORPUS_FP16 and FLMR_CORPUS_FP8 exclude each other");
  *elem = (flags & FLMR_CORPUS_FP8) ? Elem::kE4M3 : (flags & FLMR_CORPUS_FP16) ? Elem::kF16 : Elem::kBF16;
  return FLMR_OK;
}

// Packed (*soff, may be null) and padded (*poff) row offsets of n passages, relative to the first; *aligned (may be
// null): every length is a multiple of kGroup, so packed rows are stored rows.
int passage_offsets(const int32_t* h_doclens, int64_t n, std::vector<int64_t>* soff, std::vector<int64_t>* poff,
                    bool* aligned) {
  std::vector<int64_t> s(n + 1, 0), p(n + 1, 0);
  bool al = true;
  for (int64_t i = 0; i < n; ++i) {
    const int32_t len = h_doclens[i];
    if (len < 1)
      return fail(FLMR_ERR_INVALID_ARG, "passage %lld has length %d; zero-length passages have no defined MaxSim score",
                  (long long)i, len);
    s[i + 1] = s[i] + len;
    p[i + 1] = p[i] + (len + kGroup - 1) / kGroup * kGroup;
    al &= (len % kGroup == 0);
  }
  if (soff) soff->swap(s);
  poff->swap(p);
  if (aligned) *aligned = al;
  return FLMR_OK;
}

// The SM count of the device a corpus is built on, which must be an sm_90 one.
int sm90_count(int device, int* sm_count) {
  cudaDeviceProp prop;
  FLMR_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(FLMR_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is sm_90a only", device, prop.major,
                prop.minor);
  *sm_count = prop.multiProcessorCount;
  return FLMR_OK;
}

// Whether a token matrix to copy from is device (or managed) memory; device memory must be on the corpus's device.
int token_source(const void* tokens, int device, bool* is_device_ptr) {
  cudaPointerAttributes attr{};
  *is_device_ptr = (cudaPointerGetAttributes(&attr, tokens) == cudaSuccess) &&
                   (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
  cudaGetLastError();
  if (*is_device_ptr && attr.type == cudaMemoryTypeDevice && attr.device != device)
    return fail(FLMR_ERR_INVALID_ARG, "token matrix lives on device %d, corpus on %d", attr.device, device);
  return FLMR_OK;
}

// The tombstones by slot (d_dead's words) of a compacted corpus, from its tombstones by id (`dead`, as h_dead).
std::vector<uint32_t> dead_by_slot(const std::vector<int64_t>& slot_pid, int64_t pid_base,
                                   const std::vector<uint32_t>& dead) {
  const int64_t ns = static_cast<int64_t>(slot_pid.size());
  std::vector<uint32_t> out((ns + 31) / 32, 0u);
  for (int64_t s = 0; s < ns; ++s) {
    const int64_t p = slot_pid[s] - pid_base;
    if (static_cast<size_t>(p >> 5) < dead.size() && ((dead[p >> 5] >> (p & 31)) & 1u)) out[s >> 5] |= 1u << (s & 31);
  }
  return out;
}


template <typename T>
int dev_upload(T** dptr, const std::vector<T>& h, int64_t* bytes_acc) {
  const size_t bytes = std::max<size_t>(h.size(), 1) * sizeof(T);
  FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(dptr), bytes));
  if (!h.empty()) FLMR_CUDA(cudaMemcpy(*dptr, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  if (bytes_acc) *bytes_acc += static_cast<int64_t>(bytes);
  return FLMR_OK;
}

// The library's own stream-ordered memory pool (one per device) for per-call scratch: it keeps what it has
// been given (release threshold = max), so after the first call an allocation is a pointer bump in stream order —
// the default pool hands memory back to the driver at every synchronisation and re-maps it on the next call.
static int scratch_pool(cudaMemPool_t* out) {
  static cudaMemPool_t pools[64] = {};
  static std::mutex mu;
  int dev = 0;
  FLMR_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if (!pools[dev & 63]) {
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    cudaMemPool_t p = nullptr;
    FLMR_CUDA(cudaMemPoolCreate(&p, &props));
    uint64_t keep = ~0ull;
    FLMR_CUDA(cudaMemPoolSetAttribute(p, cudaMemPoolAttrReleaseThreshold, &keep));
    pools[dev & 63] = p;
  }
  *out = pools[dev & 63];
  return FLMR_OK;
}

// Per-call device scratch from the library's pool, handed back in stream order when the call has enqueued its work.
struct StreamScratch {
  cudaStream_t st;
  std::vector<void*> ptrs;
  explicit StreamScratch(cudaStream_t s) : st(s) {}
  StreamScratch(const StreamScratch&) = delete;
  StreamScratch& operator=(const StreamScratch&) = delete;
  ~StreamScratch() {
    for (void* q : ptrs) cudaFreeAsync(q, st);
  }
  template <typename T>
  int alloc(T** out, size_t bytes) {
    cudaMemPool_t pool = nullptr;
    if (int rc = scratch_pool(&pool)) return rc;
    void* q = nullptr;
    FLMR_CUDA(cudaMallocFromPoolAsync(&q, std::max<size_t>(bytes, 16), pool, st));
    ptrs.push_back(q);
    *out = static_cast<T*>(q);
    return FLMR_OK;
  }
};

// Token-balanced split of the passages into n_ctas contiguous ranges + per-tile metadata.
void build_partition(const std::vector<int64_t>& poff, int n_ctas, int tile_n,
                     std::vector<int32_t>* cta_row_begin, std::vector<int64_t>* cta_tile_base,
                     std::vector<uint32_t>* tile_end_mask, std::vector<int32_t>* tile_first_pid) {
  const int64_t n = static_cast<int64_t>(poff.size()) - 1;
  const int64_t rows = poff[n];
  std::vector<int64_t> pbeg(n_ctas + 1);
  pbeg[0] = 0;
  for (int c = 1; c < n_ctas; ++c) {
    const int64_t target = rows * c / n_ctas;
    int64_t p = std::lower_bound(poff.begin(), poff.end(), target) - poff.begin();
    p = std::min<int64_t>(std::max<int64_t>(p, pbeg[c - 1]), n);
    pbeg[c] = p;
  }
  pbeg[n_ctas] = n;
  cta_row_begin->resize(n_ctas + 1);
  cta_tile_base->resize(n_ctas + 1);
  int64_t tiles = 0;
  for (int c = 0; c <= n_ctas; ++c) {
    (*cta_row_begin)[c] = static_cast<int32_t>(poff[pbeg[c]]);
    (*cta_tile_base)[c] = tiles;
    if (c < n_ctas) tiles += (poff[pbeg[c + 1]] - poff[pbeg[c]] + tile_n - 1) / tile_n;
  }
  tile_end_mask->assign(tiles, 0u);
  tile_first_pid->assign(tiles, 0);
  for (int c = 0; c < n_ctas; ++c) {
    const int64_t r0 = poff[pbeg[c]];
    const int64_t tb = (*cta_tile_base)[c];
    const int64_t nt = (*cta_tile_base)[c + 1] - tb;
    std::vector<char> seen(nt, 0);
    for (int64_t p = pbeg[c]; p < pbeg[c + 1]; ++p) {
      const int64_t last = poff[p + 1] - 1 - r0;  // last stored row of p, relative to the CTA
      const int64_t t = last / tile_n;
      const int g = static_cast<int>((last % tile_n) / kGroup);
      (*tile_end_mask)[tb + t] |= (1u << g);
      if (!seen[t]) {
        seen[t] = 1;
        (*tile_first_pid)[tb + t] = static_cast<int32_t>(p);
      }
    }
  }
}

// ---- window planning (pure host logic; exported for tests as flmr_debug_window_plan) ------------------------------
// The slots cut into contiguous ranges, each taking as many slots as fit window_rows stored rows (poff: stored-row
// offsets of the slots).  *out receives (first slot, end slot) pairs.  A slot longer than a window cannot be scanned
// from one: FLMR_ERR_UNSUPPORTED.
int plan_windows(const std::vector<int64_t>& poff, int64_t window_rows, std::vector<std::pair<int64_t, int64_t>>* out) {
  out->clear();
  const int64_t n = static_cast<int64_t>(poff.size()) - 1;
  for (int64_t s0 = 0; s0 < n;) {
    const int64_t s1 = std::upper_bound(poff.begin() + s0, poff.end(), poff[s0] + window_rows) - poff.begin() - 1;
    if (s1 <= s0)
      return fail(FLMR_ERR_UNSUPPORTED, "passage %lld has %lld stored rows (%lld B), more than a window of %lld rows "
                  "holds", (long long)s0, (long long)(poff[s0 + 1] - poff[s0]),
                  (long long)((poff[s0 + 1] - poff[s0]) * kDim * 2), (long long)window_rows);
    out->emplace_back(s0, s1);
    s0 = s1;
  }
  return FLMR_OK;
}

// The partition of one window [s0, s1) for min(sm_total, s1 - s0) CTAs: build_partition over the window's own row
// offsets, its tiles' first slots made absolute.
void window_partition(const std::vector<int64_t>& poff, int64_t s0, int64_t s1, int sm_total, int* n_ctas,
                      std::vector<int32_t>* rb, std::vector<int64_t>* tb, std::vector<uint32_t>* em,
                      std::vector<int32_t>* fp) {
  std::vector<int64_t> wpoff(poff.begin() + s0, poff.begin() + s1 + 1);
  for (int64_t& r : wpoff) r -= poff[s0];
  *n_ctas = static_cast<int>(std::min<int64_t>(sm_total, s1 - s0));
  build_partition(wpoff, *n_ctas, kTileN, rb, tb, em, fp);
  for (int32_t& f : *fp) f += static_cast<int32_t>(s0);
}

// ---- pass planning (pure host logic; exported for tests as flmr_debug_plan_passes) -------------------
// One pass = one launch of the scan kernel over the whole shard with up to kRbMax 32-row blocks of
// queries resident (kNqMax queries at most).
enum : int { kPassAccIn = 1, kPassAccOut = 2, kPassFinal = 4, kPassPair = 8 };
struct PassPlan {
  int q_first, n_q;        // queries [q_first, q_first + n_q) are resident (pair pass: n_q PER CTA, the pass covers
                           // [q_first, q_first + 2 n_q), CTA r of every pair the r-th half)
  int row0, rows;          // their rows [row0, row0 + rows)
  int rbq, n_mtiles;       // 32-row blocks per query, 128-row MMA tiles of the pass (per CTA)
  int flags;               // kPassAccIn: add the partial scores of earlier slices; kPassAccOut: store
                           // partial scores; kPassFinal: scores complete -> top-k (+ all-scores output);
                           // kPassPair: CTA-pair pass (clusters of two CTAs share a token range)
  int group_first, acc_slot;  // row of the partial-score buffer: query group_first + acc_slot (+ i)
};

// allow_pair: CTA-pair passes (run_search decides: shards that span every SM) for as many queries as fill them —
// every CTA of a pair keeps exactly the residency a normal pass would give it, so a pair pass serves twice the
// queries per corpus pass.  Whole queries are paired only when they fill all kMtMax tiles of a CTA: with less
// residency the cross-CTA hand-back of every D stage is paid for fewer MMAs per tile.
// Pair passes always cover a PREFIX of the queries (*n_pair_queries_out); the rest gets normal passes.
void plan_passes(int n_queries, int nq, bool allow_pair, std::vector<PassPlan>* out, int* group_out,
                 int* n_pair_queries_out) {
  out->clear();
  int n_pair_q = 0;
  const int rbq_total = (nq + 31) / 32;
  if (rbq_total <= kRbMax) {
    const int qpp_max = std::min(kNqMax, kRbMax / rbq_total);
    if (allow_pair && qpp_max * rbq_total * 32 > (kMtMax - 1) * kTileM) {
      for (; n_pair_q + 2 * qpp_max <= n_queries; n_pair_q += 2 * qpp_max)
        out->push_back({n_pair_q, qpp_max, 0, nq, rbq_total, (qpp_max * rbq_total * 32 + kTileM - 1) / kTileM,
                        kPassFinal | kPassPair, n_pair_q, 0});
    }
    // whole queries resident: as many per pass as fit, spread evenly over the passes that takes (64
    // queries of one row block: 4 passes of 16 rather than 20+20+20+4, whose short last pass would be
    // HBM-bound while the others are tensor-bound)
    const int rest = n_queries - n_pair_q;
    const int n_passes = (rest + qpp_max - 1) / qpp_max;
    const int qpp = n_passes ? (rest + n_passes - 1) / n_passes : 1;
    for (int b0 = n_pair_q; b0 < n_queries; b0 += qpp) {
      const int nqp = std::min(qpp, n_queries - b0);
      out->push_back({b0, nqp, 0, nq, rbq_total, (nqp * rbq_total * 32 + kTileM - 1) / kTileM, kPassFinal,
                      b0, 0});
    }
    *group_out = 1;
    if (n_pair_queries_out) *n_pair_queries_out = n_pair_q;
    return;
  }
  // queries longer than one pass holds: rows sliced over several passes, partial scores carried through
  // HBM.  Full slices take one pass per query (pair pass: per two queries, one in each CTA); the TAIL slices of up
  // to `group` queries share one pass (Nq = 832: 3 queries = 3 full passes + 1 tail pass instead of 6; with pairs
  // 6 queries = 3 full pair passes + 1 tail pair pass).
  const int rows_per_slice = kRbMax * 32;
  const int n_slices = (nq + rows_per_slice - 1) / rows_per_slice;
  const int tail_row0 = (n_slices - 1) * rows_per_slice;
  const int tail_rows = nq - tail_row0;
  const int tail_rbq = (tail_rows + 31) / 32;
  const int g_max = std::max(1, std::min(kNqMax, kRbMax / tail_rbq));
  int group_used = 0;
  if (allow_pair) {
    const int G = 2 * g_max;                    // queries per pair group; a query's slot in the partial-score
    for (; n_pair_q + G <= n_queries; n_pair_q += G) {   // buffer = its index in the group
      const int b0 = n_pair_q;
      for (int j = 0; j < g_max; ++j)           // queries b0 + 2j (CTA 0) and b0 + 2j + 1 (CTA 1)
        for (int sl = 0; sl + 1 < n_slices; ++sl)
          out->push_back({b0 + 2 * j, 1, sl * rows_per_slice, rows_per_slice, kRbMax, rows_per_slice / kTileM,
                          kPassAccOut | (sl > 0 ? kPassAccIn : 0) | kPassPair, b0, 2 * j});
      out->push_back({b0, g_max, tail_row0, tail_rows, tail_rbq, (g_max * tail_rbq * 32 + kTileM - 1) / kTileM,
                      kPassAccIn | kPassFinal | kPassPair, b0, 0});
      group_used = G;
    }
  }
  const int rest = n_queries - n_pair_q;
  const int group = std::max(1, std::min(g_max, rest));
  for (int b0 = n_pair_q; b0 < n_queries; b0 += group) {
    const int g = std::min(group, n_queries - b0);
    for (int b = 0; b < g; ++b)
      for (int sl = 0; sl + 1 < n_slices; ++sl)
        out->push_back({b0 + b, 1, sl * rows_per_slice, rows_per_slice, kRbMax, rows_per_slice / kTileM,
                        kPassAccOut | (sl > 0 ? kPassAccIn : 0), b0, b});
    out->push_back({b0, g, tail_row0, tail_rows, tail_rbq, (g * tail_rbq * 32 + kTileM - 1) / kTileM,
                    kPassAccIn | kPassFinal, b0, 0});
    group_used = std::max(group_used, g);
  }
  *group_out = std::max(1, group_used);
  if (n_pair_queries_out) *n_pair_queries_out = n_pair_q;
}

// The scan kernels of one storage and mode (partition or listed plan): null where the storage has no such kernel.
// Every one runs ScanSmem::kBytes of dynamic shared memory; pick_scan gives its warpgroup count.
using ScanFn = void (*)(CUtensorMap, ScanParams);
struct ScanKernels {
  ScanFn two;     // two consumer warpgroups, each overlapping its own MMAs with its fold
  ScanFn three;   // three, serial loop (variant 3)
  ScanFn split;   // three, split-tile loop
  ScanFn pair;    // clusters of two CTAs (variant 4)
};
constexpr ScanKernels kScanKernels[3][2] = {   // [Elem][listed]
    {{flmr_scan_kernel<2, Elem::kBF16>, flmr_scan_kernel<3, Elem::kBF16>, flmr_scan_split_kernel<Elem::kBF16>,
      flmr_scan_kernel<2, Elem::kBF16, true>},
     {flmr_scan_listed_kernel<Elem::kBF16>, nullptr, flmr_scan_listed_split_kernel<Elem::kBF16>, nullptr}},
    {{flmr_scan_kernel<2, Elem::kF16>, nullptr, flmr_scan_split_kernel<Elem::kF16>, nullptr},
     {flmr_scan_listed_kernel<Elem::kF16>, nullptr, flmr_scan_listed_split_kernel<Elem::kF16>, nullptr}},
    {{flmr_scan_kernel<2, Elem::kE4M3>, flmr_scan_kernel<3, Elem::kE4M3>, flmr_scan_split_kernel<Elem::kE4M3>,
      nullptr},
     {flmr_scan_listed_kernel<Elem::kE4M3>, nullptr, flmr_scan_listed_split_kernel<Elem::kE4M3>, nullptr}},
};

struct ScanKernel {
  ScanFn fn;   // null: no kernel (run_search and run_listed refuse the variant)
  int wgs;
};

// The kernel a pass of `blocks` occupied 64-row query blocks runs under scan variant `variant`.  Variant 0 picks by
// the blocks: from five up (Nq = 320: five, a full row slice: six) three warpgroups with the split-tile loop (2 / 2 / 1
// or 2 / 2 / 2 blocks, each warpgroup folding one half of a tile under the MMAs of the other), below that two (each
// with two accumulators, its own MMAs overlapping its fold).  On an H100 80GB HBM3 (700 W, 200k x 180-token passages,
// median of 5, DESIGN.md 4.1), with the split loop's MMA descriptors rebuilt in regular registers, 16 x Nq = 320 took
// 6.27 ms split, 6.72 ms with the serial three-warpgroup loop and 7.98 ms with two warpgroups; 3 x Nq = 832 row slices
// 6.63 / 6.73 / 7.19 ms; a 4-block pass (4 x Nq = 256) 5.55 / 5.91 / 5.46 ms; e4m3 at five blocks 3.95 ms split,
// 5.00 ms serial.  With its descriptors in uniform registers, as here, the split loop took less again at five and six
// blocks (4 x Nq = 320 / 384) for every storage: bf16 5.62 / 6.46 ms against 6.06 / 6.88, fp16 5.59 / 6.53 against
// 6.17 / 6.91, e4m3 3.78 / 4.29 against 3.93 / 4.46.  Variants 2, 3, 4 and 6 force a kernel.  Every kernel computes
// bit-identical results.
ScanKernel pick_scan(Elem elem, bool listed, int variant, int blocks) {
  const ScanKernels& t = kScanKernels[static_cast<int>(elem)][listed];
  if (variant == 3) return {t.three, 3};
  if (variant == 4) return {t.pair, 2};
  if (variant == 6 || (variant == 0 && blocks >= 5)) return {t.split, 3};
  return {t.two, 2};
}

// One scan pass over window `win`, whose rows the tensor map `rows` describes.  pair: a CTA-pair pass (planned only
// under variant 4), which scans the resident matrix through the layout's pair partition and half-tile map instead.
// listed: p holds a listed search's plan (run_search's ListedArgs).
int launch_scan(const flmr_corpus* c, ScanParams p, bool pair, bool listed, const Window& win, const CUtensorMap& rows,
                cudaStream_t st) {
  const SlotLayout& l = c->layout;
  // the passes variant 4 leaves to single CTAs run the two-warpgroup kernel
  const int variant = g_scan_variant == 4 && !pair ? 2 : g_scan_variant;
  const ScanKernel k = pick_scan(c->elem, listed, variant, scan_blocks(p.nq_pass, p.rbq));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(pair ? 2 * l.n_pairs : win.n_ctas));
  cfg.blockDim = dim3(scan_threads(k.wgs));
  cfg.dynamicSmemBytes = ScanSmem::kBytes;
  cfg.stream = st;
  if (!listed) {   // a listed pass brings its plan's tiles
    const Partition& part = pair ? l.pair : win.cta;
    p.cta_row_begin = part.row_begin;
    p.cta_tile_base = part.tile_base;
    p.tile_end_mask = part.end_mask;
    p.tile_first_pid = part.first_pid;
  }
  cudaLaunchAttribute cluster{};
  if (pair) {
    // clusters of two CTAs share one of the n_pairs token ranges; the tensor map has a half-tile box
    cluster.id = cudaLaunchAttributeClusterDimension;
    cluster.val.clusterDim = {2, 1, 1};
    cfg.attrs = &cluster;
    cfg.numAttrs = 1;
  }
  void* args[] = {const_cast<CUtensorMap*>(pair ? &l.tmap_half : &rows), &p};
  EventPair ev{};
  if (g_profiling) {
    FLMR_CUDA(cudaEventCreate(&ev.a));
    FLMR_CUDA(cudaEventCreate(&ev.b));
    FLMR_CUDA(cudaEventRecord(ev.a, st));
  }
  cudaError_t e = cudaLaunchKernelExC(&cfg, reinterpret_cast<const void*>(k.fn), args);
  if (const cudaError_t last = cudaGetLastError(); e == cudaSuccess) e = last;   // also clears a failed launch's error
  if (e != cudaSuccess) return fail(FLMR_ERR_CUDA, "scan launch failed: %s", cudaGetErrorString(e));
  ++g_launches;
  if (g_profiling) {
    FLMR_CUDA(cudaEventRecord(ev.b, st));
    g_scan_events.push_back(ev);
  }
  return FLMR_OK;
}

// One launch stages `count` zero-padded query blocks (slot i of the workspace's staging buffer <- sp.pass[i]).
int stage_queries(flmr_workspace* ws, const void* d_q, int nq, const StageParams& sp, int count, cudaStream_t st) {
  const int threads = 256;
  const bool fp8 = ws->corpus->elem == Elem::kE4M3;
  dim3 grid((kMtMax * kTileM * (fp8 ? 8 : 16) + threads - 1) / threads, static_cast<unsigned>(count));
  (fp8 ? flmr_stage_queries_kernel<true> : flmr_stage_queries_kernel<false>)<<<grid, threads, 0, st>>>(
      reinterpret_cast<const uint4*>(d_q), reinterpret_cast<uint4*>(ws->d_qpad), nq, sp);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

// Queries [q0, q0 + nq) of a chunk of `stride` queries; `n_lists` = candidate lists per query (CTAs, or CTA pairs
// for queries that went through pair passes).  d_out_* point at the chunk's first query.
// merge_out: the output rows already hold a running top-k (a streamed corpus's earlier windows), merged in as one more
// list.
int launch_merge_keys(const flmr_corpus* c, flmr_workspace* ws, int n_lists, int stride, int q0, int nq, int k,
                      float* d_out_scores, int64_t* d_out_pids, cudaStream_t st, bool merge_out = false) {
  if (nq <= 0) return FLMR_OK;
  if ((static_cast<int64_t>(n_lists) + merge_out) * k > kMergeThreads * kMergePer)
    return fail(FLMR_ERR_UNSUPPORTED, "n_lists*k = %lld exceeds merge capacity %d",
                (long long)(n_lists + merge_out) * k, kMergeThreads * kMergePer);
  flmr_merge_kernel<<<nq, kMergeThreads, 0, st>>>(ws->d_cand_keys, nullptr, nullptr, n_lists, stride, k, k,
                                                  c->pid_base, c->d_slot_pid, d_out_scores, d_out_pids, q0, merge_out);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

// Partial-score rows of row-sliced (Nq > kRbMax * 32) queries: grown on demand, never shrunk.
int ensure_acc(flmr_workspace* ws, int64_t floats) {
  if (ws->acc_capacity >= floats) return FLMR_OK;
  if (ws->d_acc) cudaFree(ws->d_acc);
  ws->d_acc = nullptr;
  ws->acc_capacity = 0;
  FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(&ws->d_acc), static_cast<size_t>(floats) * sizeof(float)));
  ws->acc_capacity = floats;
  return FLMR_OK;
}

// A listed search (flmr_maxsim_topk_listed / flmr_maxsim_scores_listed): query b's passages are the global ids
// d_pids[h_off[b] .. h_off[b + 1]).
struct ListedArgs {
  const int64_t* h_off;   // [n_queries + 1] host CSR offsets
  const int64_t* d_off;   // the same on the device
  const int64_t* d_pids;
  float* d_scores;        // scores_listed: [h_off[n_queries]] scores aligned with d_pids; null for topk_listed
};

// The plan of one call chunk's passes, in the workspace's plan buffer (flmr_listed_plan_kernel's arrays).
struct ListedChunkPlan {
  std::vector<ListedPass> passes;
  std::vector<int64_t> u_bound, t_bound;   // per pass: union entries and tiles the buffers hold at most
  int64_t words = 0;                       // of a slot bitmap
  uint32_t* allow = nullptr;               // [n_q of the chunk][words] slot bitmaps
  ListedPass* d_passes = nullptr;
  int64_t* meta = nullptr;                 // [passes][2]: union size, tiles
  int64_t *u_cum = nullptr, *u_tile = nullptr, *cta_tile_base = nullptr;
  int32_t *u_slot = nullptr, *tile_row = nullptr, *tile_first = nullptr;
  uint32_t* tile_mask = nullptr;
};

// Plans a listed search's passes `plan` over the chunk of queries [c0, c0 + nqc): the chunk's slot bitmaps (ids outside
// the shard and ids without a slot dropped), then one planner block per pass.  Stream-ordered; no host synchronisation.
// A pass of L listed ids holds at most min(L, slots) union entries and min(L, slots) (ceil(max rows / 96) + 1) + n_ctas
// tiles (a passage starts at most ceil(its rows / 96) tiles of its run).
int plan_listed_chunk(const flmr_corpus* c, flmr_workspace* ws, const std::vector<PassPlan>& plan, int c0, int nqc,
                      const ListedArgs& la, cudaStream_t st, ListedChunkPlan* out) {
  const int64_t ns = slots(c);
  const int n_p = static_cast<int>(plan.size());
  out->words = (ns + 31) / 32;
  out->passes.resize(n_p);
  out->u_bound.resize(n_p);
  out->t_bound.resize(n_p);
  const int n_ctas = c->layout.n_ctas;
  const int64_t tiles_per = (c->layout.max_rows + kTileN - 1) / kTileN + 1;
  int64_t u_total = 0, t_total = 0;
  for (int i = 0; i < n_p; ++i) {
    const PassPlan& pp = plan[i];
    const int64_t listed = la.h_off[c0 + pp.q_first + pp.n_q] - la.h_off[c0 + pp.q_first];
    out->u_bound[i] = std::min(listed, ns);
    out->t_bound[i] = out->u_bound[i] * tiles_per + n_ctas;
    out->passes[i] = {pp.q_first, pp.n_q, u_total, static_cast<int64_t>(i) * (n_ctas + 1), t_total};
    u_total += out->u_bound[i];
    t_total += out->t_bound[i];
  }
  size_t bytes = 0;
  auto take = [&](size_t n) {
    const size_t at = bytes;
    bytes += (n + 15) / 16 * 16;
    return at;
  };
  const size_t o_allow = take(static_cast<size_t>(nqc) * out->words * 4);
  const size_t o_passes = take(n_p * sizeof(ListedPass));
  const size_t o_meta = take(2 * n_p * 8);
  const size_t o_cum = take(u_total * 8), o_tile = take(u_total * 8), o_slot = take(u_total * 4);
  const size_t o_base = take(static_cast<size_t>(n_p) * (n_ctas + 1) * 8);
  const size_t o_row = take(t_total * 4), o_mask = take(t_total * 4), o_first = take(t_total * 4);
  if (ws->plan_capacity < bytes) {
    cudaFree(ws->d_plan);   // waits for the searches still using it
    ws->d_plan = nullptr;
    ws->plan_capacity = 0;
    FLMR_CUDA(cudaMalloc(&ws->d_plan, bytes));
    ws->plan_capacity = bytes;
  }
  uint8_t* base = static_cast<uint8_t*>(ws->d_plan);
  out->allow = reinterpret_cast<uint32_t*>(base + o_allow);
  out->d_passes = reinterpret_cast<ListedPass*>(base + o_passes);
  out->meta = reinterpret_cast<int64_t*>(base + o_meta);
  out->u_cum = reinterpret_cast<int64_t*>(base + o_cum);
  out->u_tile = reinterpret_cast<int64_t*>(base + o_tile);
  out->u_slot = reinterpret_cast<int32_t*>(base + o_slot);
  out->cta_tile_base = reinterpret_cast<int64_t*>(base + o_base);
  out->tile_row = reinterpret_cast<int32_t*>(base + o_row);
  out->tile_mask = reinterpret_cast<uint32_t*>(base + o_mask);
  out->tile_first = reinterpret_cast<int32_t*>(base + o_first);
  FLMR_CUDA(cudaMemsetAsync(out->allow, 0, static_cast<size_t>(nqc) * out->words * 4, st));
  // pageable source: staged by the call, so the vector may go before the copy runs
  FLMR_CUDA(cudaMemcpyAsync(out->d_passes, out->passes.data(), n_p * sizeof(ListedPass), cudaMemcpyHostToDevice, st));
  const int64_t n_entries = la.h_off[c0 + nqc] - la.h_off[c0];
  if (n_entries > 0) {
    flmr_listed_mark_kernel<<<static_cast<unsigned>((n_entries + 255) / 256), 256, 0, st>>>(
        la.d_pids, la.d_off + c0, nqc, c->d_slot_pid, ns, c->pid_base, c->n_passages, out->words, out->allow);
    FLMR_CUDA(cudaGetLastError());
    ++g_launches;
  }
  flmr_listed_plan_kernel<<<n_p, kPlanThreads, 0, st>>>(
      out->d_passes, out->allow, out->words, c->layout.d_poff, n_ctas, out->u_slot, out->u_cum, out->u_tile,
      out->cta_tile_base, out->tile_row, out->tile_mask, out->tile_first, out->meta);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

// Shared driver of flmr_maxsim_scores / flmr_maxsim_topk (and their _allowed forms: `allow` null = unrestricted,
// else query b's bitmap starts at allow + b * allow_stride; and their _listed forms: `listed` non-null, `allow` null).
// Decode the compressed rows of window `win` of a PLAID-coded corpus, staged in ws->d_cstage[b], into the workspace's
// decoded window buffer, on `st`: one grid-stride launch of at most 8 blocks of 256 threads per SM (one wave).
int decode_window(const flmr_corpus* c, flmr_workspace* ws, const Window& win, int b, cudaStream_t st) {
  const int threads = 256;
  const int64_t want = (win.rows / kGroup + threads / 32 - 1) / (threads / 32);
  const unsigned blocks = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(want, 8ll * c->sm_total)));
  const int32_t* codes = reinterpret_cast<const int32_t*>(ws->d_cstage[b]);
  const uint8_t* residuals = ws->d_cstage[b] + c->layout.window_rows * 4;
  auto* kernel = c->elem == Elem::kF16 ? flmr_plaid_window_decode_kernel<true> : flmr_plaid_window_decode_kernel<false>;
  kernel<<<blocks, threads, 0, st>>>(codes, residuals, c->d_centroids, c->d_bucket_weights, c->codec_nbits, win.rows,
                                     reinterpret_cast<uint2*>(ws->d_win[0]));
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

int run_search(const flmr_corpus* c, flmr_workspace* ws, const void* d_q, int n_queries, int nq,
               unsigned flags, int k, const uint32_t* allow, int64_t allow_stride, float* d_all_scores,
               float* d_topk_scores, int64_t* d_topk_pids, cudaStream_t st, const ListedArgs* listed = nullptr) {
  if (!c || !ws || !d_q) return fail(FLMR_ERR_INVALID_ARG, "null corpus / workspace / query pointer");
  if (ws->corpus != c) return fail(FLMR_ERR_INVALID_ARG, "workspace belongs to a different corpus");
  if (n_queries < 0 || nq <= 0) return fail(FLMR_ERR_INVALID_ARG, "bad n_queries=%d nq=%d", n_queries, nq);
  if (k < 0 || k > kMaxK) return fail(FLMR_ERR_UNSUPPORTED, "k=%d outside [1, %d]", k, kMaxK);
  if (allow && allow_stride != 0 && allow_stride < (c->n_passages + 31) / 32)
    return fail(FLMR_ERR_INVALID_ARG, "allow_stride_words=%lld: must be 0 or >= %lld", (long long)allow_stride,
                (long long)((c->n_passages + 31) / 32));
  if (n_queries == 0) return FLMR_OK;
  if (const int code = *reinterpret_cast<volatile int*>(ws->h_status))
    return fail(FLMR_ERR_KERNEL,
                "an earlier scan on this workspace tripped the device watchdog (code %d: %s starved); "
                "the CUDA context is poisoned", code,
                code == kDevTimeoutProducer ? "TMA producer" : code == kDevTimeoutMma ? "MMA issuer" : "epilogue");
  // under variant 0 every storage has both kernels a pass may pick
  if (!pick_scan(c->elem, listed != nullptr, g_scan_variant, 0).fn)
    return fail(FLMR_ERR_UNSUPPORTED, "scan variant %d has no %s kernel", g_scan_variant, elem_name(c->elem));
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  int rc;
  // The scan works in slot space: it scans the stored passages and writes score rows of `ns` entries.  On a compacted
  // corpus the id-indexed allow bitmaps are translated to slots first, and score rows go through stream-ordered
  // scratch that flmr_expand_slot_scores_kernel spreads over the ids (-inf where an id has no slot).
  const int64_t ns = slots(c);
  const bool compacted = c->d_slot_pid != nullptr;
  StreamScratch scratch(st);
  float* d_slot_scores = nullptr;   // [min(n_queries, max_queries), ns]
  if (compacted && allow) {
    const int64_t words = (ns + 31) / 32, n_bitmaps = allow_stride ? n_queries : 1;
    uint32_t* slot_allow = nullptr;
    if ((rc = scratch.alloc(&slot_allow, static_cast<size_t>(n_bitmaps * words) * sizeof(uint32_t)))) return rc;
    const int64_t n = n_bitmaps * words;
    flmr_slot_allow_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(
        allow, allow_stride, c->d_slot_pid, c->pid_base, ns, words, n_bitmaps, slot_allow);
    FLMR_CUDA(cudaGetLastError());
    ++g_launches;
    allow = slot_allow;
    allow_stride = allow_stride ? words : 0;
  }
  if ((compacted || listed) && d_all_scores &&
      (rc = scratch.alloc(&d_slot_scores,
                          static_cast<size_t>(std::min(ws->max_queries, n_queries)) * ns * sizeof(float))))
    return rc;

  ScanParams p{};
  const SlotLayout& l = c->layout;
  p.init_val = (flags & FLMR_FLAG_RELU) ? 0.f : -INFINITY;
  p.n_passages = ns;
  p.dead = c->d_dead;   // null while no slot is deleted: the reducer then makes no extra load
  if (ws->cand_lists < l.n_ctas) {
    // the corpus grew past the CTA count this workspace was sized for (a corpus of fewer passages than SMs launches
    // one CTA per passage); cudaFree waits for the searches still using the old buffer
    cudaFree(ws->d_cand_keys);
    ws->d_cand_keys = nullptr;
    ws->cand_lists = 0;
    FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(&ws->d_cand_keys),
                         static_cast<size_t>(l.n_ctas) * ws->max_queries * kMaxK * 8));
    ws->cand_lists = l.n_ctas;
  }
  p.cand_keys = ws->d_cand_keys;
  p.q_pad = reinterpret_cast<const uint4*>(ws->d_qpad);
  p.status = ws->d_status;
  // reducer: one lane per query sums that query's row maxima when a query has at most 4 row blocks (short queries,
  // many per pass), the whole warp per (query, passage) above; a heuristic, not tuned on this architecture
  p.lane_mode_max_rbq = 4;
#ifdef FLMR_DEBUG   // timing experiments exist only in -DFLMR_DEBUG builds (tools/); the release library has no env hooks
  p.lane_mode_max_rbq = ws->dbg_lane_rbq;
#endif

  // CTA-pair passes (clusters of two CTAs stream one token range, each CTA with the residency of a normal pass, every
  // D tile fetched once and TMA-multicast into both: half the HBM / L2 traffic per query) are planned only when forced
  // (variant 4): on an H100 a pair pass of two Nq = 320 queries over 1M passages took 105.9 ms against 39.4 ms for a
  // single-CTA pass of one, so the product (variant 0) runs single-CTA passes.
  const bool allow_pair = l.n_pairs > 0 && g_scan_variant == 4;
  // a call is processed in chunks of at most ws->max_queries queries (the candidate buffer's capacity);
  // within a chunk: every pass's scan, then the merge over the chunk's queries (one launch per kind of pass)
  std::vector<PassPlan> plan;
  std::vector<int> slot;
  // The corpus is scanned window by window, each window once per call (a resident corpus has one): the windows are
  // the outer loop, the call chunks the inner one, and each chunk's top-k rows carry the running top-k from window to
  // window (the merge of a window's per-CTA lists takes the rows as one more list).  A streamed corpus's window w is
  // copied into buffer w & 1 on the workspace's copy stream; its scans wait for that copy, and the copy of window
  // w + 2 into the same buffer waits for them.  The copy stream first waits for the call's stream, and every copy is
  // waited for by a scan on it, so the call is ordered on `st` like any other.
  // A PLAID-coded corpus copies window w's codes and residuals into staging buffer w & 1 instead; `st` waits for that
  // copy, decodes the window into the one decoded buffer and records decoded_ev[w & 1], and the copy of window w + 2
  // waits for that decode, not for the scans.  Decode and scans are serial on `st` (the scan occupies every SM), so
  // one decoded buffer suffices.
  const int n_windows = static_cast<int>(l.windows.size());
  const int nbits = c->codec_nbits;
  auto copy_window = [&](int w) -> int {
    const Window& win = l.windows[w];
    const int b = w & 1;
    if (nbits) {
      const int64_t pb = kDim * nbits / 8;
      if (w >= 2) FLMR_CUDA(cudaStreamWaitEvent(ws->copy_stream, ws->decoded_ev[b], 0));
      FLMR_CUDA(cudaMemcpyAsync(ws->d_cstage[b], c->h_codes + win.row0, static_cast<size_t>(win.rows) * 4,
                                cudaMemcpyHostToDevice, ws->copy_stream));
      FLMR_CUDA(cudaMemcpyAsync(ws->d_cstage[b] + l.window_rows * 4, c->h_residuals + win.row0 * pb,
                                static_cast<size_t>(win.rows * pb), cudaMemcpyHostToDevice, ws->copy_stream));
      FLMR_CUDA(cudaEventRecord(ws->copied_ev[b], ws->copy_stream));
      return FLMR_OK;
    }
    if (w >= 2) FLMR_CUDA(cudaStreamWaitEvent(ws->copy_stream, ws->scanned_ev[b], 0));
    FLMR_CUDA(cudaMemcpyAsync(ws->d_win[b], static_cast<const char*>(c->h_stream) + win.row0 * kDim * 2,
                              static_cast<size_t>(win.rows) * kDim * 2, cudaMemcpyHostToDevice, ws->copy_stream));
    FLMR_CUDA(cudaEventRecord(ws->copied_ev[b], ws->copy_stream));
    return FLMR_OK;
  };
  if (c->streamed) {
    if (listed) return fail(FLMR_ERR_UNSUPPORTED, "a streamed corpus has no listed scan");
    FLMR_CUDA(cudaEventRecord(ws->fork_ev, st));
    FLMR_CUDA(cudaStreamWaitEvent(ws->copy_stream, ws->fork_ev, 0));
    for (int w = 0; w < std::min(n_windows, 2); ++w)
      if ((rc = copy_window(w))) return rc;
  }
  for (int w = 0; w < n_windows; ++w) {
    const Window& win = l.windows[w];
    const CUtensorMap& rows = nbits ? ws->tmap_win[0] : c->streamed ? ws->tmap_win[w & 1] : l.tmap_d;
    if (c->streamed) FLMR_CUDA(cudaStreamWaitEvent(st, ws->copied_ev[w & 1], 0));
    if (nbits) {
      if ((rc = decode_window(c, ws, win, w & 1, st))) return rc;
      FLMR_CUDA(cudaEventRecord(ws->decoded_ev[w & 1], st));
      if (w + 2 < n_windows && (rc = copy_window(w + 2))) return rc;
    }
    for (int c0 = 0; c0 < n_queries; c0 += ws->max_queries) {
      const int nqc = std::min(ws->max_queries, n_queries - c0);
      const __nv_bfloat16* d_qc = static_cast<const __nv_bfloat16*>(d_q) + static_cast<int64_t>(c0) * nq * kDim;
      float* d_all_c = d_slot_scores ? d_slot_scores
                                     : d_all_scores ? d_all_scores + static_cast<int64_t>(c0) * c->n_passages : nullptr;
      int group = 1, n_pair_q = 0;
      plan_passes(nqc, nq, allow_pair, &plan, &group, &n_pair_q);
      if (!d_all_c && nq > kRbMax * 32 && (rc = ensure_acc(ws, static_cast<int64_t>(group) * ns)))
        return rc;
      p.cand_q_stride = nqc;
      ListedChunkPlan lp;
      if (listed && (rc = plan_listed_chunk(c, ws, plan, c0, nqc, *listed, st, &lp))) return rc;
      slot.assign(plan.size(), 0);
      size_t staged_until = 0;                    // passes [0, staged_until) have their queries staged
      for (size_t pi = 0; pi < plan.size(); ++pi) {
        if (pi == staged_until) {
          // the query blocks of as many of the next passes as fit the staging buffer (a pair pass takes two slots:
          // one block per CTA of a pair) are staged by ONE launch, ahead of their scans
          StageParams sp{};
          int used = 0;
          while (staged_until < plan.size()) {
            const PassPlan& q = plan[staged_until];
            const int need = (q.flags & kPassPair) ? 2 : 1;
            if (used + need > kStageMaxPasses) break;
            slot[staged_until] = used;
            for (int r = 0; r < need; ++r)
              sp.pass[used++] = {q.q_first + r * q.n_q, q.n_q, q.row0, q.rows, q.rbq, q.n_mtiles * kTileM};
            ++staged_until;
          }
          if ((rc = stage_queries(ws, d_qc, nq, sp, used, st))) return rc;
        }
        const PassPlan& pp = plan[pi];
        // partial / final scores of query (group_first + acc_slot + i) live in row i of `acc`
        float* acc = d_all_c
                         ? d_all_c + static_cast<int64_t>(pp.group_first + pp.acc_slot) * ns
                         : (ws->d_acc ? ws->d_acc + static_cast<int64_t>(pp.acc_slot) * ns : nullptr);
        p.q_pad = reinterpret_cast<const uint4*>(ws->d_qpad) + static_cast<int64_t>(slot[pi]) * (kMtMax * kTileM * 16);
        p.n_mtiles = pp.n_mtiles;
        p.nq_pass = pp.n_q;
        p.rbq = pp.rbq;
        p.acc_in = (pp.flags & kPassAccIn) ? acc : nullptr;
        p.acc_out = ((pp.flags & kPassAccOut) || ((pp.flags & kPassFinal) && d_all_c)) ? acc : nullptr;
        p.k = (pp.flags & kPassFinal) ? k : 0;
        p.cand_q_first = pp.q_first;
        p.allow = allow ? allow + static_cast<int64_t>(c0 + pp.q_first) * allow_stride : nullptr;
        p.allow_stride = allow_stride;
        if (listed) {   // the pass's plan, and its queries' slot bitmaps
          const ListedPass& lpp = lp.passes[pi];
          p.cta_row_begin = nullptr;
          p.cta_tile_base = lp.cta_tile_base + lpp.c_off;
          p.tile_end_mask = lp.tile_mask + lpp.t_off;
          p.tile_first_pid = lp.tile_first + lpp.t_off;
          p.tile_row = lp.tile_row + lpp.t_off;
          p.allow = lp.allow + static_cast<int64_t>(pp.q_first) * lp.words;
          p.allow_stride = lp.words;
        }
        if ((rc = launch_scan(c, p, (pp.flags & kPassPair) != 0, listed != nullptr, win, rows, st))) return rc;
      }
      if (listed && d_slot_scores) {
        const int64_t n = listed->h_off[c0 + nqc] - listed->h_off[c0];
        if (n > 0) {
          flmr_listed_scores_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(
              listed->d_pids, listed->d_off + c0, nqc, c->d_slot_pid, ns, c->pid_base, c->n_passages, d_slot_scores,
              listed->d_scores);
          FLMR_CUDA(cudaGetLastError());
          ++g_launches;
        }
      } else if (d_slot_scores) {
        const int64_t n = static_cast<int64_t>(nqc) * c->n_passages;
        flmr_expand_slot_scores_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(
            d_slot_scores, ns, c->d_slot_pid, c->pid_base, c->n_passages, nqc,
            d_all_scores + static_cast<int64_t>(c0) * c->n_passages);
        FLMR_CUDA(cudaGetLastError());
        ++g_launches;
      }
      if (k > 0) {
        float* os = d_topk_scores + static_cast<int64_t>(c0) * k;
        int64_t* op = d_topk_pids + static_cast<int64_t>(c0) * k;
        // queries of pair passes have one candidate list per CTA PAIR, the others one per CTA
        if ((rc = launch_merge_keys(c, ws, l.n_pairs, nqc, 0, n_pair_q, k, os, op, st))) return rc;
        if ((rc = launch_merge_keys(c, ws, win.n_ctas, nqc, n_pair_q, nqc - n_pair_q, k, os, op, st, w > 0)))
          return rc;
      }
    }
    if (c->streamed && !nbits) {
      FLMR_CUDA(cudaEventRecord(ws->scanned_ev[w & 1], st));
      if (w + 2 < n_windows && (rc = copy_window(w + 2))) return rc;
    }
  }
  return FLMR_OK;
}

void free_layout(SlotLayout* l) {
  cudaFree(l->d_poff);
  cudaFree(l->d_doclen);
  auto free_partition = [](const Partition& q) {
    for (void* p : {static_cast<void*>(q.row_begin), static_cast<void*>(q.tile_base), static_cast<void*>(q.end_mask),
                    static_cast<void*>(q.first_pid)})
      cudaFree(p);
  };
  for (const Window& w : l->windows) free_partition(w.cta);
  free_partition(l->pair);
  *l = SlotLayout();
}

// The layout of corpus c whose stored passages (the slots: all of them until a compaction) have row offsets poff and
// lengths lens, over the token matrix d_tokens of n_rows rows (and c's e4m3 copy d_fp8 of an e4m3 corpus), into the
// empty layout *l.  A streamed corpus's windows hold c->window_bytes each; a resident corpus is one window of every
// slot, scanned straight from the matrix.  On failure nothing stays allocated.
int build_layout(const flmr_corpus* c, const __nv_bfloat16* d_tokens, int64_t n_rows, const std::vector<int64_t>& poff,
                 const int32_t* lens, SlotLayout* l) {
  // per-device function attributes of the storage's scan kernels (idempotent), set here rather than at launch time
  for (const ScanKernels& t : kScanKernels[static_cast<int>(c->elem)])
    for (ScanFn fn : {t.two, t.three, t.split, t.pair}) {
      const cudaError_t e =
          fn ? cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, ScanSmem::kBytes) : cudaSuccess;
      if (e != cudaSuccess)
        return fail(FLMR_ERR_CUDA, "cannot raise the dynamic shared memory limit to %d bytes: %s", ScanSmem::kBytes,
                    cudaGetErrorString(e));
    }
  std::vector<std::pair<int64_t, int64_t>> ranges;
  if (int rc = plan_windows(poff, c->streamed ? c->window_bytes / (kDim * 2) : n_rows, &ranges)) return rc;
  const int64_t ns = static_cast<int64_t>(poff.size()) - 1;
  l->h_poff = poff;
  l->h_doclen.assign(lens, lens + ns);
  for (int64_t s = 0; s < ns; ++s) l->max_rows = std::max(l->max_rows, poff[s + 1] - poff[s]);
  int max_ctas = c->sm_total;
#ifdef FLMR_DEBUG
  if (const char* e = getenv("FLMR_NUM_CTAS")) max_ctas = std::max(1, atoi(e));
#endif
  // a partition's arrays, uploaded into *q
  auto upload = [&](const std::vector<int32_t>& rb, const std::vector<int64_t>& tb, const std::vector<uint32_t>& em,
                    const std::vector<int32_t>& fp, Partition* q) {
    q->n_tiles = static_cast<int64_t>(em.size());
    int rc = dev_upload(&q->row_begin, rb, &l->bytes);
    if (!rc) rc = dev_upload(&q->tile_base, tb, &l->bytes);
    if (!rc) rc = dev_upload(&q->end_mask, em, &l->bytes);
    return rc ? rc : dev_upload(&q->first_pid, fp, &l->bytes);
  };
  std::vector<int32_t> rb, fp;
  std::vector<int64_t> tb;
  std::vector<uint32_t> em;
  int rc = dev_upload(&l->d_poff, l->h_poff, &l->bytes);
  if (!rc) rc = dev_upload(&l->d_doclen, l->h_doclen, &l->bytes);
  l->windows.resize(ranges.size());
  for (size_t w = 0; w < ranges.size() && !rc; ++w) {
    Window& win = l->windows[w];
    win.slot0 = ranges[w].first;
    win.slot1 = ranges[w].second;
    win.row0 = poff[win.slot0];
    win.rows = poff[win.slot1] - win.row0;
    l->window_rows = std::max(l->window_rows, win.rows);
    window_partition(poff, win.slot0, win.slot1, max_ctas, &win.n_ctas, &rb, &tb, &em, &fp);
    l->n_ctas = std::max(l->n_ctas, win.n_ctas);
    rc = upload(rb, tb, em, fp, &win.cta);
  }
  if (!rc && !c->streamed)
    rc = encode_rows_map(&l->tmap_d, c->elem == Elem::kE4M3 ? static_cast<const void*>(c->d_fp8) : d_tokens,
                         static_cast<uint64_t>(n_rows), kTileN, c->elem);
  // CTA-pair passes: their own partition + half-tile tensor map.  The product never plans pair passes (see
  // run_search); these few KB per corpus are built so flmr_debug_set_scan_variant(4) can hold the cluster kernel
  // against the single-CTA kernels on any resident bf16 corpus.
  if (!rc && !c->streamed && c->elem == Elem::kBF16 && l->n_ctas >= 2) {
    l->n_pairs = l->n_ctas / 2;
    build_partition(poff, l->n_pairs, kTileN, &rb, &tb, &em, &fp);
    rc = upload(rb, tb, em, fp, &l->pair);
    if (!rc) rc = encode_rows_map(&l->tmap_half, d_tokens, static_cast<uint64_t>(n_rows), kTileN / 2);
  }
  if (rc) free_layout(l);
  return rc;
}

// The packed (*soff) and stored (*poff) row offsets of a new corpus's passages (*aligned: as passage_offsets), refused
// when a corpus cannot hold them: a zero-length passage, 2^31 stored rows, or (window_bytes > 0: a streamed corpus) a
// passage longer than a window.
int corpus_offsets(const int32_t* h_doclens, int64_t n_passages, int64_t window_bytes, std::vector<int64_t>* soff,
                   std::vector<int64_t>* poff, bool* aligned) {
  if (int rc = passage_offsets(h_doclens, n_passages, soff, poff, aligned)) return rc;
  const int64_t n_rows = (*poff)[n_passages];
  if (n_rows + kTileN >= (1ll << 31))
    return fail(FLMR_ERR_UNSUPPORTED, "%lld stored token rows exceed the 2^31 per-shard limit; shard the corpus",
                (long long)n_rows);
  std::vector<std::pair<int64_t, int64_t>> ranges;
  return window_bytes > 0 ? plan_windows(*poff, window_bytes / (kDim * 2), &ranges) : FLMR_OK;
}

// A new corpus handle, with no matrix and no layout yet: streamed when window_bytes > 0.
int new_corpus(int device, int64_t n_passages, const std::vector<int64_t>& soff, const std::vector<int64_t>& poff,
               int64_t pid_base, Elem elem, int sm_total, int64_t window_bytes, flmr_corpus** out) {
  flmr_corpus* c = new (std::nothrow) flmr_corpus();
  if (!c) return fail(FLMR_ERR_OOM, "host allocation failed");
  c->device = device;
  c->n_passages = n_passages;
  c->n_tokens = soff[n_passages];
  c->n_rows = poff[n_passages];
  c->pid_base = pid_base;
  c->elem = elem;
  c->sm_total = sm_total;
  c->streamed = window_bytes > 0;
  c->window_bytes = window_bytes;
  *out = c;
  return FLMR_OK;
}

// The pinned, mapped host matrix of a new streamed corpus (n_rows set); d_tokens becomes its device alias.
int alloc_stream_matrix(flmr_corpus* c) {
  const size_t bytes = static_cast<size_t>(c->n_rows) * kDim * 2;
  if (const cudaError_t e = cudaHostAlloc(&c->h_stream, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
      e != cudaSuccess) {
    c->h_stream = nullptr;
    return fail(FLMR_ERR_OOM, "cudaHostAlloc(%zu B) for the streamed token matrix failed: %s", bytes,
                cudaGetErrorString(e));
  }
  FLMR_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&c->d_tokens), c->h_stream, 0));
  return FLMR_OK;
}

// The token matrix of a new corpus (n_rows set): bf16 in HBM, or (e4m3) the e4m3 copy in HBM plus the bf16 master
// in pinned, mapped host memory, whose device alias becomes d_tokens (the repack / scatter kernels write both).
int alloc_token_matrix(flmr_corpus* c) {
  const size_t rows = static_cast<size_t>(c->n_rows);
  cudaError_t e;
  if (c->elem == Elem::kE4M3) {
    if ((e = cudaHostAlloc(&c->h_master, rows * kDim * 2, cudaHostAllocMapped | cudaHostAllocPortable)) != cudaSuccess) {
      c->h_master = nullptr;
      return fail(FLMR_ERR_OOM, "cudaHostAlloc(%zu B) for the bf16 master failed: %s", rows * kDim * 2,
                  cudaGetErrorString(e));
    }
    FLMR_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&c->d_tokens), c->h_master, 0));
    if (int rc = gm_grow(&c->vm_fp8, c->device, rows * kDim)) return rc;
    c->d_fp8 = reinterpret_cast<uint8_t*>(c->vm_fp8.base);
    return FLMR_OK;
  }
  if (int rc = gm_grow(&c->vm_tokens, c->device, rows * kDim * 2)) return rc;
  c->d_tokens = reinterpret_cast<__nv_bfloat16*>(c->vm_tokens.base);
  return FLMR_OK;
}

// Packed bf16 rows of n passages (soff / poff relative to the first; host or device source) into the padded layout
// at dst, and (dst8 non-null) as e4m3 at dst8.  Synchronous.
cudaError_t pack_passages(const void* tokens, bool is_device_ptr, const std::vector<int64_t>& soff,
                          const std::vector<int64_t>& poff, const int32_t* h_doclens, int64_t n_passages, uint4* dst,
                          uint2* dst8) {
  int64_t *d_soff = nullptr, *d_poff = nullptr;
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&d_soff), soff.size() * sizeof(int64_t));
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&d_poff), poff.size() * sizeof(int64_t));
  if (e == cudaSuccess) e = cudaMemcpy(d_soff, soff.data(), soff.size() * sizeof(int64_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_poff, poff.data(), poff.size() * sizeof(int64_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && is_device_ptr) {
    const int threads = 256;
    const int64_t blocks = (n_passages * 32 + threads - 1) / threads;
    flmr_repack_kernel<<<static_cast<unsigned>(blocks), threads>>>(static_cast<const uint4*>(tokens), d_soff, d_poff,
                                                                   dst, dst8, 0, n_passages, 0);
    ++g_launches;
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
  } else if (e == cudaSuccess) {
    // host source: stage through a bounded device buffer, chunk by chunk of whole passages
    const int64_t chunk_rows = std::min<int64_t>(soff[n_passages], (256ll << 20) / (kDim * 2));
    int64_t max_len = 0;
    for (int64_t p = 0; p < n_passages; ++p) max_len = std::max<int64_t>(max_len, h_doclens[p]);
    const int64_t buf_rows = std::max(chunk_rows, max_len);
    uint4* d_stage = nullptr;
    e = cudaMalloc(reinterpret_cast<void**>(&d_stage), static_cast<size_t>(buf_rows) * kDim * 2);
    int64_t pa = 0;
    while (e == cudaSuccess && pa < n_passages) {
      int64_t pb = std::upper_bound(soff.begin() + pa, soff.end(), soff[pa] + buf_rows) - soff.begin() - 1;
      pb = std::max(pb, pa + 1);
      const int64_t rows = soff[pb] - soff[pa];
      e = cudaMemcpy(d_stage, static_cast<const char*>(tokens) + soff[pa] * kDim * 2,
                     static_cast<size_t>(rows) * kDim * 2, cudaMemcpyHostToDevice);
      if (e != cudaSuccess) break;
      const int threads = 256;
      const int64_t cnt = pb - pa;
      const int64_t blocks = (cnt * 32 + threads - 1) / threads;
      flmr_repack_kernel<<<static_cast<unsigned>(blocks), threads>>>(d_stage, d_soff, d_poff, dst, dst8, pa, cnt,
                                                                     soff[pa]);
      ++g_launches;
      e = cudaGetLastError();
      if (e == cudaSuccess) e = cudaDeviceSynchronize();
      pa = pb;
    }
    cudaFree(d_stage);
  }
  cudaFree(d_soff);
  cudaFree(d_poff);
  return e;
}

// The host twin of flmr_scatter_rows_kernel, for a streamed corpus's host matrix: packed rows [s0, s0 + n) at src go to
// their place in the padded layout at dst, a passage's last token also over its padding rows.  kRow: bytes per row
// (a PLAID-coded corpus scatters its codes and its residuals this way too).
void host_scatter_rows(const char* src, const std::vector<int64_t>& soff, const std::vector<int64_t>& poff, int64_t s0,
                       int64_t n, char* dst, int64_t kRow = kDim * 2) {
  int64_t p = std::upper_bound(soff.begin(), soff.end(), s0) - soff.begin() - 1;
  for (int64_t r = s0; r < s0 + n; ++p) {
    const int64_t take = std::min(soff[p + 1], s0 + n) - r;   // rows of passage p in this chunk
    char* d = dst + (poff[p] + (r - soff[p])) * kRow;
    memcpy(d, src + (r - s0) * kRow, static_cast<size_t>(take * kRow));
    r += take;
    if (r == soff[p + 1])
      for (int64_t j = poff[p] + (soff[p + 1] - soff[p]); j < poff[p + 1]; ++j)
        memcpy(dst + j * kRow, src + (r - 1 - s0) * kRow, kRow);
  }
}

// ---- compaction schedule (pure host logic; exported for tests as flmr_debug_compact_plan) ----------------------
// The kept passages keep their padded row blocks and their order: each run of kept rows moves down by the rows removed
// before it, so no destination lies above its source.  The moves are cut into chunks of at most `chunk_rows`
// destination rows, executed in destination order.  A chunk whose destination rows overlap its own source rows goes
// through a staging buffer (all of its rows read, then all written); any other chunk is copied directly.  Writing
// chunk i never touches a source row of a later chunk: those lie at or above chunk i's source rows, which lie at or
// above its destinations.  The staging buffer therefore never holds more than chunk_rows rows.
constexpr int64_t kCompactStageBytes = 256ll << 20;
constexpr int64_t kCompactChunkRows = kCompactStageBytes / (kDim * 2);   // a chunk of bf16 rows fills the stage

struct MovePiece {
  int64_t src, dst, rows;
  bool staged;
  int64_t chunk;
};

// runs: (first source row, rows) of each run of kept rows, ascending; their destinations are packed from row 0.
// in_place = false: the destination is another matrix (an adopted one is copied out), so every run moves, directly.
void plan_compaction(const std::vector<std::pair<int64_t, int64_t>>& runs, int64_t chunk_rows, bool in_place,
                     std::vector<MovePiece>* out) {
  out->clear();
  int64_t d = 0, chunk = 0, chunk_rows_used = 0;
  size_t chunk_first = 0;
  auto close_chunk = [&]() {
    if (chunk_rows_used == 0) return;
    // the chunk's destinations are [d - used, d); its lowest source row is its first piece's
    const bool staged = in_place && d > (*out)[chunk_first].src;
    for (size_t i = chunk_first; i < out->size(); ++i) (*out)[i].staged = staged;
    ++chunk;
    chunk_rows_used = 0;
    chunk_first = out->size();
  };
  for (const auto& run : runs) {
    int64_t src = run.first, n = run.second;
    if (in_place && src == d) {   // rows already in place (in front of the first removed passage)
      d += n;
      continue;
    }
    while (n > 0) {
      const int64_t take = std::min(n, chunk_rows - chunk_rows_used);
      out->push_back({src, d, take, false, chunk});
      src += take;
      d += take;
      n -= take;
      chunk_rows_used += take;
      if (chunk_rows_used == chunk_rows) close_chunk();
    }
  }
  close_chunk();
}

// Runs of kept rows of a corpus whose passages have padded row offsets poff, keep[s] = the passage stays.
std::vector<std::pair<int64_t, int64_t>> kept_runs(const std::vector<int64_t>& poff, const std::vector<char>& keep) {
  std::vector<std::pair<int64_t, int64_t>> runs;
  const int64_t n = static_cast<int64_t>(keep.size());
  for (int64_t s = 0; s < n;) {
    if (!keep[s]) {
      ++s;
      continue;
    }
    int64_t e = s;
    while (e < n && keep[e]) ++e;
    runs.emplace_back(poff[s], poff[e] - poff[s]);
    s = e;
  }
  return runs;
}

// Execute a compaction schedule on one matrix of `row_vecs` 16-byte vectors per row (16: bf16 / fp16, 8: e4m3):
// src and dst are the same matrix in place, or (an adopted matrix) two.  Stream-ordered on the legacy stream.
cudaError_t run_moves(const std::vector<MovePiece>& plan, const int64_t* d_pdst, const int64_t* d_psrc,
                      const uint4* src, uint4* dst, uint4* stage, int row_vecs) {
  const int threads = 256;
  for (size_t k0 = 0; k0 < plan.size();) {
    size_t k1 = k0;
    while (k1 < plan.size() && plan[k1].chunk == plan[k0].chunk) ++k1;
    const int64_t d0 = plan[k0].dst, rows = plan[k1 - 1].dst + plan[k1 - 1].rows - d0;
    const int64_t n = rows * row_vecs;
    const unsigned blocks = static_cast<unsigned>((n + threads - 1) / threads);
    if (plan[k0].staged) {   // every source row of the chunk is read before any of its destinations is written
      flmr_move_rows_kernel<<<blocks, threads>>>(src, stage, d_pdst, d_psrc, k0, k1, d0, rows, d0, row_vecs);
      ++g_launches;
      const cudaError_t e = cudaMemcpyAsync(dst + d0 * row_vecs, stage, static_cast<size_t>(n) * 16,
                                            cudaMemcpyDeviceToDevice, 0);
      if (e != cudaSuccess) return e;
    } else {
      flmr_move_rows_kernel<<<blocks, threads>>>(src, dst, d_pdst, d_psrc, k0, k1, d0, rows, 0, row_vecs);
      ++g_launches;
    }
    if (const cudaError_t e = cudaGetLastError(); e != cudaSuccess) return e;
    k0 = k1;
  }
  return cudaSuccess;
}

}  // namespace

// =================================== C ABI =============================================================
extern "C" {

const char* flmr_last_error(void) { return g_last_error.c_str(); }
int flmr_abi_version(void) { return FLMR_ABI_VERSION; }

extern "C++" {
namespace {
// flmr_corpus_create (window_bytes 0) and flmr_corpus_create_streamed (window_bytes as the caller passed it: a streamed
// call's window of no bytes is refused in its place among the checks, not taken for a resident corpus).
int corpus_create(const void* tokens, const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                  int64_t pid_base, unsigned flags, bool streamed, int64_t window_bytes, flmr_corpus_t** out) {
  if (!out) return fail(FLMR_ERR_INVALID_ARG, "out is null");
  *out = nullptr;
  if (streamed && (flags & ~FLMR_CORPUS_FP16))
    return fail(FLMR_ERR_UNSUPPORTED, "flags 0x%x: a streamed corpus is bf16 or FLMR_CORPUS_FP16, and is never adopted",
                flags);
  if (dim != kDim) return fail(FLMR_ERR_UNSUPPORTED, "dim=%d (only %d is supported)", dim, kDim);
  if (n_passages <= 0 || !tokens || !h_doclens)
    return fail(FLMR_ERR_INVALID_ARG, "empty corpus or null tokens/doclens");
  if (streamed && window_bytes < kDim * 2)
    return fail(FLMR_ERR_INVALID_ARG, "window_bytes=%lld holds no row", (long long)window_bytes);
  Elem elem;
  std::vector<int64_t> soff, poff;
  bool aligned;
  int rc;
  if ((rc = storage_from_flags(flags, &elem)) ||
      (rc = corpus_offsets(h_doclens, n_passages, window_bytes, &soff, &poff, &aligned)))   // before any allocation
    return rc;

  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  int sm_count;
  bool is_device_ptr;
  if ((rc = sm90_count(device, &sm_count)) || (rc = token_source(tokens, device, &is_device_ptr))) return rc;
  if ((flags & FLMR_CORPUS_ADOPT) && !is_device_ptr)
    return fail(FLMR_ERR_INVALID_ARG, "FLMR_CORPUS_ADOPT requires a device pointer");

  flmr_corpus* c;
  if ((rc = new_corpus(device, n_passages, soff, poff, pid_base, elem, sm_count, window_bytes, &c))) return rc;
  auto bail = [&](int code) {
    flmr_corpus_destroy(c);
    return code;
  };

  // --- token matrix residency: pinned host memory (streamed), the caller's buffer (adopted) or library HBM ---
  if (streamed) {
    rc = alloc_stream_matrix(c);
  } else if ((flags & FLMR_CORPUS_ADOPT) && aligned && (reinterpret_cast<uintptr_t>(tokens) % 16 == 0)) {
    c->d_tokens = static_cast<__nv_bfloat16*>(const_cast<void*>(tokens));
    c->adopted = true;
  } else {
    rc = alloc_token_matrix(c);
  }
  if (rc) return bail(rc);
  if (streamed && !is_device_ptr) {
    host_scatter_rows(static_cast<const char*>(tokens), soff, poff, 0, c->n_tokens, static_cast<char*>(c->h_stream));
  } else if (!c->adopted) {   // the repack kernel writes a streamed corpus's host matrix through its device alias
    const cudaError_t e = pack_passages(tokens, is_device_ptr, soff, poff, h_doclens, n_passages,
                                        reinterpret_cast<uint4*>(c->d_tokens),
                                        reinterpret_cast<uint2*>(c->d_fp8));   // d_fp8: null but for an e4m3 corpus
    if (e != cudaSuccess)
      return bail(fail(FLMR_ERR_CUDA, "corpus repack failed: %s", cudaGetErrorString(e)));
  }

  if ((rc = build_layout(c, c->d_tokens, c->n_rows, poff, h_doclens, &c->layout))) return bail(rc);
  *out = c;
  return FLMR_OK;
}
}  // namespace
}  // extern "C++"

int flmr_corpus_create(const void* tokens, const int32_t* h_doclens, int64_t n_passages, int dim,
                       int device, int64_t pid_base, unsigned flags, flmr_corpus_t** out) {
  return corpus_create(tokens, h_doclens, n_passages, dim, device, pid_base, flags, false, 0, out);
}

int flmr_corpus_create_streamed(const void* tokens, const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                int64_t pid_base, unsigned flags, int64_t window_bytes, flmr_corpus_t** out) {
  return corpus_create(tokens, h_doclens, n_passages, dim, device, pid_base, flags, true, window_bytes, out);
}

int flmr_corpus_residency(const flmr_corpus_t* c, int* streamed, int64_t* window_bytes, int64_t* host_bytes) {
  if (!c) return fail(FLMR_ERR_INVALID_ARG, "null corpus");
  if (streamed) *streamed = c->streamed ? 1 : 0;
  if (window_bytes) *window_bytes = c->streamed ? c->window_bytes : 0;
  if (host_bytes)
    *host_bytes = !c->streamed ? 0 : c->n_rows * (c->codec_nbits ? codec_row_bytes(c->codec_nbits) : kDim * 2);
  return FLMR_OK;
}

int flmr_corpus_codec(const flmr_corpus_t* c, int* nbits) {
  if (!c || !nbits) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  *nbits = c->codec_nbits;
  return FLMR_OK;
}

int flmr_corpus_destroy(flmr_corpus_t* c) {
  if (!c) return FLMR_OK;
  DeviceGuard guard(c->device);
  // no search still reads them
  if (c->vm_tokens.base || c->vm_fp8.base || c->h_stream || c->h_codes) cudaDeviceSynchronize();
  if (c->h_master) cudaFreeHost(c->h_master);   // d_tokens is its device alias
  if (c->h_stream) cudaFreeHost(c->h_stream);   // likewise
  if (c->h_codes) cudaFreeHost(c->h_codes);     // h_residuals lies in the same allocation
  gm_free(&c->vm_tokens);                       // (an adopted matrix is the caller's and has no mapping here)
  gm_free(&c->vm_fp8);
  free_layout(&c->layout);
  cudaFree(c->d_dead);
  cudaFree(c->d_slot_pid);
  cudaFree(c->d_centroids);
  cudaFree(c->d_bucket_weights);
  delete c;
  return FLMR_OK;
}

int flmr_corpus_builder_create(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                               int64_t pid_base, flmr_corpus_builder_t** out) {
  return flmr_corpus_builder_create_ex(h_doclens, n_passages, dim, device, pid_base, FLMR_CORPUS_COPY, out);
}

extern "C++" {
namespace {
// The codec of a PLAID-coded streamed corpus, as flmr_corpus_builder_create_plaid receives it.
struct PlaidCodec {
  int nbits;
  const float* centroids;   // host fp32 [n_centroids, 128]
  int64_t n_centroids;
  const float* bucket_weights;   // host fp32 [2^nbits]
};

// flmr_corpus_builder_create_ex (window_bytes = 0), flmr_corpus_builder_create_streamed (window_bytes > 0) and
// flmr_corpus_builder_create_plaid (window_bytes > 0 and a codec).
int builder_create(const int32_t* h_doclens, int64_t n_passages, int dim, int device, int64_t pid_base, unsigned flags,
                   int64_t window_bytes, flmr_corpus_builder_t** out, const PlaidCodec* codec = nullptr) {
  if (!out) return fail(FLMR_ERR_INVALID_ARG, "out is null");
  *out = nullptr;
  const bool streamed = window_bytes > 0;
  if (streamed && (flags & ~FLMR_CORPUS_FP16))
    return fail(FLMR_ERR_UNSUPPORTED, "builder flags 0x%x: a streamed corpus is bf16 or FLMR_CORPUS_FP16", flags);
  if (flags & ~(FLMR_CORPUS_FP8 | FLMR_CORPUS_FP16))
    return fail(FLMR_ERR_INVALID_ARG, "builder flags 0x%x: only FLMR_CORPUS_FP8 or FLMR_CORPUS_FP16 applies to a "
                "streamed load", flags);
  Elem elem;
  if (int rc = storage_from_flags(flags, &elem)) return rc;
  if (dim != kDim) return fail(FLMR_ERR_UNSUPPORTED, "dim=%d (only %d is supported)", dim, kDim);
  if (n_passages <= 0 || !h_doclens) return fail(FLMR_ERR_INVALID_ARG, "empty corpus or null doclens");
  if (codec) {
    const int nb = codec->nbits;
    if (nb != 1 && nb != 2 && nb != 4 && nb != 8)
      return fail(FLMR_ERR_INVALID_ARG, "nbits=%d (the PLAID codec packs 1, 2, 4 or 8 bits per dim)", nb);
    if (!codec->centroids || !codec->bucket_weights || codec->n_centroids < 1)
      return fail(FLMR_ERR_INVALID_ARG, "null centroids / bucket weights or no centroid");
  }
  flmr_corpus_builder* b = new (std::nothrow) flmr_corpus_builder();
  if (!b) return fail(FLMR_ERR_OOM, "host allocation failed");
  auto bail = [&](int code) {
    flmr_corpus_builder_destroy(b);
    return code;
  };
  b->doclens.assign(h_doclens, h_doclens + n_passages);
  if (int rc = corpus_offsets(h_doclens, n_passages, window_bytes, &b->soff, &b->poff, &b->aligned)) return bail(rc);
  DeviceGuard guard(device);
  if (!guard.ok) return bail(fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device));
  int sm_count;
  if (int rc = sm90_count(device, &sm_count)) return bail(rc);
  flmr_corpus* c;
  if (int rc = new_corpus(device, n_passages, b->soff, b->poff, pid_base, elem, sm_count, window_bytes, &c))
    return bail(rc);
  b->corpus = c;
  if (codec) {
    // the compressed arrays in the padded row layout, filled by flmr_corpus_builder_append_plaid; the tables wait for
    // finish
    const size_t bytes = static_cast<size_t>(c->n_rows) * codec_row_bytes(codec->nbits);
    void* h = nullptr;
    if (const cudaError_t e = cudaHostAlloc(&h, bytes, cudaHostAllocMapped | cudaHostAllocPortable); e != cudaSuccess)
      return bail(fail(FLMR_ERR_OOM, "cudaHostAlloc(%zu B) for the compressed rows failed: %s", bytes,
                       cudaGetErrorString(e)));
    c->codec_nbits = codec->nbits;
    c->n_centroids = codec->n_centroids;
    c->h_codes = static_cast<int32_t*>(h);
    c->h_residuals = static_cast<uint8_t*>(h) + c->n_rows * 4;
    void* d = nullptr;
    if (const cudaError_t e = cudaHostGetDevicePointer(&d, h, 0); e != cudaSuccess)
      return bail(fail(FLMR_ERR_CUDA, "cudaHostGetDevicePointer: %s", cudaGetErrorString(e)));
    c->d_codes = static_cast<const int32_t*>(d);
    c->d_residuals = static_cast<const uint8_t*>(d) + c->n_rows * 4;
    b->centroids.assign(codec->centroids, codec->centroids + codec->n_centroids * kDim);
    b->bucket_weights.assign(codec->bucket_weights, codec->bucket_weights + (1 << codec->nbits));
    *out = b;
    return FLMR_OK;
  }
  if (streamed) {
    // rows are read (or copied) straight into the host matrix, or, when passages need padding, through one pinned
    // staging buffer from which host_scatter_rows puts them in place; the device is not involved
    if (int rc = alloc_stream_matrix(c)) return bail(rc);
    const size_t buf_bytes = static_cast<size_t>(flmr_corpus_builder::kBufRows) * kDim * 2;
    if (!b->aligned) {
      if (const cudaError_t e = cudaHostAlloc(&b->h_pin[0], buf_bytes, cudaHostAllocDefault); e != cudaSuccess) {
        b->h_pin[0] = nullptr;
        return bail(fail(FLMR_ERR_OOM, "staging buffer: %s", cudaGetErrorString(e)));
      }
    }
    *out = b;
    return FLMR_OK;
  }
  if (int rc = alloc_token_matrix(c)) return bail(rc);
  // an e4m3 corpus always goes through the scatter kernel, which writes the master and the e4m3 copy
  const bool scatter = !b->aligned || elem == Elem::kE4M3;
  const size_t buf_bytes = static_cast<size_t>(flmr_corpus_builder::kBufRows) * kDim * 2;
  cudaError_t e;
  if ((e = cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking)) != cudaSuccess)
    return bail(fail(FLMR_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e)));
  for (int i = 0; i < flmr_corpus_builder::kBufs; ++i) {
    if ((e = cudaHostAlloc(&b->h_pin[i], buf_bytes, cudaHostAllocDefault)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&b->free_ev[i], cudaEventDisableTiming)) != cudaSuccess ||
        (scatter && (e = cudaMalloc(reinterpret_cast<void**>(&b->d_stage[i]), buf_bytes)) != cudaSuccess))
      return bail(fail(FLMR_ERR_OOM, "staging buffers: %s", cudaGetErrorString(e)));
  }
  if (scatter) {
    int rc;
    if ((rc = dev_upload(&b->d_soff, b->soff, nullptr)) || (rc = dev_upload(&b->d_poff, b->poff, nullptr)))
      return bail(rc);
  }
  *out = b;
  return FLMR_OK;
}
}  // namespace
}  // extern "C++"

int flmr_corpus_builder_create_ex(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                  int64_t pid_base, unsigned flags, flmr_corpus_builder_t** out) {
  return builder_create(h_doclens, n_passages, dim, device, pid_base, flags, 0, out);
}

int flmr_corpus_builder_create_streamed(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                        int64_t pid_base, unsigned flags, int64_t window_bytes,
                                        flmr_corpus_builder_t** out) {
  if (window_bytes < kDim * 2) {
    if (out) *out = nullptr;
    return fail(FLMR_ERR_INVALID_ARG, "window_bytes=%lld holds no row", (long long)window_bytes);
  }
  return builder_create(h_doclens, n_passages, dim, device, pid_base, flags, window_bytes, out);
}

int flmr_corpus_builder_create_plaid(const int32_t* h_doclens, int64_t n_passages, int dim, int device,
                                     int64_t pid_base, unsigned flags, int64_t window_bytes, int nbits,
                                     const float* h_centroids, int64_t n_centroids, const float* h_bucket_weights,
                                     flmr_corpus_builder_t** out) {
  if (window_bytes < kDim * 2) {
    if (out) *out = nullptr;
    return fail(FLMR_ERR_INVALID_ARG, "window_bytes=%lld holds no row", (long long)window_bytes);
  }
  const PlaidCodec codec{nbits, h_centroids, n_centroids, h_bucket_weights};
  return builder_create(h_doclens, n_passages, dim, device, pid_base, flags, window_bytes, out, &codec);
}

int flmr_corpus_builder_append_plaid(flmr_corpus_builder_t* b, const int32_t* h_codes, const uint8_t* h_residuals,
                                     int64_t n_rows) {
  if (!b || !h_codes || !h_residuals) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  flmr_corpus* c = b->corpus;
  if (!c->codec_nbits)
    return fail(FLMR_ERR_INVALID_ARG, "flmr_corpus_builder_append_plaid feeds the builder of a PLAID-coded corpus only");
  if (n_rows < 0 || b->rows_done + n_rows > c->n_tokens)
    return fail(FLMR_ERR_INVALID_ARG, "append of %lld rows overruns the %lld rows the doclens announce (%lld done)",
                (long long)n_rows, (long long)c->n_tokens, (long long)b->rows_done);
  for (int64_t i = 0; i < n_rows; ++i)   // every code, before any row is stored: a search never checks them
    if (h_codes[i] < 0 || h_codes[i] >= c->n_centroids)
      return fail(FLMR_ERR_INVALID_ARG, "code %d of row %lld is outside [0, %lld)", h_codes[i],
                  (long long)(b->rows_done + i), (long long)c->n_centroids);
  timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  host_scatter_rows(reinterpret_cast<const char*>(h_codes), b->soff, b->poff, b->rows_done, n_rows,
                    reinterpret_cast<char*>(c->h_codes), 4);
  host_scatter_rows(reinterpret_cast<const char*>(h_residuals), b->soff, b->poff, b->rows_done, n_rows,
                    reinterpret_cast<char*>(c->h_residuals), kDim * c->codec_nbits / 8);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  b->fill_s += (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
  b->rows_done += n_rows;
  return FLMR_OK;
}

extern "C++" {
namespace {
// Feed `n_rows` packed rows through the staging ring; `fill(dst, row0, rows)` writes rows [row0, row0 + rows) of
// this append into pinned memory (memcpy from a host buffer, or pread from a file).
template <typename Fill>
int builder_feed(flmr_corpus_builder* b, int64_t n_rows, Fill fill) {
  flmr_corpus* c = b->corpus;
  if (c->codec_nbits)
    return fail(FLMR_ERR_INVALID_ARG, "the builder of a PLAID-coded corpus takes flmr_corpus_builder_append_plaid");
  if (n_rows < 0 || b->rows_done + n_rows > c->n_tokens)
    return fail(FLMR_ERR_INVALID_ARG, "append of %lld rows overruns the %lld rows the doclens announce (%lld done)",
                (long long)n_rows, (long long)c->n_tokens, (long long)b->rows_done);
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  if (c->streamed) {   // straight into the host matrix (aligned), or through the staging buffer and host_scatter_rows
    char* matrix = static_cast<char*>(c->h_stream);
    for (int64_t r0 = 0; r0 < n_rows; r0 += flmr_corpus_builder::kBufRows) {
      const int64_t rows = std::min<int64_t>(flmr_corpus_builder::kBufRows, n_rows - r0);
      void* dst = b->aligned ? matrix + b->rows_done * kDim * 2 : b->h_pin[0];
      timespec t0, t1;
      clock_gettime(CLOCK_MONOTONIC, &t0);
      if (int rc = fill(dst, r0, rows)) return rc;
      clock_gettime(CLOCK_MONOTONIC, &t1);
      b->fill_s += (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
      if (!b->aligned) host_scatter_rows(static_cast<const char*>(b->h_pin[0]), b->soff, b->poff, b->rows_done, rows,
                                         matrix);
      b->rows_done += rows;
    }
    return FLMR_OK;
  }
  for (int64_t r0 = 0; r0 < n_rows; r0 += flmr_corpus_builder::kBufRows) {
    const int64_t rows = std::min<int64_t>(flmr_corpus_builder::kBufRows, n_rows - r0);
    const int i = b->next;
    b->next = (b->next + 1) % flmr_corpus_builder::kBufs;
    FLMR_CUDA(cudaEventSynchronize(b->free_ev[i]));          // the DMA that last read this buffer is done
    timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    if (int rc = fill(b->h_pin[i], r0, rows)) return rc;
    clock_gettime(CLOCK_MONOTONIC, &t1);
    b->fill_s += (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
    const size_t bytes = static_cast<size_t>(rows) * kDim * 2;
    const int64_t s0 = b->rows_done;
    if (b->aligned && c->elem != Elem::kE4M3) {   // packed order == stored order: straight into place
      FLMR_CUDA(cudaMemcpyAsync(c->d_tokens + s0 * kDim, b->h_pin[i], bytes, cudaMemcpyHostToDevice, b->stream));
    } else {
      FLMR_CUDA(cudaMemcpyAsync(b->d_stage[i], b->h_pin[i], bytes, cudaMemcpyHostToDevice, b->stream));
      const int threads = 256;
      flmr_scatter_rows_kernel<<<static_cast<unsigned>((rows * 16 + threads - 1) / threads), threads, 0, b->stream>>>(
          b->d_stage[i], b->d_soff, b->d_poff, reinterpret_cast<uint4*>(c->d_tokens),
          reinterpret_cast<uint2*>(c->d_fp8), s0, rows, c->n_passages);
      FLMR_CUDA(cudaGetLastError());
      ++g_launches;
    }
    FLMR_CUDA(cudaEventRecord(b->free_ev[i], b->stream));
    b->rows_done += rows;
  }
  return FLMR_OK;
}
}  // namespace
}  // extern "C++"

int flmr_corpus_builder_append(flmr_corpus_builder_t* b, const void* h_tokens_bf16, int64_t n_rows) {
  if (!b || !h_tokens_bf16) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  const char* src = static_cast<const char*>(h_tokens_bf16);
  return builder_feed(b, n_rows, [&](void* dst, int64_t r0, int64_t rows) {
    memcpy(dst, src + r0 * kDim * 2, static_cast<size_t>(rows) * kDim * 2);
    return FLMR_OK;
  });
}

int flmr_corpus_builder_append_file(flmr_corpus_builder_t* b, const char* path, int64_t byte_offset, int64_t n_rows) {
  if (!b || !path) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  const int fd = open(path, O_RDONLY);
  if (fd < 0) return fail(FLMR_ERR_INVALID_ARG, "cannot open %s: %s", path, strerror(errno));
  // the file is read straight into pinned memory by a few threads (pread is thread-safe): no intermediate copy
  const int rc = builder_feed(b, n_rows, [&](void* dst, int64_t r0, int64_t rows) {
    constexpr int kThreads = 8;
    const int64_t total = rows * kDim * 2, per = (total + kThreads - 1) / kThreads;
    int errs[kThreads] = {};
    std::thread th[kThreads];
    for (int t = 0; t < kThreads; ++t)
      th[t] = std::thread([&, t]() {
        int64_t a = t * per, e = std::min<int64_t>(total, a + per);
        while (a < e) {
          const ssize_t got = pread(fd, static_cast<char*>(dst) + a, static_cast<size_t>(e - a),
                                    byte_offset + r0 * kDim * 2 + a);
          if (got <= 0) {
            errs[t] = got == 0 ? -1 : errno;
            return;
          }
          a += got;
        }
      });
    for (auto& x : th) x.join();
    for (int e : errs)
      if (e) return fail(FLMR_ERR_INVALID_ARG, "short read from %s (%s)", path, e < 0 ? "end of file" : strerror(e));
    return static_cast<int>(FLMR_OK);
  });
  close(fd);
  return rc;
}

int flmr_corpus_builder_finish(flmr_corpus_builder_t* b, flmr_corpus_t** out, double* host_fill_seconds) {
  if (!b || !out) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  flmr_corpus* c = b->corpus;
  if (b->rows_done != c->n_tokens)
    return fail(FLMR_ERR_INVALID_ARG, "%lld rows appended, the doclens announce %lld", (long long)b->rows_done,
                (long long)c->n_tokens);
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  if (b->stream) FLMR_CUDA(cudaStreamSynchronize(b->stream));   // a streamed load wrote the host matrix itself
  if (c->codec_nbits && !c->d_centroids) {   // a PLAID-coded corpus: its codec tables go to HBM
    int64_t bytes = 0;
    int rc = dev_upload(&c->d_centroids, b->centroids, &bytes);
    if (!rc) rc = dev_upload(&c->d_bucket_weights, b->bucket_weights, &bytes);
    if (rc) {
      cudaFree(c->d_centroids);
      cudaFree(c->d_bucket_weights);
      c->d_centroids = c->d_bucket_weights = nullptr;
      return rc;
    }
    c->codec_hbm_bytes = bytes;
  }
  if (int rc = build_layout(c, c->d_tokens, c->n_rows, b->poff, b->doclens.data(), &c->layout)) return rc;
  if (host_fill_seconds) *host_fill_seconds = b->fill_s;
  b->corpus = nullptr;     // ownership passes to the caller
  flmr_corpus_builder_destroy(b);
  *out = c;
  return FLMR_OK;
}

int flmr_corpus_builder_destroy(flmr_corpus_builder_t* b) {
  if (!b) return FLMR_OK;
  if (b->stream) cudaStreamSynchronize(b->stream);
  for (int i = 0; i < flmr_corpus_builder::kBufs; ++i) {
    if (b->h_pin[i]) cudaFreeHost(b->h_pin[i]);
    if (b->d_stage[i]) cudaFree(b->d_stage[i]);
    if (b->free_ev[i]) cudaEventDestroy(b->free_ev[i]);
  }
  cudaFree(b->d_soff);
  cudaFree(b->d_poff);
  if (b->stream) cudaStreamDestroy(b->stream);
  if (b->corpus) flmr_corpus_destroy(b->corpus);
  delete b;
  return FLMR_OK;
}

int flmr_corpus_info(const flmr_corpus_t* c, flmr_corpus_info_t* out) {
  if (!c || !out) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  out->n_passages = c->n_passages;
  out->n_tokens = c->n_tokens;
  out->n_rows = c->n_rows;
  out->pid_base = c->pid_base;
  out->dim = kDim;
  out->device = c->device;
  out->n_ctas = c->layout.n_ctas;
  out->adopted = c->adopted ? 1 : 0;
  out->n_tiles = 0;
  for (const Window& w : c->layout.windows) out->n_tiles += w.cta.n_tiles;
  out->hbm_bytes = hbm_bytes(c);
  return FLMR_OK;
}

int flmr_corpus_storage(const flmr_corpus_t* c, int* storage, int64_t* host_bytes) {
  if (!c) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  const bool e4m3 = c->elem == Elem::kE4M3;
  if (storage) *storage = e4m3 ? 1 : c->elem == Elem::kF16 ? 2 : 0;   // the ABI's codes, not the Elem values
  if (host_bytes) *host_bytes = e4m3 ? c->n_rows * kDim * 2 : 0;
  return FLMR_OK;
}

int flmr_corpus_append(flmr_corpus_t* c, const void* tokens, const int32_t* h_doclens, int64_t n_passages,
                       int64_t* first_pid) {
  if (!c || !tokens || !h_doclens) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  if (c->streamed) return fail(FLMR_ERR_UNSUPPORTED, "a streamed corpus cannot be appended to");
  if (n_passages <= 0) return fail(FLMR_ERR_INVALID_ARG, "n_passages=%lld must be >= 1", (long long)n_passages);
  const int64_t old_n = c->n_passages, old_rows = c->n_rows;
  // the new passages, relative to their first: packed (soff) and padded (poff) row offsets
  std::vector<int64_t> soff, poff;
  if (int rc = passage_offsets(h_doclens, n_passages, &soff, &poff, nullptr)) return rc;
  const int64_t new_n = old_n + n_passages, new_rows = old_rows + poff[n_passages];
  // the partition stores first passage ids and CTA row starts as int32, the scan's top-k key a 32-bit ~local id
  if (new_n > 0x7fffffffll)
    return fail(FLMR_ERR_UNSUPPORTED, "%lld passages exceed the 2^31 per-shard limit; shard the corpus", (long long)new_n);
  if (new_rows + kTileN >= (1ll << 31))
    return fail(FLMR_ERR_UNSUPPORTED, "%lld stored token rows exceed the 2^31 per-shard limit; shard the corpus",
                (long long)new_rows);
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  bool is_device_ptr;
  if (int rc = token_source(tokens, c->device, &is_device_ptr)) return rc;
  // searches enqueued before this call (any stream) finish on the corpus as it was
  FLMR_CUDA(cudaDeviceSynchronize());

  // --- 1. room for the new rows: mapped behind the library-owned matrices, which stay where they are ---
  const size_t row_bytes = static_cast<size_t>(kDim) * 2;
  const bool e4m3 = c->elem == Elem::kE4M3;
  if (e4m3) {
    if (int rc = gm_grow(&c->vm_fp8, c->device, static_cast<size_t>(new_rows) * kDim)) return rc;
    // the bf16 master is pinned host memory: reallocated and copied (old + new size are held for the copy)
    void* h = nullptr;
    cudaError_t e = cudaHostAlloc(&h, static_cast<size_t>(new_rows) * row_bytes,
                                  cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess)
      return fail(FLMR_ERR_OOM, "cudaHostAlloc(%zu B) for the bf16 master failed: %s",
                  static_cast<size_t>(new_rows) * row_bytes, cudaGetErrorString(e));
    __nv_bfloat16* d_alias = nullptr;
    if ((e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&d_alias), h, 0)) != cudaSuccess) {
      cudaFreeHost(h);
      return fail(FLMR_ERR_CUDA, "cudaHostGetDevicePointer: %s", cudaGetErrorString(e));
    }
    memcpy(h, c->h_master, static_cast<size_t>(old_rows) * row_bytes);
    cudaFreeHost(c->h_master);
    c->h_master = h;
    c->d_tokens = d_alias;
  } else if (c->adopted) {
    // the caller's buffer is copied into library memory once; from here on it is no longer referenced
    GrowableMatrix g;
    int rc = gm_grow(&g, c->device, static_cast<size_t>(new_rows) * row_bytes);
    cudaError_t e = cudaSuccess;
    if (!rc && (e = cudaMemcpy(reinterpret_cast<void*>(g.base), c->d_tokens, static_cast<size_t>(old_rows) * row_bytes,
                               cudaMemcpyDeviceToDevice)) != cudaSuccess)
      rc = fail(FLMR_ERR_CUDA, "copying the adopted token matrix failed: %s", cudaGetErrorString(e));
    if (rc) {
      gm_free(&g);
      return rc;
    }
    c->vm_tokens = g;
    c->d_tokens = reinterpret_cast<__nv_bfloat16*>(g.base);
    c->adopted = false;
  } else {
    if (int rc = gm_grow(&c->vm_tokens, c->device, static_cast<size_t>(new_rows) * row_bytes)) return rc;
  }

  // --- 2. the new rows into place (bf16, and e4m3 for an fp8 corpus), behind the old ones ---
  cudaError_t e = pack_passages(tokens, is_device_ptr, soff, poff, h_doclens, n_passages,
                                reinterpret_cast<uint4*>(c->d_tokens + old_rows * kDim),
                                e4m3 ? reinterpret_cast<uint2*>(c->d_fp8 + old_rows * kDim) : nullptr);
  if (e != cudaSuccess) return fail(FLMR_ERR_CUDA, "packing the appended passages failed: %s", cudaGetErrorString(e));

  // --- 3. layout and tombstones for the grown corpus, then swapped in ---
  std::vector<int64_t> all_poff(c->layout.h_poff);
  for (int64_t p = 1; p <= n_passages; ++p) all_poff.push_back(old_rows + poff[p]);
  std::vector<int32_t> all_len(c->layout.h_doclen);
  all_len.insert(all_len.end(), h_doclens, h_doclens + n_passages);
  std::vector<int64_t> slot_pid(c->h_slot_pid);
  std::vector<uint32_t> dead(c->h_dead);
  uint32_t* d_dead = nullptr;
  int64_t* d_slot_pid = nullptr;
  // compacted: the new passages take the next slots and the next ids (h_dead is never empty after a compaction)
  const bool compacted = !slot_pid.empty();
  if (compacted)
    for (int64_t p = 0; p < n_passages; ++p) slot_pid.push_back(c->pid_base + old_n + p);
  if (!dead.empty()) dead.resize((new_n + 31) / 32, 0u);
  int rc = compacted ? dev_upload(&d_slot_pid, slot_pid, nullptr) : FLMR_OK;
  if (!rc && c->d_dead)   // d_dead exists once anything is deleted, except right after a compaction
    rc = dev_upload(&d_dead, compacted ? dead_by_slot(slot_pid, c->pid_base, dead) : dead, nullptr);
  SlotLayout layout;
  if (!rc) rc = build_layout(c, c->d_tokens, new_rows, all_poff, all_len.data(), &layout);
  if (rc) {
    cudaFree(d_dead);
    cudaFree(d_slot_pid);
    return rc;
  }
  free_layout(&c->layout);
  cudaFree(c->d_dead);
  cudaFree(c->d_slot_pid);
  c->layout = std::move(layout);
  c->d_dead = d_dead;
  c->d_slot_pid = d_slot_pid;
  c->h_slot_pid.swap(slot_pid);
  c->h_dead.swap(dead);
  c->n_passages = new_n;
  c->n_tokens += soff[n_passages];
  c->n_rows = new_rows;
  if (first_pid) *first_pid = c->pid_base + old_n;
  return FLMR_OK;
}

int flmr_corpus_delete(flmr_corpus_t* c, const int64_t* h_pids, int64_t n) {
  if (!c || n < 0 || (n > 0 && !h_pids)) return fail(FLMR_ERR_INVALID_ARG, "null argument or negative count");
  for (int64_t i = 0; i < n; ++i) {   // the whole list is checked before anything changes
    const int64_t p = h_pids[i] - c->pid_base;
    if (p < 0 || p >= c->n_passages)
      return fail(FLMR_ERR_INVALID_ARG, "passage id %lld is outside this shard [%lld, %lld)", (long long)h_pids[i],
                  (long long)c->pid_base, (long long)(c->pid_base + c->n_passages));
  }
  std::vector<uint32_t> dead(c->h_dead);
  dead.resize((c->n_passages + 31) / 32, 0u);
  int64_t added = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t p = h_pids[i] - c->pid_base;
    const uint32_t bit = 1u << (p & 31);
    added += (dead[p >> 5] & bit) == 0;
    dead[p >> 5] |= bit;
  }
  if (added == 0) return FLMR_OK;   // already deleted (or nothing to do): no change, no bitmap allocated
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  // a compacted corpus: the device bitmap is indexed by slot (a newly deleted id always has one: a compacted-away id
  // was deleted already)
  const std::vector<uint32_t> words = c->h_slot_pid.empty() ? dead : dead_by_slot(c->h_slot_pid, c->pid_base, dead);
  // searches enqueued before this call (any stream) finish with the old bitmap
  FLMR_CUDA(cudaDeviceSynchronize());
  const size_t bytes = words.size() * sizeof(uint32_t);
  if (!c->d_dead) FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->d_dead), bytes));
  FLMR_CUDA(cudaMemcpy(c->d_dead, words.data(), bytes, cudaMemcpyHostToDevice));
  c->h_dead.swap(dead);
  c->n_deleted += added;
  return FLMR_OK;
}

int flmr_corpus_deleted(const flmr_corpus_t* c, int64_t* n_deleted, int64_t* h_pids, int64_t capacity) {
  if (!c || !n_deleted) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  *n_deleted = c->n_deleted;
  if (!h_pids) return FLMR_OK;
  if (capacity < c->n_deleted)
    return fail(FLMR_ERR_INVALID_ARG, "capacity %lld < %lld deleted ids", (long long)capacity,
                (long long)c->n_deleted);
  int64_t j = 0;
  for (size_t w = 0; w < c->h_dead.size(); ++w)
    for (uint32_t bits = c->h_dead[w]; bits; bits &= bits - 1)
      h_pids[j++] = c->pid_base + static_cast<int64_t>(w) * 32 + __builtin_ctz(bits);
  return FLMR_OK;
}

int flmr_corpus_compact(flmr_corpus_t* c, int64_t* n_removed, int64_t* bytes_released) {
  if (n_removed) *n_removed = 0;
  if (bytes_released) *bytes_released = 0;
  if (!c) return fail(FLMR_ERR_INVALID_ARG, "null corpus");
  if (c->streamed) return fail(FLMR_ERR_UNSUPPORTED, "a streamed corpus cannot be compacted");
  const int64_t ns = slots(c);
  // --- 1. which slots stay: their ids, offsets and lengths in the compacted corpus ---
  std::vector<char> keep(ns, 1);
  int64_t removed = 0;
  for (int64_t s = 0; s < ns; ++s) {
    const int64_t p = c->h_slot_pid.empty() ? s : c->h_slot_pid[s] - c->pid_base;
    if (static_cast<size_t>(p >> 5) < c->h_dead.size() && ((c->h_dead[p >> 5] >> (p & 31)) & 1u)) {
      keep[s] = 0;
      ++removed;
    }
  }
  if (removed == 0) return FLMR_OK;   // nothing deleted since the last compaction: the corpus is already compact
  if (removed == ns)
    return fail(FLMR_ERR_INVALID_ARG, "every passage of the shard is deleted; a corpus keeps at least one passage");
  std::vector<int64_t> slot_pid, poff(1, 0);
  std::vector<int32_t> lens;
  slot_pid.reserve(ns - removed);
  lens.reserve(ns - removed);
  poff.reserve(ns - removed + 1);
  for (int64_t s = 0; s < ns; ++s) {
    if (!keep[s]) continue;
    slot_pid.push_back(c->h_slot_pid.empty() ? c->pid_base + s : c->h_slot_pid[s]);
    lens.push_back(c->layout.h_doclen[s]);
    poff.push_back(poff.back() + (c->layout.h_poff[s + 1] - c->layout.h_poff[s]));
  }
  int64_t n_tokens = 0;
  for (int32_t l : lens) n_tokens += l;
  const int64_t new_rows = poff.back();
  std::vector<MovePiece> plan;
  plan_compaction(kept_runs(c->layout.h_poff, keep), kCompactChunkRows, !c->adopted, &plan);

  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  // searches enqueued before this call (any stream) finish on the corpus as it was
  FLMR_CUDA(cudaDeviceSynchronize());

  // --- 2. everything that can fail on allocation, before a row moves: the matrix an adopted corpus is copied into,
  // the schedule on the device, the staging buffer, and the slot -> id map and layout of the compacted corpus ---
  const bool e4m3 = c->elem == Elem::kE4M3;
  const size_t row_bytes = hbm_row_bytes(c->elem);   // of the matrix in HBM
  GrowableMatrix copy;          // an adopted corpus: the library-owned matrix its live rows go to
  __nv_bfloat16* d_tokens = c->d_tokens;   // where the rows end up
  int64_t *d_slot_pid = nullptr, *d_pdst = nullptr, *d_psrc = nullptr;
  uint4* stage = nullptr;
  SlotLayout layout;
  auto release = [&](int code) {
    free_layout(&layout);
    cudaFree(d_slot_pid);
    gm_free(&copy);
    cudaFree(d_pdst);
    cudaFree(d_psrc);
    cudaFree(stage);
    return code;
  };
  int rc = FLMR_OK;
  if (c->adopted) {
    if ((rc = gm_grow(&copy, c->device, static_cast<size_t>(new_rows) * row_bytes))) return release(rc);
    d_tokens = reinterpret_cast<__nv_bfloat16*>(copy.base);
  }
  {
    std::vector<int64_t> pdst(plan.size()), psrc(plan.size());
    int64_t stage_rows = 0;
    for (size_t i = 0; i < plan.size(); ++i) {
      pdst[i] = plan[i].dst;
      psrc[i] = plan[i].src;
    }
    for (size_t k0 = 0; k0 < plan.size();) {
      size_t k1 = k0;
      while (k1 < plan.size() && plan[k1].chunk == plan[k0].chunk) ++k1;
      if (plan[k0].staged) stage_rows = std::max(stage_rows, plan[k1 - 1].dst + plan[k1 - 1].rows - plan[k0].dst);
      k0 = k1;
    }
    if (!plan.empty() && ((rc = dev_upload(&d_pdst, pdst, nullptr)) || (rc = dev_upload(&d_psrc, psrc, nullptr))))
      return release(rc);
    if (stage_rows > 0) {
      const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&stage), static_cast<size_t>(stage_rows) * row_bytes);
      if (e != cudaSuccess)
        return release(fail(FLMR_ERR_OOM, "compaction staging buffer (%lld rows): %s", (long long)stage_rows,
                            cudaGetErrorString(e)));
    }
  }
  if ((rc = dev_upload(&d_slot_pid, slot_pid, nullptr)) ||
      (rc = build_layout(c, d_tokens, new_rows, poff, lens.data(), &layout)))
    return release(rc);

  // --- 3. the rows move: the HBM matrix on the device, the pinned bf16 master of an e4m3 corpus on the host ---
  cudaError_t e = cudaSuccess;
  if (!plan.empty()) {
    uint4* rows = reinterpret_cast<uint4*>(e4m3 ? static_cast<void*>(c->d_fp8) : c->d_tokens);   // in HBM
    e = run_moves(plan, d_pdst, d_psrc, rows, e4m3 ? rows : reinterpret_cast<uint4*>(d_tokens), stage,
                  static_cast<int>(row_bytes / 16));
    if (e4m3) {   // ordered memmove in place: every destination lies at or below its source, earlier pieces first
      char* m = static_cast<char*>(c->h_master);
      for (const MovePiece& mp : plan)
        memmove(m + mp.dst * kDim * 2, m + mp.src * kDim * 2, static_cast<size_t>(mp.rows) * kDim * 2);
    }
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return release(fail(FLMR_ERR_CUDA, "compaction row move failed: %s", cudaGetErrorString(e)));
  cudaFree(d_pdst);
  cudaFree(d_psrc);
  cudaFree(stage);

  // --- 4. physical memory wholly behind the new end goes back to the device; the handle takes the new state ---
  size_t released = 0;
  if (c->adopted) {
    c->vm_tokens = copy;          // the caller's buffer is no longer referenced
    c->d_tokens = d_tokens;
    c->adopted = false;
  } else {
    released = gm_shrink(e4m3 ? &c->vm_fp8 : &c->vm_tokens, static_cast<size_t>(new_rows) * row_bytes);
  }
  free_layout(&c->layout);
  cudaFree(c->d_dead);
  cudaFree(c->d_slot_pid);
  c->layout = std::move(layout);
  c->d_dead = nullptr;          // every deleted slot is removed
  c->d_slot_pid = d_slot_pid;
  c->h_slot_pid.swap(slot_pid);
  c->n_tokens = n_tokens;
  c->n_rows = new_rows;
  if (n_removed) *n_removed = removed;
  if (bytes_released) *bytes_released = static_cast<int64_t>(released);
  return FLMR_OK;
}

int flmr_corpus_stored(const flmr_corpus_t* c, int64_t* n_stored_passages, int64_t* mapped_device_bytes) {
  if (!c) return fail(FLMR_ERR_INVALID_ARG, "null corpus");
  if (n_stored_passages) *n_stored_passages = slots(c);
  if (mapped_device_bytes) *mapped_device_bytes = static_cast<int64_t>(c->vm_tokens.mapped + c->vm_fp8.mapped);
  return FLMR_OK;
}

int flmr_workspace_create(const flmr_corpus_t* c, int max_queries, int max_nq,
                          flmr_workspace_t** out) {
  if (!c || !out) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  if (max_queries < 1 || max_nq < 1)
    return fail(FLMR_ERR_INVALID_ARG, "max_queries=%d / max_nq=%d must be >= 1", max_queries, max_nq);
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  flmr_workspace* ws = new (std::nothrow) flmr_workspace();
  if (!ws) return fail(FLMR_ERR_OOM, "host allocation failed");
  ws->corpus = c;
  ws->device = c->device;
  ws->max_queries = max_queries;
  ws->max_nq = max_nq;
  auto bail = [&](int code) {
    flmr_workspace_destroy(ws);
    return code;
  };
  cudaError_t e;
  const size_t qbytes = static_cast<size_t>(kStageMaxPasses) * kMtMax * kTileM * kDim * 2;   // 10 MB
  if ((e = cudaMalloc(reinterpret_cast<void**>(&ws->d_qpad), qbytes)) != cudaSuccess ||
      (e = cudaMemset(ws->d_qpad, 0, qbytes)) != cudaSuccess ||
      (e = cudaMalloc(reinterpret_cast<void**>(&ws->d_cand_keys),
                      static_cast<size_t>(c->layout.n_ctas) * max_queries * kMaxK * 8)) != cudaSuccess ||
      (e = cudaHostAlloc(reinterpret_cast<void**>(&ws->h_status), sizeof(int), cudaHostAllocMapped)) != cudaSuccess ||
      (e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&ws->d_status), ws->h_status, 0)) != cudaSuccess)
    return bail(fail(FLMR_ERR_CUDA, "workspace allocation failed: %s", cudaGetErrorString(e)));
  ws->cand_lists = c->layout.n_ctas;
  *ws->h_status = 0;
  if (c->streamed) {   // the window buffers (two, or one for a one-window plan; zeroed: rows a tile reads past its
                       // window's end are finite), their tensor maps, the copy stream and its events
    const size_t wbytes = static_cast<size_t>(c->layout.window_rows) * kDim * 2;
    const int n_bufs = c->layout.windows.size() > 1 ? 2 : 1;
    // a PLAID-coded corpus: one decoded window buffer, and n_bufs staging buffers of compressed rows
    const bool coded = c->codec_nbits > 0;
    const size_t sbytes = coded ? static_cast<size_t>(c->layout.window_rows * codec_row_bytes(c->codec_nbits)) : 0;
    for (int i = 0; i < n_bufs; ++i) {
      const bool win_buf = !coded || i == 0;
      if ((win_buf && (e = cudaMalloc(reinterpret_cast<void**>(&ws->d_win[i]), wbytes)) != cudaSuccess) ||
          (win_buf && (e = cudaMemset(ws->d_win[i], 0, wbytes)) != cudaSuccess) ||
          (coded && (e = cudaMalloc(reinterpret_cast<void**>(&ws->d_cstage[i]), sbytes)) != cudaSuccess) ||
          (coded && (e = cudaEventCreateWithFlags(&ws->decoded_ev[i], cudaEventDisableTiming)) != cudaSuccess) ||
          (e = cudaEventCreateWithFlags(&ws->copied_ev[i], cudaEventDisableTiming)) != cudaSuccess ||
          (e = cudaEventCreateWithFlags(&ws->scanned_ev[i], cudaEventDisableTiming)) != cudaSuccess)
        return bail(fail(e == cudaErrorMemoryAllocation ? FLMR_ERR_OOM : FLMR_ERR_CUDA,
                         "window buffers: %s", cudaGetErrorString(e)));
      if (!win_buf) continue;
      if (int rc = encode_rows_map(&ws->tmap_win[i], ws->d_win[i], static_cast<uint64_t>(c->layout.window_rows),
                                   kTileN, c->elem))
        return bail(rc);
    }
    if ((e = cudaStreamCreateWithFlags(&ws->copy_stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaEventCreateWithFlags(&ws->fork_ev, cudaEventDisableTiming)) != cudaSuccess)
      return bail(fail(FLMR_ERR_CUDA, "copy stream: %s", cudaGetErrorString(e)));
  }
  if (max_nq > kRbMax * 32) {   // row-sliced queries expected: size their partial-score rows now
    std::vector<PassPlan> plan;
    int group = 1;
    plan_passes(max_queries, max_nq, c->layout.n_pairs > 0, &plan, &group, nullptr);
    if (int rc = ensure_acc(ws, static_cast<int64_t>(group) * c->n_passages)) return bail(rc);
  }
#ifdef FLMR_DEBUG
  if (const char* e = getenv("FLMR_LANE_RBQ")) ws->dbg_lane_rbq = atoi(e);
#endif
  *out = ws;
  return FLMR_OK;
}

int flmr_workspace_destroy(flmr_workspace_t* ws) {
  if (!ws) return FLMR_OK;
  DeviceGuard guard(ws->device);
  cudaFree(ws->d_qpad);
  cudaFree(ws->d_cand_keys);
  cudaFree(ws->d_acc);
  cudaFree(ws->d_plan);
  if (ws->h_status) cudaFreeHost(ws->h_status);
  if (ws->copy_stream) cudaStreamSynchronize(ws->copy_stream);
  for (int i = 0; i < 2; ++i) {
    cudaFree(ws->d_win[i]);   // waits for the scans still reading it
    cudaFree(ws->d_cstage[i]);
    if (ws->copied_ev[i]) cudaEventDestroy(ws->copied_ev[i]);
    if (ws->scanned_ev[i]) cudaEventDestroy(ws->scanned_ev[i]);
    if (ws->decoded_ev[i]) cudaEventDestroy(ws->decoded_ev[i]);
  }
  if (ws->fork_ev) cudaEventDestroy(ws->fork_ev);
  if (ws->copy_stream) cudaStreamDestroy(ws->copy_stream);
  delete ws;
  return FLMR_OK;
}

int flmr_workspace_status(const flmr_workspace_t* ws, int* out) {
  if (!ws || !out) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  *out = ws->h_status ? *reinterpret_cast<volatile int*>(ws->h_status) : 0;
  return FLMR_OK;
}

int flmr_maxsim_scores(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q,
                       int n_queries, int nq, unsigned flags, float* d_out_scores, void* stream) {
  return flmr_maxsim_scores_allowed(corpus, ws, d_q, n_queries, nq, flags, nullptr, 0, d_out_scores, stream);
}

int flmr_maxsim_scores_allowed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries,
                               int nq, unsigned flags, const uint32_t* d_allow, int64_t allow_stride_words,
                               float* d_out_scores, void* stream) {
  if (!d_out_scores) return fail(FLMR_ERR_INVALID_ARG, "d_out_scores is null");
  return run_search(corpus, ws, d_q, n_queries, nq, flags, 0, d_allow, allow_stride_words, d_out_scores, nullptr,
                    nullptr, static_cast<cudaStream_t>(stream));
}

int flmr_maxsim_topk(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q,
                     int n_queries, int nq, int k, unsigned flags, float* d_out_scores,
                     int64_t* d_out_pids, void* stream) {
  return flmr_maxsim_topk_allowed(corpus, ws, d_q, n_queries, nq, k, flags, nullptr, 0, d_out_scores, d_out_pids,
                                  stream);
}

int flmr_maxsim_topk_allowed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries,
                             int nq, int k, unsigned flags, const uint32_t* d_allow, int64_t allow_stride_words,
                             float* d_out_scores, int64_t* d_out_pids, void* stream) {
  if (!d_out_scores || !d_out_pids) return fail(FLMR_ERR_INVALID_ARG, "output pointer is null");
  if (k < 1) return fail(FLMR_ERR_INVALID_ARG, "k=%d must be >= 1", k);
  return run_search(corpus, ws, d_q, n_queries, nq, flags, k, d_allow, allow_stride_words, nullptr, d_out_scores,
                    d_out_pids, static_cast<cudaStream_t>(stream));
}

extern "C++" {
namespace {
// Checks a listed call's lists and runs it: the offsets go to the device (stream-ordered scratch), then run_search.
int run_listed(const flmr_corpus* c, flmr_workspace* ws, const void* d_q, int n_queries, int nq, unsigned flags,
               int k, const int64_t* h_off, const int64_t* d_pids, float* d_scores, float* d_topk_scores,
               int64_t* d_topk_pids, cudaStream_t st) {
  if (!c || !ws) return fail(FLMR_ERR_INVALID_ARG, "null corpus / workspace");
  if (c->streamed) return fail(FLMR_ERR_UNSUPPORTED, "a streamed corpus has no listed scan; use the _allowed calls");
  if (n_queries < 0) return fail(FLMR_ERR_INVALID_ARG, "bad n_queries=%d", n_queries);
  if (!h_off) return fail(FLMR_ERR_INVALID_ARG, "h_list_offsets is null");
  if (h_off[0] < 0) return fail(FLMR_ERR_INVALID_ARG, "h_list_offsets[0] = %lld < 0", (long long)h_off[0]);
  for (int b = 0; b < n_queries; ++b)
    if (h_off[b + 1] < h_off[b])
      return fail(FLMR_ERR_INVALID_ARG, "h_list_offsets decreases at query %d", b);
  if (h_off[n_queries] > h_off[0] && !d_pids) return fail(FLMR_ERR_INVALID_ARG, "d_list_pids is null");
  if (!pick_scan(c->elem, true, g_scan_variant, 0).fn)   // as in run_search
    return fail(FLMR_ERR_UNSUPPORTED, "scan variant %d has no plan-mode (listed) kernel", g_scan_variant);
  if (n_queries == 0) return FLMR_OK;
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  StreamScratch scratch(st);
  int64_t* d_off = nullptr;
  if (int rc = scratch.alloc(&d_off, (n_queries + 1) * sizeof(int64_t))) return rc;
  FLMR_CUDA(cudaMemcpyAsync(d_off, h_off, (n_queries + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  const ListedArgs la{h_off, d_off, d_pids, d_scores};
  return run_search(c, ws, d_q, n_queries, nq, flags, k, nullptr, 0, d_scores, d_topk_scores, d_topk_pids, st, &la);
}
}  // namespace
}

int flmr_maxsim_topk_listed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries, int nq,
                            int k, unsigned flags, const int64_t* h_list_offsets, const int64_t* d_list_pids,
                            float* d_out_scores, int64_t* d_out_pids, void* stream) {
  if (!d_out_scores || !d_out_pids) return fail(FLMR_ERR_INVALID_ARG, "output pointer is null");
  if (k < 1) return fail(FLMR_ERR_INVALID_ARG, "k=%d must be >= 1", k);
  return run_listed(corpus, ws, d_q, n_queries, nq, flags, k, h_list_offsets, d_list_pids, nullptr, d_out_scores,
                    d_out_pids, static_cast<cudaStream_t>(stream));
}

int flmr_maxsim_scores_listed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, const void* d_q, int n_queries,
                              int nq, unsigned flags, const int64_t* h_list_offsets, const int64_t* d_list_pids,
                              float* d_out_scores, void* stream) {
  if (!d_out_scores) return fail(FLMR_ERR_INVALID_ARG, "d_out_scores is null");
  return run_listed(corpus, ws, d_q, n_queries, nq, flags, 0, h_list_offsets, d_list_pids, d_out_scores, nullptr,
                    nullptr, static_cast<cudaStream_t>(stream));
}

int flmr_debug_listed_plan(const flmr_corpus_t* c, flmr_workspace_t* ws, int n_queries, int nq,
                           const int64_t* h_list_offsets, const int64_t* d_list_pids, int64_t* h_out,
                           int64_t capacity, int64_t* n_out) {
  if (!c || !ws || !h_list_offsets || !n_out || n_queries < 1 || nq < 1)
    return fail(FLMR_ERR_INVALID_ARG, "bad argument");
  if (ws->corpus != c) return fail(FLMR_ERR_INVALID_ARG, "workspace belongs to a different corpus");
  if (c->streamed) return fail(FLMR_ERR_UNSUPPORTED, "a streamed corpus has no listed scan");
  if (n_queries > ws->max_queries)
    return fail(FLMR_ERR_INVALID_ARG, "n_queries=%d > the workspace's max_queries=%d", n_queries, ws->max_queries);
  for (int b = 0; b < n_queries; ++b)
    if (h_list_offsets[b + 1] < h_list_offsets[b] || h_list_offsets[b] < 0)
      return fail(FLMR_ERR_INVALID_ARG, "bad h_list_offsets at query %d", b);
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  cudaStream_t st = nullptr;
  std::vector<PassPlan> plan;
  int group = 1;
  plan_passes(n_queries, nq, false, &plan, &group, nullptr);
  int64_t* d_off = nullptr;
  FLMR_CUDA(cudaMalloc(&d_off, (n_queries + 1) * sizeof(int64_t)));
  FLMR_CUDA(cudaMemcpy(d_off, h_list_offsets, (n_queries + 1) * sizeof(int64_t), cudaMemcpyHostToDevice));
  const ListedArgs la{h_list_offsets, d_off, d_list_pids, nullptr};
  ListedChunkPlan lp;
  int rc = plan_listed_chunk(c, ws, plan, 0, n_queries, la, st, &lp);
  if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = fail(FLMR_ERR_CUDA, "planner failed");
  cudaFree(d_off);
  if (rc) return rc;
  // per pass: q_first, n_q, n_ctas, union size, tiles, tile bound, the union's slots, cta_tile_base [n_ctas + 1],
  // then per tile its start row, end mask and first slot
  const int n_p = static_cast<int>(plan.size());
  std::vector<int64_t> meta(2 * n_p), out{n_p};
  FLMR_CUDA(cudaMemcpy(meta.data(), lp.meta, meta.size() * 8, cudaMemcpyDeviceToHost));
  for (int i = 0; i < n_p; ++i) {
    const ListedPass& q = lp.passes[i];
    const int64_t nu = meta[2 * i], nt = meta[2 * i + 1];
    if (nt > lp.t_bound[i] || nu > lp.u_bound[i])
      return fail(FLMR_ERR_KERNEL, "pass %d: plan of %lld tiles exceeds its bound %lld", i, (long long)nt,
                  (long long)lp.t_bound[i]);
    out.insert(out.end(), {q.q_first, q.n_q, c->layout.n_ctas, nu, nt, lp.t_bound[i]});
    std::vector<int32_t> slots_(nu), row(nt), first(nt);
    std::vector<int64_t> base(c->layout.n_ctas + 1);
    std::vector<uint32_t> mask(nt);
    FLMR_CUDA(cudaMemcpy(slots_.data(), lp.u_slot + q.u_off, nu * 4, cudaMemcpyDeviceToHost));
    FLMR_CUDA(cudaMemcpy(base.data(), lp.cta_tile_base + q.c_off, base.size() * 8, cudaMemcpyDeviceToHost));
    FLMR_CUDA(cudaMemcpy(row.data(), lp.tile_row + q.t_off, nt * 4, cudaMemcpyDeviceToHost));
    FLMR_CUDA(cudaMemcpy(mask.data(), lp.tile_mask + q.t_off, nt * 4, cudaMemcpyDeviceToHost));
    FLMR_CUDA(cudaMemcpy(first.data(), lp.tile_first + q.t_off, nt * 4, cudaMemcpyDeviceToHost));
    out.insert(out.end(), slots_.begin(), slots_.end());
    out.insert(out.end(), base.begin(), base.end());
    out.insert(out.end(), row.begin(), row.end());
    out.insert(out.end(), mask.begin(), mask.end());
    out.insert(out.end(), first.begin(), first.end());
  }
  *n_out = static_cast<int64_t>(out.size());
  if (h_out) {
    if (static_cast<int64_t>(out.size()) > capacity)
      return fail(FLMR_ERR_INVALID_ARG, "capacity %lld < %zu", (long long)capacity, out.size());
    std::copy(out.begin(), out.end(), h_out);
  }
  return FLMR_OK;
}

int flmr_topk_merge(const float* d_in_scores, const int64_t* d_in_pids, int n_lists, int n_queries,
                    int k_in, int k_out, float* d_out_scores, int64_t* d_out_pids, int device,
                    void* stream) {
  if (!d_in_scores || !d_in_pids || !d_out_scores || !d_out_pids)
    return fail(FLMR_ERR_INVALID_ARG, "null pointer");
  if (n_lists < 1 || n_queries < 0 || k_in < 1 || k_out < 1 || k_out > kMaxK)
    return fail(FLMR_ERR_INVALID_ARG, "bad merge shape n_lists=%d n_queries=%d k_in=%d k_out=%d",
                n_lists, n_queries, k_in, k_out);
  if (static_cast<int64_t>(n_lists) * k_in > kMergeThreads * kMergePer)
    return fail(FLMR_ERR_UNSUPPORTED, "n_lists*k_in = %lld exceeds merge capacity %d",
                (long long)n_lists * k_in, kMergeThreads * kMergePer);
  if (n_queries == 0) return FLMR_OK;
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  flmr_merge_kernel<<<n_queries, kMergeThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      nullptr, d_in_scores, d_in_pids, n_lists, n_queries, k_in, k_out, 0, nullptr, d_out_scores, d_out_pids, 0);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

extern "C++" {
namespace {
thread_local int g_merge_path = 0;   // 0 = by peer capability, 1 = stage every list (flmr_debug_set_merge_path)

// How the home device reads lists on `peer`: 1 through peer access (enabled here the first time), 0 through a staged
// copy.  Decided once per ordered device pair for the process, under a lock.
int peer_readable(int home, int peer, int n_dev, bool* out) {
  static std::mutex mu;
  static std::vector<signed char> state;   // [home * n_dev + peer]: -1 undecided, 0 staged, 1 peer reads
  std::lock_guard<std::mutex> lock(mu);
  if (state.size() < static_cast<size_t>(n_dev) * n_dev) state.assign(static_cast<size_t>(n_dev) * n_dev, -1);
  signed char& s = state[static_cast<size_t>(home) * n_dev + peer];
  if (s < 0) {
    int can = 0;
    FLMR_CUDA(cudaDeviceCanAccessPeer(&can, home, peer));
    if (can) {
      DeviceGuard guard(home);
      if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", home);
      const cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();   // enabled earlier by someone else in this process: not an error, and not left behind
      } else if (e != cudaSuccess) {
        return fail(FLMR_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d -> %d) failed: %s", home, peer, cudaGetErrorString(e));
      }
    }
    s = can ? 1 : 0;
  }
  *out = s == 1;
  return FLMR_OK;
}

// One event per device and host thread, recorded on a source stream and waited for at once, so one suffices.
int device_event(int device, cudaEvent_t* out) {
  thread_local std::vector<cudaEvent_t> events;
  if (events.size() <= static_cast<size_t>(device)) events.resize(device + 1, nullptr);
  if (!events[device]) {
    DeviceGuard guard(device);
    if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
    FLMR_CUDA(cudaEventCreateWithFlags(&events[device], cudaEventDisableTiming));
  }
  *out = events[device];
  return FLMR_OK;
}
}  // namespace
}  // extern "C++"

int flmr_topk_merge_devices(const float* const* d_scores, const int64_t* const* d_pids, const int* devices,
                            void* const* src_streams, int n_lists, int n_queries, int k_in, int k_out,
                            float* d_out_scores, int64_t* d_out_pids, void* stream) {
  if (!d_scores || !d_pids || !devices || !src_streams || !d_out_scores || !d_out_pids)
    return fail(FLMR_ERR_INVALID_ARG, "null array or output pointer");
  if (n_lists < 1 || n_queries < 0 || k_in < 1 || k_out < 1 || k_out > kMaxK)
    return fail(FLMR_ERR_INVALID_ARG, "bad merge shape n_lists=%d n_queries=%d k_in=%d k_out=%d",
                n_lists, n_queries, k_in, k_out);
  if (static_cast<int64_t>(k_out) > static_cast<int64_t>(n_lists) * k_in)
    return fail(FLMR_ERR_INVALID_ARG, "k_out=%d exceeds the n_lists*k_in = %lld entries merged", k_out,
                (long long)n_lists * k_in);
  if (n_lists > kMergeMaxLists)
    return fail(FLMR_ERR_UNSUPPORTED, "n_lists=%d exceeds %d lists", n_lists, kMergeMaxLists);
  if (static_cast<int64_t>(n_lists) * k_in > kMergeThreads * kMergePer)
    return fail(FLMR_ERR_UNSUPPORTED, "n_lists*k_in = %lld exceeds merge capacity %d",
                (long long)n_lists * k_in, kMergeThreads * kMergePer);
  for (int i = 0; i < n_lists; ++i) {
    if (!d_scores[i] || !d_pids[i]) return fail(FLMR_ERR_INVALID_ARG, "list %d is null", i);
    if (devices[i] < 0) return fail(FLMR_ERR_INVALID_ARG, "list %d: device %d", i, devices[i]);
  }
  if (n_queries == 0) return FLMR_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int n_dev = 0, home = 0;
  FLMR_CUDA(cudaGetDeviceCount(&n_dev));
  for (int i = 0; i < n_lists; ++i)
    if (devices[i] >= n_dev) return fail(FLMR_ERR_INVALID_ARG, "list %d: device %d of %d", i, devices[i], n_dev);
  FLMR_CUDA(cudaStreamGetDevice(st, &home));
  DeviceGuard guard(home);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", home);
  // the merge reads list i once src_streams[i] has produced it: its event, waited for on `stream`
  for (int i = 0; i < n_lists; ++i) {
    cudaStream_t src = static_cast<cudaStream_t>(src_streams[i]);
    if (src == st && devices[i] == home) continue;
    cudaEvent_t ev = nullptr;
    if (int rc = device_event(devices[i], &ev)) return rc;
    {
      DeviceGuard on_src(devices[i]);
      if (!on_src.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", devices[i]);
      FLMR_CUDA(cudaEventRecord(ev, src));
    }
    FLMR_CUDA(cudaStreamWaitEvent(st, ev, 0));
  }
  // lists on the home device are read in place, lists on a peer the home device can read through peer access;
  // the others are copied into one stream-ordered staging buffer on the home device first
  MergeLists lists;
  std::vector<int> staged;
  for (int i = 0; i < n_lists; ++i) {
    lists.scores[i] = d_scores[i];
    lists.pids[i] = d_pids[i];
    bool direct = devices[i] == home;
    if (!direct)
      if (int rc = peer_readable(home, devices[i], n_dev, &direct)) return rc;
    if (g_merge_path == 1 || !direct) staged.push_back(i);
  }
  const size_t list_elems = static_cast<size_t>(n_queries) * k_in;
  char* stage = nullptr;
  if (!staged.empty()) {
    const size_t bytes = staged.size() * list_elems * (sizeof(float) + sizeof(int64_t));
    FLMR_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&stage), bytes, st));
    int64_t* sp = reinterpret_cast<int64_t*>(stage);
    float* ss = reinterpret_cast<float*>(sp + staged.size() * list_elems);
    for (size_t j = 0; j < staged.size(); ++j) {
      const int i = staged[j];
      FLMR_CUDA(cudaMemcpyPeerAsync(ss + j * list_elems, home, d_scores[i], devices[i], list_elems * sizeof(float), st));
      FLMR_CUDA(cudaMemcpyPeerAsync(sp + j * list_elems, home, d_pids[i], devices[i], list_elems * sizeof(int64_t), st));
      lists.scores[i] = ss + j * list_elems;
      lists.pids[i] = sp + j * list_elems;
    }
  }
  const size_t smem = static_cast<size_t>(n_lists) * k_in * sizeof(int64_t);   // the candidates' pids
  cudaError_t launched = cudaFuncSetAttribute(flmr_merge_lists_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              static_cast<int>(smem));
  if (launched == cudaSuccess) {
    flmr_merge_lists_kernel<<<n_queries, kMergeThreads, smem, st>>>(lists, n_lists, k_in, k_out, d_out_scores,
                                                                    d_out_pids);
    launched = cudaGetLastError();
  }
  if (stage) FLMR_CUDA(cudaFreeAsync(stage, st));   // stream-ordered: released after the kernel has read it
  if (launched != cudaSuccess) return fail(FLMR_ERR_CUDA, "merge launch failed: %s", cudaGetErrorString(launched));
  ++g_launches;
  return FLMR_OK;
}

int flmr_debug_set_merge_path(int path) {
  if (path < 0 || path > 1)
    return fail(FLMR_ERR_INVALID_ARG, "path must be 0 (by peer capability) or 1 (stage every list)");
  g_merge_path = path;
  return FLMR_OK;
}

extern "C++" {
namespace {
template <bool kF16>
int plaid_decode(const int32_t* d_codes, const uint8_t* d_residuals, int64_t n_tokens, const float* d_centroids,
                 int64_t n_centroids, const float* d_bucket_weights, int nbits, int dim, int normalize,
                 void* d_out_bf16, int device, void* stream) {
  if (!d_codes || !d_residuals || !d_centroids || !d_bucket_weights || !d_out_bf16)
    return fail(FLMR_ERR_INVALID_ARG, "null pointer");
  if (dim != kDim) return fail(FLMR_ERR_UNSUPPORTED, "dim=%d (only %d is supported)", dim, kDim);
  if (nbits != 1 && nbits != 2 && nbits != 4 && nbits != 8)
    return fail(FLMR_ERR_INVALID_ARG, "nbits=%d (the PLAID codec packs 1, 2, 4 or 8 bits per dim)", nbits);
  if (n_tokens < 0 || n_centroids < 1) return fail(FLMR_ERR_INVALID_ARG, "bad sizes");
  if (n_tokens == 0) return FLMR_OK;
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // "a code was out of range" flag: one pinned + mapped word per host thread, reused by every call
  thread_local int* h_bad = nullptr;
  if (!h_bad) FLMR_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&h_bad), sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable));
  int* d_bad = nullptr;
  FLMR_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&d_bad), h_bad, 0));
  *reinterpret_cast<volatile int*>(h_bad) = 0;
  cudaError_t e = cudaSuccess;
  const int threads = 256;
  const int64_t want = (n_tokens * 32 + threads - 1) / threads;
  int sms = 0;
  FLMR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  const int blocks = static_cast<int>(std::min<int64_t>(want, static_cast<int64_t>(sms) * 16));
  if (e == cudaSuccess) {
    flmr_plaid_decode_kernel<kF16><<<blocks, threads, 0, st>>>(d_codes, d_residuals, d_centroids,
                                                             d_bucket_weights, nbits, normalize, n_tokens,
                                                             n_centroids, static_cast<uint2*>(d_out_bf16), d_bad);
    ++g_launches;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  const int bad = *reinterpret_cast<volatile int*>(h_bad);
  if (e != cudaSuccess) return fail(FLMR_ERR_CUDA, "plaid decode failed: %s", cudaGetErrorString(e));
  if (bad) return fail(FLMR_ERR_INVALID_ARG, "a centroid code is outside [0, %lld)", (long long)n_centroids);
  return FLMR_OK;
}
}  // namespace
}  // extern "C++"

int flmr_plaid_decode(const int32_t* d_codes, const uint8_t* d_residuals, int64_t n_tokens,
                      const float* d_centroids, int64_t n_centroids, const float* d_bucket_weights,
                      int nbits, int dim, int normalize, void* d_out_bf16, int device, void* stream) {
  return plaid_decode<false>(d_codes, d_residuals, n_tokens, d_centroids, n_centroids, d_bucket_weights, nbits, dim,
                             normalize, d_out_bf16, device, stream);
}

int flmr_plaid_decode_fp16(const int32_t* d_codes, const uint8_t* d_residuals, int64_t n_tokens,
                           const float* d_centroids, int64_t n_centroids, const float* d_bucket_weights,
                           int nbits, int dim, int normalize, void* d_out_fp16, int device, void* stream) {
  return plaid_decode<true>(d_codes, d_residuals, n_tokens, d_centroids, n_centroids, d_bucket_weights, nbits, dim,
                            normalize, d_out_fp16, device, stream);
}

// PLAID encode (flmr_plaid_encode_kernel.cuh): one persistent CTA per SM over 256-row token tiles, nothing
// synchronised, so the call can be captured in a CUDA graph.
int flmr_plaid_encode(const void* d_x, int64_t n, const void* d_centroids, int K, const float* d_cutoffs, int nbits,
                      int32_t* d_codes, uint8_t* d_residuals, float* d_best, int device, void* stream) {
  if (!d_x || !d_centroids || !d_codes || (d_residuals && !d_cutoffs)) return fail(FLMR_ERR_INVALID_ARG, "null pointer");
  if (nbits != 1 && nbits != 2 && nbits != 4 && nbits != 8)
    return fail(FLMR_ERR_INVALID_ARG, "nbits=%d (the PLAID codec packs 1, 2, 4 or 8 bits per dim)", nbits);
  if (K < 1) return fail(FLMR_ERR_INVALID_ARG, "K=%d: at least one centroid is needed", K);
  if (n < 0) return fail(FLMR_ERR_INVALID_ARG, "n=%lld", (long long)n);
  if ((reinterpret_cast<uintptr_t>(d_x) | reinterpret_cast<uintptr_t>(d_centroids)) & 15u)
    return fail(FLMR_ERR_INVALID_ARG, "d_x and d_centroids must be 16-byte aligned");
  if (d_residuals && (reinterpret_cast<uintptr_t>(d_residuals) & 3u))
    return fail(FLMR_ERR_INVALID_ARG, "d_residuals must be 4-byte aligned");
  if (n == 0) return FLMR_OK;
  if (n + kEncRows >= (1ll << 31)) return fail(FLMR_ERR_UNSUPPORTED, "n=%lld tokens: split the call below 2^31", (long long)n);
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  CUtensorMap tmap_x, tmap_c;
  if (int rc = encode_rows_map(&tmap_x, d_x, static_cast<uint64_t>(n), 128, Elem::kF16)) return rc;
  if (int rc = encode_rows_map(&tmap_c, d_centroids, static_cast<uint64_t>(K), kEncTileC, Elem::kF16)) return rc;
  static std::once_flag attr_once[64];
  cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once[device & 63], [&]() {
    attr_err = cudaFuncSetAttribute(flmr_plaid_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncSmemBytes);
  });
  if (attr_err != cudaSuccess)
    return fail(FLMR_ERR_CUDA, "cannot raise the dynamic shared memory limit: %s", cudaGetErrorString(attr_err));
  int sms = 0;
  FLMR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  PlaidEncodeParams prm{};
  prm.centroids = static_cast<const __half*>(d_centroids);
  prm.cutoffs = d_cutoffs;
  prm.codes = d_codes;
  prm.residuals = d_residuals;
  prm.best = d_best;
  prm.n = n;
  prm.K = K;
  prm.nbits = nbits;
  prm.n_tiles = static_cast<int32_t>((n + kEncRows - 1) / kEncRows);
  prm.status = nullptr;
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(prm.n_tiles, sms));
  flmr_plaid_encode_kernel<<<grid, kEncThreads, kEncSmemBytes, static_cast<cudaStream_t>(stream)>>>(tmap_x, tmap_c, prm);
  cudaError_t e = cudaGetLastError();
  ++g_launches;
  if (e != cudaSuccess) return fail(FLMR_ERR_CUDA, "flmr_plaid_encode_kernel launch failed: %s", cudaGetErrorString(e));
  return FLMR_OK;
}

int flmr_topk_select(const float* d_scores, int n_queries, int64_t n, int k, int64_t pid_base,
                     float* d_out_scores, int64_t* d_out_pids, int device, void* stream) {
  if (!d_scores || !d_out_scores || !d_out_pids) return fail(FLMR_ERR_INVALID_ARG, "null pointer");
  if (n_queries < 0 || n < 1 || k < 1) return fail(FLMR_ERR_INVALID_ARG, "bad shape n_queries=%d n=%lld k=%d", n_queries, (long long)n, k);
  if (k > kSelectMaxK) return fail(FLMR_ERR_UNSUPPORTED, "k=%d exceeds the selection capacity %d", k, kSelectMaxK);
  if (n >= (1ll << 32)) return fail(FLMR_ERR_UNSUPPORTED, "rows of 2^32 or more scores are not supported");
  if (n_queries == 0) return FLMR_OK;
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  flmr_select_kernel<<<n_queries, kSelectThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      d_scores, n, k, pid_base, d_out_scores, d_out_pids);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

int flmr_corpus_gather(const flmr_corpus_t* c, const int64_t* d_pids, int64_t n_pids, int nd_max,
                       void* d_out_bf16, uint8_t* d_mask, void* stream) {
  if (!c || !d_pids || !d_out_bf16) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  if (n_pids < 0 || nd_max < 1) return fail(FLMR_ERR_INVALID_ARG, "bad shape n_pids=%lld nd_max=%d", (long long)n_pids, nd_max);
  if (n_pids == 0) return FLMR_OK;
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  const int threads = 256;
  const int64_t blocks = (n_pids * nd_max * 32 + threads - 1) / threads;
  if (blocks > 0x7fffffffll) return fail(FLMR_ERR_UNSUPPORTED, "gather of %lld x %d rows is too large", (long long)n_pids, nd_max);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  StreamScratch scratch(st);
  if (c->d_slot_pid) {   // compacted: the gather reads slots, each id's found by binary search in the slot map
    int64_t* slot_ids = nullptr;
    if (int rc = scratch.alloc(&slot_ids, static_cast<size_t>(n_pids) * sizeof(int64_t))) return rc;
    flmr_slot_ids_kernel<<<static_cast<unsigned>((n_pids + threads - 1) / threads), threads, 0, st>>>(
        d_pids, n_pids, c->d_slot_pid, slots(c), c->pid_base, slot_ids);
    FLMR_CUDA(cudaGetLastError());
    ++g_launches;
    d_pids = slot_ids;
  }
  if (c->codec_nbits) {   // a PLAID-coded corpus: decoded from its mapped host arrays
    auto* kernel = c->elem == Elem::kF16 ? flmr_plaid_gather_kernel<true> : flmr_plaid_gather_kernel<false>;
    kernel<<<static_cast<unsigned>(blocks), threads, 0, st>>>(
        c->d_codes, c->d_residuals, c->d_centroids, c->d_bucket_weights, c->codec_nbits, c->layout.d_poff,
        c->layout.d_doclen, c->d_dead, d_pids, n_pids, nd_max, slots(c), c->pid_base, static_cast<uint2*>(d_out_bf16),
        d_mask);
    FLMR_CUDA(cudaGetLastError());
    ++g_launches;
    return FLMR_OK;
  }
  flmr_gather_kernel<<<static_cast<unsigned>(blocks), threads, 0, st>>>(
      reinterpret_cast<const uint2*>(c->d_tokens), c->layout.d_poff, c->layout.d_doclen, c->d_dead, d_pids, n_pids,
      nd_max, slots(c), c->pid_base, static_cast<uint2*>(d_out_bf16), d_mask);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

// ---- the wgmma route of the arg-max forward (flmr_train_tc_kernel.cuh) ----------------------------------------
thread_local int g_argmax_path = 0;   // 0 = by size, 1 = warp-MMA kernel, 2 = wgmma kernel (flmr_debug_set_argmax_path)

static int argmax_tc(const void* d_q, int n_queries, int nq, const void* d_docs, const uint8_t* d_mask, int n_per,
                     int stride_b, int nd, int32_t* d_argmax, float* d_rowmax, Elem elem, cudaStream_t st) {
  const int64_t n_total = stride_b ? static_cast<int64_t>(n_queries) * n_per : n_per;
  const int nd_c = (nd + kTcTile - 1) / kTcTile * kTcTile;
  if (n_total * nd_c + kTcTile >= (1ll << 31) || static_cast<int64_t>(n_queries) * nq + kTcTile >= (1ll << 31))
    return fail(FLMR_ERR_UNSUPPORTED, "arg-max operands exceed 2^31 rows");
  // stream-ordered scratch: packed documents, their index maps and lengths (freed in stream order below)
  const size_t b_dc = static_cast<size_t>(n_total) * nd_c * kDim * 2;
  const size_t b_map = static_cast<size_t>(n_total) * nd_c * sizeof(int32_t);
  const size_t b_len = static_cast<size_t>(n_total) * sizeof(int32_t);
  char* scratch = nullptr;
  cudaMemPool_t pool = nullptr;
  if (int rc = scratch_pool(&pool)) return rc;
  FLMR_CUDA(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&scratch), b_dc + b_map + b_len + 256, pool, st));
  uint4* dc = reinterpret_cast<uint4*>(scratch);
  int32_t* idx_map = reinterpret_cast<int32_t*>(scratch + b_dc);
  int32_t* doc_len = reinterpret_cast<int32_t*>(scratch + b_dc + b_map);
  auto done = [&](int code) {
    cudaFreeAsync(scratch, st);
    return code;
  };
  flmr_compact_docs_kernel<<<static_cast<unsigned>(n_total), 256, 0, st>>>(
      static_cast<const uint4*>(d_docs), d_mask, nd, nd_c, dc, idx_map, doc_len);
  ++g_launches;
  CUtensorMap tmap_q, tmap_d;
  int rc;
  if ((rc = encode_rows_map(&tmap_q, d_q, static_cast<uint64_t>(n_queries) * nq, kTcTile, elem))) return done(rc);
  if ((rc = encode_rows_map(&tmap_d, dc, static_cast<uint64_t>(n_total) * nd_c, kTcTile, elem))) return done(rc);
  const bool f16 = elem == Elem::kF16;
  auto* kernel = f16 ? flmr_argmax_tc_f16_kernel : flmr_argmax_tc_kernel;
  static std::once_flag attr_once[2][64];
  int dev = 0;
  cudaGetDevice(&dev);
  cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once[f16][dev & 63], [&]() {
    attr_err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmemBytes);
  });
  if (attr_err != cudaSuccess)
    return done(fail(FLMR_ERR_CUDA, "cannot raise the dynamic shared memory limit: %s", cudaGetErrorString(attr_err)));
  const int n_tiles = (nq + kTcTile - 1) / kTcTile;
  // documents per CTA: a CTA pays a fixed set-up (barriers, query tile, pipeline fill) before its first MMA, modelled
  // as ~17 chunks of 128 tokens; pick the split with the shortest modelled makespan (waves of one CTA per SM x
  // per-CTA time): many documents per CTA unless that leaves SMs idle
  int sms = 0;
  FLMR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int64_t pairs_q = static_cast<int64_t>(n_queries) * n_tiles;
  int dpc = 1;
  double best_t = 1e30;
  for (int d = 1; d <= 32 && d <= std::max(1, n_per); ++d) {
    const int64_t ctas = pairs_q * ((n_per + d - 1) / d);
    const double t = static_cast<double>((ctas + sms - 1) / sms) * (5.0 + d * 0.3 * (nd_c / kTcTile));
    if (t < best_t) {
      best_t = t;
      dpc = d;
    }
  }
  ArgmaxTcParams prm{};
  prm.doc_len = doc_len;
  prm.idx_map = idx_map;
  prm.arg = d_argmax;
  prm.rowmax = d_rowmax;
  prm.nq = nq;
  prm.nd_c = nd_c;
  prm.n_per = n_per;
  prm.stride_b = stride_b;
  prm.docs_per_cta = dpc;
  prm.status = nullptr;
  dim3 grid(static_cast<unsigned>((n_per + dpc - 1) / dpc), static_cast<unsigned>(n_tiles),
            static_cast<unsigned>(n_queries));
  kernel<<<grid, kTcThreads, kTcSmemBytes, st>>>(tmap_q, tmap_d, prm);
  cudaError_t e = cudaGetLastError();
  ++g_launches;
  if (e != cudaSuccess)
    return done(fail(FLMR_ERR_CUDA, "%s launch failed: %s", f16 ? "flmr_argmax_tc_f16_kernel" : "flmr_argmax_tc_kernel",
                     cudaGetErrorString(e)));
  return done(FLMR_OK);
}

// n_per documents per query; stride_b = 0: all queries meet documents [0, n_per) (all pairs),
// stride_b = n_per: query b meets documents [b * n_per, (b + 1) * n_per) (block diagonal).  elem: the element type of
// both operands (Elem::kBF16 or Elem::kF16), which picks the kernels' bf16 or fp16 instantiations.
static int argmax_impl(const void* d_q, int n_queries, int nq, const void* d_docs, const uint8_t* d_mask,
                       int n_per, int stride_b, int nd, int32_t* d_argmax, float* d_rowmax, Elem elem, int device,
                       void* stream) {
  if (!d_q || !d_docs || !d_mask || !d_argmax) return fail(FLMR_ERR_INVALID_ARG, "null pointer");
  if (n_queries < 0 || n_per < 0 || nq <= 0 || nd <= 0)
    return fail(FLMR_ERR_INVALID_ARG, "bad shape n_queries=%d nq=%d n_docs=%d nd=%d", n_queries, nq, n_per, nd);
  if (n_queries > 65535 || n_per > 65535)
    return fail(FLMR_ERR_UNSUPPORTED, "n_queries / n_docs above 65535 (training-sized batches only)");
  if (n_queries == 0 || n_per == 0) return FLMR_OK;
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  // wgmma route when the contraction is worth a TMA pipeline (>= 16M query-row x token pairs and full
  // tiles), warp-MMA kernel below that: a RAG re-score of 5 passages stays on the small kernel
  const double pairs = static_cast<double>(n_queries) * n_per * nq * nd;
  const bool tc_ok = n_queries <= 65535 && (nq + kTcTile - 1) / kTcTile <= 65535;
  if (tc_ok && (g_argmax_path == 2 || (g_argmax_path == 0 && nq >= 64 && nd >= 128 && pairs >= 16e6)))
    return argmax_tc(d_q, n_queries, nq, d_docs, d_mask, n_per, stride_b, nd, d_argmax, d_rowmax, elem,
                     static_cast<cudaStream_t>(stream));
  dim3 grid(static_cast<unsigned>((nq + kArgTile - 1) / kArgTile), static_cast<unsigned>(n_per),
            static_cast<unsigned>(n_queries));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool f16 = elem == Elem::kF16;
#ifdef FLMR_DEBUG
  // debug builds: FLMR_ARGMAX_SIMT=1 selects the plain-FMA twin (cross-check / A-B timing)
  const char* simt = getenv("FLMR_ARGMAX_SIMT");
  if (simt && atoi(simt)) {
    if (f16)
      flmr_argmax_f16_kernel<<<grid, kArgThreads, 0, st>>>(static_cast<const __half*>(d_q),
                                                           static_cast<const __half*>(d_docs), d_mask, nq, nd, n_per,
                                                           stride_b, d_argmax, d_rowmax);
    else
      flmr_argmax_kernel<<<grid, kArgThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(d_q),
                                                       static_cast<const __nv_bfloat16*>(d_docs), d_mask, nq, nd,
                                                       n_per, stride_b, d_argmax, d_rowmax);
    FLMR_CUDA(cudaGetLastError());
    ++g_launches;
    return FLMR_OK;
  }
#endif
  if (f16)
    flmr_argmax_mma_f16_kernel<<<grid, kMmaThreads, 0, st>>>(static_cast<const __half*>(d_q),
                                                             static_cast<const __half*>(d_docs), d_mask, nq, nd,
                                                             n_per, stride_b, d_argmax, d_rowmax);
  else
    flmr_argmax_mma_kernel<<<grid, kMmaThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(d_q),
                                                         static_cast<const __nv_bfloat16*>(d_docs), d_mask, nq, nd,
                                                         n_per, stride_b, d_argmax, d_rowmax);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

static int backward_impl(const void* d_q, int n_queries, int nq, const void* d_docs, int n_per, int stride_b,
                         int nd, const int32_t* d_argmax, const float* d_grad, float* d_dq, float* d_dd, Elem elem,
                         int device, void* stream) {
  if (n_queries < 0 || n_per < 0 || nq <= 0 || nd <= 0)
    return fail(FLMR_ERR_INVALID_ARG, "bad shape n_queries=%d nq=%d n_docs=%d nd=%d", n_queries, nq, n_per, nd);
  // without documents dQ is zeroed and nothing else is read: empty operands may come as null pointers (an empty
  // torch tensor has none)
  if (n_queries > 0 && n_per > 0 && (!d_q || !d_docs || !d_argmax || !d_grad))
    return fail(FLMR_ERR_INVALID_ARG, "null pointer");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int threads = 256;
  const int64_t n_docs_total = stride_b ? static_cast<int64_t>(n_queries) * n_per : n_per;
  const bool f16 = elem == Elem::kF16;
  if (d_dq && n_queries > 0) {
    const int64_t warps = static_cast<int64_t>(n_queries) * nq;
    if (n_per == 0) {
      FLMR_CUDA(cudaMemsetAsync(d_dq, 0, static_cast<size_t>(warps) * kDim * sizeof(float), st));
    } else {
      const unsigned blocks = static_cast<unsigned>((warps * 32 + threads - 1) / threads);
      if (f16)
        flmr_bwd_dq_f16_kernel<<<blocks, threads, 0, st>>>(static_cast<const __half*>(d_docs), d_argmax, d_grad,
                                                           n_queries, nq, n_per, nd, stride_b, d_dq);
      else
        flmr_bwd_dq_kernel<<<blocks, threads, 0, st>>>(static_cast<const __nv_bfloat16*>(d_docs), d_argmax, d_grad,
                                                       n_queries, nq, n_per, nd, stride_b, d_dq);
      FLMR_CUDA(cudaGetLastError());
      ++g_launches;
    }
  }
  if (d_dd && n_docs_total > 0) {
    FLMR_CUDA(cudaMemsetAsync(d_dd, 0, static_cast<size_t>(n_docs_total) * nd * kDim * sizeof(float), st));
    const int64_t warps = static_cast<int64_t>(n_queries) * n_per * nq;
    if (warps > 0) {
      if ((warps * 32 + threads - 1) / threads > 0x7fffffffll)
        return fail(FLMR_ERR_UNSUPPORTED, "backward grid too large (%lld warps)", (long long)warps);
      const unsigned blocks = static_cast<unsigned>((warps * 32 + threads - 1) / threads);
      if (f16)
        flmr_bwd_dd_f16_kernel<<<blocks, threads, 0, st>>>(static_cast<const __half*>(d_q), d_argmax, d_grad,
                                                           n_queries, nq, n_per, nd, stride_b, d_dd);
      else
        flmr_bwd_dd_kernel<<<blocks, threads, 0, st>>>(static_cast<const __nv_bfloat16*>(d_q), d_argmax, d_grad,
                                                       n_queries, nq, n_per, nd, stride_b, d_dd);
      FLMR_CUDA(cudaGetLastError());
      ++g_launches;
    }
  }
  return FLMR_OK;
}

int flmr_maxsim_argmax(const void* d_q, int n_queries, int nq, const void* d_docs,
                       const uint8_t* d_mask, int n_docs, int nd, int32_t* d_argmax, float* d_rowmax,
                       int device, void* stream) {
  return argmax_impl(d_q, n_queries, nq, d_docs, d_mask, n_docs, 0, nd, d_argmax, d_rowmax, Elem::kBF16, device,
                     stream);
}

int flmr_maxsim_argmax_fp16(const void* d_q, int n_queries, int nq, const void* d_docs,
                            const uint8_t* d_mask, int n_docs, int nd, int32_t* d_argmax, float* d_rowmax,
                            int device, void* stream) {
  return argmax_impl(d_q, n_queries, nq, d_docs, d_mask, n_docs, 0, nd, d_argmax, d_rowmax, Elem::kF16, device,
                     stream);
}

int flmr_maxsim_backward(const void* d_q, int n_queries, int nq, const void* d_docs, int n_docs, int nd,
                         const int32_t* d_argmax, const float* d_grad, float* d_dq, float* d_dd,
                         int device, void* stream) {
  return backward_impl(d_q, n_queries, nq, d_docs, n_docs, 0, nd, d_argmax, d_grad, d_dq, d_dd, Elem::kBF16, device,
                       stream);
}

int flmr_maxsim_backward_fp16(const void* d_q, int n_queries, int nq, const void* d_docs, int n_docs, int nd,
                              const int32_t* d_argmax, const float* d_grad, float* d_dq, float* d_dd,
                              int device, void* stream) {
  return backward_impl(d_q, n_queries, nq, d_docs, n_docs, 0, nd, d_argmax, d_grad, d_dq, d_dd, Elem::kF16, device,
                       stream);
}

int flmr_ib_loss(const float* d_rowmax, int n_queries, int n_docs, int nq, int nway, int label0,
                 float* d_scores, float* d_loss_per_query, float* d_dscores, int device, void* stream) {
  if (!d_rowmax || !d_scores || !d_loss_per_query || !d_dscores) return fail(FLMR_ERR_INVALID_ARG, "null pointer");
  if (n_queries < 1 || n_docs < 1 || nq < 1 || nway < 1 || label0 < 0 ||
      static_cast<int64_t>(label0) + static_cast<int64_t>(n_queries - 1) * nway >= n_docs)
    return fail(FLMR_ERR_INVALID_ARG, "bad shape n_queries=%d n_docs=%d nq=%d nway=%d label0=%d", n_queries, n_docs,
                nq, nway, label0);
  if (static_cast<size_t>(n_docs) * sizeof(float) > 200 * 1024)
    return fail(FLMR_ERR_UNSUPPORTED, "%d documents per query exceed the loss kernel's shared memory", n_docs);
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  const size_t smem = static_cast<size_t>(n_docs) * sizeof(float);
  // the 48 KiB a launch may use without opting in covers static + dynamic shared memory: the kernel's static
  // reduction buffer counts too (12,288 documents = exactly 48 KiB of scores failed to launch).  Opt in to the whole
  // 200 KiB the check above admits, so that concurrent callers never lower the limit under each other's launches.
  if (smem + kIbThreads / 32 * sizeof(float) > 48 * 1024)
    FLMR_CUDA(cudaFuncSetAttribute(flmr_ib_loss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  flmr_ib_loss_kernel<<<n_queries, kIbThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      d_rowmax, n_queries, n_docs, nq, nway, label0, d_scores, d_loss_per_query, d_dscores);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

int flmr_maxsim_argmax_grouped(const void* d_q, int n_queries, int nq, const void* d_docs,
                               const uint8_t* d_mask, int docs_per_query, int nd, int32_t* d_argmax,
                               float* d_rowmax, int device, void* stream) {
  if (docs_per_query < 1) return fail(FLMR_ERR_INVALID_ARG, "docs_per_query=%d must be >= 1", docs_per_query);
  return argmax_impl(d_q, n_queries, nq, d_docs, d_mask, docs_per_query, docs_per_query, nd, d_argmax, d_rowmax,
                     Elem::kBF16, device, stream);
}

int flmr_maxsim_argmax_grouped_fp16(const void* d_q, int n_queries, int nq, const void* d_docs,
                                    const uint8_t* d_mask, int docs_per_query, int nd, int32_t* d_argmax,
                                    float* d_rowmax, int device, void* stream) {
  if (docs_per_query < 1) return fail(FLMR_ERR_INVALID_ARG, "docs_per_query=%d must be >= 1", docs_per_query);
  return argmax_impl(d_q, n_queries, nq, d_docs, d_mask, docs_per_query, docs_per_query, nd, d_argmax, d_rowmax,
                     Elem::kF16, device, stream);
}

int flmr_maxsim_backward_grouped(const void* d_q, int n_queries, int nq, const void* d_docs,
                                 int docs_per_query, int nd, const int32_t* d_argmax, const float* d_grad,
                                 float* d_dq, float* d_dd, int device, void* stream) {
  if (docs_per_query < 1) return fail(FLMR_ERR_INVALID_ARG, "docs_per_query=%d must be >= 1", docs_per_query);
  return backward_impl(d_q, n_queries, nq, d_docs, docs_per_query, docs_per_query, nd, d_argmax, d_grad, d_dq,
                       d_dd, Elem::kBF16, device, stream);
}

int flmr_maxsim_backward_grouped_fp16(const void* d_q, int n_queries, int nq, const void* d_docs,
                                      int docs_per_query, int nd, const int32_t* d_argmax, const float* d_grad,
                                      float* d_dq, float* d_dd, int device, void* stream) {
  if (docs_per_query < 1) return fail(FLMR_ERR_INVALID_ARG, "docs_per_query=%d must be >= 1", docs_per_query);
  return backward_impl(d_q, n_queries, nq, d_docs, docs_per_query, docs_per_query, nd, d_argmax, d_grad, d_dq,
                       d_dd, Elem::kF16, device, stream);
}

int flmr_debug_maxsim_scores_simt(const flmr_corpus_t* c, const void* d_q, int n_queries, int nq,
                                  unsigned flags, float* d_out_scores, void* stream) {
  if (!c || !d_q || !d_out_scores) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  if (c->codec_nbits) return fail(FLMR_ERR_UNSUPPORTED, "a PLAID-coded corpus holds no rows for the SIMT kernel");
  if (n_queries <= 0 || nq <= 0) return fail(FLMR_ERR_INVALID_ARG, "bad shape");
  if (c->n_passages > 0x7fffffffll || n_queries > 65535)
    return fail(FLMR_ERR_UNSUPPORTED, "SIMT cross-check grid too large");
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  const int threads = nq >= 256 ? 256 : (nq > 128 ? 256 : 128);
  const int64_t ns = slots(c);
  dim3 grid(static_cast<unsigned>(ns), static_cast<unsigned>(n_queries));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const float init = (flags & FLMR_FLAG_RELU) ? 0.f : -INFINITY;
  StreamScratch scratch(st);
  // a compacted corpus: slot-indexed rows into scratch, then spread over the ids as flmr_maxsim_scores does
  float* out = d_out_scores;
  if (c->d_slot_pid) {
    if (int rc = scratch.alloc(&out, static_cast<size_t>(n_queries) * ns * sizeof(float))) return rc;
  }
  const SlotLayout& l = c->layout;
  if (c->elem != Elem::kE4M3) {
    auto* kernel = c->elem == Elem::kF16 ? flmr_simt_maxsim_kernel<Elem::kF16> : flmr_simt_maxsim_kernel<Elem::kBF16>;
    kernel<<<grid, threads, 0, st>>>(c->d_tokens, l.d_poff, l.d_doclen, c->d_dead, d_q, nq, init, out, ns);
    FLMR_CUDA(cudaGetLastError());
    ++g_launches;
  } else {
    // e4m3 corpus: MaxSim of e4m3(Q) against the e4m3 matrix, the queries rounded into stream-ordered scratch
    const int64_t n_chunks = static_cast<int64_t>(n_queries) * nq * (kDim / 8);
    __nv_bfloat16* q8 = nullptr;
    if (int rc = scratch.alloc(&q8, static_cast<size_t>(n_chunks) * 16)) return rc;
    flmr_round_e4m3_kernel<<<static_cast<unsigned>((n_chunks + 255) / 256), 256, 0, st>>>(
        static_cast<const uint4*>(d_q), reinterpret_cast<uint4*>(q8), n_chunks);
    flmr_simt_maxsim_kernel<Elem::kE4M3><<<grid, threads, 0, st>>>(c->d_fp8, l.d_poff, l.d_doclen, c->d_dead, q8, nq,
                                                                   init, out, ns);
    const cudaError_t e = cudaGetLastError();
    g_launches += 2;
    if (e != cudaSuccess) return fail(FLMR_ERR_CUDA, "SIMT cross-check launch failed: %s", cudaGetErrorString(e));
  }
  if (c->d_slot_pid) {
    const int64_t n = static_cast<int64_t>(n_queries) * c->n_passages;
    flmr_expand_slot_scores_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(
        out, ns, c->d_slot_pid, c->pid_base, c->n_passages, n_queries, d_out_scores);
    FLMR_CUDA(cudaGetLastError());
    ++g_launches;
  }
  return FLMR_OK;
}

int flmr_debug_set_scan_variant(int variant) {
  if (variant != 0 && variant != 2 && variant != 3 && variant != 4 && variant != 6)
    return fail(FLMR_ERR_INVALID_ARG, "variant must be 0 (default), 2 or 3 (epilogue warpgroups), 4 (CTA-pair "
                "experiment) or 6 (three warpgroups, split-tile loop)");
  g_scan_variant = variant;
  return FLMR_OK;
}

int flmr_debug_set_argmax_path(int path) {
  if (path < 0 || path > 2) return fail(FLMR_ERR_INVALID_ARG, "path must be 0 (by size), 1 (warp-MMA) or 2 (wgmma)");
  g_argmax_path = path;
  return FLMR_OK;
}

int flmr_debug_build_partition(const int32_t* h_doclens, int64_t n_passages, int n_ctas,
                               int32_t* cta_row_begin, int64_t* cta_tile_base,
                               uint32_t* tile_end_mask, int32_t* tile_first_pid,
                               int64_t tile_capacity, int64_t* n_tiles_out) {
  if (!h_doclens || n_passages <= 0 || n_ctas < 1 || !cta_row_begin || !cta_tile_base || !n_tiles_out)
    return fail(FLMR_ERR_INVALID_ARG, "bad argument");
  std::vector<int64_t> poff;
  if (int rc = passage_offsets(h_doclens, n_passages, nullptr, &poff, nullptr)) return rc;
  n_ctas = static_cast<int>(std::min<int64_t>(n_ctas, n_passages));
  std::vector<int32_t> rb, fp;
  std::vector<int64_t> tb;
  std::vector<uint32_t> em;
  build_partition(poff, n_ctas, kTileN, &rb, &tb, &em, &fp);
  *n_tiles_out = static_cast<int64_t>(em.size());
  std::copy(rb.begin(), rb.end(), cta_row_begin);
  std::copy(tb.begin(), tb.end(), cta_tile_base);
  if (tile_end_mask && tile_first_pid) {
    if (static_cast<int64_t>(em.size()) > tile_capacity)
      return fail(FLMR_ERR_INVALID_ARG, "tile_capacity %lld < %zu tiles", (long long)tile_capacity, em.size());
    std::copy(em.begin(), em.end(), tile_end_mask);
    std::copy(fp.begin(), fp.end(), tile_first_pid);
  }
  return FLMR_OK;
}

int flmr_debug_window_plan(const int32_t* h_doclens, int64_t n_passages, int64_t window_bytes, int n_ctas,
                           int64_t* out_windows, int64_t capacity, int64_t* n_windows_out, int32_t* cta_row_begin,
                           int64_t* cta_tile_base, uint32_t* tile_end_mask, int32_t* tile_first_pid,
                           int64_t tile_capacity, int64_t* n_tiles_out) {
  if (!h_doclens || n_passages <= 0 || n_ctas < 1 || !n_windows_out) return fail(FLMR_ERR_INVALID_ARG, "bad argument");
  if (window_bytes < kDim * 2) return fail(FLMR_ERR_INVALID_ARG, "window_bytes=%lld holds no row", (long long)window_bytes);
  std::vector<int64_t> poff;
  if (int rc = passage_offsets(h_doclens, n_passages, nullptr, &poff, nullptr)) return rc;
  std::vector<std::pair<int64_t, int64_t>> ranges;
  if (int rc = plan_windows(poff, window_bytes / (kDim * 2), &ranges)) return rc;
  const int64_t nw = static_cast<int64_t>(ranges.size());
  *n_windows_out = nw;
  if (!out_windows) return FLMR_OK;
  if (capacity < nw) return fail(FLMR_ERR_INVALID_ARG, "capacity %lld < %lld windows", (long long)capacity, (long long)nw);
  std::vector<int32_t> all_rb, all_fp;
  std::vector<int64_t> all_tb;
  std::vector<uint32_t> all_em;
  for (int64_t w = 0; w < nw; ++w) {
    const int64_t s0 = ranges[w].first, s1 = ranges[w].second;
    int nc = 0;
    std::vector<int32_t> rb, fp;
    std::vector<int64_t> tb;
    std::vector<uint32_t> em;
    window_partition(poff, s0, s1, n_ctas, &nc, &rb, &tb, &em, &fp);
    int64_t* o = out_windows + 6 * w;
    o[0] = s0;
    o[1] = s1;
    o[2] = poff[s0];
    o[3] = poff[s1] - poff[s0];
    o[4] = nc;
    o[5] = static_cast<int64_t>(em.size());
    all_rb.insert(all_rb.end(), rb.begin(), rb.end());
    all_tb.insert(all_tb.end(), tb.begin(), tb.end());
    all_em.insert(all_em.end(), em.begin(), em.end());
    all_fp.insert(all_fp.end(), fp.begin(), fp.end());
  }
  if (n_tiles_out) *n_tiles_out = static_cast<int64_t>(all_em.size());
  if (cta_row_begin && cta_tile_base && tile_end_mask && tile_first_pid) {
    if (static_cast<int64_t>(all_em.size()) > tile_capacity || static_cast<int64_t>(all_rb.size()) > tile_capacity)
      return fail(FLMR_ERR_INVALID_ARG, "tile_capacity %lld < %zu tiles or %zu CTA entries", (long long)tile_capacity,
                  all_em.size(), all_rb.size());
    std::copy(all_rb.begin(), all_rb.end(), cta_row_begin);
    std::copy(all_tb.begin(), all_tb.end(), cta_tile_base);
    std::copy(all_em.begin(), all_em.end(), tile_end_mask);
    std::copy(all_fp.begin(), all_fp.end(), tile_first_pid);
  }
  return FLMR_OK;
}

int flmr_debug_plan_passes(int n_queries, int nq, int allow_pair, int32_t* out_plan, int capacity, int* n_passes_out) {
  if (n_queries < 0 || nq <= 0 || !n_passes_out) return fail(FLMR_ERR_INVALID_ARG, "bad argument");
  std::vector<PassPlan> plan;
  int group = 1;
  plan_passes(n_queries, nq, allow_pair != 0, &plan, &group, nullptr);
  *n_passes_out = static_cast<int>(plan.size());
  if (out_plan) {
    if (static_cast<int>(plan.size()) > capacity)
      return fail(FLMR_ERR_INVALID_ARG, "capacity %d < %zu passes", capacity, plan.size());
    for (size_t i = 0; i < plan.size(); ++i) {
      const PassPlan& q = plan[i];
      const int32_t row[8] = {q.q_first, q.n_q, q.row0, q.rows, q.rbq, q.n_mtiles, q.flags, q.group_first + q.acc_slot};
      std::copy(row, row + 8, out_plan + i * 8);
    }
  }
  return FLMR_OK;
}

int flmr_debug_compact_plan(const int32_t* h_doclens, int64_t n_passages, const int64_t* h_deleted, int64_t n_deleted,
                            int64_t chunk_rows, int64_t* out_moves, int64_t capacity, int64_t* n_moves_out) {
  if (!h_doclens || n_passages <= 0 || n_deleted < 0 || (n_deleted > 0 && !h_deleted) || chunk_rows < 0 ||
      !n_moves_out)
    return fail(FLMR_ERR_INVALID_ARG, "bad argument");
  std::vector<int64_t> poff;
  if (int rc = passage_offsets(h_doclens, n_passages, nullptr, &poff, nullptr)) return rc;
  std::vector<char> keep(n_passages, 1);
  for (int64_t i = 0; i < n_deleted; ++i) {
    if (h_deleted[i] < 0 || h_deleted[i] >= n_passages)
      return fail(FLMR_ERR_INVALID_ARG, "deleted passage %lld outside [0, %lld)", (long long)h_deleted[i],
                  (long long)n_passages);
    keep[h_deleted[i]] = 0;
  }
  std::vector<MovePiece> plan;
  plan_compaction(kept_runs(poff, keep), chunk_rows ? chunk_rows : kCompactChunkRows, true, &plan);
  *n_moves_out = static_cast<int64_t>(plan.size());
  if (out_moves) {
    if (static_cast<int64_t>(plan.size()) > capacity)
      return fail(FLMR_ERR_INVALID_ARG, "capacity %lld < %zu moves", (long long)capacity, plan.size());
    for (size_t i = 0; i < plan.size(); ++i) {
      const int64_t row[5] = {plan[i].src, plan[i].dst, plan[i].rows, plan[i].staged ? 1 : 0, plan[i].chunk};
      std::copy(row, row + 5, out_moves + i * 5);
    }
  }
  return FLMR_OK;
}

int flmr_comm_unique_id(void* out_id_128_bytes) {
  if (!out_id_128_bytes) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  const NcclApi* api = nullptr;
  if (int rc = load_nccl(&api)) return rc;
  FLMR_NCCL(api, api->GetUniqueId(out_id_128_bytes));
  return FLMR_OK;
}

int flmr_comm_create(const void* id_128_bytes, int rank, int world_size, int device, flmr_comm_t** out) {
  if (!id_128_bytes || !out) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  if (world_size < 1 || rank < 0 || rank >= world_size)
    return fail(FLMR_ERR_INVALID_ARG, "bad rank %d / world size %d", rank, world_size);
  const NcclApi* api = nullptr;
  if (int rc = load_nccl(&api)) return rc;
  DeviceGuard guard(device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", device);
  flmr_comm* c = new (std::nothrow) flmr_comm();
  if (!c) return fail(FLMR_ERR_OOM, "host allocation failed");
  NcclId id;
  memcpy(id.internal, id_128_bytes, sizeof id.internal);
  const int r = api->CommInitRank(&c->nccl, world_size, id, rank);
  if (r != 0) {
    delete c;
    return fail(FLMR_ERR_CUDA, "ncclCommInitRank failed: %s", api->GetErrorString(r));
  }
  c->rank = rank;
  c->world = world_size;
  c->device = device;
  c->owned = true;
  *out = c;
  return FLMR_OK;
}

int flmr_comm_adopt(void* nccl_comm, int device, flmr_comm_t** out) {
  if (!nccl_comm || !out) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  const NcclApi* api = nullptr;
  if (int rc = load_nccl(&api)) return rc;
  flmr_comm* c = new (std::nothrow) flmr_comm();
  if (!c) return fail(FLMR_ERR_OOM, "host allocation failed");
  c->nccl = nccl_comm;
  c->device = device;
  int r = api->CommCount(nccl_comm, &c->world);
  if (r == 0) r = api->CommUserRank(nccl_comm, &c->rank);
  if (r != 0) {
    delete c;
    return fail(FLMR_ERR_CUDA, "ncclCommCount / ncclCommUserRank failed: %s", api->GetErrorString(r));
  }
  *out = c;
  return FLMR_OK;
}

int flmr_comm_destroy(flmr_comm_t* c) {
  if (!c) return FLMR_OK;
  DeviceGuard guard(c->device);
  cudaFree(c->d_send_s);
  cudaFree(c->d_send_p);
  cudaFree(c->d_recv_s);
  cudaFree(c->d_recv_p);
  if (c->owned && c->nccl) {
    const NcclApi* api = nullptr;
    if (load_nccl(&api) == FLMR_OK) api->CommDestroy(c->nccl);
  }
  delete c;
  return FLMR_OK;
}

int flmr_comm_info(const flmr_comm_t* c, int* rank, int* world_size) {
  if (!c) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  if (rank) *rank = c->rank;
  if (world_size) *world_size = c->world;
  return FLMR_OK;
}

int flmr_topk_exchange(flmr_comm_t* c, const float* d_scores, const int64_t* d_pids, int n_queries, int k_in,
                       int k_out, float* d_out_scores, int64_t* d_out_pids, void* stream) {
  if (!c || !d_scores || !d_pids || !d_out_scores || !d_out_pids) return fail(FLMR_ERR_INVALID_ARG, "null argument");
  if (n_queries < 0 || k_in < 1 || k_out < 1 || k_out > kMaxK)
    return fail(FLMR_ERR_INVALID_ARG, "bad shape n_queries=%d k_in=%d k_out=%d", n_queries, k_in, k_out);
  if (static_cast<int64_t>(c->world) * k_in > kMergeThreads * kMergePer)
    return fail(FLMR_ERR_UNSUPPORTED, "world*k_in = %lld exceeds merge capacity %d", (long long)c->world * k_in,
                kMergeThreads * kMergePer);
  if (n_queries == 0) return FLMR_OK;
  const NcclApi* api = nullptr;
  if (int rc = load_nccl(&api)) return rc;
  DeviceGuard guard(c->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", c->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = static_cast<int64_t>(n_queries) * k_in;
  if (c->capacity < n) {   // (grown only when a call brings more entries than any before: not on the steady path)
    cudaFree(c->d_recv_s);
    cudaFree(c->d_recv_p);
    c->d_recv_s = nullptr;
    c->d_recv_p = nullptr;
    c->capacity = 0;
    FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->d_recv_s), static_cast<size_t>(n) * c->world * sizeof(float)));
    FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->d_recv_p), static_cast<size_t>(n) * c->world * sizeof(int64_t)));
    c->capacity = n;
  }
  // one exchange step: both all-gathers in ONE NCCL group (a single fused launch on the wire), then the merge
  FLMR_NCCL(api, api->GroupStart());
  int r1 = api->AllGather(d_scores, c->d_recv_s, static_cast<size_t>(n), kNcclFloat32, c->nccl, st);
  int r2 = api->AllGather(d_pids, c->d_recv_p, static_cast<size_t>(n), kNcclInt64, c->nccl, st);
  FLMR_NCCL(api, api->GroupEnd());
  if (r1 != 0 || r2 != 0)
    return fail(FLMR_ERR_CUDA, "ncclAllGather failed: %s", api->GetErrorString(r1 ? r1 : r2));
  flmr_merge_kernel<<<n_queries, kMergeThreads, 0, st>>>(nullptr, c->d_recv_s, c->d_recv_p, c->world, n_queries,
                                                        k_in, k_out, 0, nullptr, d_out_scores, d_out_pids, 0);
  FLMR_CUDA(cudaGetLastError());
  ++g_launches;
  return FLMR_OK;
}

int flmr_maxsim_topk_sharded(const flmr_corpus_t* corpus, flmr_workspace_t* ws, flmr_comm_t* comm, const void* d_q,
                             int n_queries, int nq, int k, unsigned flags, float* d_out_scores,
                             int64_t* d_out_pids, void* stream) {
  return flmr_maxsim_topk_sharded_allowed(corpus, ws, comm, d_q, n_queries, nq, k, flags, nullptr, 0, d_out_scores,
                                          d_out_pids, stream);
}

int flmr_maxsim_topk_sharded_allowed(const flmr_corpus_t* corpus, flmr_workspace_t* ws, flmr_comm_t* comm,
                                     const void* d_q, int n_queries, int nq, int k, unsigned flags,
                                     const uint32_t* d_allow, int64_t allow_stride_words, float* d_out_scores,
                                     int64_t* d_out_pids, void* stream) {
  if (!comm) return fail(FLMR_ERR_INVALID_ARG, "comm is null");
  if (!d_out_scores || !d_out_pids) return fail(FLMR_ERR_INVALID_ARG, "output pointer is null");
  if (k < 1 || k > kMaxK) return fail(FLMR_ERR_INVALID_ARG, "k=%d outside [1, %d]", k, kMaxK);
  if (corpus && corpus->device != comm->device)
    return fail(FLMR_ERR_INVALID_ARG, "corpus on device %d, communicator on device %d", corpus->device, comm->device);
  if (n_queries <= 0) return n_queries == 0 ? FLMR_OK : fail(FLMR_ERR_INVALID_ARG, "bad n_queries=%d", n_queries);
  DeviceGuard guard(comm->device);
  if (!guard.ok) return fail(FLMR_ERR_CUDA, "cudaSetDevice(%d) failed", comm->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = static_cast<int64_t>(n_queries) * k;
  if (comm->send_capacity < n) {   // sized apart from the receive buffers, which flmr_topk_exchange alone may grow
    cudaFree(comm->d_send_s);
    cudaFree(comm->d_send_p);
    comm->d_send_s = nullptr;
    comm->d_send_p = nullptr;
    comm->send_capacity = 0;
    FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(&comm->d_send_s), static_cast<size_t>(n) * sizeof(float)));
    FLMR_CUDA(cudaMalloc(reinterpret_cast<void**>(&comm->d_send_p), static_cast<size_t>(n) * sizeof(int64_t)));
    comm->send_capacity = n;
  }
  // this rank's shard (the fused scan fills short lists with (-inf, -1), which the merge ignores)
  if (int rc = run_search(corpus, ws, d_q, n_queries, nq, flags, k, d_allow, allow_stride_words, nullptr,
                          comm->d_send_s, comm->d_send_p, st))
    return rc;
  return flmr_topk_exchange(comm, comm->d_send_s, comm->d_send_p, n_queries, k, k, d_out_scores, d_out_pids, stream);
}

int64_t flmr_launch_count(int reset) {
  const int64_t v = g_launches;
  if (reset) g_launches = 0;
  return v;
}

int flmr_set_profiling(int enable) {
  g_profiling = enable != 0;
  return FLMR_OK;
}

int flmr_scan_kernel_stats(double* total_ms, int64_t* launches, int reset) {
  double tot = 0.0;
  int64_t n = 0;
  for (auto& ev : g_scan_events) {
    float ms = 0.f;
    if (cudaEventSynchronize(ev.b) == cudaSuccess && cudaEventElapsedTime(&ms, ev.a, ev.b) == cudaSuccess) {
      tot += ms;
      ++n;
    }
  }
  if (total_ms) *total_ms = tot;
  if (launches) *launches = n;
  if (reset) {
    for (auto& ev : g_scan_events) {
      cudaEventDestroy(ev.a);
      cudaEventDestroy(ev.b);
    }
    g_scan_events.clear();
  }
  return FLMR_OK;
}

}  // extern "C"
