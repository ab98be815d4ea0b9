// common.cuh -- shared helpers: error plumbing, candidate loads, shared-memory carving, PTX wrappers for sm_90a
// (mbarrier, bulk copy (TMA engine), warpgroup MMA), fp16 split, packed arg-max keys.
#pragma once

#include <assert.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/baybe_b200.h"

namespace bb {

// ------------------------------------------------------------------------------------------
// error plumbing (thread-local message, integer status)
// ------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);

#define BB_CHECK_ARG(cond, ...)        \
  do {                                 \
    if (!(cond)) {                     \
      bb::set_error(__VA_ARGS__);      \
      return BB_ERR_INVALID;           \
    }                                  \
  } while (0)

#define BB_CHECK_SUPPORTED(cond, ...)  \
  do {                                 \
    if (!(cond)) {                     \
      bb::set_error(__VA_ARGS__);      \
      return BB_ERR_UNSUPPORTED;       \
    }                                  \
  } while (0)

#define BB_CUDA(call)                                                                     \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      bb::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,                  \
                    cudaGetErrorString(e_));                                              \
      return BB_ERR_CUDA;                                                                 \
    }                                                                                     \
  } while (0)

#define BB_LAUNCH_CHECK() BB_CUDA(cudaGetLastError())

// SM count and opt-in shared-memory limit of the current device, queried once per device (not per launch).
static inline int device_limits(int* sms, int* max_smem) {
  constexpr int kMaxDev = 64;
  static int c_sms[kMaxDev], c_smem[kMaxDev];
  static bool c_ok[kMaxDev];
  int dev = 0;
  BB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDev || !c_ok[dev]) {
    int a = 0, b = 0;
    BB_CUDA(cudaDeviceGetAttribute(&b, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    BB_CUDA(cudaDeviceGetAttribute(&a, cudaDevAttrMultiProcessorCount, dev));
    if (dev < 0 || dev >= kMaxDev) {
      *sms = a;
      *max_smem = b;
      return BB_OK;
    }
    c_sms[dev] = a;
    c_smem[dev] = b;
    c_ok[dev] = true;
  }
  *sms = c_sms[dev];
  *max_smem = c_smem[dev];
  return BB_OK;
}

// Opt a kernel into the full dynamic shared-memory carve-out once per device (function-local static per
// instantiation site), instead of one cudaFuncSetAttribute per launch.  The 227 KB a block may opt in to include the
// kernel's static shared memory, so the dynamic limit is what that leaves.
#define BB_SMEM_OPTIN_ONCE(kernel)                                                                         \
  do {                                                                                                     \
    static unsigned long long done_mask_ = 0ull;                                                           \
    int dev_ = 0;                                                                                          \
    BB_CUDA(cudaGetDevice(&dev_));                                                                         \
    if (dev_ < 0 || dev_ >= 64 || !((done_mask_ >> dev_) & 1ull)) {                                        \
      cudaFuncAttributes fa_;                                                                              \
      BB_CUDA(cudaFuncGetAttributes(&fa_, kernel));                                                        \
      BB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,                    \
                                   227 * 1024 - (int)fa_.sharedSizeBytes));                                \
      if (dev_ >= 0 && dev_ < 64) done_mask_ |= 1ull << dev_;                                              \
    }                                                                                                      \
  } while (0)

constexpr int kTileM = 128;     // candidates per tile = two 64-row warpgroup MMAs
constexpr int kChunk = 64;      // training points per K chunk = one 128-byte swizzle row of fp16
constexpr int kSMs = 132;       // H100 SXM: grid caps of the grid-stride kernels

// candidate layouts beyond bb_layout, internal to the single-launch host pass: level codes expanded while staging
constexpr int kLayoutCodes4 = 16, kLayoutCodes8 = 17;

static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// ------------------------------------------------------------------------------------------
// candidate loads for the four layouts of bb_layout
// ------------------------------------------------------------------------------------------
template <int LAYOUT>
__device__ __forceinline__ float load_x(const void* __restrict__ x, int64_t row, int col,
                                        int64_t ld) {
  if constexpr (LAYOUT == BB_ROW_MAJOR_F32) {
    return __ldg(reinterpret_cast<const float*>(x) + row * ld + col);
  } else if constexpr (LAYOUT == BB_COL_MAJOR_F32) {
    return __ldg(reinterpret_cast<const float*>(x) + (int64_t)col * ld + row);
  } else if constexpr (LAYOUT == BB_ROW_MAJOR_F64) {
    return (float)__ldg(reinterpret_cast<const double*>(x) + row * ld + col);
  } else {
    return (float)__ldg(reinterpret_cast<const double*>(x) + (int64_t)col * ld + row);
  }
}

// load_x with the layout known only at run time
__device__ __forceinline__ float load_x_any(const void* __restrict__ x, int layout, int64_t row, int col, int64_t ld) {
  switch (layout) {
    case BB_ROW_MAJOR_F32: return load_x<BB_ROW_MAJOR_F32>(x, row, col, ld);
    case BB_COL_MAJOR_F32: return load_x<BB_COL_MAJOR_F32>(x, row, col, ld);
    case BB_ROW_MAJOR_F64: return load_x<BB_ROW_MAJOR_F64>(x, row, col, ld);
    default: return load_x<BB_COL_MAJOR_F64>(x, row, col, ld);
  }
}

// ------------------------------------------------------------------------------------------
// Dynamic shared memory, carved in order: a buffer starts where the previous one ends and spans a whole multiple of
// its alignment, so the buffers of the largest alignment go first (the base is 1024-byte aligned).  A kernel's carve
// function runs on the host with base = null to size the launch, and in the kernel to place the buffers, so the
// byte count and the pointers come from the same code.  The host run asserts that every buffer starts on its
// alignment, so a carve that takes a more aligned buffer after a less aligned one fails at its first launch.  (The
// kernels do not round the offset up themselves: that arithmetic raises k_fused's spills.)
// ------------------------------------------------------------------------------------------
struct SmemCarver {
  uint8_t* base;
  size_t bytes = 0;
  template <class T>
  __host__ __device__ __forceinline__ T* take(size_t n, size_t align = 16) {
#ifndef __CUDA_ARCH__
    assert(bytes % align == 0 && "carve the buffers of larger alignment first");
#endif
    uint8_t* p = base + bytes;  // plain pointer arithmetic: nvcc keeps seeing a shared-memory address
    bytes += (n + align - 1) / align * align;
    return reinterpret_cast<T*>(p);
  }
};

// ------------------------------------------------------------------------------------------
// kernel epilogues k(r^2) -- the scaled squared distance t already carries the family's
// constant (5 r^2 for Matern-5/2, 3 r^2 for 3/2, r^2 for 1/2, r^2 log2(e)/2 for RBF), folded
// into the lengthscale by bb_model_build.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float fast_sqrt(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

template <int FAMILY>
__device__ __forceinline__ float kernel_from_t(float t) {
  t = fmaxf(t, 0.0f);
  if constexpr (FAMILY == BB_KERNEL_RBF) {
    return fast_ex2(-t);
  } else if constexpr (FAMILY == BB_KERNEL_MATERN12) {
    float s = fast_sqrt(t);
    return fast_ex2(-kLog2e * s);
  } else if constexpr (FAMILY == BB_KERNEL_MATERN32) {
    float s = fast_sqrt(t);
    return (1.0f + s) * fast_ex2(-kLog2e * s);
  } else {
    float s = fast_sqrt(t);
    float poly = fmaf(t, (1.0f / 3.0f), s) + 1.0f;
    return poly * fast_ex2(-kLog2e * s);
  }
}

// ------------------------------------------------------------------------------------------
// packed (score, lowest-index) keys: signed-int64 max == (max score, then min index); -0.0 packs as +0.0, so
// the two zeros tie and the lower index wins, as in torch.argmax.  NaN scores are skipped by every caller.
// ------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int64_t pack_key(float score, uint32_t local_idx) {
  uint32_t u;
#ifdef __CUDA_ARCH__
  u = __float_as_uint(score);
#else
  memcpy(&u, &score, 4);
#endif
  if (u == 0x80000000u) u = 0u;
  int32_t s = (int32_t)u;
  s ^= (s >> 31) & 0x7fffffff;  // total order as signed int
  return (int64_t)(((uint64_t)(uint32_t)s << 32) | (uint64_t)(0xffffffffu - local_idx));
}
constexpr int64_t kEmptyKey = INT64_MIN;

// ------------------------------------------------------------------------------------------
// PTX: shared-memory addresses, mbarrier, fences, bulk copies (TMA engine)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 1-D bulk copy global -> shared through the TMA engine (UBLKCP), completion on an mbarrier.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ------------------------------------------------------------------------------------------
// PTX: warpgroup MMA (wgmma, sm_90a).  Operands are K-major fp16 tiles in shared memory; the fp32
// accumulator lives in the registers of the issuing warpgroup (128 threads).
// ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major swizzled tile whose 8-row groups are contiguous:
// K2 = 64 -> 128-byte rows / 128B swizzle, K2 = 32 -> 64-byte rows / 64B swizzle.  Advancing the
// start address by 32 bytes (two 16-byte units) steps K by 16 inside the swizzle atom.
template <int K2>
__device__ __forceinline__ uint64_t make_wg_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3ffff) >> 4);          // start address, 16-byte units
  d |= (uint64_t)1 << 16;                               // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)((K2 == 64 ? 1024 : 512) >> 4) << 32;  // stride byte offset between 8-row groups
  d |= (uint64_t)(K2 == 64 ? 1 : 2) << 62;              // 1: 128B swizzle, 2: 64B swizzle
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 x 64] += A[64 x 16] * B[64 x 16]^T, fp16 operands, fp32 accumulate.  Fragment of thread t
// (warp w = t / 32 of the warpgroup, lane l): d[i] is row 16 w + l / 4 + 8 ((i / 2) & 1), column
// 8 (i / 4) + 2 (l & 3) + (i & 1).
__device__ __forceinline__ void wgmma_64x64(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b));
}
// Same with A from registers: a[0..3] are the packed fp16 pairs of the A fragment, which has the layout of the
// accumulator fragment of columns 16 k .. 16 k + 15 (a[0] = d[8k..8k+1], a[1] = d[8k+2..3], a[2] = d[8k+4..5],
// a[3] = d[8k+6..7]): an accumulator converts into the next MMA's A operand without leaving the registers.
__device__ __forceinline__ void wgmma_64x64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, 1, 1, 1, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b));
}
// Named barrier over the 128 threads of warpgroup `wg` (ids 2.. are free; 0 is __syncthreads, 1 bar_compute).
__device__ __forceinline__ void bar_wg(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }

// Byte offset of 16-byte chunk `c16` (0..7) of row `r` inside a 128B-swizzled tile whose rows are
// 128 bytes (64 fp16): Swizzle<3,4,3> -- XOR the chunk index with (row mod 8).
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t r, uint32_t c16) {
  return r * 128u + ((c16 ^ (r & 7u)) << 4);
}

// K-major tiles whose rows hold K2 fp16 (K2 = 64 -> 128-byte rows / SWIZZLE_128B, K2 = 32 ->
// 64-byte rows / SWIZZLE_64B).  8-row groups are contiguous (SBO = 8 * row bytes).
template <int K2>
__host__ __device__ __forceinline__ uint32_t swk_offset(uint32_t r, uint32_t c16) {
  if constexpr (K2 == 64) return r * 128u + ((c16 ^ (r & 7u)) << 4);
  else return r * 64u + ((c16 ^ ((r >> 1) & 3u)) << 4);  // Swizzle<2,4,3>: bits[5:4] ^= bits[8:7]
}
// fp16 hi/lo split of a non-negative-or-signed fp32 value: x ~= hi + lo, relative error 2^-22.
__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  __half2 h = __floats2half2_rn(x0, x1);
  float2 hf = __half22float2(h);
  __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

}  // namespace bb
