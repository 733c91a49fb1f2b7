// common.cuh -- shared host/device helpers for libsmaat_b200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/smaat_b200.h"

namespace smaat {

// ---------------------------------------------------------------------------------------
// host-side error plumbing: nothing throws across the C ABI
// ---------------------------------------------------------------------------------------
extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

int fail(int code, const char* fmt, ...);

#define SMAAT_REQUIRE(cond, ...)                                    \
  do {                                                              \
    if (!(cond)) return ::smaat::fail(SMAAT_E_BADARG, __VA_ARGS__); \
  } while (0)

// After a kernel launch: count it and surface launch-configuration errors.
#define SMAAT_LAUNCH_CHECK(name)                                                              \
  do {                                                                                        \
    ::smaat::g_launches.fetch_add(1, std::memory_order_relaxed);                              \
    cudaError_t e__ = cudaGetLastError();                                                     \
    if (e__ != cudaSuccess)                                                                   \
      return ::smaat::fail(SMAAT_E_CUDA, "%s: launch failed: %s", name, cudaGetErrorString(e__)); \
  } while (0)

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Driver entry point for TMA descriptors, resolved at run time through cudart so that the
// library links (and loads on a CPU-only box) without libcuda.
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

// Build a fp32 tiled tensor map.  dims/strides innermost first; strides in BYTES for dims 1..rank-1.
int make_tmap_f32(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, CUtensorMapSwizzle swizzle, const char* who);
// the same for any element type (the bf16 weight packs of SMAAT_PW_BF16: CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)
int make_tmap(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle, const char* who);

int num_sms();

// True the first time a call site sees the current device (`mask` is the call site's function-local static): per-device
// one-time setup such as cudaFuncSetAttribute, which applies to the current device only.
inline bool first_use_on_device(std::atomic<uint64_t>& mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const uint64_t bit = 1ull << (dev & 63);
  return (mask.fetch_or(bit, std::memory_order_relaxed) & bit) == 0;
}

// ---------------------------------------------------------------------------------------
// device-side PTX wrappers (mbarrier, TMA, fences)
// ---------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                   smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// bf16 activations (the serving forward's bf16 storage route) are raw uint16_t bits: widened exactly, rounded to nearest even
__device__ __forceinline__ float bf16_f32(uint16_t h) { return __uint_as_float((uint32_t)h << 16); }
__device__ __forceinline__ uint16_t f32_bf16(float v) {
  uint16_t r;
  asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(v));
  return r;
}
__device__ __forceinline__ uint32_t f32x2_bf16x2(float lo, float hi) {   // lo at the lower address
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float4 bf16x4_f32(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xffff0000u));
}
// Activation loads and stores in the storage type T (float or uint16_t bf16), as fp32 values: one element, or four
// consecutive ones (a 16-byte fp32 / 8-byte bf16 access, which must be aligned to its size)
template <typename T>
__device__ __forceinline__ float ld_act(const T* p) {
  if constexpr (sizeof(T) == 4) return __ldg(p);
  else return bf16_f32(__ldg(reinterpret_cast<const unsigned short*>(p)));
}
template <typename T>
__device__ __forceinline__ float4 ld_act4(const T* p) {
  if constexpr (sizeof(T) == 4) return __ldg(reinterpret_cast<const float4*>(p));
  else return bf16x4_f32(__ldg(reinterpret_cast<const uint2*>(p)));
}
template <typename T>
__device__ __forceinline__ void st_act(T* p, float v) {
  if constexpr (sizeof(T) == 4) *p = v;
  else *p = f32_bf16(v);
}
template <typename T>
__device__ __forceinline__ void st_act4(T* p, float4 v) {
  if constexpr (sizeof(T) == 4) *reinterpret_cast<float4*>(p) = v;
  else *reinterpret_cast<uint2*>(p) = make_uint2(f32x2_bf16x2(v.x, v.y), f32x2_bf16x2(v.z, v.w));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
#endif  // __CUDACC__

}  // namespace smaat
