// datasets.cu -- the arithmetic of the precipitation dataset builder: the number of rain pixels in every frame.
//
// Replaces the per-frame `np.sum(images[i] > 0)` of the reference's create_datasets.py:79-82 (the host decides every
// rain threshold from the same counts).  `v > 0.0f` under IEEE ordered comparison is tested on the bit pattern,
// 0 < bits <= 0x7f800000 as int32: +0, negative values (sign bit set: -0, -inf, negative NaNs) and NaNs above +inf are
// not counted, positive denormals and +inf are.  No floating-point instruction touches the value, so no compiler flag
// (flush-to-zero among them) can change a count.  Counts are exact integers, whatever the reduction order.
//
// One CTA per frame (grid-strided over the frames): 16-byte loads when every frame starts 16-byte aligned (frames aligned
// and plane % 4 == 0), 4-byte loads otherwise; a warp-shuffle and shared-memory reduction, one store per frame.
#include "common.cuh"

namespace smaat {

constexpr int kRainThreads = 512;

__device__ __forceinline__ int is_rain(int b) { return (b > 0) & (b <= 0x7f800000); }

template <bool VEC>
__global__ void __launch_bounds__(kRainThreads) rain_pixels_kernel(const float* __restrict__ frames, int64_t n_frames,
                                                                   int plane, int32_t* __restrict__ counts) {
  __shared__ int warp_part[kRainThreads / 32];
  for (int64_t f = blockIdx.x; f < n_frames; f += gridDim.x) {
    const float* src = frames + f * (int64_t)plane;
    int c = 0;
    if constexpr (VEC) {
      const int4* s4 = reinterpret_cast<const int4*>(src);
      const int n4 = plane >> 2;
      int p = threadIdx.x;
#pragma unroll 1
      for (; p + 3 * kRainThreads < n4; p += 4 * kRainThreads) {   // four 16-byte loads in flight per thread
        int4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = __ldcs(s4 + p + u * kRainThreads);
#pragma unroll
        for (int u = 0; u < 4; ++u) c += is_rain(v[u].x) + is_rain(v[u].y) + is_rain(v[u].z) + is_rain(v[u].w);
      }
      for (; p < n4; p += kRainThreads) {
        const int4 v = __ldcs(s4 + p);
        c += is_rain(v.x) + is_rain(v.y) + is_rain(v.z) + is_rain(v.w);
      }
    } else {
      const int* s = reinterpret_cast<const int*>(src);
      for (int p = threadIdx.x; p < plane; p += kRainThreads) c += is_rain(__ldcs(s + p));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x < 32) {
      c = threadIdx.x < kRainThreads / 32 ? warp_part[threadIdx.x] : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (threadIdx.x == 0) counts[f] = c;
    }
    __syncthreads();   // warp_part is rewritten by the next frame
  }
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_rain_pixels_fwd(const float* frames, int64_t n_frames, int64_t plane, int32_t* counts, void* stream) {
  SMAAT_REQUIRE(frames && counts && n_frames >= 1 && plane >= 1 && plane < (int64_t(1) << 31),
                "rain_pixels: bad arguments (frames=%p counts=%p n_frames=%lld plane=%lld; need non-null pointers, "
                "n_frames >= 1, 1 <= plane < 2^31)",
                (const void*)frames, (void*)counts, (long long)n_frames, (long long)plane);
  int64_t blocks = n_frames;
  const int64_t cap = (int64_t)num_sms() * 4;   // as many CTAs as can be resident
  if (blocks > cap) blocks = cap;
  if (aligned16(frames) && plane % 4 == 0)
    rain_pixels_kernel<true><<<(unsigned)blocks, kRainThreads, 0, (cudaStream_t)stream>>>(frames, n_frames, (int)plane, counts);
  else
    rain_pixels_kernel<false><<<(unsigned)blocks, kRainThreads, 0, (cudaStream_t)stream>>>(frames, n_frames, (int)plane, counts);
  SMAAT_LAUNCH_CHECK("smaat_rain_pixels_fwd");
  return SMAAT_OK;
}
