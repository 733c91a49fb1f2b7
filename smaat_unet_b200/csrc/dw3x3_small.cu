// dw3x3_small.cu -- depthwise 3x3 forward for SMALL planes whose rows TMA cannot describe (W % 4 != 0), e.g. the 18 x 18
// bottleneck of SmaAt-UNet (down4 / up1: 16 384 planes of 324 floats at B = 32).
//
// Same arithmetic as dw3x3.cu (reference models/layers.py:38-44,48).  The generic LDG loader there spends one CTA and a
// block-wide barrier per plane; here one WARP owns one (b, c) plane: 8 planes per CTA, the plane (+ zero border = padding 1)
// is staged in the warp's own shared-memory tile with coalesced loads, warp-level sync only, and every lane then produces
// outputs pixel by pixel (coalesced stores of the K output planes).  Optional relu(scale*x+shift) on load (train-mode
// BN+ReLU of the producer) and virtual concat like the main kernel.
#include "common.cuh"

namespace smaat {

constexpr int DWS_WARPS = 8;
constexpr int DWS_MAX_PIXELS = 1024;   // plane size limit (tile <= 34 x 34 floats per warp)

template <int K, bool PRO>
__global__ void __launch_bounds__(32 * DWS_WARPS) dw3x3_small_kernel(const float* __restrict__ x0, int C0, int64_t bs0,
                                                                    const float* __restrict__ x1, int C1, int64_t bs1,
                                                                    const float* __restrict__ w, const float* __restrict__ bias,
                                                                    const float* __restrict__ in_scale,
                                                                    const float* __restrict__ in_shift, float* __restrict__ y,
                                                                    int64_t planes, int H, int W) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t plane = (int64_t)blockIdx.x * DWS_WARPS + warp;
  if (plane >= planes) return;   // whole warp leaves together; only __syncwarp below
  const int Cin = C0 + C1;
  const int b = (int)(plane / Cin), c = (int)(plane - (int64_t)b * Cin);
  const int P = H * W, TW = W + 2;
  float* tile = sm + warp * ((H + 2) * TW);
  const float* src = (c < C0) ? x0 + (int64_t)b * bs0 + (int64_t)c * P : x1 + (int64_t)b * bs1 + (int64_t)(c - C0) * P;
  // zero border (= the conv's padding), then the plane
  for (int i = lane; i < TW; i += 32) { tile[i] = 0.f; tile[(H + 1) * TW + i] = 0.f; }
  for (int i = lane; i < H; i += 32) { tile[(i + 1) * TW] = 0.f; tile[(i + 1) * TW + W + 1] = 0.f; }
  float ps = 1.f, pt = 0.f;
  if (PRO) { ps = __ldg(in_scale + c); pt = __ldg(in_shift + c); }
  for (int i = lane; i < P; i += 32) {
    const int r = i / W, cc = i - r * W;
    float v = __ldg(src + i);
    if (PRO) v = fmaxf(fmaf(v, ps, pt), 0.f);
    tile[(r + 1) * TW + cc + 1] = v;
  }
  float wr[K][9], br[K];
#pragma unroll
  for (int kk = 0; kk < K; ++kk) {
#pragma unroll
    for (int t = 0; t < 9; ++t) wr[kk][t] = __ldg(w + ((int64_t)c * K + kk) * 9 + t);
    br[kk] = bias ? __ldg(bias + (int64_t)c * K + kk) : 0.f;
  }
  __syncwarp();
  float* dst = y + ((int64_t)b * Cin + c) * K * P;
  for (int i = lane; i < P; i += 32) {
    const int r = i / W, cc = i - r * W;
    const float* t0 = tile + r * TW + cc;   // top-left of the 3x3 window
    float win[9];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) win[dy * 3 + dx] = t0[dy * TW + dx];
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
      float a = br[kk];
#pragma unroll
      for (int t = 0; t < 9; ++t) a = fmaf(wr[kk][t], win[t], a);
      dst[(int64_t)kk * P + i] = a;
    }
  }
}

// 1 = not applicable (caller uses the general kernel), else SMAAT_OK / error code
int dw3x3_small_try(const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1, const float* w, const float* bias,
                    const float* in_scale, const float* in_shift, float* y, int B, int H, int W, int k, cudaStream_t st) {
  if (!(k == 1 || k == 2 || k == 4) || (int64_t)H * W > DWS_MAX_PIXELS || W > 62 || H > 62) return 1;
  const int64_t planes = (int64_t)B * (C0 + C1);
  const int64_t grid = ceil_div64(planes, DWS_WARPS);
  SMAAT_REQUIRE(grid < (1ll << 31), "dw3x3(small): grid too large");
  const size_t smem = (size_t)DWS_WARPS * (H + 2) * (W + 2) * sizeof(float);
  if (smem > 48 * 1024) return 1;
  const bool pro = in_scale != nullptr;
  const unsigned g = (unsigned)grid, thr = 32 * DWS_WARPS;
  if (k == 1) {
    if (pro) dw3x3_small_kernel<1, true><<<g, thr, smem, st>>>(x0, C0, bs0, x1, C1, bs1, w, bias, in_scale, in_shift, y, planes, H, W);
    else dw3x3_small_kernel<1, false><<<g, thr, smem, st>>>(x0, C0, bs0, x1, C1, bs1, w, bias, in_scale, in_shift, y, planes, H, W);
  } else if (k == 2) {
    if (pro) dw3x3_small_kernel<2, true><<<g, thr, smem, st>>>(x0, C0, bs0, x1, C1, bs1, w, bias, in_scale, in_shift, y, planes, H, W);
    else dw3x3_small_kernel<2, false><<<g, thr, smem, st>>>(x0, C0, bs0, x1, C1, bs1, w, bias, in_scale, in_shift, y, planes, H, W);
  } else {
    if (pro) dw3x3_small_kernel<4, true><<<g, thr, smem, st>>>(x0, C0, bs0, x1, C1, bs1, w, bias, in_scale, in_shift, y, planes, H, W);
    else dw3x3_small_kernel<4, false><<<g, thr, smem, st>>>(x0, C0, bs0, x1, C1, bs1, w, bias, in_scale, in_shift, y, planes, H, W);
  }
  SMAAT_LAUNCH_CHECK("smaat_dw3x3_fwd");
  return SMAAT_OK;
}

}  // namespace smaat
