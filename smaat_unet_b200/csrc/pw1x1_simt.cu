// pw1x1_simt.cu -- pointwise 1x1 conv as an exact-fp32 CUDA-core GEMM with the fused
// per-channel affine (+ReLU) epilogue and optional BatchNorm statistics.
//
// Replaces DepthwiseSeparableConv.pointwise + eval BatchNorm2d + ReLU
// (reference models/layers.py:45,49; parts_ds.py:25-26,34-35) in SMAAT_PW_FP32_SIMT mode.
// This is the exact-product path: the strict-tolerance parity anchor on the GPU, and the
// kernel for shapes the tensor-core path does not take (P % 4 != 0, K % 4 != 0).  The fast path
// is pw1x1_tc.cu.  Per image: Y[Cout x P] = W[Cout x K] * X[K x P].
#include "common.cuh"

namespace smaat {

constexpr int PW_BM = 64;   // out channels per CTA
constexpr int PW_BN = 128;  // pixels per CTA
constexpr int PW_BK = 16;

template <bool VECX, bool VECW>
__global__ void __launch_bounds__(256) pw1x1_simt_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                                         float* __restrict__ y, int64_t y_bstride, double* __restrict__ stats,
                                                         int K, int Cout, int P, int relu) {
  __shared__ __align__(16) float Xs[PW_BK][PW_BN];
  __shared__ __align__(16) float Ws[PW_BK][PW_BM + 4];

  const int tid = threadIdx.x;
  const int tx = tid & 31;  // pixel quad
  const int ty = tid >> 5;  // out-channel octet (warp index)
  const int p0 = blockIdx.x * PW_BN;
  const int o0 = blockIdx.y * PW_BM;
  const int b = blockIdx.z;
  const float* xb = x + (int64_t)b * K * P;

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += PW_BK) {
    // X tile: PW_BK rows x 128 px
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int idx = tid + it * 256;  // 0..511 float4 slots
      const int r = idx >> 5, q = idx & 31;
      const int kk = k0 + r, pp = p0 + q * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kk < K) {
        const float* src = xb + (int64_t)kk * P + pp;
        if (VECX && pp + 3 < P) {
          v = __ldg(reinterpret_cast<const float4*>(src));
        } else {
          if (pp < P) v.x = __ldg(src);
          if (pp + 1 < P) v.y = __ldg(src + 1);
          if (pp + 2 < P) v.z = __ldg(src + 2);
          if (pp + 3 < P) v.w = __ldg(src + 3);
        }
      }
      *reinterpret_cast<float4*>(&Xs[r][q * 4]) = v;
    }
    // W tile: 64 out-channels x 16 k, stored k-major
    {
      const int o = tid >> 2, kq = tid & 3;
      const int oo = o0 + o, kk = k0 + kq * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (oo < Cout) {
        const float* src = w + (int64_t)oo * K + kk;
        if (VECW && kk + 3 < K) {
          v = __ldg(reinterpret_cast<const float4*>(src));
        } else {
          if (kk < K) v.x = __ldg(src);
          if (kk + 1 < K) v.y = __ldg(src + 1);
          if (kk + 2 < K) v.z = __ldg(src + 2);
          if (kk + 3 < K) v.w = __ldg(src + 3);
        }
      }
      Ws[kq * 4 + 0][o] = v.x;
      Ws[kq * 4 + 1][o] = v.y;
      Ws[kq * 4 + 2][o] = v.z;
      Ws[kq * 4 + 3][o] = v.w;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < PW_BK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&Ws[kk][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&Ws[kk][ty * 8 + 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Xs[kk][tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }

  const int pp = p0 + tx * 4;
  float* yb = y + (int64_t)b * y_bstride;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int oo = o0 + ty * 8 + i;  // warp-uniform
    if (oo >= Cout) break;
    const float s = scale ? __ldg(scale + oo) : 1.f;
    const float t = shift ? __ldg(shift + oo) : 0.f;
    float v[4];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float pre = fmaf(acc[i][j], s, t);
      if (pp + j < P) {
        s1 += pre;
        s2 = fmaf(pre, pre, s2);
      }
      v[j] = relu ? fmaxf(pre, 0.f) : pre;
    }
    float* dst = yb + (int64_t)oo * P + pp;
    if (VECX && pp + 3 < P && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
      *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (pp + j < P) dst[j] = v[j];
    }
    if (stats) {
      s1 = warp_sum(s1);
      s2 = warp_sum(s2);
      if (tx == 0) {
        atomicAdd(stats + oo, (double)s1);
        atomicAdd(stats + Cout + oo, (double)s2);
      }
    }
  }
}

int pw1x1_simt_launch(const float* x, const float* w, const float* scale, const float* shift, float* y, int64_t y_bstride,
                      double* stats, int B, int K, int Cout, int P, int relu, cudaStream_t st) {
  dim3 grid(ceil_div(P, PW_BN), ceil_div(Cout, PW_BM), B);
  SMAAT_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "pw1x1(simt): grid too large");
  const bool vx = (P % 4 == 0) && aligned16(x);
  const bool vw = (K % 4 == 0) && aligned16(w);
  if (vx && vw)
    pw1x1_simt_kernel<true, true><<<grid, 256, 0, st>>>(x, w, scale, shift, y, y_bstride, stats, K, Cout, P, relu);
  else if (vx)
    pw1x1_simt_kernel<true, false><<<grid, 256, 0, st>>>(x, w, scale, shift, y, y_bstride, stats, K, Cout, P, relu);
  else if (vw)
    pw1x1_simt_kernel<false, true><<<grid, 256, 0, st>>>(x, w, scale, shift, y, y_bstride, stats, K, Cout, P, relu);
  else
    pw1x1_simt_kernel<false, false><<<grid, 256, 0, st>>>(x, w, scale, shift, y, y_bstride, stats, K, Cout, P, relu);
  SMAAT_LAUNCH_CHECK("smaat_pw1x1_fwd(simt)");
  return SMAAT_OK;
}

}  // namespace smaat
