// glue.cu -- the memory-bound glue between the DS-conv blocks: BN folding, MaxPool2d(2),
// OutConv, tf32 weight split, bf16 weight pack (bilinear x2 + pad lives in upsample.cu).  All are streaming kernels
// (no reuse beyond what L1/L2 give for free); coalesced 128-bit accesses where alignment allows.
#include "common.cuh"

namespace smaat {

// ---- eval BatchNorm -> (scale, shift) -------------------------------------------------------
__global__ void bn_fold_kernel(const float* __restrict__ g, const float* __restrict__ bta, const float* __restrict__ rm,
                               const float* __restrict__ rv, const float* __restrict__ cb, float eps,
                               float* __restrict__ scale, float* __restrict__ shift, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  // 1/sqrt via IEEE sqrt + division: matches torch's (x - mean) / sqrt(var + eps) * gamma to ~1 ulp
  const float s = g[c] / sqrtf(rv[c] + eps);
  scale[c] = s;
  shift[c] = fmaf((cb ? cb[c] : 0.f) - rm[c], s, bta[c]);
}

// ---- tf32 split ---------------------------------------------------------------------------------
__global__ void split_tf32_kernel(const float* __restrict__ src, float* __restrict__ hi, float* __restrict__ lo, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = src[i];
  const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
  hi[i] = h;
  lo[i] = v - h;
}

// ---- bf16 weight pack (SMAAT_PW_BF16) --------------------------------------------------------------
// out[r][c] = bf16_rn(w[r][src]), src = the physical k of logical k c in its group of 16 (tc_common.cuh bf16_frag), zero past
// cols.  One thread per output pair: one bf16x2 store
__global__ void pack_bf16_kernel(const float* __restrict__ w, uint32_t* __restrict__ out, int rows, int cols, int cols_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // pair index
  const int half = cols_out >> 1;
  if (i >= (int64_t)rows * half) return;
  const int r = (int)(i / half), c = 2 * (int)(i - (int64_t)r * half);
  float v[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int l = (c + e) & 15;
    const int src = ((c + e) & ~15) | (l & 8) | ((l & 1) << 2) | ((l >> 1) & 3);
    v[e] = src < cols ? w[(int64_t)r * cols + src] : 0.f;
  }
  uint32_t p;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p) : "f"(v[1]), "f"(v[0]));
  out[i] = p;
}

// ---- MaxPool2d(2) ---------------------------------------------------------------------------------
// One thread -> two horizontally adjacent outputs (float4 row loads, float2 store) when W % 4 == 0.
template <bool VEC>
__global__ void __launch_bounds__(256) maxpool2_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t N, int H,
                                                       int W, int Ho, int Wo) {
  const int wq = VEC ? (Wo >> 1) : Wo;  // work items per output row
  const int64_t total = N * (int64_t)Ho * wq;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % wq);
    const int64_t t = i / wq;
    const int oy = (int)(t % Ho);
    const int64_t n = t / Ho;
    const float* r0 = x + (n * H + 2 * oy) * (int64_t)W;
    if (VEC) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(r0 + 4 * q));
      const float4 b = __ldg(reinterpret_cast<const float4*>(r0 + W + 4 * q));
      float2 o;
      o.x = fmaxf(fmaxf(a.x, a.y), fmaxf(b.x, b.y));
      o.y = fmaxf(fmaxf(a.z, a.w), fmaxf(b.z, b.w));
      *reinterpret_cast<float2*>(y + (n * Ho + oy) * (int64_t)Wo + 2 * q) = o;
    } else {
      const float* s = r0 + 2 * q;
      y[(n * Ho + oy) * (int64_t)Wo + q] = fmaxf(fmaxf(__ldg(s), __ldg(s + 1)), fmaxf(__ldg(s + W), __ldg(s + W + 1)));
    }
  }
}

// ---- OutConv: 1x1, Cin -> ncls (small) -------------------------------------------------------------
// HBM-bound on the Cin-channel read (SURVEY 8a row a12: 680 MB -> 10.6 MB).  One thread owns 4
// consecutive pixels and NC classes; loops over Cin with coalesced float4 loads; weights in smem.
// TA: the storage type of x and y (float, or uint16_t bf16 in the serving forward's bf16 route: fp32 accumulation, each logit
// rounded once)
template <int NC, bool VEC, typename TA = float>
__global__ void __launch_bounds__(256) outconv_kernel(const TA* __restrict__ x, const float* __restrict__ w,
                                                      const float* __restrict__ bias, TA* __restrict__ y, int Cin, int ncls,
                                                      int P) {
  extern __shared__ float wsm[];  // [NC][Cin]
  const int cls0 = blockIdx.y * NC;
  const int b = blockIdx.z;
  for (int i = threadIdx.x; i < NC * Cin; i += blockDim.x) {
    const int j = i / Cin, c = i - j * Cin;
    wsm[i] = (cls0 + j < ncls) ? __ldg(w + (int64_t)(cls0 + j) * Cin + c) : 0.f;
  }
  __syncthreads();
  const int pp = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (pp >= P) return;
  float acc[NC][4];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const float bj = (bias && cls0 + j < ncls) ? __ldg(bias + cls0 + j) : 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[j][q] = bj;
  }
  const TA* xb = x + (int64_t)b * Cin * P + pp;
#pragma unroll 4
  for (int c = 0; c < Cin; ++c) {
    float4 v;
    if (VEC) {
      v = ld_act4(xb + (int64_t)c * P);
    } else {
      const TA* s = xb + (int64_t)c * P;
      v.x = ld_act(s);
      v.y = (pp + 1 < P) ? ld_act(s + 1) : 0.f;
      v.z = (pp + 2 < P) ? ld_act(s + 2) : 0.f;
      v.w = (pp + 3 < P) ? ld_act(s + 3) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      const float wj = wsm[j * Cin + c];
      acc[j][0] = fmaf(wj, v.x, acc[j][0]);
      acc[j][1] = fmaf(wj, v.y, acc[j][1]);
      acc[j][2] = fmaf(wj, v.z, acc[j][2]);
      acc[j][3] = fmaf(wj, v.w, acc[j][3]);
    }
  }
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    if (cls0 + j >= ncls) break;
    TA* dst = y + ((int64_t)b * ncls + cls0 + j) * P + pp;
    if (VEC) {
      st_act4(dst, make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]));
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (pp + q < P) st_act(dst + q, acc[j][q]);
    }
  }
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_bn_fold(const float* gamma, const float* beta, const float* rm, const float* rv, const float* conv_bias,
                             float eps, float* scale, float* shift, int C, void* stream) {
  SMAAT_REQUIRE(gamma && beta && rm && rv && scale && shift && C > 0, "bn_fold: bad arguments");
  bn_fold_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(gamma, beta, rm, rv, conv_bias, eps, scale, shift, C);
  SMAAT_LAUNCH_CHECK("smaat_bn_fold");
  return SMAAT_OK;
}

extern "C" int smaat_split_tf32(const float* src, float* hi, float* lo, int64_t n, void* stream) {
  SMAAT_REQUIRE(src && hi && lo && n > 0, "split_tf32: bad arguments");
  split_tf32_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(src, hi, lo, n);
  SMAAT_LAUNCH_CHECK("smaat_split_tf32");
  return SMAAT_OK;
}

extern "C" int smaat_pack_bf16(const float* w, uint16_t* out, int rows, int cols, int cols_out, void* stream) {
  SMAAT_REQUIRE(w && out && rows > 0 && cols > 0, "pack_bf16: bad arguments rows=%d cols=%d", rows, cols);
  SMAAT_REQUIRE(cols_out == (cols + 31) / 32 * 32, "pack_bf16: cols_out=%d must be cols=%d rounded up to 32", cols_out, cols);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3u) == 0, "pack_bf16: out must be 4-byte aligned");
  const int64_t pairs = (int64_t)rows * (cols_out / 2);
  pack_bf16_kernel<<<(unsigned)ceil_div64(pairs, 256), 256, 0, (cudaStream_t)stream>>>(w, reinterpret_cast<uint32_t*>(out), rows, cols,
                                                                                        cols_out);
  SMAAT_LAUNCH_CHECK("smaat_pack_bf16");
  return SMAAT_OK;
}

extern "C" int smaat_maxpool2_fwd(const float* x, float* y, int64_t N, int H, int W, void* stream) {
  SMAAT_REQUIRE(x && y && N > 0 && H >= 2 && W >= 2, "maxpool2: bad arguments N=%lld H=%d W=%d", (long long)N, H, W);
  const int Ho = H / 2, Wo = W / 2;
  const bool vec = (W % 4 == 0) && aligned16(x) && ((reinterpret_cast<uintptr_t>(y) & 7u) == 0);
  const int64_t items = N * (int64_t)Ho * (vec ? Wo / 2 : Wo);
  const int64_t blocks = ceil_div64(items, 256);
  const unsigned grid = (unsigned)(blocks < (int64_t)num_sms() * 64 ? blocks : (int64_t)num_sms() * 64);
  if (vec)
    maxpool2_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, N, H, W, Ho, Wo);
  else
    maxpool2_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, N, H, W, Ho, Wo);
  SMAAT_LAUNCH_CHECK("smaat_maxpool2_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_outconv_fwd(const float* x, const float* w, const float* bias, float* y, int B, int Cin, int ncls, int P,
                                 void* stream) {
  SMAAT_REQUIRE(x && w && y && B > 0 && Cin > 0 && ncls > 0 && P > 0, "outconv: bad arguments");
  SMAAT_REQUIRE(B <= 65535, "outconv: batch too large for grid.z");
  const bool vec = (P % 4 == 0) && aligned16(x) && aligned16(y);
  cudaStream_t st = (cudaStream_t)stream;
  const int threads = 128;
  const unsigned gx = (unsigned)ceil_div(ceil_div(P, 4), threads);
  if (ncls <= 2) {
    constexpr int NC = 2;
    dim3 grid(gx, ceil_div(ncls, NC), B);
    const size_t smem = (size_t)NC * Cin * sizeof(float);
    if (vec) outconv_kernel<NC, true><<<grid, threads, smem, st>>>(x, w, bias, y, Cin, ncls, P);
    else outconv_kernel<NC, false><<<grid, threads, smem, st>>>(x, w, bias, y, Cin, ncls, P);
  } else {
    constexpr int NC = 8;
    dim3 grid(gx, ceil_div(ncls, NC), B);
    const size_t smem = (size_t)NC * Cin * sizeof(float);
    SMAAT_REQUIRE(smem <= 48 * 1024, "outconv: Cin=%d too large", Cin);
    if (vec) outconv_kernel<NC, true><<<grid, threads, smem, st>>>(x, w, bias, y, Cin, ncls, P);
    else outconv_kernel<NC, false><<<grid, threads, smem, st>>>(x, w, bias, y, Cin, ncls, P);
  }
  SMAAT_LAUNCH_CHECK("smaat_outconv_fwd");
  return SMAAT_OK;
}

/* smaat_outconv_fwd from bf16 activations to bf16 logits (the serving forward's bf16 route): the same fp32 accumulation, each
 * logit rounded to bf16 once. */
extern "C" int smaat_outconv_bf16_fwd(const void* x, const float* w, const float* bias, void* y, int B, int Cin, int ncls, int P,
                                      void* stream) {
  SMAAT_REQUIRE(x && w && y && B > 0 && Cin > 0 && ncls > 0 && P > 0, "outconv_bf16: bad arguments");
  SMAAT_REQUIRE(B <= 65535, "outconv_bf16: batch too large for grid.z");
  SMAAT_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 1u) == 0, "outconv_bf16: x and y must be 2-byte aligned");
  const uint16_t* xb = static_cast<const uint16_t*>(x);
  uint16_t* yb = static_cast<uint16_t*>(y);
  const bool vec = (P % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 7u) == 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int threads = 128;
  const unsigned gx = (unsigned)ceil_div(ceil_div(P, 4), threads);
  if (ncls <= 2) {
    constexpr int NC = 2;
    dim3 grid(gx, ceil_div(ncls, NC), B);
    const size_t smem = (size_t)NC * Cin * sizeof(float);
    if (vec) outconv_kernel<NC, true, uint16_t><<<grid, threads, smem, st>>>(xb, w, bias, yb, Cin, ncls, P);
    else outconv_kernel<NC, false, uint16_t><<<grid, threads, smem, st>>>(xb, w, bias, yb, Cin, ncls, P);
  } else {
    constexpr int NC = 8;
    dim3 grid(gx, ceil_div(ncls, NC), B);
    const size_t smem = (size_t)NC * Cin * sizeof(float);
    SMAAT_REQUIRE(smem <= 48 * 1024, "outconv_bf16: Cin=%d too large", Cin);
    if (vec) outconv_kernel<NC, true, uint16_t><<<grid, threads, smem, st>>>(xb, w, bias, yb, Cin, ncls, P);
    else outconv_kernel<NC, false, uint16_t><<<grid, threads, smem, st>>>(xb, w, bias, yb, Cin, ncls, P);
  }
  SMAAT_LAUNCH_CHECK("smaat_outconv_bf16_fwd");
  return SMAAT_OK;
}
