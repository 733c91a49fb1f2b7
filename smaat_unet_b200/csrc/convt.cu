// convt.cu -- UpDS(bilinear=False): nn.ConvTranspose2d(in, in // 2, kernel_size=2, stride=2) + F.pad to the skip size
// (reference models/unet_parts_depthwise_separable.py:72-73, 76-81).
//
// With kernel = stride = 2 the transposed convolution has no overlapping taps: output pixel (2i + dy, 2j + dx) of channel o is
//   bias[o] + sum_c x[c, i, j] * W[c, o, dy, dx]
// i.e. ONE pointwise GEMM from Cin to 4 * Cout "packed" channels (dy, dx, o) -- run by the wgmma pointwise kernel
// (pw1x1_tc.cu) on a repacked weight -- followed by a 2x2 pixel shuffle.  This file holds the three data-movement kernels
// around that GEMM: weight repack, pixel shuffle (+ bias + pad), and their transposes for the backward pass.
#include "common.cuh"

namespace smaat {

// W (Cin, Cout, 2, 2) -> Wp (4 Cout, Cin), row (2 dy + dx) Cout + o.  UNPACK: the transpose, ACCUMULATING into W's layout
// (weight gradient) and folding the packed bias gradient (4 Cout) into db (Cout).
template <bool UNPACK>
__global__ void convt2x2_repack_kernel(const float* __restrict__ src, float* __restrict__ dst, const float* __restrict__ dbp,
                                       float* __restrict__ db, int Cin, int Cout) {
  const int64_t n = (int64_t)Cin * Cout * 4;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    // i indexes W's layout: ((c * Cout + o) * 2 + dy) * 2 + dx
    const int t = (int)(i & 3);
    const int64_t co = i >> 2;
    const int o = (int)(co % Cout), c = (int)(co / Cout);
    const int64_t ip = ((int64_t)t * Cout + o) * Cin + c;
    if (UNPACK) dst[i] += src[ip];
    else dst[ip] = src[i];
  }
  if (UNPACK && db && i < Cout) db[i] += (dbp[i] + dbp[Cout + i]) + (dbp[2 * Cout + i] + dbp[3 * Cout + i]);
}

// t (B, 4 Cout, H, W) -> y (B, Cout, Ho, Wo): y[b, o, 2i + dy + pad_t, 2j + dx + pad_l] = t[b, (2 dy + dx) Cout + o, i, j] + bias[o];
// the pad frame is written as zeros.  One thread = one output row pair-of-columns (float2 store, two coalesced plane reads).
__global__ void __launch_bounds__(256) pixel_shuffle2_pad_kernel(const float* __restrict__ t, const float* __restrict__ bias,
                                                                 float* __restrict__ y, int64_t y_bstride, int B, int Cout, int H, int W,
                                                                 int Ho, int Wo, int pad_t, int pad_l) {
  const int64_t P = (int64_t)H * W;
  const int wq = (Wo + 1) >> 1;
  const int64_t total = (int64_t)B * Cout * Ho * wq;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int q = (int)(idx % wq);
    int64_t r = idx / wq;
    const int oy = (int)(r % Ho);
    r /= Ho;
    const int o = (int)(r % Cout), b = (int)(r / Cout);
    const int uy = oy - pad_t;
    float v[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int ux = 2 * q + e - pad_l;
      if (uy >= 0 && uy < 2 * H && ux >= 0 && ux < 2 * W) {
        const int tap = ((uy & 1) << 1) | (ux & 1);
        v[e] = __ldg(t + ((int64_t)b * 4 * Cout + (int64_t)tap * Cout + o) * P + (int64_t)(uy >> 1) * W + (ux >> 1)) + (bias ? __ldg(bias + o) : 0.f);
      }
    }
    float* d = y + (int64_t)b * y_bstride + ((int64_t)o * Ho + oy) * Wo + 2 * q;
    d[0] = v[0];
    if (2 * q + 1 < Wo) d[1] = v[1];
  }
}

// backward of the shuffle: dt[b, (2 dy + dx) Cout + o, i, j] = g[b, o, 2i + dy + pad_t, 2j + dx + pad_l]
__global__ void __launch_bounds__(256) pixel_shuffle2_pad_bwd_kernel(const float* __restrict__ g, int64_t g_bstride, float* __restrict__ dt,
                                                                     int B, int Cout, int H, int W, int Ho, int Wo, int pad_t, int pad_l) {
  const int64_t P = (int64_t)H * W;
  const int64_t total = (int64_t)B * 4 * Cout * P;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % W);
    int64_t r = idx / W;
    const int i = (int)(r % H);
    r /= H;
    const int pc = (int)(r % (4 * Cout)), b = (int)(r / (4 * Cout));
    const int tap = pc / Cout, o = pc - tap * Cout;
    const int oy = 2 * i + (tap >> 1) + pad_t, ox = 2 * j + (tap & 1) + pad_l;
    dt[idx] = __ldg(g + (int64_t)b * g_bstride + ((int64_t)o * Ho + oy) * Wo + ox);
  }
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_convt2x2_pack_weight(const float* w, float* wp, int Cin, int Cout, void* stream) {
  SMAAT_REQUIRE(w && wp && Cin > 0 && Cout > 0, "convt2x2_pack_weight: bad arguments");
  const int64_t n = (int64_t)Cin * Cout * 4;
  convt2x2_repack_kernel<false><<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(w, wp, nullptr, nullptr, Cin, Cout);
  SMAAT_LAUNCH_CHECK("smaat_convt2x2_pack_weight");
  return SMAAT_OK;
}

extern "C" int smaat_convt2x2_unpack_wgrad(const float* dwp, const float* dbp, float* dw, float* db, int Cin, int Cout, void* stream) {
  SMAAT_REQUIRE(dwp && dw && Cin > 0 && Cout > 0 && (!db || dbp), "convt2x2_unpack_wgrad: bad arguments");
  const int64_t n = (int64_t)Cin * Cout * 4;
  convt2x2_repack_kernel<true><<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(dwp, dw, dbp, db, Cin, Cout);
  SMAAT_LAUNCH_CHECK("smaat_convt2x2_unpack_wgrad");
  return SMAAT_OK;
}

extern "C" int smaat_pixel_shuffle2_pad_fwd(const float* t, const float* bias, float* y, int64_t y_bstride, int B, int Cout, int H, int W,
                                            int Ho, int Wo, void* stream) {
  SMAAT_REQUIRE(t && y && B > 0 && Cout > 0 && H > 0 && W > 0, "pixel_shuffle2_pad: bad arguments");
  SMAAT_REQUIRE(Ho >= 2 * H && Wo >= 2 * W, "pixel_shuffle2_pad: target %dx%d smaller than 2x source %dx%d (crop unsupported)", Ho, Wo, H, W);
  SMAAT_REQUIRE(y_bstride >= (int64_t)Cout * Ho * Wo, "pixel_shuffle2_pad: y batch stride too small");
  const int pad_t = (Ho - 2 * H) / 2, pad_l = (Wo - 2 * W) / 2;       // F.pad(x1, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])
  const int64_t total = (int64_t)B * Cout * Ho * ((Wo + 1) / 2);
  const int64_t blocks = ceil_div64(total, 256);
  pixel_shuffle2_pad_kernel<<<(unsigned)(blocks < (int64_t)num_sms() * 32 ? blocks : (int64_t)num_sms() * 32), 256, 0, (cudaStream_t)stream>>>(
      t, bias, y, y_bstride, B, Cout, H, W, Ho, Wo, pad_t, pad_l);
  SMAAT_LAUNCH_CHECK("smaat_pixel_shuffle2_pad_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_pixel_shuffle2_pad_bwd(const float* g, int64_t g_bstride, float* dt, int B, int Cout, int H, int W, int Ho, int Wo,
                                            void* stream) {
  SMAAT_REQUIRE(g && dt && B > 0 && Cout > 0 && H > 0 && W > 0 && Ho >= 2 * H && Wo >= 2 * W, "pixel_shuffle2_pad_bwd: bad arguments");
  const int pad_t = (Ho - 2 * H) / 2, pad_l = (Wo - 2 * W) / 2;
  const int64_t total = (int64_t)B * 4 * Cout * H * W;
  const int64_t blocks = ceil_div64(total, 256);
  pixel_shuffle2_pad_bwd_kernel<<<(unsigned)(blocks < (int64_t)num_sms() * 32 ? blocks : (int64_t)num_sms() * 32), 256, 0, (cudaStream_t)stream>>>(
      g, g_bstride, dt, B, Cout, H, W, Ho, Wo, pad_t, pad_l);
  SMAAT_LAUNCH_CHECK("smaat_pixel_shuffle2_pad_bwd");
  return SMAAT_OK;
}
