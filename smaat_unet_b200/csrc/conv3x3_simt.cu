// conv3x3_simt.cu -- dense 3x3 conv, padding 1, on the CUDA cores (exact fp32 products), and the C-ABI entry points of the
// dense 3x3 conv family: weight packing, forward (routed to this kernel or to conv3x3_tc.cu) and weight gradient.
//
// Replaces nn.Conv2d(Cin, Cout, 3, padding=1) (+ eval BatchNorm2d + ReLU) of DoubleConv (reference models/unet_parts.py:16-21)
// and its weight gradient in SMAAT_PW_FP32_SIMT mode -- the exact-product anchor of the module tests -- and for shapes the
// tensor-core kernels (conv3x3_tc.cu, conv3x3_wgrad_tc.cu) decline (W % 4 != 0, Cout < 8, unaligned pointers).  Correct
// rather than fast.
//
// Packed weight (both kernels): wp[o][tap][kc], kc = C0p + C1p, Cxp = Cx rounded up to 32; channel c of x0 sits at kc = c,
// channel c of x1 at kc = C0p + c, the padding is zero.  The flip_transpose form packs W'[c][o][2-dy][2-dx] for the input
// gradient (rows = the forward's Cin, one source of Cout channels).
#include "common.cuh"

namespace smaat {

bool conv3x3_tc_eligible(const float* x0, int64_t bs0, const float* x1, int C1, int64_t bs1, const float* wp, const float* wp_lo,
                         int W, int Cout);
int conv3x3_tc_launch(const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1, const float* wp, const float* wp_lo,
                      const float* scale, const float* shift, float* y, int64_t y_bstride, double* stats, int B, int H, int W, int Cout,
                      int relu, int mode, cudaStream_t st);
int conv3x3_wgrad_tc_launch(const float* dz, const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1, float* dW,
                            int B, int H, int W, int Cout, bool x3, cudaStream_t st);

static inline int pad32(int c) { return (c + 31) / 32 * 32; }

// w: (Cout, Cin, 3, 3).  Plain: rows = Cout, sources (C0, C1).  Flipped: rows = Cin = C0 + C1, one source of Cout channels.
__global__ void conv3x3_pack_kernel(const float* __restrict__ w, float* __restrict__ wp, int Cout, int C0, int C1, int flip,
                                    int rows, int c0p, int kc) {
  const int64_t n = (int64_t)rows * 9 * kc;
  const int Cin = C0 + C1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % kc);
    const int tap = (int)((i / kc) % 9);
    const int r = (int)(i / (9 * (int64_t)kc));
    float v = 0.f;
    if (!flip) {
      const int c = k < c0p ? (k < C0 ? k : -1) : (k - c0p < C1 ? C0 + k - c0p : -1);
      if (c >= 0) v = w[((int64_t)r * Cin + c) * 9 + tap];
    } else if (k < Cout) {
      v = w[((int64_t)k * Cin + r) * 9 + (8 - tap)];   // W'[r][k][dy][dx] = W[k][r][2-dy][2-dx]
    }
    wp[i] = v;
  }
}

constexpr int C3S_BM = 64;   // out channels per CTA
constexpr int C3S_BN = 128;  // pixels per CTA
constexpr int C3S_BK = 16;

__global__ void __launch_bounds__(256) conv3x3_simt_kernel(const float* __restrict__ x0, int64_t bs0, const float* __restrict__ x1,
                                                           int64_t bs1, int C0, int C1, int c0p, int kc, const float* __restrict__ wp,
                                                           const float* __restrict__ scale, const float* __restrict__ shift,
                                                           float* __restrict__ y, int64_t y_bstride, double* __restrict__ stats,
                                                           int H, int W, int Cout, int relu) {
  __shared__ __align__(16) float Xs[C3S_BK][C3S_BN];
  __shared__ __align__(16) float Ws[C3S_BK][C3S_BM + 4];
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const int P = H * W;
  const int p0 = blockIdx.x * C3S_BN, o0 = blockIdx.y * C3S_BM, b = blockIdx.z;
  const float* xb0 = x0 + (int64_t)b * bs0;
  const float* xb1 = x1 ? x1 + (int64_t)b * bs1 : nullptr;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int tap = 0; tap < 9; ++tap) {
    const int dy = tap / 3 - 1, dx = tap % 3 - 1;
    for (int k0 = 0; k0 < kc; k0 += C3S_BK) {
      for (int idx = tid; idx < C3S_BK * C3S_BN; idx += 256) {
        const int r = idx / C3S_BN, q = idx % C3S_BN;
        const int k = k0 + r, pp = p0 + q;
        float v = 0.f;
        if (pp < P) {
          const int yy = pp / W + dy, xx = pp % W + dx;
          if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
            if (k < c0p) {
              if (k < C0) v = __ldg(xb0 + (int64_t)k * P + yy * W + xx);
            } else if (k - c0p < C1) {
              v = __ldg(xb1 + (int64_t)(k - c0p) * P + yy * W + xx);
            }
          }
        }
        Xs[r][q] = v;
      }
      for (int idx = tid; idx < C3S_BK * C3S_BM; idx += 256) {
        const int o = idx / C3S_BK, r = idx % C3S_BK;
        Ws[r][o] = (o0 + o < Cout) ? __ldg(wp + ((int64_t)(o0 + o) * 9 + tap) * kc + k0 + r) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < C3S_BK; ++kk) {
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
  }

  const int pp = p0 + tx * 4;
  float* yb = y + (int64_t)b * y_bstride;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int oo = o0 + ty * 8 + i;  // warp-uniform
    if (oo >= Cout) break;
    const float s = scale ? __ldg(scale + oo) : 1.f;
    const float t = shift ? __ldg(shift + oo) : 0.f;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float pre = fmaf(acc[i][j], s, t);
      if (pp + j < P) {
        s1 += pre;
        s2 = fmaf(pre, pre, s2);
        yb[(int64_t)oo * P + pp + j] = relu ? fmaxf(pre, 0.f) : pre;
      }
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

// dW[o][c][tap] += sum_{b,p} dz[b,o,p] * in[b,c,p + shift(tap)].  CTA: 32 output x 32 input channels, all 9 taps; it walks
// 32-pixel row segments (b, row, segment) with a grid stride and merges into dW with one fp32 atomic per weight at the end.
constexpr int C3W_T = 32;
constexpr int C3W_SEG = 32;

__global__ void __launch_bounds__(256) conv3x3_wgrad_simt_kernel(const float* __restrict__ dz, const float* __restrict__ x0, int64_t bs0,
                                                                 const float* __restrict__ x1, int64_t bs1, int C0, int C1,
                                                                 float* __restrict__ dW, int B, int H, int W, int Cout) {
  __shared__ float Ds[C3W_T][C3W_SEG + 1];
  __shared__ float Xs[C3W_T][3][C3W_SEG + 3];
  const int tid = threadIdx.x;
  const int c = tid & 31, og = tid >> 5;   // thread: input channel c0 + c, output channels o0 + 4 og .. + 3
  const int c0 = blockIdx.x * C3W_T, o0 = blockIdx.y * C3W_T;
  const int Cin = C0 + C1, P = H * W;
  const int nseg = (W + C3W_SEG - 1) / C3W_SEG;
  const int64_t nchunk = (int64_t)B * H * nseg;
  float acc[4][9];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 9; ++j) acc[i][j] = 0.f;

  for (int64_t ch = blockIdx.z; ch < nchunk; ch += gridDim.z) {
    const int seg = (int)(ch % nseg);
    const int row = (int)((ch / nseg) % H);
    const int b = (int)(ch / ((int64_t)nseg * H));
    const int xs = seg * C3W_SEG;
    for (int idx = tid; idx < C3W_T * C3W_SEG; idx += 256) {
      const int o = idx / C3W_SEG, q = idx % C3W_SEG;
      const int oo = o0 + o, xx = xs + q;
      Ds[o][q] = (oo < Cout && xx < W) ? __ldg(dz + ((int64_t)b * Cout + oo) * P + row * W + xx) : 0.f;
    }
    for (int idx = tid; idx < C3W_T * 3 * (C3W_SEG + 2); idx += 256) {
      const int cc = idx / (3 * (C3W_SEG + 2)), r = (idx / (C3W_SEG + 2)) % 3, q = idx % (C3W_SEG + 2);
      const int ci = c0 + cc, yy = row + r - 1, xx = xs + q - 1;
      float v = 0.f;
      if (ci < Cin && yy >= 0 && yy < H && xx >= 0 && xx < W) {
        v = ci < C0 ? __ldg(x0 + (int64_t)b * bs0 + (int64_t)ci * P + yy * W + xx)
                    : __ldg(x1 + (int64_t)b * bs1 + (int64_t)(ci - C0) * P + yy * W + xx);
      }
      Xs[cc][r][q] = v;
    }
    __syncthreads();
    for (int q = 0; q < C3W_SEG; ++q) {
      float xv[9];
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) xv[tap] = Xs[c][tap / 3][q + tap % 3];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float d = Ds[4 * og + i][q];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) acc[i][tap] = fmaf(d, xv[tap], acc[i][tap]);
      }
    }
    __syncthreads();
  }
  const int ci = c0 + c;
  if (ci >= Cin) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int oo = o0 + 4 * og + i;
    if (oo >= Cout) continue;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) atomicAdd(dW + ((int64_t)oo * Cin + ci) * 9 + tap, acc[i][tap]);
  }
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_conv3x3_pack_weight(const float* w, float* wp, int Cout, int C0, int C1, int flip_transpose, void* stream) {
  SMAAT_REQUIRE(w && wp, "conv3x3_pack_weight: null pointer");
  SMAAT_REQUIRE(Cout > 0 && C0 > 0 && C1 >= 0, "conv3x3_pack_weight: bad shape Cout=%d C0=%d C1=%d", Cout, C0, C1);
  const int rows = flip_transpose ? C0 + C1 : Cout;
  const int c0p = flip_transpose ? pad32(Cout) : pad32(C0);
  const int kc = flip_transpose ? c0p : c0p + pad32(C1);
  const int64_t n = (int64_t)rows * 9 * kc;
  const int grid = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  conv3x3_pack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, wp, Cout, C0, C1, flip_transpose, rows, c0p, kc);
  SMAAT_LAUNCH_CHECK("smaat_conv3x3_pack_weight");
  return SMAAT_OK;
}

extern "C" int smaat_conv3x3_tc_eligible(const float* x0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                         const float* wp, int W, int Cout) {
  return conv3x3_tc_eligible(x0, x0_bstride, x1, C1, x1_bstride, wp, nullptr, W, Cout) ? 1 : 0;
}

extern "C" int smaat_conv3x3_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                 const float* wp, const float* wp_lo, const float* scale, const float* shift, float* y,
                                 int64_t y_bstride, double* stats, int B, int H, int W, int Cout, int relu, int mode, void* stream) {
  SMAAT_REQUIRE(x0 && wp && y, "conv3x3: null pointer");
  SMAAT_REQUIRE(B > 0 && C0 > 0 && C1 >= 0 && H > 0 && W > 0 && Cout > 0, "conv3x3: bad shape B=%d C0=%d C1=%d H=%d W=%d Cout=%d", B, C0,
                C1, H, W, Cout);
  SMAAT_REQUIRE(C1 == 0 || x1, "conv3x3: C1=%d but x1 is null", C1);
  SMAAT_REQUIRE(x0_bstride >= (int64_t)C0 * H * W && (C1 == 0 || x1_bstride >= (int64_t)C1 * H * W), "conv3x3: input batch stride too small");
  SMAAT_REQUIRE(y_bstride >= (int64_t)Cout * H * W, "conv3x3: y batch stride %lld < Cout*H*W", (long long)y_bstride);
  cudaStream_t st = (cudaStream_t)stream;
  switch (mode) {
    case SMAAT_PW_FP32_SIMT: {
      dim3 grid(ceil_div(H * W, C3S_BN), ceil_div(Cout, C3S_BM), B);
      SMAAT_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "conv3x3(simt): grid too large");
      const int c0p = pad32(C0);
      conv3x3_simt_kernel<<<grid, 256, 0, st>>>(x0, x0_bstride, C1 ? x1 : nullptr, x1_bstride, C0, C1, c0p, c0p + pad32(C1), wp, scale,
                                                shift, y, y_bstride, stats, H, W, Cout, relu);
      SMAAT_LAUNCH_CHECK("smaat_conv3x3_fwd(simt)");
      return SMAAT_OK;
    }
    case SMAAT_PW_TF32:
    case SMAAT_PW_BF16:
      return conv3x3_tc_launch(x0, C0, x0_bstride, x1, C1, x1_bstride, wp, nullptr, scale, shift, y, y_bstride, stats, B, H, W, Cout, relu,
                               mode, st);
    case SMAAT_PW_TF32X3:
      return conv3x3_tc_launch(x0, C0, x0_bstride, x1, C1, x1_bstride, wp, wp_lo, scale, shift, y, y_bstride, stats, B, H, W, Cout, relu,
                               mode, st);
    default:
      return fail(SMAAT_E_BADARG, "conv3x3: unknown mode %d", mode);
  }
}

extern "C" int smaat_conv3x3_bwd_weight(const float* dz, const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1,
                                        int64_t x1_bstride, float* dW, int B, int H, int W, int Cout, int mode, void* stream) {
  SMAAT_REQUIRE(dz && x0 && dW, "conv3x3_bwd_weight: null pointer");
  SMAAT_REQUIRE(B > 0 && C0 > 0 && C1 >= 0 && H > 0 && W > 0 && Cout > 0, "conv3x3_bwd_weight: bad shape");
  SMAAT_REQUIRE(C1 == 0 || x1, "conv3x3_bwd_weight: C1=%d but x1 is null", C1);
  SMAAT_REQUIRE(mode >= SMAAT_PW_FP32_SIMT && mode <= SMAAT_PW_TF32X3, "conv3x3_bwd_weight: unknown mode %d", mode);
  if (mode != SMAAT_PW_FP32_SIMT)
    return conv3x3_wgrad_tc_launch(dz, x0, C0, x0_bstride, C1 ? x1 : nullptr, C1, x1_bstride, dW, B, H, W, Cout,
                                   mode == SMAAT_PW_TF32X3, (cudaStream_t)stream);
  const int gx = ceil_div(C0 + C1, C3W_T), gy = ceil_div(Cout, C3W_T);
  const int64_t nchunk = (int64_t)B * H * ceil_div(W, C3W_SEG);
  // enough CTAs to fill the GPU twice over, each walking many row segments (fewer atomics per weight)
  int64_t gz = (2 * (int64_t)num_sms() + gx * gy - 1) / ((int64_t)gx * gy);
  if (gz < 1) gz = 1;
  if (gz > nchunk) gz = nchunk;
  if (gz > 65535) gz = 65535;
  SMAAT_REQUIRE(gy <= 65535, "conv3x3_bwd_weight: grid too large");
  conv3x3_wgrad_simt_kernel<<<dim3(gx, gy, (unsigned)gz), 256, 0, (cudaStream_t)stream>>>(dz, x0, x0_bstride, C1 ? x1 : nullptr,
                                                                                          x1_bstride, C0, C1, dW, B, H, W, Cout);
  SMAAT_LAUNCH_CHECK("smaat_conv3x3_bwd_weight(simt)");
  return SMAAT_OK;
}
