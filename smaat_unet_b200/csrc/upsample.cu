// upsample.cu -- nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True) + F.pad to the skip size
// (reference models/unet_parts_depthwise_separable.py:64,78-81), forward.
//
// Write-bound (output 4x the input): algorithmic bytes = 4*B*C*(H*W + Ho*Wo).  One CTA produces a 48 x 72 output tile
// of one plane, separably, through shared memory:
//   * the per-column / per-row source index and the two lerp weights are computed ONCE per CTA into small tables
//     (pad rows/columns get weights 0), so the per-pixel work has no index arithmetic;
//   * the <= 26 x 38 source patch is staged with clamped coordinates (the clamp is torch's x1 = min(x0+1, W-1));
//   * phase 1: horizontal lerp of every staged source row at the tile's 72 output columns (2 LDS + 2 FP each);
//   * phase 2: vertical lerp, 4 output columns per thread: 2 LDS.128 + 8 FP + one 128-bit store.
// Index math follows torch's area_pixel_compute_source_index for align_corners=True: src = dst*(in-1)/(out-1),
// and the blend keeps torch's association w_y0*(w_x0*v00 + w_x1*v01) + w_y1*(w_x0*v10 + w_x1*v11).
#include "common.cuh"

namespace smaat {

constexpr int UP_TY = 48, UP_TX = 72;          // output tile
constexpr int UP_SR = 27, UP_SC = 40;          // staged source patch (rows, cols) incl. the +1 neighbours
constexpr int UP_SP = UP_SC + 1;               // pitch
constexpr int UP_THREADS = (UP_TX / 4) * 12;   // 18 column quads x 12 row lanes = 216

template <bool VEC>
__global__ void __launch_bounds__(UP_THREADS) upsample2x_pad_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                    int64_t y_bstride, int C, int H, int W, int Ho, int Wo,
                                                                    int pad_t, int pad_l, float ry, float rx, int tiles_x) {
  __shared__ float src[UP_SR * UP_SP];
  __shared__ __align__(16) float hs[UP_SR][UP_TX];
  __shared__ int cidx[UP_TX], ridx[UP_TY];
  __shared__ float cw0[UP_TX], cw1[UP_TX], rw0[UP_TY], rw1[UP_TY];
  const int c = blockIdx.y, b = blockIdx.z;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
  const int oy_t = ty * UP_TY, ox_t = tx * UP_TX;
  const int tid = threadIdx.x;
  // first source column / row any output of this tile can touch
  const int xa = min((int)(rx * (float)max(ox_t - pad_l, 0)), W - 1);
  const int ya = min((int)(ry * (float)max(oy_t - pad_t, 0)), H - 1);
  if (tid < UP_TX) {
    const int ux = ox_t + tid - pad_l;
    const bool in = (ux >= 0) && (ux < 2 * W) && (ox_t + tid < Wo);
    const float sx = rx * (float)max(ux, 0);
    const int x0 = min((int)sx, W - 1);
    const float lx = sx - (float)x0;
    cidx[tid] = min(max(x0 - xa, 0), UP_SC - 2);
    cw0[tid] = in ? 1.f - lx : 0.f;
    cw1[tid] = in ? lx : 0.f;
  } else if (tid < UP_TX + UP_TY) {
    const int r = tid - UP_TX;
    const int uy = oy_t + r - pad_t;
    const bool in = (uy >= 0) && (uy < 2 * H) && (oy_t + r < Ho);
    const float sy = ry * (float)max(uy, 0);
    const int y0 = min((int)sy, H - 1);
    const float ly = sy - (float)y0;
    ridx[r] = min(max(y0 - ya, 0), UP_SR - 2);
    rw0[r] = in ? 1.f - ly : 0.f;
    rw1[r] = in ? ly : 0.f;
  }
  const float* plane = x + ((int64_t)b * C + c) * H * W;
  for (int i = tid; i < UP_SR * UP_SC; i += UP_THREADS) {
    const int r = i / UP_SC, cc = i - r * UP_SC;
    src[r * UP_SP + cc] = __ldg(plane + (int64_t)min(ya + r, H - 1) * W + min(xa + cc, W - 1));
  }
  __syncthreads();
  // phase 1: hs[r][j] = w_x0 * src[r][x0] + w_x1 * src[r][x0 + 1]
  for (int i = tid; i < UP_SR * UP_TX; i += UP_THREADS) {
    const int r = i / UP_TX, j = i - r * UP_TX;
    const float* s = src + r * UP_SP + cidx[j];
    hs[r][j] = cw0[j] * s[0] + cw1[j] * s[1];
  }
  __syncthreads();
  // phase 2: out[r][4q..4q+3] = w_y0 * hs[y0][..] + w_y1 * hs[y0 + 1][..]
  const int q = tid % (UP_TX / 4), rl = tid / (UP_TX / 4);
  const int ox = ox_t + 4 * q;
  if (ox >= Wo) return;
  float* dst = y + (int64_t)b * y_bstride + (int64_t)c * Ho * Wo + ox;
#pragma unroll
  for (int r = rl; r < UP_TY; r += 12) {
    const int oy = oy_t + r;
    if (oy >= Ho) break;
    const int y0 = ridx[r];
    const float w0 = rw0[r], w1 = rw1[r];
    const float4 a = *reinterpret_cast<const float4*>(&hs[y0][4 * q]);
    const float4 bb = *reinterpret_cast<const float4*>(&hs[y0 + 1][4 * q]);
    const float o0 = w0 * a.x + w1 * bb.x, o1 = w0 * a.y + w1 * bb.y, o2 = w0 * a.z + w1 * bb.z, o3 = w0 * a.w + w1 * bb.w;
    float* d = dst + (int64_t)oy * Wo;
    if (VEC) {
      *reinterpret_cast<float4*>(d) = make_float4(o0, o1, o2, o3);
    } else {
      d[0] = o0;
      if (ox + 1 < Wo) d[1] = o1;
      if (ox + 2 < Wo) d[2] = o2;
      if (ox + 3 < Wo) d[3] = o3;
    }
  }
}

// ---- streaming variant (128-bit stores, no shared memory, no barriers) ------------------------------------------------
// A thread owns 4 consecutive output columns and walks UPS_ROWS consecutive output rows of one plane.  Its 4 columns need at
// most 4 consecutive source columns (src = dst * (W-1)/(2W-1) < dst / 2 + 1): the horizontally blended source row
// h[j] = w_x0[j] * v[x0[j]] + w_x1[j] * v[x0[j] + 1] is kept in registers for source rows y0 and y0 + 1 and recomputed only when
// the walk crosses into the next source row (every ~2 output rows): ~2.5 scalar loads (L1 / L2 hits: the source is 4x smaller
// than the output and every value is read by ~4 neighbouring threads), 16 flops and one 128-bit store per 4 outputs.
// TI / TO: the storage types of x and y (float, or uint16_t bf16 in the serving forward's bf16 route: the blend runs in fp32 and
// each output is rounded to bf16 once)
constexpr int UPS_ROWS = 8;
template <typename TI = float, typename TO = float>
__global__ void __launch_bounds__(256) upsample2x_pad_stream_kernel(const TI* __restrict__ x, TO* __restrict__ y, int64_t y_bstride,
                                                                    int C, int H, int W, int Ho, int Wo, int pad_t, int pad_l, float ry,
                                                                    float rx, int quads, int row_groups, int64_t planes) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int q = (int)(t % quads);
  const int64_t t2 = t / quads;
  const int rg = (int)(t2 % row_groups);
  const int64_t plane_id = t2 / row_groups;            // b * C + c
  if (plane_id >= planes) return;
  const int b = (int)(plane_id / C), c = (int)(plane_id - (int64_t)b * C);
  const int ox = 4 * q;
  // per-column source index / weights (torch: area_pixel_compute_source_index, align_corners=True); pad columns -> weight 0
  int xi[4];
  float wx0[4], wx1[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int ux = ox + j - pad_l;
    const bool in = (ux >= 0) && (ux < 2 * W);
    const float sx = rx * (float)max(ux, 0);
    const int x0 = min((int)sx, W - 1);
    const float lx = sx - (float)x0;
    xi[j] = x0;
    wx0[j] = in ? 1.f - lx : 0.f;
    wx1[j] = in ? lx : 0.f;
  }
  const TI* plane = x + ((int64_t)b * C + c) * H * W;
  auto hrow = [&](int yy, float (&h)[4]) {
    const TI* r = plane + (int64_t)yy * W;
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = wx0[j] * ld_act(r + xi[j]) + wx1[j] * ld_act(r + min(xi[j] + 1, W - 1));
  };
  TO* dst = y + (int64_t)b * y_bstride + (int64_t)c * Ho * Wo + ox;
  float h0[4], h1[4];
  int cur = -1;                                        // source row held in h0 (h1 = row min(cur + 1, H - 1))
  const int oy0 = rg * UPS_ROWS;
#pragma unroll
  for (int r = 0; r < UPS_ROWS; ++r) {
    const int oy = oy0 + r;
    if (oy >= Ho) break;
    const int uy = oy - pad_t;
    const bool in = (uy >= 0) && (uy < 2 * H);
    const float sy = ry * (float)max(uy, 0);
    const int y0 = min((int)sy, H - 1);
    const float ly = sy - (float)y0;
    const float w0 = in ? 1.f - ly : 0.f, w1 = in ? ly : 0.f;
    if (y0 != cur) {
      if (y0 == cur + 1 && cur >= 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) h0[j] = h1[j];
      } else {
        hrow(y0, h0);
      }
      hrow(min(y0 + 1, H - 1), h1);
      cur = y0;
    }
    st_act4(dst + (int64_t)oy * Wo,
            make_float4(w0 * h0[0] + w1 * h1[0], w0 * h0[1] + w1 * h1[1], w0 * h0[2] + w1 * h1[2], w0 * h0[3] + w1 * h1[3]));
  }
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_upsample2x_pad_fwd(const float* x, float* y, int64_t y_bstride, int B, int C, int H, int W, int Ho, int Wo,
                                        void* stream) {
  SMAAT_REQUIRE(x && y && B > 0 && C > 0 && H > 0 && W > 0, "upsample2x: bad arguments");
  SMAAT_REQUIRE(Ho >= 2 * H && Wo >= 2 * W, "upsample2x: target %dx%d smaller than 2x source %dx%d (negative pad = crop unsupported)",
                Ho, Wo, H, W);
  SMAAT_REQUIRE(y_bstride >= (int64_t)C * Ho * Wo, "upsample2x: y batch stride too small");
  SMAAT_REQUIRE(C <= 65535 && B <= 65535, "upsample2x: C/B too large for grid.y/z");
  const int pad_t = (Ho - 2 * H) / 2, pad_l = (Wo - 2 * W) / 2;
  const float ry = (2 * H > 1) ? (float)(H - 1) / (float)(2 * H - 1) : 0.f;
  const float rx = (2 * W > 1) ? (float)(W - 1) / (float)(2 * W - 1) : 0.f;
  const bool vec = (Wo % 4 == 0) && aligned16(y) && (y_bstride % 4 == 0);
  if (vec) {   // Wo % 4 == 0 and aligned: every thread stores whole 128-bit quads
    const int quads = Wo / 4, row_groups = ceil_div(Ho, UPS_ROWS);
    const int64_t threads = (int64_t)quads * row_groups * C * B;
    SMAAT_REQUIRE(ceil_div64(threads, 256) < (1ll << 31), "upsample2x: grid too large");
    upsample2x_pad_stream_kernel<float, float><<<(unsigned)ceil_div64(threads, 256), 256, 0, (cudaStream_t)stream>>>(
        x, y, y_bstride, C, H, W, Ho, Wo, pad_t, pad_l, ry, rx, quads, row_groups, (int64_t)B * C);
    SMAAT_LAUNCH_CHECK("smaat_upsample2x_pad_fwd");
    return SMAAT_OK;
  }
  const int tiles_x = ceil_div(Wo, UP_TX), tiles_y = ceil_div(Ho, UP_TY);
  dim3 grid(tiles_x * tiles_y, C, B);
  if (vec)
    upsample2x_pad_kernel<true><<<grid, UP_THREADS, 0, (cudaStream_t)stream>>>(x, y, y_bstride, C, H, W, Ho, Wo, pad_t, pad_l, ry, rx,
                                                                              tiles_x);
  else
    upsample2x_pad_kernel<false><<<grid, UP_THREADS, 0, (cudaStream_t)stream>>>(x, y, y_bstride, C, H, W, Ho, Wo, pad_t, pad_l, ry, rx,
                                                                               tiles_x);
  SMAAT_LAUNCH_CHECK("smaat_upsample2x_pad_fwd");
  return SMAAT_OK;
}

/* smaat_upsample2x_pad_fwd with a bf16 output (the serving forward's bf16 route), from an fp32 (x_bf16 = 0: the 36 x 36 level
 * into up2) or a bf16 x.  Needs Wo % 4 == 0, an 8-byte aligned y and y_bstride % 4 == 0 (every thread stores 4 outputs at once):
 * SMAAT_E_UNSUPPORTED otherwise. */
extern "C" int smaat_upsample2x_pad_bf16_fwd(const void* x, int x_bf16, void* y, int64_t y_bstride, int B, int C, int H, int W, int Ho,
                                             int Wo, void* stream) {
  SMAAT_REQUIRE(x && y && B > 0 && C > 0 && H > 0 && W > 0, "upsample2x_bf16: bad arguments");
  SMAAT_REQUIRE(Ho >= 2 * H && Wo >= 2 * W, "upsample2x_bf16: target %dx%d smaller than 2x source %dx%d (negative pad = crop unsupported)",
                Ho, Wo, H, W);
  SMAAT_REQUIRE(y_bstride >= (int64_t)C * Ho * Wo, "upsample2x_bf16: y batch stride too small");
  if (Wo % 4 != 0 || (reinterpret_cast<uintptr_t>(y) & 7u) || y_bstride % 4 != 0)
    return fail(SMAAT_E_UNSUPPORTED, "upsample2x_bf16: needs Wo %% 4 == 0, an 8-byte aligned output and a batch stride that is a "
                                     "multiple of 4 (Wo=%d)", Wo);
  const int pad_t = (Ho - 2 * H) / 2, pad_l = (Wo - 2 * W) / 2;
  const float ry = (2 * H > 1) ? (float)(H - 1) / (float)(2 * H - 1) : 0.f;
  const float rx = (2 * W > 1) ? (float)(W - 1) / (float)(2 * W - 1) : 0.f;
  const int quads = Wo / 4, row_groups = ceil_div(Ho, UPS_ROWS);
  const int64_t threads = (int64_t)quads * row_groups * C * B;
  SMAAT_REQUIRE(ceil_div64(threads, 256) < (1ll << 31), "upsample2x_bf16: grid too large");
  const unsigned grid = (unsigned)ceil_div64(threads, 256);
  uint16_t* yb = static_cast<uint16_t*>(y);
  if (x_bf16)
    upsample2x_pad_stream_kernel<uint16_t, uint16_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
        static_cast<const uint16_t*>(x), yb, y_bstride, C, H, W, Ho, Wo, pad_t, pad_l, ry, rx, quads, row_groups, (int64_t)B * C);
  else
    upsample2x_pad_stream_kernel<float, uint16_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
        static_cast<const float*>(x), yb, y_bstride, C, H, W, Ho, Wo, pad_t, pad_l, ry, rx, quads, row_groups, (int64_t)B * C);
  SMAAT_LAUNCH_CHECK("smaat_upsample2x_pad_bf16_fwd");
  return SMAAT_OK;
}
