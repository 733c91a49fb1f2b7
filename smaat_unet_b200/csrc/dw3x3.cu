// dw3x3.cu -- depthwise 3x3 (padding 1, groups = Cin, k outputs per input channel), forward.
//
// Replaces DepthwiseSeparableConv.depthwise (reference models/layers.py:38-44,48).
// HBM-bound: algorithmic bytes = 4*B*H*W*Cin*(1+k) (SURVEY 8d).  One CTA owns one
// TH x TW output tile of one (b, cin) plane:
//   * the (TH+2) x (TW+8) input halo tile is staged in shared memory by ONE TMA
//     (cp.async.bulk.tensor.4d) whose out-of-bounds zero fill IS the conv's padding=1; the box
//     starts at column x0-4 because the inner TMA coordinate must be 16-byte aligned;
//   * each thread walks an RH-row strip of 4 output columns with a 3-row register window
//     (1 LDS.128 + 2 LDS.32 per input row), producing k output planes, 128-bit stores;
//   * many small CTAs per SM (<= ~14 KB smem each) keep enough bytes in flight to cover
//     HBM latency without an intra-CTA pipeline.
// The input may be the virtual concat of two tensors (UpDS: cat([skip, up]), parts_ds.py:85)
// and may get relu(scale*x+shift) applied on load (train-mode BN+ReLU of the producer).
// An LDG loader variant covers W % 4 != 0 (TMA needs 16-byte row pitch) and serves as the
// on-GPU cross-check of the TMA path (tests force both).
#include "common.cuh"

namespace smaat {

struct DwParams {
  const float* x0;
  const float* x1;
  int C0, C1;
  int64_t bs0, bs1;
  const float* w;
  const float* bias;
  const float* in_scale;
  const float* in_shift;
  float* y;
  int B, H, W, k;
  int TW, TH, BW, BH;
  int tiles_x, tiles_y;
};

template <int K, int RH, bool USE_TMA, bool PRO, bool VEC>
__global__ void __launch_bounds__(256) dw3x3_kernel(const __grid_constant__ CUtensorMap map0,
                                                    const __grid_constant__ CUtensorMap map1, const DwParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tile = reinterpret_cast<float*>(smem_raw);
  __shared__ __align__(8) uint64_t bar;

  const int tiles = p.tiles_x * p.tiles_y;
  const int tile_id = blockIdx.x % tiles;
  const int plane = blockIdx.x / tiles;  // b * Cin + c
  const int Cin = p.C0 + p.C1;
  const int b = plane / Cin;
  const int c = plane - b * Cin;
  const int ty = tile_id / p.tiles_x;
  const int tx = tile_id - ty * p.tiles_x;
  const int x0 = tx * p.TW;
  const int y0 = ty * p.TH;
  const int tid = threadIdx.x;
  const int BW = p.BW, BH = p.BH;

  if (USE_TMA) {
    if (tid == 0) {
      mbar_init(&bar, 1);
      fence_barrier_init();
      mbar_arrive_expect_tx(&bar, (uint32_t)(BW * BH * sizeof(float)));
      if (c < p.C0)
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
                "r"(smem_u32(tile)),
            "l"(reinterpret_cast<uint64_t>(&map0)), "r"(smem_u32(&bar)), "r"(x0 - 4), "r"(y0 - 1), "r"(c), "r"(b)
            : "memory");
      else
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
                "r"(smem_u32(tile)),
            "l"(reinterpret_cast<uint64_t>(&map1)), "r"(smem_u32(&bar)), "r"(x0 - 4), "r"(y0 - 1), "r"(c - p.C0), "r"(b)
            : "memory");
    }
  } else {
    const float* src = (c < p.C0) ? p.x0 + (int64_t)b * p.bs0 + (int64_t)c * p.H * p.W
                                  : p.x1 + (int64_t)b * p.bs1 + (int64_t)(c - p.C0) * p.H * p.W;
    float s = 1.f, t = 0.f;
    if (PRO) {
      s = __ldg(p.in_scale + c);
      t = __ldg(p.in_shift + c);
    }
    for (int i = tid; i < BW * BH; i += blockDim.x) {
      const int r = i / BW, cc = i - r * BW;
      const int gy = y0 - 1 + r, gx = x0 - 4 + cc;
      float v = 0.f;
      if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) {
        v = __ldg(src + (int64_t)gy * p.W + gx);
        if (PRO) v = fmaxf(fmaf(v, s, t), 0.f);
      }
      tile[i] = v;
    }
  }

  // weights / bias of the k output planes fed by this input channel (overlaps the TMA)
  constexpr int KMAX = (K > 0) ? K : 1;
  float wr[KMAX][9];
  float br[KMAX];
  if (K > 0) {
#pragma unroll
    for (int kk = 0; kk < KMAX; ++kk) {
      const int o = c * K + kk;
#pragma unroll
      for (int t = 0; t < 9; ++t) wr[kk][t] = __ldg(p.w + (int64_t)o * 9 + t);
      br[kk] = p.bias ? __ldg(p.bias + o) : 0.f;
    }
  }

  if (USE_TMA) {
    __syncthreads();  // barrier init by thread 0 must be visible before anyone polls it
    mbar_wait(&bar, 0);
    // PRO: relu(scale*x+shift) is applied while the register window is loaded (below); the zero padding stays zero
  } else {
    __syncthreads();
  }

  const int nsx = p.TW >> 2;
  const int nsy = p.TH / RH;
  const int kout = (K > 0) ? K : p.k;
  float* ybase = p.y + ((int64_t)b * Cin * kout + (int64_t)c * kout) * p.H * p.W;

  for (int s = tid; s < nsx * nsy; s += blockDim.x) {
    const int sy = s / nsx, sx = s - sy * nsx;
    const int col = sx << 2;
    const int row0 = sy * RH;
    const int gx = x0 + col;
    if (gx >= p.W) continue;
    if (y0 + row0 >= p.H) continue;

    for (int kk0 = 0; kk0 < kout; kk0 += KMAX) {
      if (K == 0) {  // generic k: one output plane per pass, weights fetched per pass
        const int o = c * kout + kk0;
#pragma unroll
        for (int t = 0; t < 9; ++t) wr[0][t] = __ldg(p.w + (int64_t)o * 9 + t);
        br[0] = p.bias ? __ldg(p.bias + o) : 0.f;
      }
      float win[3][6];
      // smem column of global x is x - (x0 - 4): the 4 outputs at col..col+3 read smem cols col+3..col+8
      const float* trow = tile + row0 * BW + col + 3;
      // TMA path + PRO: activation on load; rows / edge columns outside the image are the conv's zero padding
      const bool tma_pro = USE_TMA && PRO;
      float ps = 1.f, pt = 0.f;
      if (tma_pro) { ps = __ldg(p.in_scale + c); pt = __ldg(p.in_shift + c); }
      const bool lpad = (gx == 0), rpad = (gx + 4 >= p.W);
      auto load_row = [&](float* wl, int r) {   // r = tile row relative to row0 (0 .. RH+1); image row y0 + row0 + r - 1
        const float4 a = *reinterpret_cast<const float4*>(trow + r * BW + 1);
        wl[0] = trow[r * BW]; wl[1] = a.x; wl[2] = a.y; wl[3] = a.z; wl[4] = a.w; wl[5] = trow[r * BW + 5];
        if (tma_pro) {
          const int gyr = y0 + row0 + r - 1;
          const bool rowin = (gyr >= 0) && (gyr < p.H);
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            const bool in = rowin && !(q == 0 && lpad) && !(q == 5 && rpad) && (q == 0 || q == 5 || gx + q - 1 < p.W);
            wl[q] = in ? fmaxf(fmaf(wl[q], ps, pt), 0.f) : 0.f;
          }
        }
      };
#pragma unroll
      for (int r = 0; r < 2; ++r) load_row(win[r], r);
#pragma unroll
      for (int i = 0; i < RH; ++i) {
        load_row(win[(i + 2) % 3], i + 2);
        const int gy = y0 + row0 + i;
        if (gy < p.H) {
          const float* r0 = win[i % 3];
          const float* r1 = win[(i + 1) % 3];
          const float* r2 = win[(i + 2) % 3];
#pragma unroll
          for (int kk = 0; kk < KMAX; ++kk) {
            float o4[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float a = br[kk];
              a = fmaf(wr[kk][0], r0[j], a); a = fmaf(wr[kk][1], r0[j + 1], a); a = fmaf(wr[kk][2], r0[j + 2], a);
              a = fmaf(wr[kk][3], r1[j], a); a = fmaf(wr[kk][4], r1[j + 1], a); a = fmaf(wr[kk][5], r1[j + 2], a);
              a = fmaf(wr[kk][6], r2[j], a); a = fmaf(wr[kk][7], r2[j + 1], a); a = fmaf(wr[kk][8], r2[j + 2], a);
              o4[j] = a;
            }
            float* dst = ybase + (int64_t)(kk0 + kk) * p.H * p.W + (int64_t)gy * p.W + gx;
            if (VEC && gx + 3 < p.W) {
              *reinterpret_cast<float4*>(dst) = make_float4(o4[0], o4[1], o4[2], o4[3]);
            } else {
#pragma unroll
              for (int j = 0; j < 4; ++j)
                if (gx + j < p.W) dst[j] = o4[j];
            }
          }
        }
      }
    }
  }
}

// Tile heuristic: TW = widest multiple-of-4 divisor of W up to 96 (else 64 with a ragged
// edge); TH = RH * strip_rows minimising (row waste) x (halo overhead), CTA <= 256 threads.
static void pick_tile(int H, int W, int* TW, int* TH, int* RH) {
  int tw = 0;
  if (W % 4 == 0) {
    for (int c = 96; c >= 16; c -= 4)
      if (W % c == 0) {
        tw = c;
        break;
      }
  }
  if (tw == 0) tw = (W >= 64) ? 64 : ((W + 3) / 4) * 4;
  const int rh = (H >= 32) ? 8 : 4;
  const int nsx = tw / 4;
  int best_sr = 1;
  double best = 1e30;
  for (int sr = 1; sr <= 16; ++sr) {
    if (nsx * sr > 256 && sr > 1) break;
    const int th = sr * rh;
    const double rows = (double)ceil_div(H, th) * th / H;
    const double halo = (double)(th + 2) / th;
    const double small = (nsx * sr < 64) ? 1.0 + 0.15 * (64 - nsx * sr) / 64.0 : 1.0;  // tiny CTAs cost launch slots
    const double cost = rows * halo * small;
    if (cost < best - 1e-9) {
      best = cost;
      best_sr = sr;
    }
    if (th >= H) break;
  }
  *TW = tw;
  *TH = best_sr * rh;
  *RH = rh;
}

void dw_pick_tile(int H, int W, int* TW, int* TH, int* RH) { pick_tile(H, W, TW, TH, RH); }  // shared with dw3x3_bwd.cu

// dw3x3_small.cu: returns 1 when not applicable
int dw3x3_small_try(const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1, const float* w, const float* bias,
                    const float* in_scale, const float* in_shift, float* y, int B, int H, int W, int k, cudaStream_t st);

template <int K, int RH, bool USE_TMA, bool PRO, bool VEC>
static int launch_dw(const CUtensorMap& m0, const CUtensorMap& m1, const DwParams& p, int threads, size_t smem,
                     int64_t grid, cudaStream_t st) {
  auto kern = dw3x3_kernel<K, RH, USE_TMA, PRO, VEC>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "dw3x3: smem attribute: %s", cudaGetErrorString(e));
  }
  kern<<<(unsigned)grid, threads, smem, st>>>(m0, m1, p);
  SMAAT_LAUNCH_CHECK("smaat_dw3x3_fwd");
  return SMAAT_OK;
}

template <int K, int RH, bool USE_TMA>
static int dispatch_dw2(const CUtensorMap& m0, const CUtensorMap& m1, const DwParams& p, bool pro, bool vec, int threads,
                        size_t smem, int64_t grid, cudaStream_t st) {
  if (pro) {
    if (vec) return launch_dw<K, RH, USE_TMA, true, true>(m0, m1, p, threads, smem, grid, st);
    return launch_dw<K, RH, USE_TMA, true, false>(m0, m1, p, threads, smem, grid, st);
  }
  if (vec) return launch_dw<K, RH, USE_TMA, false, true>(m0, m1, p, threads, smem, grid, st);
  return launch_dw<K, RH, USE_TMA, false, false>(m0, m1, p, threads, smem, grid, st);
}

template <int K>
static int dispatch_dw(const CUtensorMap& m0, const CUtensorMap& m1, const DwParams& p, int rh, bool tma, bool pro, bool vec,
                       int threads, size_t smem, int64_t grid, cudaStream_t st) {
  if (rh == 8) {
    if (tma) return dispatch_dw2<K, 8, true>(m0, m1, p, pro, vec, threads, smem, grid, st);
    return dispatch_dw2<K, 8, false>(m0, m1, p, pro, vec, threads, smem, grid, st);
  }
  if (tma) return dispatch_dw2<K, 4, true>(m0, m1, p, pro, vec, threads, smem, grid, st);
  return dispatch_dw2<K, 4, false>(m0, m1, p, pro, vec, threads, smem, grid, st);
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_dw3x3_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                               const float* w, const float* bias, const float* in_scale, const float* in_shift, float* y,
                               int B, int H, int W, int k, int loader, void* stream) {
  SMAAT_REQUIRE(x0 && w && y, "dw3x3: null pointer");
  SMAAT_REQUIRE(B > 0 && C0 > 0 && C1 >= 0 && H > 0 && W > 0 && k > 0, "dw3x3: bad shape B=%d C0=%d C1=%d H=%d W=%d k=%d", B,
                C0, C1, H, W, k);
  SMAAT_REQUIRE(C1 == 0 || x1, "dw3x3: C1=%d but x1 is null", C1);
  SMAAT_REQUIRE((in_scale == nullptr) == (in_shift == nullptr), "dw3x3: in_scale/in_shift must both be given or both null");
  SMAAT_REQUIRE(x0_bstride >= (int64_t)C0 * H * W, "dw3x3: x0 batch stride %lld < C0*H*W", (long long)x0_bstride);
  SMAAT_REQUIRE(C1 == 0 || x1_bstride >= (int64_t)C1 * H * W, "dw3x3: x1 batch stride too small");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);

  DwParams p;
  p.x0 = x0; p.x1 = x1; p.C0 = C0; p.C1 = C1; p.bs0 = x0_bstride; p.bs1 = x1_bstride;
  p.w = w; p.bias = bias; p.in_scale = in_scale; p.in_shift = in_shift; p.y = y;
  p.B = B; p.H = H; p.W = W; p.k = k;
  int rh;
  pick_tile(H, W, &p.TW, &p.TH, &rh);
  p.BW = p.TW + 8;  // box starts at x0-4: TMA needs a 16-byte aligned inner coordinate (measured: x0-1 traps)
  p.BH = p.TH + 2;
  p.tiles_x = ceil_div(W, p.TW);
  p.tiles_y = ceil_div(H, p.TH);

  const bool vec = (W % 4 == 0) && aligned16(y);
  bool tma_ok = (W % 4 == 0) && aligned16(x0) && (x0_bstride % 4 == 0) && p.BW <= 256 && p.BH <= 256 &&
                (C1 == 0 || (aligned16(x1) && (x1_bstride % 4 == 0)));
  SMAAT_REQUIRE(loader >= 0 && loader <= 2, "dw3x3: loader must be 0 (auto), 1 (ldg) or 2 (tma)");
  SMAAT_REQUIRE(!(loader == 2 && !tma_ok), "dw3x3: TMA loader forced but ineligible (W %% 4 = %d, alignment)", W % 4);
  const bool use_tma = (loader == 1) ? false : tma_ok;
  if (loader == 0 && !tma_ok) {   // small planes TMA cannot describe (e.g. 18 x 18): one warp per plane (dw3x3_small.cu)
    const int r = dw3x3_small_try(x0, C0, x0_bstride, x1, C1, x1_bstride, w, bias, in_scale, in_shift, y, B, H, W, k, st);
    if (r != 1) return r;
  }

  CUtensorMap m0, m1;
  memset(&m0, 0, sizeof(m0));
  memset(&m1, 0, sizeof(m1));
  if (use_tma) {
    const uint32_t box[4] = {(uint32_t)p.BW, (uint32_t)p.BH, 1u, 1u};
    {
      const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C0, (uint64_t)B};
      const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)x0_bstride * 4};
      int r = make_tmap_f32(&m0, x0, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "dw3x3(x0)");
      if (r) return r;
    }
    if (C1 > 0) {
      const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C1, (uint64_t)B};
      const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)x1_bstride * 4};
      int r = make_tmap_f32(&m1, x1, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "dw3x3(x1)");
      if (r) return r;
    } else {
      m1 = m0;
    }
  }

  const int nstrips = (p.TW / 4) * (p.TH / rh);
  int threads = ((nstrips < 256 ? nstrips : 256) + 31) / 32 * 32;
  const size_t smem = (size_t)p.BW * p.BH * sizeof(float);
  const int64_t grid = (int64_t)B * (C0 + C1) * p.tiles_x * p.tiles_y;
  SMAAT_REQUIRE(grid < (1ll << 31), "dw3x3: grid too large (%lld CTAs)", (long long)grid);
  const bool pro = in_scale != nullptr;

  if (k == 1) return dispatch_dw<1>(m0, m1, p, rh, use_tma, pro, vec, threads, smem, grid, st);
  if (k == 2) return dispatch_dw<2>(m0, m1, p, rh, use_tma, pro, vec, threads, smem, grid, st);
  if (k == 4) return dispatch_dw<4>(m0, m1, p, rh, use_tma, pro, vec, threads, smem, grid, st);
  return dispatch_dw<0>(m0, m1, p, rh, use_tma, pro, vec, threads, smem, grid, st);
}
