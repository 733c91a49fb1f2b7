// dw3x3_bwd.cu -- depthwise 3x3 backward, smem-tiled (replaces the naive per-element versions).
//
// Backward of DepthwiseSeparableConv.depthwise (reference models/layers.py:38-44,48):
//   input : dx[b,c,i,j]  = sum_kk sum_{dy,dx} w[c*k+kk][dy][dx] * dd[b, c*k+kk, i-dy+1, j-dx+1]
//   weight: dW[o][dy][dx] += sum_{b,i,j} dd[b,o,i,j] * in[b,o/k,i+dy-1,j+dx-1],  db[o] += sum dd
// One CTA per (plane, TH x TW tile): the halo tile(s) are staged in shared memory once (coalesced loads,
// zero fill = padding), so every global element is read once instead of 9-18 times.  The weight kernel
// keeps 10*k partial sums per thread, block-reduces them and merges tiles with fp32 atomics.
#include "common.cuh"

namespace smaat {

constexpr int DB_TH = 32;     // tile rows
constexpr int DB_KMAX = 4;    // kernels_per_layer supported by the tiled kernels

static int pick_tw(int W) {
  if (W % 4 == 0)
    for (int c = 96; c >= 16; c -= 4)
      if (W % c == 0) return c;
  return W >= 64 ? 64 : ((W + 3) / 4) * 4;
}

__global__ void __launch_bounds__(256) dw3x3_bwd_input_tiled(const float* __restrict__ dd, const float* __restrict__ w,
                                                             float* __restrict__ dx0, int C0, int64_t bs0,
                                                             float* __restrict__ dx1, int C1, int64_t bs1, int H, int W, int k,
                                                             int TW, int tiles_x, int tiles_y) {
  extern __shared__ float sm[];  // [k][DB_TH+2][TW+2]
  const int Cin = C0 + C1;
  const int tiles = tiles_x * tiles_y;
  const int plane = blockIdx.x / tiles, tile = blockIdx.x % tiles;
  const int b = plane / Cin, c = plane - b * Cin;
  const int y0 = (tile / tiles_x) * DB_TH, x0 = (tile % tiles_x) * TW;
  const int SW = TW + 2, SH = DB_TH + 2;
  const int P = H * W;
  const float* g = dd + ((int64_t)b * Cin + c) * k * P;
  for (int i = threadIdx.x; i < k * SH * SW; i += blockDim.x) {
    const int kk = i / (SH * SW), r = (i / SW) % SH, cc = i % SW;
    const int gy = y0 - 1 + r, gx = x0 - 1 + cc;
    sm[i] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(g + (int64_t)kk * P + (int64_t)gy * W + gx) : 0.f;
  }
  __shared__ float ws[DB_KMAX * 9];
  if (threadIdx.x < k * 9) ws[threadIdx.x] = __ldg(w + (int64_t)c * k * 9 + threadIdx.x);
  __syncthreads();
  float* dst = (c < C0) ? dx0 + (int64_t)b * bs0 + (int64_t)c * P : dx1 + (int64_t)b * bs1 + (int64_t)(c - C0) * P;
  for (int i = threadIdx.x; i < DB_TH * TW; i += blockDim.x) {
    const int y = i / TW, x = i - y * TW;
    const int gy = y0 + y, gx = x0 + x;
    if (gy >= H || gx >= W) continue;
    float acc = 0.f;
    for (int kk = 0; kk < k; ++kk) {
      const float* t = sm + (kk * SH + y + 1) * SW + x + 1;   // centre
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dxx = 0; dxx < 3; ++dxx) acc = fmaf(ws[kk * 9 + dy * 3 + dxx], t[(1 - dy) * SW + (1 - dxx)], acc);
    }
    dst[(int64_t)gy * W + gx] = acc;
  }
}

__global__ void __launch_bounds__(256) dw3x3_bwd_weight_tiled(const float* __restrict__ dd, const float* __restrict__ x0p, int C0,
                                                              int64_t bs0, const float* __restrict__ x1p, int C1, int64_t bs1,
                                                              const float* __restrict__ in_scale, const float* __restrict__ in_shift,
                                                              float* __restrict__ dw, float* __restrict__ db, int H, int W, int k,
                                                              int TW, int tiles_x, int tiles_y) {
  extern __shared__ float sm[];  // [DB_TH+2][TW+2] input halo tile (activation applied, zero padding)
  const int Cin = C0 + C1;
  const int tiles = tiles_x * tiles_y;
  const int plane = blockIdx.x / tiles, tile = blockIdx.x % tiles;
  const int b = plane / Cin, c = plane - b * Cin;
  const int y0 = (tile / tiles_x) * DB_TH, x0 = (tile % tiles_x) * TW;
  const int SW = TW + 2, SH = DB_TH + 2;
  const int P = H * W;
  const float* src = (c < C0) ? x0p + (int64_t)b * bs0 + (int64_t)c * P : x1p + (int64_t)b * bs1 + (int64_t)(c - C0) * P;
  const bool pro = in_scale != nullptr;
  const float s = pro ? __ldg(in_scale + c) : 1.f, t = pro ? __ldg(in_shift + c) : 0.f;
  for (int i = threadIdx.x; i < SH * SW; i += blockDim.x) {
    const int r = i / SW, cc = i - r * SW;
    const int gy = y0 - 1 + r, gx = x0 - 1 + cc;
    float v = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      v = __ldg(src + (int64_t)gy * W + gx);
      if (pro) v = fmaxf(fmaf(v, s, t), 0.f);
    }
    sm[i] = v;
  }
  __syncthreads();
  float acc[DB_KMAX][10];
#pragma unroll
  for (int kk = 0; kk < DB_KMAX; ++kk)
#pragma unroll
    for (int q = 0; q < 10; ++q) acc[kk][q] = 0.f;
  const float* g = dd + ((int64_t)b * Cin + c) * k * P;
  for (int i = threadIdx.x; i < DB_TH * TW; i += blockDim.x) {
    const int y = i / TW, x = i - y * TW;
    const int gy = y0 + y, gx = x0 + x;
    if (gy >= H || gx >= W) continue;
    const float* tl = sm + y * SW + x;  // top-left of the 3x3 window
    float win[9];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dxx = 0; dxx < 3; ++dxx) win[dy * 3 + dxx] = tl[dy * SW + dxx];
#pragma unroll
    for (int kk = 0; kk < DB_KMAX; ++kk) {
      if (kk < k) {
        const float gv = __ldg(g + (int64_t)kk * P + (int64_t)gy * W + gx);
#pragma unroll
        for (int q = 0; q < 9; ++q) acc[kk][q] = fmaf(gv, win[q], acc[kk][q]);
        acc[kk][9] += gv;
      }
    }
  }
  __shared__ float red[DB_KMAX * 10][8];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
  for (int kk = 0; kk < DB_KMAX; ++kk) {
    if (kk < k) {
#pragma unroll
      for (int q = 0; q < 10; ++q) {
        const float v = warp_sum(acc[kk][q]);
        if (lane == 0) red[kk * 10 + q][wp] = v;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < k * 10) {
    float v = 0.f;
    for (int i = 0; i < 8; ++i) v += red[threadIdx.x][i];
    const int kk = threadIdx.x / 10, q = threadIdx.x % 10;
    const int o = c * k + kk;
    if (q < 9) atomicAdd(dw + (int64_t)o * 9 + q, v);
    else if (db) atomicAdd(db + o, v);
  }
}

// ---------------------------------------------------------------------------------------------
// TMA variants (W % 4 == 0, k in {1, 2, 4}): same structure as the forward kernel (dw3x3.cu) -- the halo
// tile arrives by one bulk tensor copy per plane (out-of-bounds zero fill = padding), each thread walks
// an RH-row strip of 4 columns with a 3-row register window, 128-bit global accesses.
//   input : K gradient planes -> 1 dx plane, flipped taps.      bytes = 4*B*P*Cin*(k+1)
//   weight: 1 input plane (TMA) x K gradient planes (LDG.128) -> 10*K partial sums per thread.
// ---------------------------------------------------------------------------------------------
void dw_pick_tile(int H, int W, int* TW, int* TH, int* RH);   // dw3x3.cu

struct DwbParams {
  const float* g;          // dd [B][Cin*k][H][W]
  const float* w;
  float* dx0; float* dx1;
  int C0, C1;
  int64_t bs0, bs1;
  const float* in_scale; const float* in_shift;
  float* dw; float* db;
  int H, W;
  int TW, TH, BW, BH, plane_floats;
  int tiles_x, tiles_y;
};

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

__device__ __forceinline__ void load_row6(float* wl, const float* src) {
  const float4 a = *reinterpret_cast<const float4*>(src + 1);
  wl[0] = src[0]; wl[1] = a.x; wl[2] = a.y; wl[3] = a.z; wl[4] = a.w; wl[5] = src[5];
}

template <int K, int RH>
__global__ void __launch_bounds__(256) dw3x3_bwd_input_tma(const __grid_constant__ CUtensorMap mapg, const DwbParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tile = reinterpret_cast<float*>(smem_raw);   // [K][plane_floats]
  __shared__ __align__(8) uint64_t bar;
  const int tiles = p.tiles_x * p.tiles_y;
  const int tile_id = blockIdx.x % tiles, plane = blockIdx.x / tiles;
  const int Cin = p.C0 + p.C1;
  const int b = plane / Cin, c = plane - b * Cin;
  const int ty = tile_id / p.tiles_x, tx = tile_id - ty * p.tiles_x;
  const int x0 = tx * p.TW, y0 = ty * p.TH;
  const int tid = threadIdx.x, BW = p.BW;
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar, (uint32_t)(K * BW * p.BH * sizeof(float)));
#pragma unroll
    for (int kk = 0; kk < K; ++kk) tma_load_4d(tile + kk * p.plane_floats, &mapg, &bar, x0 - 4, y0 - 1, c * K + kk, b);
  }
  float wr[K][9];   // flipped taps: dx[i,j] = sum w[dy][dx] * dd[i+1-dy][j+1-dx]
#pragma unroll
  for (int kk = 0; kk < K; ++kk)
#pragma unroll
    for (int t = 0; t < 9; ++t) wr[kk][t] = __ldg(p.w + (int64_t)(c * K + kk) * 9 + 8 - t);
  __syncthreads();
  mbar_wait(&bar, 0);

  const int P = p.H * p.W;
  float* dst0 = (c < p.C0) ? p.dx0 + (int64_t)b * p.bs0 + (int64_t)c * P : p.dx1 + (int64_t)b * p.bs1 + (int64_t)(c - p.C0) * P;
  const int nsx = p.TW >> 2, nsy = p.TH / RH;
  for (int s = tid; s < nsx * nsy; s += blockDim.x) {
    const int sy = s / nsx, sx = s - sy * nsx;
    const int col = sx << 2, row0 = sy * RH;
    const int gx = x0 + col;
    if (gx >= p.W || y0 + row0 >= p.H) continue;
    float win[K][3][6];
    const float* trow = tile + row0 * BW + col + 3;
#pragma unroll
    for (int kk = 0; kk < K; ++kk)
#pragma unroll
      for (int r = 0; r < 2; ++r) load_row6(win[kk][r], trow + kk * p.plane_floats + r * BW);
#pragma unroll
    for (int i = 0; i < RH; ++i) {
#pragma unroll
      for (int kk = 0; kk < K; ++kk) load_row6(win[kk][(i + 2) % 3], trow + kk * p.plane_floats + (i + 2) * BW);
      const int gy = y0 + row0 + i;
      if (gy < p.H) {
        float o4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float a = 0.f;
#pragma unroll
          for (int kk = 0; kk < K; ++kk) {
            const float* r0 = win[kk][i % 3];
            const float* r1 = win[kk][(i + 1) % 3];
            const float* r2 = win[kk][(i + 2) % 3];
            a = fmaf(wr[kk][0], r0[j], a); a = fmaf(wr[kk][1], r0[j + 1], a); a = fmaf(wr[kk][2], r0[j + 2], a);
            a = fmaf(wr[kk][3], r1[j], a); a = fmaf(wr[kk][4], r1[j + 1], a); a = fmaf(wr[kk][5], r1[j + 2], a);
            a = fmaf(wr[kk][6], r2[j], a); a = fmaf(wr[kk][7], r2[j + 1], a); a = fmaf(wr[kk][8], r2[j + 2], a);
          }
          o4[j] = a;
        }
        *reinterpret_cast<float4*>(dst0 + (int64_t)gy * p.W + gx) = make_float4(o4[0], o4[1], o4[2], o4[3]);
      }
    }
  }
}

template <int K, int RH, bool PRO>
__global__ void __launch_bounds__(256) dw3x3_bwd_weight_tma(const __grid_constant__ CUtensorMap map0,
                                                            const __grid_constant__ CUtensorMap map1,
                                                            const __grid_constant__ CUtensorMap mapg, const DwbParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tile = reinterpret_cast<float*>(smem_raw);   // [BH][BW] input halo tile
  float* gt = tile + p.plane_floats;                  // [K][TH][TW] gradient tiles (one TMA box, K planes deep)
  __shared__ __align__(8) uint64_t bar;
  __shared__ float red[K * 10][8];
  const int tiles = p.tiles_x * p.tiles_y;
  const int tile_id = blockIdx.x % tiles, plane = blockIdx.x / tiles;
  const int Cin = p.C0 + p.C1;
  const int b = plane / Cin, c = plane - b * Cin;
  const int ty = tile_id / p.tiles_x, tx = tile_id - ty * p.tiles_x;
  const int x0 = tx * p.TW, y0 = ty * p.TH;
  const int tid = threadIdx.x, BW = p.BW, BH = p.BH;
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bar, (uint32_t)((BW * BH + K * p.TW * p.TH) * sizeof(float)));
    if (c < p.C0) tma_load_4d(tile, &map0, &bar, x0 - 4, y0 - 1, c, b);
    else tma_load_4d(tile, &map1, &bar, x0 - 4, y0 - 1, c - p.C0, b);
    tma_load_4d(gt, &mapg, &bar, x0, y0, c * K, b);   // all bytes in flight by bulk copy: no per-thread load latency
  }
  __syncthreads();
  mbar_wait(&bar, 0);
  // PRO: relu(scale*x+shift) of the producer's BatchNorm is applied while the register window is loaded; positions
  // outside the image are the conv's zero padding and stay zero
  float ps = 1.f, pt = 0.f;
  if (PRO) { ps = __ldg(p.in_scale + c); pt = __ldg(p.in_shift + c); }
  float acc[K][10];
#pragma unroll
  for (int kk = 0; kk < K; ++kk)
#pragma unroll
    for (int q = 0; q < 10; ++q) acc[kk][q] = 0.f;
  const int nsx = p.TW >> 2, nsy = p.TH / RH;
  const int gplane = p.TW * p.TH;
  for (int s = tid; s < nsx * nsy; s += blockDim.x) {
    const int sy = s / nsx, sx = s - sy * nsx;
    const int col = sx << 2, row0 = sy * RH;
    const int gx = x0 + col;
    if (gx >= p.W || y0 + row0 >= p.H) continue;
    float win[3][6];
    const float* trow = tile + row0 * BW + col + 3;
    const float* grow = gt + row0 * p.TW + col;
    const bool lpad = (gx == 0), rpad = (gx + 4 >= p.W);
    auto load_row = [&](float* wl, int r) {   // r: tile row relative to row0; image row y0 + row0 + r - 1
      load_row6(wl, trow + r * BW);
      if (PRO) {
        const int gyr = y0 + row0 + r - 1;
        const bool rowin = (gyr >= 0) && (gyr < p.H);
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const bool in = rowin && !(q == 0 && lpad) && !(q == 5 && rpad);
          wl[q] = in ? fmaxf(fmaf(wl[q], ps, pt), 0.f) : 0.f;
        }
      }
    };
    load_row(win[0], 0);
    load_row(win[1], 1);
#pragma unroll
    for (int i = 0; i < RH; ++i) {
      load_row(win[(i + 2) % 3], i + 2);
      const int gy = y0 + row0 + i;
      if (gy < p.H) {
        const float* r0 = win[i % 3];
        const float* r1 = win[(i + 1) % 3];
        const float* r2 = win[(i + 2) % 3];
#pragma unroll
        for (int kk = 0; kk < K; ++kk) {
          const float4 g4 = *reinterpret_cast<const float4*>(grow + kk * gplane + i * p.TW);   // rows past H: TMA zero fill
          const float gv[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[kk][0] = fmaf(gv[j], r0[j], acc[kk][0]); acc[kk][1] = fmaf(gv[j], r0[j + 1], acc[kk][1]);
            acc[kk][2] = fmaf(gv[j], r0[j + 2], acc[kk][2]);
            acc[kk][3] = fmaf(gv[j], r1[j], acc[kk][3]); acc[kk][4] = fmaf(gv[j], r1[j + 1], acc[kk][4]);
            acc[kk][5] = fmaf(gv[j], r1[j + 2], acc[kk][5]);
            acc[kk][6] = fmaf(gv[j], r2[j], acc[kk][6]); acc[kk][7] = fmaf(gv[j], r2[j + 1], acc[kk][7]);
            acc[kk][8] = fmaf(gv[j], r2[j + 2], acc[kk][8]);
            acc[kk][9] += gv[j];
          }
        }
      }
    }
  }
  const int lane = tid & 31, wp = tid >> 5;
#pragma unroll
  for (int kk = 0; kk < K; ++kk)
#pragma unroll
    for (int q = 0; q < 10; ++q) {
      const float v = warp_sum(acc[kk][q]);
      if (lane == 0) red[kk * 10 + q][wp] = v;
    }
  __syncthreads();
  auto flush = [&](int r) {   // sum r of the K * 10
    const int nw = (blockDim.x + 31) >> 5;
    float v = 0.f;
    for (int i = 0; i < nw; ++i) v += red[r][i];
    const int kk = r / 10, q = r - kk * 10;
    const int o = c * K + kk;
    if (q < 9) atomicAdd(p.dw + (int64_t)o * 9 + q, v);
    else if (p.db) atomicAdd(p.db + o, v);
  };
  // small planes launch a single warp: one sum per thread up to K = 3, a second pass at K = 4 (40 sums)
  if constexpr (K * 10 <= 32) {
    if (tid < K * 10) flush(tid);
  } else {
    for (int r = tid; r < K * 10; r += blockDim.x) flush(r);
  }
}

static bool dwb_tma_geometry(int H, int W, DwbParams* p, int* rh, int* threads) {
  if (W % 4 != 0) return false;
  dw_pick_tile(H, W, &p->TW, &p->TH, rh);
  p->BW = p->TW + 8;
  p->BH = p->TH + 2;
  if (p->BW > 256 || p->BH > 256) return false;
  p->plane_floats = (p->BW * p->BH + 31) / 32 * 32;   // 128-byte aligned plane pitch in shared memory
  p->tiles_x = ceil_div(W, p->TW);
  p->tiles_y = ceil_div(H, p->TH);
  p->H = H; p->W = W;
  const int nstrips = (p->TW / 4) * (p->TH / *rh);
  *threads = ((nstrips < 256 ? nstrips : 256) + 31) / 32 * 32;
  return true;
}

template <typename Kern>
static int dwb_set_smem(Kern kern, size_t smem, const char* what) {
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "%s: smem attribute: %s", what, cudaGetErrorString(e));
  }
  return SMAAT_OK;
}

template <int K, int RH>
static int launch_dwb_input(const CUtensorMap& mg, const DwbParams& p, int64_t grid, int threads, cudaStream_t st) {
  const size_t smem = (size_t)K * p.plane_floats * sizeof(float);
  auto kern = dw3x3_bwd_input_tma<K, RH>;
  if (int r = dwb_set_smem(kern, smem, "dw3x3_bwd_input")) return r;
  kern<<<(unsigned)grid, threads, smem, st>>>(mg, p);
  SMAAT_LAUNCH_CHECK("smaat_dw3x3_bwd_input");
  return SMAAT_OK;
}

template <int K, int RH, bool PRO>
static int launch_dwb_weight(const CUtensorMap& m0, const CUtensorMap& m1, const CUtensorMap& mg, const DwbParams& p, int64_t grid,
                             int threads, cudaStream_t st) {
  const size_t smem = ((size_t)p.plane_floats + (size_t)K * p.TW * p.TH) * sizeof(float);   // input halo tile + K gradient tiles
  auto kern = dw3x3_bwd_weight_tma<K, RH, PRO>;
  if (int r = dwb_set_smem(kern, smem, "dw3x3_bwd_weight")) return r;
  kern<<<(unsigned)grid, threads, smem, st>>>(m0, m1, mg, p);
  SMAAT_LAUNCH_CHECK("smaat_dw3x3_bwd_weight");
  return SMAAT_OK;
}

// returns 1 when the TMA variant is not applicable (caller falls back), else SMAAT_OK / error
static int dwb_input_try_tma(const float* dd, const float* w, float* dx0, int C0, int64_t bs0, float* dx1, int C1, int64_t bs1,
                             int B, int H, int W, int k, cudaStream_t st) {
  DwbParams p;
  memset(&p, 0, sizeof(p));
  int rh, threads;
  if (!(k == 1 || k == 2 || k == 4) || !dwb_tma_geometry(H, W, &p, &rh, &threads)) return 1;
  if (!aligned16(dd) || !aligned16(dx0) || bs0 % 4 != 0 || (C1 > 0 && (!aligned16(dx1) || bs1 % 4 != 0))) return 1;
  const int Cin = C0 + C1;
  p.g = dd; p.w = w; p.dx0 = dx0; p.dx1 = dx1; p.C0 = C0; p.C1 = C1; p.bs0 = bs0; p.bs1 = bs1;
  CUtensorMap mg;
  memset(&mg, 0, sizeof(mg));
  const uint32_t box[4] = {(uint32_t)p.BW, (uint32_t)p.BH, 1u, 1u};
  const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)Cin * k, (uint64_t)B};
  const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)Cin * k * H * W * 4};
  if (int r = make_tmap_f32(&mg, dd, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "dw3x3_bwd_input(dd)")) return r;
  const int64_t grid = (int64_t)B * Cin * p.tiles_x * p.tiles_y;
  SMAAT_REQUIRE(grid < (1ll << 31), "dw3x3_bwd_input: grid too large");
  if (k == 1) return rh == 8 ? launch_dwb_input<1, 8>(mg, p, grid, threads, st) : launch_dwb_input<1, 4>(mg, p, grid, threads, st);
  if (k == 2) return rh == 8 ? launch_dwb_input<2, 8>(mg, p, grid, threads, st) : launch_dwb_input<2, 4>(mg, p, grid, threads, st);
  return rh == 8 ? launch_dwb_input<4, 8>(mg, p, grid, threads, st) : launch_dwb_input<4, 4>(mg, p, grid, threads, st);
}

static int dwb_weight_try_tma(const float* dd, const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1,
                              const float* in_scale, const float* in_shift, float* dw, float* db, int B, int H, int W, int k,
                              cudaStream_t st) {
  DwbParams p;
  memset(&p, 0, sizeof(p));
  int rh, threads;
  if (!(k == 1 || k == 2 || k == 4) || !dwb_tma_geometry(H, W, &p, &rh, &threads)) return 1;
  if (!aligned16(dd) || !aligned16(x0) || bs0 % 4 != 0 || (C1 > 0 && (!aligned16(x1) || bs1 % 4 != 0))) return 1;
  p.g = dd; p.C0 = C0; p.C1 = C1; p.bs0 = bs0; p.bs1 = bs1; p.in_scale = in_scale; p.in_shift = in_shift; p.dw = dw; p.db = db;
  CUtensorMap m0, m1;
  memset(&m0, 0, sizeof(m0));
  memset(&m1, 0, sizeof(m1));
  const uint32_t box[4] = {(uint32_t)p.BW, (uint32_t)p.BH, 1u, 1u};
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C0, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)bs0 * 4};
    if (int r = make_tmap_f32(&m0, x0, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "dw3x3_bwd_weight(x0)")) return r;
  }
  if (C1 > 0) {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C1, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)bs1 * 4};
    if (int r = make_tmap_f32(&m1, x1, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "dw3x3_bwd_weight(x1)")) return r;
  } else {
    m1 = m0;
  }
  CUtensorMap mg;   // gradient planes: one box = TW x TH x k planes of this input channel
  memset(&mg, 0, sizeof(mg));
  {
    const int Cin = C0 + C1;
    const uint32_t gbox[4] = {(uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)k, 1u};
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)Cin * k, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)Cin * k * H * W * 4};
    if (int r = make_tmap_f32(&mg, dd, 4, dims, str, gbox, CU_TENSOR_MAP_SWIZZLE_NONE, "dw3x3_bwd_weight(dd)")) return r;
  }
  const int64_t grid = (int64_t)B * (C0 + C1) * p.tiles_x * p.tiles_y;
  SMAAT_REQUIRE(grid < (1ll << 31), "dw3x3_bwd_weight: grid too large");
  const bool pro = in_scale != nullptr;
#define SMAAT_DWB_W(KK, RR) \
  (pro ? launch_dwb_weight<KK, RR, true>(m0, m1, mg, p, grid, threads, st) : launch_dwb_weight<KK, RR, false>(m0, m1, mg, p, grid, threads, st))
  if (k == 1) return rh == 8 ? SMAAT_DWB_W(1, 8) : SMAAT_DWB_W(1, 4);
  if (k == 2) return rh == 8 ? SMAAT_DWB_W(2, 8) : SMAAT_DWB_W(2, 4);
  return rh == 8 ? SMAAT_DWB_W(4, 8) : SMAAT_DWB_W(4, 4);
#undef SMAAT_DWB_W
}

int dw3x3_bwd_input_tiled_launch(const float* dd, const float* w, float* dx0, int C0, int64_t bs0, float* dx1, int C1, int64_t bs1,
                                 int B, int H, int W, int k, cudaStream_t st) {
  {
    const int r = dwb_input_try_tma(dd, w, dx0, C0, bs0, dx1, C1, bs1, B, H, W, k, st);
    if (r != 1) return r;
  }
  const int TW = pick_tw(W);
  const int tiles_x = ceil_div(W, TW), tiles_y = ceil_div(H, DB_TH);
  const int64_t grid = (int64_t)B * (C0 + C1) * tiles_x * tiles_y;
  SMAAT_REQUIRE(grid < (1ll << 31), "dw3x3_bwd_input: grid too large");
  const size_t smem = (size_t)k * (DB_TH + 2) * (TW + 2) * sizeof(float);
  dw3x3_bwd_input_tiled<<<(unsigned)grid, 256, smem, st>>>(dd, w, dx0, C0, bs0, dx1, C1, bs1, H, W, k, TW, tiles_x, tiles_y);
  SMAAT_LAUNCH_CHECK("smaat_dw3x3_bwd_input");
  return SMAAT_OK;
}

int dw3x3_bwd_weight_tiled_launch(const float* dd, const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1,
                                  const float* in_scale, const float* in_shift, float* dw, float* db, int B, int H, int W, int k,
                                  cudaStream_t st) {
  {
    const int r = dwb_weight_try_tma(dd, x0, C0, bs0, x1, C1, bs1, in_scale, in_shift, dw, db, B, H, W, k, st);
    if (r != 1) return r;
  }
  const int TW = pick_tw(W);
  const int tiles_x = ceil_div(W, TW), tiles_y = ceil_div(H, DB_TH);
  const int64_t grid = (int64_t)B * (C0 + C1) * tiles_x * tiles_y;
  SMAAT_REQUIRE(grid < (1ll << 31), "dw3x3_bwd_weight: grid too large");
  const size_t smem = (size_t)(DB_TH + 2) * (TW + 2) * sizeof(float);
  dw3x3_bwd_weight_tiled<<<(unsigned)grid, 256, smem, st>>>(dd, x0, C0, bs0, x1, C1, bs1, in_scale, in_shift, dw, db, H, W, k, TW,
                                                            tiles_x, tiles_y);
  SMAAT_LAUNCH_CHECK("smaat_dw3x3_bwd_weight");
  return SMAAT_OK;
}

}  // namespace smaat
