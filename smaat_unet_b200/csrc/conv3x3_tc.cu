// conv3x3_tc.cu -- dense 3x3 conv, padding 1, as an implicit GEMM on the Hopper tensor cores (wgmma, tf32, fp32 accumulate
// in registers), fused with the per-channel affine (+ReLU) epilogue and optional BatchNorm batch statistics.
//
// Replaces nn.Conv2d(Cin, Cout, 3, padding=1) + eval BatchNorm2d + ReLU of DoubleConv (reference models/unet_parts.py:16-21).
// The same kernel runs the input gradient: dX = conv3x3(dZ, W') with W'[c][o][dy][dx] = W[o][c][2-dy][2-dx]
// (smaat_conv3x3_pack_weight with flip_transpose), no affine, no ReLU.
//
// GEMM view, per tile:  D[128 pixels x N_TILE channels] += A[128 px x K] * B[N_TILE x K]^T,  K = 9 * Cin
//   M: a PH x PW = 128-pixel patch of one image (PW 32 or 16, whichever wastes fewer pixels on this layer's H x W).
//   N: Cout in passes of N_TILE (64 or 128, chosen from Cout alone: the tile shapes never depend on B, so results are
//      bit-identical across batch sizes).
//   K: walked as (32-channel chunk, tap).  Chunks never straddle the virtual concat [x0 | x1]: each source is padded to a
//      multiple of 32 channels in the packed weight ([Cout][tap][C0p | C1p], K-major), and the TMA zero fill past a source's
//      last channel meets zero weights.
//   A: per chunk, warp 0 loads ONE halo box of BH x (PW + 8) x 32 channels (box origin (x0 - 4, y0 - 1): the inner TMA
//      coordinate must be 16-byte aligned; out-of-bounds zero fill is the padding).  All 9 taps read their shifted window
//      straight from that box: each consumer thread loads its register-A fragment at the tap's offset (design "registers
//      from the halo box"; the producers never copy windows).  A fragment register holds 8 consecutive pixels of one row
//      for 4 channel rows; the box is BH = PH + 3 rows tall so that the channel pitch BH * (PW + 8) is 8 or 24 mod 32 words:
//      the 32 lanes of every fragment load then hit 32 different banks, at any tap.  (The alternative, producer warps
//      copying each shifted window into a swizzled [k][pixel] ring, was not built, so no measurement chose between them.)
//   B: warp 1 streams the packed weight of one (chunk, tap) per stage as a 128-byte-swizzled K-major box [N_TILE x 32]
//      (hi, and lo in TF32X3 mode), through its own ring: one halo chunk feeds 9 weight stages.
// TF32X3: the activations are split into tf32 hi/lo in registers, the weights arrive pre-split (smaat_split_tf32 of the
// packed weight); three MMAs (hi*hi + lo*hi + hi*lo) per k-step.
// BF16: the activations are rounded to bf16 in registers (two k8 fragments -> one k16 fragment, tc_common.cuh bf16_frag), the
// weights arrive as smaat_pack_bf16 of the packed weight (every (chunk, tap) box starts on a multiple of 32 columns, so the
// pack's k permutation lines up with the fragments); 64-byte swizzled boxes, one m64nNk16 MMA per 16 k.
//
// Persistent: one CTA per SM loops over tiles (channel pass fastest, so consecutive tiles re-read the same halo from L2).
// Warps 4-11 = two consumer warpgroups (64 pixels each).  Epilogue as pw1x1_tc.cu: affine/ReLU -> batch-strided NCHW stores,
// BatchNorm sums from the raw accumulators in fp64 shared-memory partials (pixels outside the image masked), the affine
// applied analytically at the flush.  Statistics work for every Cout (passes of N_TILE flush separately).
#include "tc_common.cuh"

namespace smaat {

struct C3Params {
  const float* scale;
  const float* shift;
  float* y;
  int64_t y_bstride;
  double* stats;
  int H, W, Cout, relu;
  int c0p;        // x0's channels padded to 32: the packed-weight channel offset of x1's chunks
  int kc;         // channels per tap in the packed weight (c0p + c1p)
  int nch0, nch;  // chunks read from x0, chunks in total
  int tiles_x, tiles_y, tiles_n, total_tiles;
};

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

template <int N_TILE, int PW, Prec P>
struct C3Cfg {
  static constexpr bool X3 = P == Prec::TF32X3;
  static constexpr int PH = TC_BM / PW;
  static constexpr int BW = PW + 8;
  static constexpr int BH = PH + 3;                 // one spare row: see the bank note in the header
  static constexpr int CP = BH * BW;                // channel pitch of the halo box (words)
  static_assert(CP % 32 == 8 || CP % 32 == 24, "halo channel pitch must keep fragment loads conflict-free");
  static constexpr int IS = 2;                      // halo ring depth
  static constexpr int IN_BYTES = TC_BK * CP * 4;
  static_assert((IS * IN_BYTES) % 1024 == 0, "weight ring must start 1 KB aligned");
  static constexpr int WB_BYTES = N_TILE * TC_BK * (P == Prec::BF16 ? 2 : 4);
  static constexpr int WST_BYTES = (X3 ? 2 : 1) * WB_BYTES;
  // weight ring depth; BF16 keeps TF32's (its stages are half the size: the barrier block holds no more)
  static constexpr int WS = (96 * 1024) / ((X3 ? 2 : 1) * N_TILE * TC_BK * 4);
  static constexpr int OFF_W = IS * IN_BYTES;
  static constexpr int OFF_BAR = OFF_W + WS * WST_BYTES;
  static constexpr int BAR_BYTES = 256;
  static_assert(8 * 2 * (IS + WS) <= BAR_BYTES, "barriers");
  static constexpr int AFF_N = 1024;
  static constexpr int OFF_AFF = OFF_BAR + BAR_BYTES;
  static constexpr int OFF_SACC = OFF_AFF + 2 * AFF_N * 4;
  static constexpr int SACC_BYTES = 8 * 2 * N_TILE * 8;
  static constexpr int TOTAL = OFF_SACC + SACC_BYTES + 1024;
  static_assert(TOTAL <= 227 * 1024, "shared memory budget");
  static constexpr int THREADS = 384;
};

template <int N_TILE, int PW, Prec P>
__global__ void __launch_bounds__(384, 1)
    conv3x3_tc_kernel(const __grid_constant__ CUtensorMap map_x0, const __grid_constant__ CUtensorMap map_x1,
                      const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo, const C3Params p) {
  using L = C3Cfg<N_TILE, PW, P>;
  constexpr bool X3 = L::X3;
  constexpr int PH = L::PH, BW = L::BW, CP = L::CP, IS = L::IS, WS = L::WS;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* in_full = bars;
  uint64_t* in_empty = bars + IS;
  uint64_t* w_full = bars + 2 * IS;
  uint64_t* w_empty = bars + 2 * IS + WS;
  float* aff = reinterpret_cast<float*>(smem + L::OFF_AFF);  // [2][AFF_N] scale | shift

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_x0);
    tma_prefetch_desc(&map_x1);
    tma_prefetch_desc(&map_w);
    if (X3) tma_prefetch_desc(&map_wlo);
    for (int s = 0; s < IS; ++s) {
      mbar_init(&in_full[s], 1);
      mbar_init(&in_empty[s], 8);
    }
    for (int s = 0; s < WS; ++s) {
      mbar_init(&w_full[s], 1);
      mbar_init(&w_empty[s], 8);
    }
    fence_barrier_init();
  }
  for (int c = threadIdx.x; c < L::AFF_N; c += blockDim.x) {
    aff[c] = (c < p.Cout && p.scale) ? __ldg(p.scale + c) : 1.f;
    aff[L::AFF_N + c] = (c < p.Cout && p.shift) ? __ldg(p.shift + c) : 0.f;
  }
  __syncthreads();

  auto decode = [&](int tile, int& b, int& y0, int& x0, int& n0) {
    const int tn = tile % p.tiles_n;
    int r = tile / p.tiles_n;
    const int tx = r % p.tiles_x;
    r /= p.tiles_x;
    const int ty = r % p.tiles_y;
    b = r / p.tiles_y;
    x0 = tx * PW;
    y0 = ty * PH;
    n0 = tn * N_TILE;
  };

  if (warp == 0) {
    // ===== TMA: one halo box per 32-channel chunk =====
    if (lane == 0) {
      uint32_t gc = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int b, y0, x0, n0;
        decode(tile, b, y0, x0, n0);
        for (int i = 0; i < p.nch; ++i, ++gc) {
          const int s = gc % IS;
          mbar_wait(&in_empty[s], ((gc / IS) & 1u) ^ 1u);
          mbar_arrive_expect_tx(&in_full[s], L::IN_BYTES);
          const bool second = i >= p.nch0;
          const int cc = (second ? i - p.nch0 : i) * TC_BK;
          tma_load_4d(smem + s * L::IN_BYTES, second ? &map_x1 : &map_x0, &in_full[s], x0 - 4, y0 - 1, cc, b);
        }
      }
    }
    return;
  }
  if (warp == 1) {
    // ===== TMA: packed weights of one (chunk, tap) per stage =====
    if (lane == 0) {
      uint32_t gc = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int b, y0, x0, n0;
        decode(tile, b, y0, x0, n0);
        for (int i = 0; i < p.nch; ++i) {
          const int kofs = i < p.nch0 ? i * TC_BK : p.c0p + (i - p.nch0) * TC_BK;
          for (int tap = 0; tap < 9; ++tap, ++gc) {
            const int s = gc % WS;
            mbar_wait(&w_empty[s], ((gc / WS) & 1u) ^ 1u);
            mbar_arrive_expect_tx(&w_full[s], L::WST_BYTES);
            unsigned char* dst = smem + L::OFF_W + s * L::WST_BYTES;
            tma_load_2d(dst, &map_w, &w_full[s], tap * p.kc + kofs, n0);
            if (X3) tma_load_2d(dst + L::WB_BYTES, &map_wlo, &w_full[s], tap * p.kc + kofs, n0);
          }
        }
      }
    }
    return;
  }
  if (warp < 4) return;

  // ===== consumer warpgroups 1, 2 =====
  const int wg = (warp >> 2) - 1, wq = warp & 3, cw = warp - 4;
  const int g = lane >> 2, t = lane & 3;
  const int m0 = 64 * wg + 16 * wq + g, m1 = m0 + 8;   // accumulator rows g / g + 8: 8 consecutive pixels of one patch row
  const int h0 = m0 / PW, w0 = m0 % PW, h1 = m1 / PW, w1 = m1 % PW;
  // halo word offset of the thread's pixels at tap (0, 0), channel row t: box column 0 is image column x0 - 4
  const int base0 = t * CP + h0 * BW + w0 + 3, base1 = t * CP + h1 * BW + w1 + 3;
  const float act_lo = p.relu ? 0.f : -INFINITY;
  const int64_t HW = (int64_t)p.H * p.W;

  double* sacc = reinterpret_cast<double*>(smem + L::OFF_SACC) + cw * 2 * N_TILE;
  int stat_n0 = -1;
  if (p.stats) {
    for (int c = lane; c < 2 * N_TILE; c += 32) sacc[c] = 0.0;
    __syncwarp();
  }
  double stat_npix = 0.0;
  auto flush_stats = [&](int n0f) {
    __syncwarp();
    for (int c = lane; c < N_TILE; c += 32) {
      if (n0f + c < p.Cout) {
        const double sc = (double)aff[(n0f + c) & (L::AFF_N - 1)], sh = (double)aff[L::AFF_N + ((n0f + c) & (L::AFF_N - 1))];
        const double S1 = sacc[c], S2 = sacc[N_TILE + c];
        atomicAdd(p.stats + n0f + c, sc * S1 + stat_npix * sh);
        atomicAdd(p.stats + p.Cout + n0f + c, sc * sc * S2 + 2.0 * sc * sh * S1 + stat_npix * sh * sh);
      }
      sacc[c] = 0.0;
      sacc[N_TILE + c] = 0.0;
    }
    stat_npix = 0.0;
    __syncwarp();
  };

  uint32_t ic = 0, wc = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    int b, y0, x0, n0;
    decode(tile, b, y0, x0, n0);
    if (p.stats && n0 != stat_n0) {
      if (stat_n0 >= 0) flush_stats(stat_n0);
      stat_n0 = n0;
    }
    float acc[N_TILE / 2];
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) acc[i] = 0.f;
    for (int i = 0; i < p.nch; ++i, ++ic) {
      const int s = ic % IS;
      mbar_wait(&in_full[s], (ic / IS) & 1u);
      const float* hb = reinterpret_cast<const float*>(smem + s * L::IN_BYTES);
#pragma unroll 1
      for (int tap = 0; tap < 9; ++tap, ++wc) {
        const int ws = wc % WS;
        mbar_wait(&w_full[ws], (wc / WS) & 1u);
        const unsigned char* wst = smem + L::OFF_W + ws * L::WST_BYTES;
        const uint64_t bd0 = make_b_desc<P>(smem_u32(wst));
        const uint64_t bl0 = make_kmajor_desc(smem_u32(wst + L::WB_BYTES));
        const float* at = hb + (tap / 3) * BW + (tap % 3);
        if constexpr (P == Prec::BF16) {
          // both k16 fragments are written before the fence: registers an MMA reads may not change after it
          uint32_t af[TC_BK / 16][4];
#pragma unroll
          for (int s2 = 0; s2 < TC_BK / 16; ++s2) {
            const float* a0 = at + 16 * s2 * CP;
            const float* a1 = a0 + 8 * CP;
            const float v0[4] = {a0[base0], a0[base1], a0[base0 + 4 * CP], a0[base1 + 4 * CP]};
            const float v1[4] = {a1[base0], a1[base1], a1[base0 + 4 * CP], a1[base1 + 4 * CP]};
            bf16_frag(v0, v1, af[s2]);
          }
          wgmma_fence();
#pragma unroll
          for (int s2 = 0; s2 < TC_BK / 16; ++s2) Wgmma<N_TILE>::rs_bf16(acc, af[s2], bd0 + (uint64_t)(2 * s2), 1u);
        } else {
#pragma unroll
          for (int kk = 0; kk < TC_BK / 8; ++kk) {
            const float* ak = at + 8 * kk * CP;
            const float v[4] = {ak[base0], ak[base1], ak[base0 + 4 * CP], ak[base1 + 4 * CP]};
            uint32_t ahi[4], alo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float h = X3 ? tf32_hi(v[e]) : v[e];
              ahi[e] = __float_as_uint(h);
              alo[e] = __float_as_uint(v[e] - h);
            }
            wgmma_fence();
            Wgmma<N_TILE>::rs(acc, ahi, bd0 + (uint64_t)(2 * kk), 1u);
            if (X3) {
              Wgmma<N_TILE>::rs(acc, alo, bd0 + (uint64_t)(2 * kk), 1u);
              Wgmma<N_TILE>::rs(acc, ahi, bl0 + (uint64_t)(2 * kk), 1u);
            }
          }
        }
        wgmma_commit();
        wgmma_wait0();
        wgmma_keep(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&w_empty[ws]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&in_empty[s]);
    }

    // ----- epilogue: rows g / g + 8 are pixels (y0 + h0, x0 + w0) / (y0 + h1, x0 + w1), columns n0 + 8j + 2t + {0, 1}
    const int py0 = y0 + h0, px0 = x0 + w0, py1 = y0 + h1, px1 = x0 + w1;
    const bool v0 = py0 < p.H && px0 < p.W, v1 = py1 < p.H && px1 < p.W;
    const int64_t o0 = (int64_t)py0 * p.W + px0, o1 = (int64_t)py1 * p.W + px1;
    float* yb = p.y + (int64_t)b * p.y_bstride;
#pragma unroll
    for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = n0 + 8 * j + 2 * t + e;
        if (c < p.Cout) {
          const float sc = aff[c & (L::AFF_N - 1)], sh = aff[L::AFF_N + (c & (L::AFF_N - 1))];
          float* yc = yb + (int64_t)c * HW;
          if (v0) yc[o0] = fmaxf(fmaf(acc[4 * j + e], sc, sh), act_lo);
          if (v1) yc[o1] = fmaxf(fmaf(acc[4 * j + 2 + e], sc, sh), act_lo);
        }
      }
    }
    if (p.stats) {
      // raw accumulators of pixels outside the image are NOT zero (their windows overlap the image): mask them
#pragma unroll
      for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float a = v0 ? acc[4 * j + e] : 0.f, bb = v1 ? acc[4 * j + 2 + e] : 0.f;
          const float s1 = frag_colsum(a + bb), s2 = frag_colsum(fmaf(a, a, bb * bb));
          if (lane < 4) {
            const int col = 8 * j + 2 * t + e;
            sacc[col] += (double)s1;
            sacc[N_TILE + col] += (double)s2;
          }
        }
      }
      const int nv = __popc(__ballot_sync(0xffffffffu, v0)) + __popc(__ballot_sync(0xffffffffu, v1));
      stat_npix += (double)(nv / 4);
    }
  }
  if (p.stats && stat_n0 >= 0) flush_stats(stat_n0);
}

template <int N_TILE, int PW, Prec P>
static int launch_c3(const CUtensorMap& m0, const CUtensorMap& m1, const CUtensorMap& mw, const CUtensorMap& mwl, C3Params p, int B,
                     cudaStream_t st) {
  using L = C3Cfg<N_TILE, PW, P>;
  auto kern = conv3x3_tc_kernel<N_TILE, PW, P>;
  static std::atomic<uint64_t> attr_mask{0};
  if (first_use_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "conv3x3(tc): smem attribute (%d B): %s", L::TOTAL, cudaGetErrorString(e));
  }
  p.tiles_x = ceil_div(p.W, PW);
  p.tiles_y = ceil_div(p.H, L::PH);
  p.tiles_n = ceil_div(p.Cout, N_TILE);
  const int64_t total = (int64_t)B * p.tiles_x * p.tiles_y * p.tiles_n;
  SMAAT_REQUIRE(total < (1ll << 31), "conv3x3(tc): too many tiles");
  p.total_tiles = (int)total;
  const int grid = p.total_tiles < num_sms() ? p.total_tiles : num_sms();
  kern<<<grid, L::THREADS, L::TOTAL, st>>>(m0, m1, mw, mwl, p);
  SMAAT_LAUNCH_CHECK("smaat_conv3x3_fwd(tc)");
  return SMAAT_OK;
}

// Patch width with the fewest computed pixels for this layer (ties: 32).
static int c3_pick_pw(int H, int W) {
  const int64_t c32 = (int64_t)ceil_div(W, 32) * 32 * ceil_div(H, 4) * 4;
  const int64_t c16 = (int64_t)ceil_div(W, 16) * 16 * ceil_div(H, 8) * 8;
  return c16 < c32 ? 16 : 32;
}

bool conv3x3_tc_eligible(const float* x0, int64_t bs0, const float* x1, int C1, int64_t bs1, const float* wp, const float* wp_lo,
                         int W, int Cout) {
  if (W % 4 != 0 || Cout < 8 || !aligned16(x0) || bs0 % 4 != 0) return false;
  if (C1 > 0 && (!aligned16(x1) || bs1 % 4 != 0)) return false;
  return aligned16(wp) && (wp_lo == nullptr || aligned16(wp_lo));
}

int conv3x3_tc_launch(const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1, const float* wp, const float* wp_lo,
                      const float* scale, const float* shift, float* y, int64_t y_bstride, double* stats, int B, int H, int W, int Cout,
                      int relu, int mode, cudaStream_t st) {
  const bool x3 = mode == SMAAT_PW_TF32X3, bf16 = mode == SMAAT_PW_BF16;
  if (!conv3x3_tc_eligible(x0, bs0, x1, C1, bs1, wp, wp_lo, W, Cout))
    return fail(SMAAT_E_UNSUPPORTED, "conv3x3(tc): needs W %% 4 == 0, Cout >= 8, 16-byte aligned pointers and batch strides "
                "(W=%d Cout=%d); use SMAAT_PW_FP32_SIMT", W, Cout);
  SMAAT_REQUIRE(!x3 || wp_lo, "conv3x3(tc): TF32X3 needs wp_lo (smaat_split_tf32 of the packed weight)");
  SMAAT_REQUIRE(Cout <= 1024 || (!scale && !shift), "conv3x3(tc): Cout=%d > 1024 with an epilogue affine", Cout);
  const int pw = c3_pick_pw(H, W);
  const int ph = TC_BM / pw;
  const int n_tile = Cout > 64 ? 128 : 64;
  const int c0p = (C0 + TC_BK - 1) / TC_BK * TC_BK, c1p = (C1 + TC_BK - 1) / TC_BK * TC_BK;
  const int kc = c0p + c1p;

  CUtensorMap m0, m1, mw, mwl;
  const uint32_t box[4] = {(uint32_t)(pw + 8), (uint32_t)(ph + 3), (uint32_t)TC_BK, 1u};
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C0, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)bs0 * 4};
    int r = make_tmap_f32(&m0, x0, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "conv3x3(x0)");
    if (r) return r;
    m1 = m0;
  }
  if (C1 > 0) {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C1, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)bs1 * 4};
    int r = make_tmap_f32(&m1, x1, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "conv3x3(x1)");
    if (r) return r;
  }
  {
    // 9 kc is a multiple of 32: the bf16 pack of wp has wp's row length
    const uint64_t dims[2] = {(uint64_t)9 * kc, (uint64_t)Cout};
    const uint64_t str[2] = {0, (uint64_t)9 * kc * (bf16 ? 2 : 4)};
    const uint32_t wbox[2] = {(uint32_t)TC_BK, (uint32_t)n_tile};
    int r = bf16 ? make_tmap(&mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, wp, 2, dims, str, wbox, CU_TENSOR_MAP_SWIZZLE_64B, "conv3x3(w bf16)")
                 : make_tmap_f32(&mw, wp, 2, dims, str, wbox, CU_TENSOR_MAP_SWIZZLE_128B, "conv3x3(w)");
    if (r) return r;
    mwl = mw;
    if (x3) {
      r = make_tmap_f32(&mwl, wp_lo, 2, dims, str, wbox, CU_TENSOR_MAP_SWIZZLE_128B, "conv3x3(w_lo)");
      if (r) return r;
    }
  }
  C3Params p;
  p.scale = scale; p.shift = shift; p.y = y; p.y_bstride = y_bstride; p.stats = stats;
  p.H = H; p.W = W; p.Cout = Cout; p.relu = relu;
  p.c0p = c0p; p.kc = kc;
  p.nch0 = c0p / TC_BK; p.nch = kc / TC_BK;
  p.tiles_x = p.tiles_y = p.tiles_n = p.total_tiles = 0;

#define C3_DISPATCH(NT, PWv)                                                                     \
  return x3 ? launch_c3<NT, PWv, Prec::TF32X3>(m0, m1, mw, mwl, p, B, st)                           \
            : bf16 ? launch_c3<NT, PWv, Prec::BF16>(m0, m1, mw, mwl, p, B, st)                      \
                   : launch_c3<NT, PWv, Prec::TF32>(m0, m1, mw, mwl, p, B, st)
  if (n_tile == 128) {
    if (pw == 32) { C3_DISPATCH(128, 32); }
    C3_DISPATCH(128, 16);
  }
  if (pw == 32) { C3_DISPATCH(64, 32); }
  C3_DISPATCH(64, 16);
#undef C3_DISPATCH
}

}  // namespace smaat
