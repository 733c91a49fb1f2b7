// pw1x1_tc.cu -- pointwise 1x1 conv on the Hopper tensor cores (wgmma, tf32, fp32 accumulate in registers), fused with the
// per-channel affine (+ReLU) epilogue and optional BatchNorm statistics.
//
// Replaces DepthwiseSeparableConv.pointwise + eval BatchNorm2d + ReLU
// (reference models/layers.py:45,49; parts_ds.py:25-26,34-35): the only dense contraction
// on the SmaAt-UNet forward path.
//
// Mapping (per image b):  D[128 pixels x N_TILE channels] += A[128 px x 8] * B[N_TILE x 8]^T
//   A = activations X[b] ([K][P], pixels contiguous): consumed as it lies in HBM, no transpose.  TMA boxes of 32 k-rows x
//       32 px (4 boxes = 128 pixels) with the 128-byte swizzle; each consumer thread loads its A fragment into registers
//       (tf32 wgmma reads only K-major operands from shared memory, this one is MN-major) -- conflict-free, see tc_common.cuh;
//   B = weights W ([Cout][K], K contiguous) -> K-major SW128 operand, one TMA box of N_TILE rows x 32 k;
//   D in registers of two consumer warpgroups (64 pixels each).
// TF32X3 mode (fp32-grade accuracy): the activations are split into a tf32 "hi" part and the "lo" remainder in registers,
// the weights arrive pre-split; three MMAs (hi*hi + lo*hi + hi*lo) per k-step accumulate into the same registers.
// BF16 mode: the activations are rounded to bf16 in registers, the weights arrive as a smaat_pack_bf16 pack ([Cout][K rounded
// up to 32], K-major, 64-byte rows: TMA SWIZZLE_64B); one m64nNk16 MMA per 16 k.
//
// Persistent: one CTA per SM loops over output tiles (tile = blockIdx.x + i*gridDim.x; consecutive tiles share the activation
// tile and differ in the channel tile, so the re-read hits L2).  Warp 0 = TMA producer, running ahead across tile boundaries
// through a STAGES-deep shared-memory ring, so the loads of the next tile overlap the epilogue of this one; warpgroups 1-2 =
// MMA + epilogue.  mbarriers: full (TMA bytes) / empty (8 consumer warps done reading) per stage.  The k loop keeps one
// chunk's MMAs in flight while the previous chunk retires and its stage is released (two register-A fragment sets in turn;
// setmaxnreg moves warpgroup 0's spare registers to the consumers for them).
#include <stdlib.h>

#include "tc_common.cuh"

namespace smaat {

struct PwTcParams {
  const float* scale;
  const float* shift;
  float* y;
  int64_t y_bstride;
  double* stats;
  int K, Cout, P, relu;
  int tiles_m, tiles_n, total_tiles;
};

template <int N_TILE, int STAGES, Prec P>
struct PwTcCfg {
  static constexpr bool X3 = P == Prec::TF32X3;
  static constexpr int A_BYTES = TC_BM * TC_BK * 4;   // 16 KB: 4 blocks x (32 k-rows x 128 B)
  static constexpr int B_BYTES = N_TILE * TC_BK * (P == Prec::BF16 ? 2 : 4);  // N_TILE rows x 128 B (bf16: 64 B)
  static constexpr int STAGE_BYTES = A_BYTES + (X3 ? 2 : 1) * B_BYTES;
  static constexpr int OFF_B = A_BYTES;
  static constexpr int OFF_BLO = A_BYTES + B_BYTES;  // X3 only
  static constexpr int BAR_BYTES = 256;
  static constexpr int AFF_N = 512;                                      // per-channel epilogue affine staged in smem
  static constexpr int SACC_BYTES = 8 * 2 * N_TILE * 8;                  // per-consumer-warp fp64 BatchNorm partial sums
  static constexpr int TOTAL = STAGES * STAGE_BYTES + BAR_BYTES + 2 * AFF_N * 4 + SACC_BYTES + 1024;  // + alignment slack
  static constexpr uint32_t TX_BYTES = A_BYTES + (X3 ? 2 : 1) * B_BYTES;
  static constexpr int THREADS = 384;
  // setmaxnreg split of the 3 x 168 registers per thread the CTA launches with (__launch_bounds__(384, 1))
  static constexpr int REGS_TMA = 40, REGS_MMA = 232;
  static_assert(REGS_TMA + 2 * REGS_MMA <= 3 * 168, "register budget");
  // the consumers hold two stages (chunk i in flight, chunk i - 1 retiring): the TMA warp needs a third to run ahead
  static_assert(STAGES >= 3, "ring depth");
  static_assert(TOTAL <= 227 * 1024, "shared memory budget");
};

template <int N_TILE, int STAGES, Prec P>
__global__ void __launch_bounds__(384, 1)
    pw1x1_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const __grid_constant__ CUtensorMap map_wlo, const PwTcParams p) {
  using L = PwTcCfg<N_TILE, STAGES, P>;
  constexpr bool X3 = L::X3;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  // 1 KB alignment: 128-byte swizzle atoms.  Offset arithmetic on the __shared__ array (not a uintptr_t round trip) keeps the
  // accesses LDS/STS instead of generic LD/ST.
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * L::STAGE_BYTES);
  float* aff = reinterpret_cast<float*>(smem + STAGES * L::STAGE_BYTES + L::BAR_BYTES);  // [2][AFF_N] scale | shift
  uint64_t* full_bar = bars;            // [STAGES] TMA bytes landed
  uint64_t* empty_bar = bars + STAGES;  // [STAGES] the 8 consumer warps finished with the stage

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler too
  const int lane = threadIdx.x & 31;
  const int nk = (p.K + TC_BK - 1) / TC_BK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_x);
    tma_prefetch_desc(&map_w);
    if (X3) tma_prefetch_desc(&map_wlo);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    fence_barrier_init();
  }
  // epilogue affine of the channels this CTA can touch (padded with identity; all-identity when no affine is given,
  // which is why indices may wrap for Cout > AFF_N)
  for (int c = threadIdx.x; c < L::AFF_N; c += blockDim.x) {
    aff[c] = (c < p.Cout && p.scale) ? __ldg(p.scale + c) : 1.f;
    aff[L::AFF_N + c] = (c < p.Cout && p.shift) ? __ldg(p.shift + c) : 0.f;
  }
  __syncthreads();

  if (warp < 4) {
    // warpgroup 0 keeps few registers: the consumers' two register-A fragment sets need them (all four warps reallocate)
    regs_dealloc<L::REGS_TMA>();
    // ===== TMA producer =====
    if (warp == 0 && lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int tn = tile % p.tiles_n;
        const int rest = tile / p.tiles_n;
        const int tm = rest % p.tiles_m;
        const int b = rest / p.tiles_m;
        const int p0 = tm * TC_BM, n0 = tn * N_TILE;
        for (int i = 0; i < nk; ++i, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1u;
          mbar_wait(&empty_bar[s], ph ^ 1u);
          unsigned char* st = smem + s * L::STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[s], L::TX_BYTES);
          const int k0 = i * TC_BK;
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_load_3d(st + j * (TC_BK * 128), &map_x, &full_bar[s], p0 + 32 * j, k0, b);
          tma_load_2d(st + L::OFF_B, &map_w, &full_bar[s], k0, n0);
          if (X3) tma_load_2d(st + L::OFF_BLO, &map_wlo, &full_bar[s], k0, n0);
        }
      }
    }
    return;
  }
  regs_alloc<L::REGS_MMA>();

  // ===== consumer warpgroups 1, 2: MMAs into register accumulators, then affine/ReLU -> NCHW stores =====
  const int wg = (warp >> 2) - 1, wq = warp & 3, cw = warp - 4;   // cw: consumer warp 0..7
  const int g = lane >> 2, t = lane & 3;
  const int m0 = tc_row_pixel(wg, wq, 0, g), m1 = tc_row_pixel(wg, wq, 1, g);
  const float act_lo = p.relu ? 0.f : -INFINITY;  // ReLU as a branch-free max()
  // BatchNorm batch statistics: this warp's fp64 partial sums [2][N_TILE] live in shared memory across the CTA's tiles
  // (lanes 0..3 own the columns of their fragment group: no atomics) and reach HBM once per n-tile change / at the end
  double* sacc = reinterpret_cast<double*>(smem + STAGES * L::STAGE_BYTES + L::BAR_BYTES + 2 * L::AFF_N * 4) + cw * 2 * N_TILE;
  int stat_n0 = -1;
  if (p.stats) {
    for (int c = lane; c < 2 * N_TILE; c += 32) sacc[c] = 0.0;
    __syncwarp();
  }
  double stat_npix = 0.0;   // valid pixels this warp has accumulated since the last flush (warp-uniform)
  auto flush_stats = [&](int n0f) {
    __syncwarp();
    for (int c = lane; c < N_TILE; c += 32) {
      if (n0f + c < p.Cout) {
        // z = sc * acc + sh:  sum z = sc*S1 + n*sh,  sum z^2 = sc^2*S2 + 2*sc*sh*S1 + n*sh^2
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

  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const int tn = tile % p.tiles_n;
    const int rest = tile / p.tiles_n;
    const int tm = rest % p.tiles_m;
    const int b = rest / p.tiles_m;
    const int n0 = tn * N_TILE;
    if (p.stats && n0 != stat_n0) {
      if (stat_n0 >= 0) flush_stats(stat_n0);
      stat_n0 = n0;
    }
    float acc[N_TILE / 2];
#pragma unroll
    for (int i = 0; i < N_TILE / 2; ++i) acc[i] = 0.f;
    // Pipelined k loop: chunk i's MMAs are issued as one group, then the wait leaves that group in flight and retires chunk
    // i - 1, whose stage goes back to the TMA warp.  Chunk i's fragments must stay untouched until it retires, so two
    // fragment sets alternate (the loop is unrolled by 2; no control-flow path may load a set whose chunk is still in
    // flight, or ptxas serialises the MMAs: the odd tail is outside the loop)
    auto release = [&](uint32_t c) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[c % STAGES]);
    };
    auto chunk = [&](AFrags<P>& cur, AFrags<P>& prev, int i) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1u);
      const unsigned char* st = smem + s * L::STAGE_BYTES;
      load_a_frags<P, TC_BK / 8>(st, 0, t, m0, m1, cur);
      mma_a_frags<N_TILE, P, TC_BK / 8>(acc, cur, make_b_desc<P>(smem_u32(st + L::OFF_B)),
                                        make_kmajor_desc(smem_u32(st + L::OFF_BLO)), 0);
      wgmma_wait<1>();
      wgmma_keep(prev);
      if (i > 0) release(it - 1);
      ++it;
    };
    AFrags<P> fa, fb;
    int i = 0;
    for (; i + 1 < nk; i += 2) {
      chunk(fa, fb, i);
      chunk(fb, fa, i + 1);
    }
    if (i < nk) chunk(fa, fb, i);
    // the tile's last chunk retires before the epilogue; its stage is released first, so TMA runs on through the epilogue
    wgmma_wait0();
    wgmma_keep(acc);
    wgmma_keep(fa);
    wgmma_keep(fb);
    release(it - 1);

    // ----- epilogue: rows g / g + 8 are pixels m0 / m1, columns n0 + 8j + 2t + {0, 1}
    const int pix0 = tm * TC_BM + m0, pix1 = tm * TC_BM + m1;
    const bool v0 = pix0 < p.P, v1 = pix1 < p.P;
    float* yb = p.y + (int64_t)b * p.y_bstride;
#pragma unroll
    for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = n0 + 8 * j + 2 * t + e;
        if (c < p.Cout) {
          const float sc = aff[c & (L::AFF_N - 1)], sh = aff[L::AFF_N + (c & (L::AFF_N - 1))];
          float* yc = yb + (int64_t)c * p.P;
          if (v0) yc[pix0] = fmaxf(fmaf(acc[4 * j + e], sc, sh), act_lo);
          if (v1) yc[pix1] = fmaxf(fmaf(acc[4 * j + 2 + e], sc, sh), act_lo);
        }
      }
    }
    if (p.stats) {
      // BatchNorm batch statistics from the RAW accumulators.  Pixels past P and channels past Cout are exact zeros (TMA zero
      // fill), so no masks; the epilogue affine is applied analytically when the sums are flushed.
#pragma unroll
      for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float a = acc[4 * j + e], bb = acc[4 * j + 2 + e];
          const float s1 = frag_colsum(a + bb), s2 = frag_colsum(fmaf(a, a, bb * bb));
          if (lane < 4) {
            const int col = 8 * j + 2 * t + e;
            sacc[col] += (double)s1;
            sacc[N_TILE + col] += (double)s2;
          }
        }
      }
      const int nv = __popc(__ballot_sync(0xffffffffu, v0)) + __popc(__ballot_sync(0xffffffffu, v1));
      stat_npix += (double)(nv / 4);   // each pixel row is held by the 4 lanes of its fragment group
    }
  }
  if (p.stats && stat_n0 >= 0) flush_stats(stat_n0);
}

template <int N_TILE, int STAGES, Prec P>
static int launch_tc(const CUtensorMap& mx, const CUtensorMap& mw, const CUtensorMap& mwl, PwTcParams p, int B, cudaStream_t st) {
  using L = PwTcCfg<N_TILE, STAGES, P>;
  auto kern = pw1x1_tc_kernel<N_TILE, STAGES, P>;
  static std::atomic<uint64_t> attr_mask{0};   // cudaFuncSetAttribute is per device
  if (first_use_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "pw1x1(tc): smem attribute (%d B): %s", L::TOTAL, cudaGetErrorString(e));
    int r = check_reg_budget((const void*)kern, L::THREADS, L::REGS_TMA + 2 * L::REGS_MMA, "pw1x1(tc)");
    if (r) return r;
  }
  p.tiles_m = ceil_div(p.P, TC_BM);
  p.tiles_n = ceil_div(p.Cout, N_TILE);
  const int64_t total = (int64_t)B * p.tiles_m * p.tiles_n;
  SMAAT_REQUIRE(total < (1ll << 31), "pw1x1(tc): too many tiles");
  p.total_tiles = (int)total;
  const int grid = p.total_tiles < num_sms() ? p.total_tiles : num_sms();
  kern<<<grid, L::THREADS, L::TOTAL, st>>>(mx, mw, mwl, p);
  SMAAT_LAUNCH_CHECK("smaat_pw1x1_fwd(tc)");
  return SMAAT_OK;
}

bool pw1x1_tc_eligible(const float* x, const float* w, const float* w_lo, int K, int Cout, int P) {
  return (P % 4 == 0) && (K % 4 == 0) && aligned16(x) && aligned16(w) && (w_lo == nullptr || aligned16(w_lo)) && Cout >= 8;
}

// mode: SMAAT_PW_TF32, SMAAT_PW_TF32X3 (w the tf32 hi parts, w_lo the lo parts) or SMAAT_PW_BF16 (w the smaat_pack_bf16 pack of
// the (Cout, K) weight: (Cout, K rounded up to 32) bf16)
int pw1x1_tc_launch(const float* x, const float* w, const float* w_lo, const float* scale, const float* shift, float* y,
                    int64_t y_bstride, double* stats, int B, int K, int Cout, int P, int relu, int mode, cudaStream_t st) {
  const bool x3 = mode == SMAAT_PW_TF32X3, bf16 = mode == SMAAT_PW_BF16;
  SMAAT_REQUIRE(pw1x1_tc_eligible(x, w, w_lo, K, Cout, P), "pw1x1(tc): needs P %% 4 == 0, K %% 4 == 0 and 16-byte aligned x/w");
  SMAAT_REQUIRE(!x3 || w_lo, "pw1x1(tc): TF32X3 needs w_lo (see smaat_split_tf32)");
  SMAAT_REQUIRE(Cout <= 512 || (!scale && !shift), "pw1x1(tc): Cout=%d > 512 with an epilogue affine (smem staging holds 512 channels)", Cout);
  // the tile shape depends on the layer only, never on the batch: results stay bit-identical across batch sizes.  N_TILE is
  // at most 128: the accumulators of a 64 x N_TILE warpgroup tile live in registers (N_TILE / 2 per thread).
  const int n_tile = Cout > 64 ? 128 : 64;

  CUtensorMap mx, mw, mwl;
  {
    const uint64_t dims[3] = {(uint64_t)P, (uint64_t)K, (uint64_t)B};
    const uint64_t str[3] = {0, (uint64_t)P * 4, (uint64_t)K * P * 4};
    const uint32_t box[3] = {32u, (uint32_t)TC_BK, 1u};
    int r = make_tmap_f32(&mx, x, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "pw1x1(x)");
    if (r) return r;
  }
  {
    const uint64_t kw = bf16 ? (uint64_t)(K + TC_BK - 1) / TC_BK * TC_BK : (uint64_t)K;   // the bf16 pack's row length
    const uint64_t dims[2] = {kw, (uint64_t)Cout};
    const uint64_t str[2] = {0, kw * (bf16 ? 2 : 4)};
    const uint32_t box[2] = {(uint32_t)TC_BK, (uint32_t)n_tile};
    int r = bf16 ? make_tmap(&mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, w, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B, "pw1x1(w bf16)")
                 : make_tmap_f32(&mw, w, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "pw1x1(w)");
    if (r) return r;
    mwl = mw;
    if (x3) {
      r = make_tmap_f32(&mwl, w_lo, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "pw1x1(w_lo)");
      if (r) return r;
    }
  }
  PwTcParams p;
  p.scale = scale; p.shift = shift; p.y = y; p.y_bstride = y_bstride; p.stats = stats;
  p.K = K; p.Cout = Cout; p.P = P; p.relu = relu;
  p.tiles_m = p.tiles_n = p.total_tiles = 0;

  // one persistent CTA per SM: the smem ring takes ~150-200 KB of the 227 KB.  BF16 keeps TF32's depths (its stages are
  // smaller: 24 / 20 KB instead of 32 / 24 KB)
  if (x3) {
    if (n_tile == 128) return launch_tc<128, 4, Prec::TF32X3>(mx, mw, mwl, p, B, st);
    return launch_tc<64, 5, Prec::TF32X3>(mx, mw, mwl, p, B, st);
  }
  if (bf16) {
    if (n_tile == 128) return launch_tc<128, 5, Prec::BF16>(mx, mw, mwl, p, B, st);
    return launch_tc<64, 6, Prec::BF16>(mx, mw, mwl, p, B, st);
  }
  if (n_tile == 128) return launch_tc<128, 5, Prec::TF32>(mx, mw, mwl, p, B, st);
  return launch_tc<64, 6, Prec::TF32>(mx, mw, mwl, p, B, st);
}

}  // namespace smaat
