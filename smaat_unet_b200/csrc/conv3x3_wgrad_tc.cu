// conv3x3_wgrad_tc.cu -- weight gradient of the dense 3x3 conv (padding 1) on the Hopper tensor cores (wgmma, tf32):
//   dW[o][c][dy][dx] += sum_{b,y,x} dz[b,o,y,x] * in[b,c,y+dy-1,x+dx-1]      (zero outside the image)
//
// Backward of nn.Conv2d(Cin, Cout, 3, padding=1) of DoubleConv (reference models/unet_parts.py:16,19); `in` may be the
// virtual concat [x0 | x1] of Up (unet_parts.py:63).  As in pw1x1_wgrad_tc.cu both operands have the reduction dimension
// (pixels) contiguous, so both are K-major and the tensor core reads both from shared memory; split-K over
// (image, row, 32-pixel segment) chunks with fp32 atomics into dW, which is written in the nn.Conv2d layout.
//   A = dz: TMA box of 32 px x 1 row x 128 output channels, SWIZZLE_128B -> [128 o][32 px] K-major (two warpgroups x 64 rows).
//       Loaded once per chunk and used for the three taps of the CTA's kernel row dy.
//   B = the input, shifted per tap: warp 0 stages ONE halo row per chunk (TMA box (32 + 8) px x 1 row x 64 channels, origin
//       (x0 - 4, y + dy - 1); out-of-bounds zero fill is the padding), and the 256 consumer threads copy the three dx-shifted
//       windows of it into 128B-swizzled K-major tiles [64 c][32 px] (as tf32 hi + lo in TF32X3 mode).
//   D: three m64n64 accumulators per warpgroup (one per dx), in registers.
// Pixels past the image width are zero in the dz box, so every product they take part in vanishes: no masks.  Channel tiles
// never straddle the concat (tiles over x0's channels, then over x1's); rows / columns of D past Cout / the source's channels
// are never stored.  The grid is (o tile, c tile, dy, pixel split): dz is read three times, once per kernel row.
#include "tc_common.cuh"

namespace smaat {

struct C3wParams {
  float* dW;
  int C0, C1, Cout, W, H, B;
  int tiles_o, tiles_c0, tiles_c;     // channel tiles of x0, of x0 and x1 together
  int nseg, total_chunks, chunks_per_split;
};

__device__ __forceinline__ void tma_load_4d_w(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

template <bool X3>
struct C3wCfg {
  static constexpr int NT = 64;                       // input channels per tile (N)
  static constexpr int A_BYTES = TC_BM * 128;         // [128 o][32 px]
  static constexpr int HALO_W = 40;
  static constexpr int HALO_BYTES = NT * HALO_W * 4;  // [64 c][40 px]
  static constexpr int STAGE_BYTES = A_BYTES + HALO_BYTES;
  static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
  static constexpr int STAGES = 4;
  static constexpr int BT_BYTES = NT * 128;           // one tap's [64 c][32 px] tile
  static constexpr int OFF_ALO = STAGES * STAGE_BYTES;
  static constexpr int OFF_B = OFF_ALO + (X3 ? A_BYTES : 0);
  static constexpr int OFF_BLO = OFF_B + 3 * BT_BYTES;
  static constexpr int OFF_BAR = OFF_BLO + (X3 ? 3 * BT_BYTES : 0);
  static constexpr int TOTAL = OFF_BAR + 256 + 1024;
  static_assert(TOTAL <= 227 * 1024, "shared memory budget");
  static constexpr uint32_t TX = STAGE_BYTES;
};

template <bool X3>
__global__ void __launch_bounds__(384, 1)
    conv3x3_wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_x0,
                            const __grid_constant__ CUtensorMap map_x1, const C3wParams p) {
  using L = C3wCfg<X3>;
  constexpr int STAGES = L::STAGES, NT = L::NT;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  // work item: (o tile, c tile, kernel row dy, pixel split)
  int r = blockIdx.x;
  const int to = r % p.tiles_o;
  r /= p.tiles_o;
  const int tc = r % p.tiles_c;
  r /= p.tiles_c;
  const int dy = r % 3;
  const int split = r / 3;
  const int o0 = to * TC_BM;
  const bool second = tc >= p.tiles_c0;
  const int cs0 = (second ? tc - p.tiles_c0 : tc) * NT;   // first channel of the tile inside its source
  const int csrc = second ? p.C1 : p.C0;
  const int cglob0 = (second ? p.C0 : 0) + cs0;            // its channel index in the concat
  const int ch_lo = split * p.chunks_per_split;
  const int ch_hi = min(p.total_chunks, ch_lo + p.chunks_per_split);
  const int nchunks = ch_hi - ch_lo;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_dz);
    tma_prefetch_desc(second ? &map_x1 : &map_x0);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      for (int i = 0; i < nchunks; ++i) {
        const int s = i % STAGES;
        mbar_wait(&empty_bar[s], ((i / STAGES) & 1u) ^ 1u);
        const int ch = ch_lo + i;
        const int seg = ch % p.nseg;
        const int y = (ch / p.nseg) % p.H;
        const int b = ch / (p.nseg * p.H);
        unsigned char* st = smem + s * L::STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[s], L::TX);
        tma_load_4d_w(st, &map_dz, &full_bar[s], seg * 32, y, o0, b);
        tma_load_4d_w(st + L::A_BYTES, second ? &map_x1 : &map_x0, &full_bar[s], seg * 32 - 4, y + dy - 1, cs0, b);
      }
    }
    return;
  }
  if (warp < 4 || nchunks <= 0) return;

  const int wg = (warp >> 2) - 1, wq = warp & 3;
  const int ct = threadIdx.x - 128;   // 0..255
  float acc[3][NT / 2];
#pragma unroll
  for (int d = 0; d < 3; ++d)
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[d][i] = 0.f;

  for (int i = 0; i < nchunks; ++i) {
    const int s = i % STAGES;
    mbar_wait(&full_bar[s], (i / STAGES) & 1u);
    unsigned char* st = smem + s * L::STAGE_BYTES;
    const float* halo = reinterpret_cast<const float*>(st + L::A_BYTES);
    // the three dx-shifted windows of the halo row -> K-major SW128 tiles (tf32 hi / lo in X3 mode)
#pragma unroll 4
    for (int idx = ct; idx < 3 * NT * 32; idx += 256) {
      const int px = idx & 31, c = (idx >> 5) % NT, dx = idx / (NT * 32);
      const float v = halo[c * L::HALO_W + px + dx + 3];     // box column 0 is image column x0 - 4
      const uint32_t off = (uint32_t)(dx * L::BT_BYTES) + kmajor_offset(c, px);
      const float h = X3 ? tf32_hi(v) : v;
      *reinterpret_cast<float*>(smem + L::OFF_B + off) = h;
      if (X3) *reinterpret_cast<float*>(smem + L::OFF_BLO + off) = v - h;
    }
    if (X3) {   // split the dz tile into hi (in place) + lo
      float4* a4 = reinterpret_cast<float4*>(st);
      float4* l4 = reinterpret_cast<float4*>(smem + L::OFF_ALO);
#pragma unroll 4
      for (int idx = ct; idx < L::A_BYTES / 16; idx += 256) {
        const float4 v = a4[idx];
        float4 h, l;
        h.x = tf32_hi(v.x); h.y = tf32_hi(v.y); h.z = tf32_hi(v.z); h.w = tf32_hi(v.w);
        l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
        a4[idx] = h;
        l4[idx] = l;
      }
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor-core (async) proxy
    consumer_sync();
    const uint32_t a_addr = smem_u32(st) + (uint32_t)(wg * 64 * 128);
    const uint64_t ad0 = make_kmajor_desc(a_addr);
    const uint64_t al0 = make_kmajor_desc(smem_u32(smem + L::OFF_ALO) + (uint32_t)(wg * 64 * 128));
    wgmma_fence();
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const uint64_t bd0 = make_kmajor_desc(smem_u32(smem + L::OFF_B + dx * L::BT_BYTES));
      const uint64_t bl0 = make_kmajor_desc(smem_u32(smem + L::OFF_BLO + dx * L::BT_BYTES));
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        Wgmma<NT>::ss(acc[dx], ad0 + (uint64_t)(2 * kk), bd0 + (uint64_t)(2 * kk), 1u);
        if (X3) {
          Wgmma<NT>::ss(acc[dx], al0 + (uint64_t)(2 * kk), bd0 + (uint64_t)(2 * kk), 1u);
          Wgmma<NT>::ss(acc[dx], ad0 + (uint64_t)(2 * kk), bl0 + (uint64_t)(2 * kk), 1u);
        }
      }
    }
    wgmma_commit();
    wgmma_wait0();
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) wgmma_keep(acc[dx]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
    consumer_sync();   // both warpgroups are done with the shifted tiles before the next chunk overwrites them
  }

  // epilogue: D row = output channel o, column = input channel c (of the source), one accumulator per dx
  const int g = lane >> 2, t = lane & 3;
  const int Cin = p.C0 + p.C1;
#pragma unroll
  for (int e2 = 0; e2 < 2; ++e2) {
    const int o = o0 + 64 * wg + 16 * wq + g + 8 * e2;
    if (o >= p.Cout) continue;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int cl = 8 * j + 2 * t + e;
        if (cs0 + cl >= csrc) continue;
        float* dst = p.dW + ((int64_t)o * Cin + cglob0 + cl) * 9 + 3 * dy;
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) atomicAdd(dst + dx, acc[dx][4 * j + 2 * e2 + e]);
      }
    }
  }
}

bool conv3x3_wgrad_tc_eligible(const float* dz, const float* x0, int64_t bs0, const float* x1, int C1, int64_t bs1, int W) {
  if (W % 4 != 0 || !aligned16(dz) || !aligned16(x0) || bs0 % 4 != 0) return false;
  return C1 == 0 || (aligned16(x1) && bs1 % 4 == 0);
}

template <bool X3>
static int launch_c3w(const CUtensorMap& mz, const CUtensorMap& m0, const CUtensorMap& m1, C3wParams p, cudaStream_t st) {
  using L = C3wCfg<X3>;
  auto kern = conv3x3_wgrad_tc_kernel<X3>;
  static std::atomic<uint64_t> attr_mask{0};
  if (first_use_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "conv3x3_wgrad(tc): smem attribute: %s", cudaGetErrorString(e));
  }
  const int64_t tiles = (int64_t)p.tiles_o * p.tiles_c * 3;
  int64_t splits = ceil_div64(2 * (int64_t)num_sms(), tiles);     // ~2 waves of CTAs
  const int64_t min_chunks = 16;                                   // amortise the atomics of a slice
  if (splits > ceil_div64(p.total_chunks, min_chunks)) splits = ceil_div64(p.total_chunks, min_chunks);
  if (splits < 1) splits = 1;
  p.chunks_per_split = (int)ceil_div64(p.total_chunks, splits);
  splits = ceil_div64(p.total_chunks, p.chunks_per_split);
  SMAAT_REQUIRE(tiles * splits < (1ll << 31), "conv3x3_wgrad(tc): grid too large");
  kern<<<(unsigned)(tiles * splits), 384, L::TOTAL, st>>>(mz, m0, m1, p);
  SMAAT_LAUNCH_CHECK("smaat_conv3x3_bwd_weight(tc)");
  return SMAAT_OK;
}

int conv3x3_wgrad_tc_launch(const float* dz, const float* x0, int C0, int64_t bs0, const float* x1, int C1, int64_t bs1, float* dW,
                            int B, int H, int W, int Cout, bool x3, cudaStream_t st) {
  if (!conv3x3_wgrad_tc_eligible(dz, x0, bs0, x1, C1, bs1, W))
    return fail(SMAAT_E_UNSUPPORTED, "conv3x3_bwd_weight(tc): needs W %% 4 == 0, 16-byte aligned pointers and batch strides (W=%d); "
                "use SMAAT_PW_FP32_SIMT", W);
  constexpr int NT = C3wCfg<false>::NT;
  CUtensorMap mz, m0, m1;
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)Cout, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)Cout * H * W * 4};
    const uint32_t box[4] = {32u, 1u, (uint32_t)TC_BM, 1u};
    int r = make_tmap_f32(&mz, dz, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "conv3x3_wgrad(dz)");
    if (r) return r;
  }
  const uint32_t hbox[4] = {(uint32_t)C3wCfg<false>::HALO_W, 1u, (uint32_t)NT, 1u};
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C0, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)bs0 * 4};
    int r = make_tmap_f32(&m0, x0, 4, dims, str, hbox, CU_TENSOR_MAP_SWIZZLE_NONE, "conv3x3_wgrad(x0)");
    if (r) return r;
    m1 = m0;
  }
  if (C1 > 0) {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C1, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4, (uint64_t)bs1 * 4};
    int r = make_tmap_f32(&m1, x1, 4, dims, str, hbox, CU_TENSOR_MAP_SWIZZLE_NONE, "conv3x3_wgrad(x1)");
    if (r) return r;
  }
  C3wParams p;
  p.dW = dW; p.C0 = C0; p.C1 = C1; p.Cout = Cout; p.W = W; p.H = H; p.B = B;
  p.tiles_o = ceil_div(Cout, TC_BM);
  p.tiles_c0 = ceil_div(C0, NT);
  p.tiles_c = p.tiles_c0 + (C1 > 0 ? ceil_div(C1, NT) : 0);
  p.nseg = ceil_div(W, 32);
  const int64_t total = (int64_t)B * H * p.nseg;
  SMAAT_REQUIRE(total < (1ll << 31), "conv3x3_wgrad(tc): too many pixel chunks");
  p.total_chunks = (int)total;
  p.chunks_per_split = 0;
  return x3 ? launch_c3w<true>(mz, m0, m1, p, st) : launch_c3w<false>(mz, m0, m1, p, st);
}

}  // namespace smaat
