// pw1x1_wgrad_tc.cu -- pointwise 1x1 weight gradient on the Hopper tensor cores (wgmma, tf32):
//   dW[o][c] += sum_{b,p} dz[b,o,p] * d[b,c,p]        (Cout x K outputs, reduction over B*H*W pixels)
//
// Backward of DepthwiseSeparableConv.pointwise (reference models/layers.py:45,49).  Both operands have
// the reduction dimension (pixels) contiguous in NCHW, i.e. both are K-major for the MMA and both are read by
// the tensor core straight from shared memory:
//   A = dz viewed [B*Cout rows][P]  -> TMA box 128 rows x 32 px, SWIZZLE_128B (two consumer warpgroups x 64 rows)
//   B = d  viewed [B*K    rows][P]  -> TMA box N_TILE rows x 32 px, SWIZZLE_128B
//   D[128 x N_TILE] in registers accumulates over this CTA's slice of the (image, 32-pixel chunk) list;
// the slice results are merged into dW with fp32 atomics (split-K over pixels: the output is tiny,
// the reduction is B*P = millions long).  Rows of A beyond Cout / rows of B beyond K inside a box
// belong to neighbouring channels or images: they only produce D rows/columns that are never stored.
// TF32X3: the consumer warpgroups split BOTH landed tiles into tf32 hi (in place) + lo, three MMAs per
// k-step (hi*hi + lo*hi + hi*lo) -> fp32-grade gradients; TF32: one MMA on the raw fp32 tiles.
#include "tc_common.cuh"

namespace smaat {

// A = the operand on the M side (rows), B = the operand on the N side (columns).  Normally A = dz (Cout rows per
// image) and B = d (K rows); for Cout <= 64 the roles are swapped so the 128-row A box is not half empty (transposed = 1:
// D is dW^T).
struct WgParams {
  float* dW;
  int K, Cout, P, B;       // K = rows of the B-side operand per image, Cout = rows of the A-side operand per image
  int ldw, transposed;     // dW row pitch; 1 when D holds dW^T
  int chunks_per_img, total_chunks, chunks_per_split, tiles_o, tiles_c;
};

template <int N_TILE, bool X3>
struct WgCfg {
  static constexpr int A_BYTES = TC_BM * 128;     // 128 rows x 32 px
  static constexpr int B_BYTES = N_TILE * 128;
  static constexpr int STAGE_BYTES = (X3 ? 2 : 1) * (A_BYTES + B_BYTES);
  static constexpr int OFF_B = A_BYTES;
  static constexpr int OFF_LO = A_BYTES + B_BYTES;  // lo copies of [A | B] (X3)
  static constexpr int STAGES = (200 * 1024) / STAGE_BYTES > 6 ? 6 : (200 * 1024) / STAGE_BYTES;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 512 + 1024;
  static constexpr uint32_t TX = A_BYTES + B_BYTES;
  static constexpr int THREADS = 384;
  static_assert(STAGES >= 2, "pipeline depth");
};

template <int N_TILE, bool X3>
__global__ void __launch_bounds__(384, 1)
    pw1x1_wgrad_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_d, const WgParams p) {
  using L = WgCfg<N_TILE, X3>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * L::STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp-uniform for the compiler
  // work item: (o tile, c tile, pixel split)
  const int tile = blockIdx.x % (p.tiles_o * p.tiles_c);
  const int split = blockIdx.x / (p.tiles_o * p.tiles_c);
  const int o0 = (tile % p.tiles_o) * TC_BM;
  const int c0 = (tile / p.tiles_o) * N_TILE;
  const int ch_lo = split * p.chunks_per_split;
  const int ch_hi = min(p.total_chunks, ch_lo + p.chunks_per_split);
  const int nchunks = ch_hi - ch_lo;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_dz);
    tma_prefetch_desc(&map_d);
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
        const int b = ch / p.chunks_per_img;
        const int p0 = (ch - b * p.chunks_per_img) * 32;
        unsigned char* st = smem + s * L::STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[s], L::TX);
        tma_load_2d(st, &map_dz, &full_bar[s], p0, b * p.Cout + o0);
        tma_load_2d(st + L::OFF_B, &map_d, &full_bar[s], p0, b * p.K + c0);
      }
    }
    return;
  }
  if (warp < 4 || nchunks <= 0) return;

  // ===== consumer warpgroups 1, 2: warpgroup wg owns D rows 64 wg .. 64 wg + 63 =====
  const int wg = (warp >> 2) - 1, wq = warp & 3;
  const int ct = threadIdx.x - 128;   // 0..255
  float acc[N_TILE / 2];
#pragma unroll
  for (int i = 0; i < N_TILE / 2; ++i) acc[i] = 0.f;
  for (int i = 0; i < nchunks; ++i) {
    const int s = i % STAGES;
    mbar_wait(&full_bar[s], (i / STAGES) & 1u);
    unsigned char* st = smem + s * L::STAGE_BYTES;
    if (X3) {
      // split [A | B] into hi (in place) and lo; the named barrier makes the whole B split visible to both warpgroups
      float4* a4 = reinterpret_cast<float4*>(st);
      float4* l4 = reinterpret_cast<float4*>(st + L::OFF_LO);
#pragma unroll 4
      for (int idx = ct; idx < (L::A_BYTES + L::B_BYTES) / 16; idx += 256) {
        const float4 v = a4[idx];
        float4 h, l;
        h.x = tf32_hi(v.x); h.y = tf32_hi(v.y); h.z = tf32_hi(v.z); h.w = tf32_hi(v.w);
        l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
        a4[idx] = h;
        l4[idx] = l;
      }
      fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor-core (async) proxy
      consumer_sync();
    }
    const uint32_t a_addr = smem_u32(st) + (uint32_t)(wg * 64 * 128);
    const uint64_t ad0 = make_kmajor_desc(a_addr), bd0 = make_kmajor_desc(smem_u32(st + L::OFF_B));
    const uint64_t al0 = make_kmajor_desc(a_addr + L::OFF_LO), bl0 = make_kmajor_desc(smem_u32(st + L::OFF_LO + L::OFF_B));
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      Wgmma<N_TILE>::ss(acc, ad0 + (uint64_t)(2 * kk), bd0 + (uint64_t)(2 * kk), 1u);
      if (X3) {
        Wgmma<N_TILE>::ss(acc, al0 + (uint64_t)(2 * kk), bd0 + (uint64_t)(2 * kk), 1u);
        Wgmma<N_TILE>::ss(acc, ad0 + (uint64_t)(2 * kk), bl0 + (uint64_t)(2 * kk), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait0();
    wgmma_keep(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }

  // epilogue: D row = output channel o, column = input channel c
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int e2 = 0; e2 < 2; ++e2) {
    const int o = o0 + 64 * wg + 16 * wq + g + 8 * e2;
    if (o >= p.Cout) continue;
#pragma unroll
    for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = c0 + 8 * j + 2 * t + e;
        if (c >= p.K) continue;
        const float v = acc[4 * j + 2 * e2 + e];
        if (p.transposed) atomicAdd(p.dW + (int64_t)c * p.ldw + o, v);   // D[o][c] = dW[c][o]
        else atomicAdd(p.dW + (int64_t)o * p.ldw + c, v);
      }
    }
  }
}

template <int N_TILE, bool X3>
static int launch_wg(const CUtensorMap& mz, const CUtensorMap& md, WgParams p, cudaStream_t st) {
  using L = WgCfg<N_TILE, X3>;
  auto kern = pw1x1_wgrad_kernel<N_TILE, X3>;
  static std::atomic<uint64_t> attr_mask{0};   // cudaFuncSetAttribute is per device
  if (first_use_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL);
    if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "pw1x1_wgrad: smem attribute: %s", cudaGetErrorString(e));
  }
  p.tiles_o = ceil_div(p.Cout, TC_BM);
  p.tiles_c = ceil_div(p.K, N_TILE);
  p.chunks_per_img = ceil_div(p.P, 32);
  p.total_chunks = p.B * p.chunks_per_img;
  const int tiles = p.tiles_o * p.tiles_c;
  int splits = ceil_div(num_sms() * 2, tiles);                 // ~2 waves of CTAs
  const int min_chunks = 16;                                    // amortise the atomics of a slice
  if (splits > ceil_div(p.total_chunks, min_chunks)) splits = ceil_div(p.total_chunks, min_chunks);
  if (splits < 1) splits = 1;
  p.chunks_per_split = ceil_div(p.total_chunks, splits);
  splits = ceil_div(p.total_chunks, p.chunks_per_split);
  kern<<<tiles * splits, L::THREADS, L::TOTAL, st>>>(mz, md, p);
  SMAAT_LAUNCH_CHECK("smaat_pw1x1_bwd_weight(tc)");
  return SMAAT_OK;
}

bool pw1x1_wgrad_tc_eligible(const float* dz, const float* d, int K, int Cout, int P) {
  return (P % 4 == 0) && aligned16(dz) && aligned16(d) && Cout >= 8 && K >= 8;
}

int pw1x1_wgrad_tc_launch(const float* dz, const float* d, float* dW, int B, int K, int Cout, int P, bool x3, cudaStream_t st) {
  CUtensorMap mz, md;
  const int ldw = K;
  int transposed = 0;
  if (Cout <= 64 && K > Cout) {   // put the longer operand on the 128-row M side
    const float* t = dz; dz = d; d = t;
    const int ti = K; K = Cout; Cout = ti;
    transposed = 1;
  }
  const int n_tile = K > 64 ? 128 : 64;   // accumulators in registers: N_TILE / 2 per thread
  {
    const uint64_t dims[2] = {(uint64_t)P, (uint64_t)B * Cout};
    const uint64_t str[2] = {0, (uint64_t)P * 4};
    const uint32_t box[2] = {32u, (uint32_t)TC_BM};
    int r = make_tmap_f32(&mz, dz, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "pw1x1_wgrad(dz)");
    if (r) return r;
  }
  {
    const uint64_t dims[2] = {(uint64_t)P, (uint64_t)B * K};
    const uint64_t str[2] = {0, (uint64_t)P * 4};
    const uint32_t box[2] = {32u, (uint32_t)n_tile};
    int r = make_tmap_f32(&md, d, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "pw1x1_wgrad(d)");
    if (r) return r;
  }
  WgParams p;
  p.dW = dW; p.K = K; p.Cout = Cout; p.P = P; p.B = B; p.ldw = ldw; p.transposed = transposed;
  p.chunks_per_img = p.total_chunks = p.chunks_per_split = p.tiles_o = p.tiles_c = 0;
  if (x3) {
    if (n_tile == 128) return launch_wg<128, true>(mz, md, p, st);
    return launch_wg<64, true>(mz, md, p, st);
  }
  if (n_tile == 128) return launch_wg<128, false>(mz, md, p, st);
  return launch_wg<64, false>(mz, md, p, st);
}

}  // namespace smaat

namespace smaat {
// db[c] += sum_{b,p} x[b,c,p]
__global__ void __launch_bounds__(256) channel_sum_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int C, int P,
                                                          int chunks) {
  const int c = blockIdx.y;
  const int64_t n = (int64_t)B * P;
  const int64_t per = (n + chunks - 1) / chunks;
  const int64_t lo = (int64_t)blockIdx.x * per, hi = min(n, lo + per);
  float s = 0.f;
  for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const int64_t b = i / P, pp = i - b * P;
    s += __ldg(x + (b * C + c) * (int64_t)P + pp);
  }
  __shared__ float red[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int i = 0; i < 8; ++i) v += red[i];
    atomicAdd(out + c, v);
  }
}
}  // namespace smaat

using namespace smaat;

/* Tensor-core variant of smaat_pw1x1_bwd_weight (mode SMAAT_PW_TF32 or SMAAT_PW_TF32X3); returns
 * SMAAT_E_UNSUPPORTED for shapes TMA cannot describe (P % 4 != 0): use smaat_pw1x1_bwd_weight then. */
extern "C" int smaat_pw1x1_bwd_weight_tc(const float* dz, const float* d, float* dW, float* db, int B, int K, int Cout, int P,
                                         int mode, void* stream) {
  SMAAT_REQUIRE(dz && d && dW && B > 0 && K > 0 && Cout > 0 && P > 0, "pw1x1_bwd_weight_tc: bad arguments");
  SMAAT_REQUIRE(mode == SMAAT_PW_TF32 || mode == SMAAT_PW_TF32X3, "pw1x1_bwd_weight_tc: mode must be TF32 or TF32X3");
  if (!pw1x1_wgrad_tc_eligible(dz, d, K, Cout, P)) return fail(SMAAT_E_UNSUPPORTED, "pw1x1_bwd_weight_tc: shape not TMA-describable");
  cudaStream_t st = (cudaStream_t)stream;
  int r = pw1x1_wgrad_tc_launch(dz, d, dW, B, K, Cout, P, mode == SMAAT_PW_TF32X3, st);
  if (r) return r;
  if (db) {
    SMAAT_REQUIRE(Cout <= 65535, "pw1x1_bwd_weight_tc: Cout too large");
    int chunks = (int)ceil_div64((int64_t)B * P, 256 * 64);
    const int maxc = ceil_div(num_sms() * 8, Cout);
    if (chunks > maxc) chunks = maxc;
    if (chunks < 1) chunks = 1;
    channel_sum_kernel<<<dim3(chunks, Cout), 256, 0, st>>>(dz, db, B, Cout, P, chunks);
    SMAAT_LAUNCH_CHECK("smaat_pw1x1_bwd_weight_tc(bias)");
  }
  return SMAAT_OK;
}
