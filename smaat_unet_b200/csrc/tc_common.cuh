// tc_common.cuh -- Hopper warpgroup-MMA (wgmma) helpers shared by the tensor-core kernels (pw1x1_tc.cu, pw1x1_wgrad_tc.cu,
// dsconv_fused.cu).
//
// tf32 wgmma takes shared-memory operands only K-major.  The activations of the forward kernels lie pixels-contiguous (NCHW),
// i.e. MN-major for the pixel-rows operand, so that operand goes through registers: each thread loads its A fragment from a
// 128B-swizzled [k][32 px] tile (what TMA SWIZZLE_128B writes, or what the depthwise producers write) and issues the RS form.
// (The fused DS conv's producers can instead write their result K-major, for the tensor core to read: kmajor_offset.)
// The weights ([Cout][K], K contiguous) are the K-major B operand, read by the tensor core through a descriptor.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace smaat {

constexpr int TC_BM = 128;  // pixels per tile: two consumer warpgroups x m64
constexpr int TC_BK = 32;   // k per stage (one 128-byte swizzle row of fp32)

// Operand precision of a tensor-core instance: one tf32 pass (SMAAT_PW_TF32), the 3xTF32 split (SMAAT_PW_TF32X3), or bf16
// operands with fp32 accumulation (SMAAT_PW_BF16: A rounded to bf16 in registers, B a smaat_pack_bf16 pack, one
// m64nNk16 MMA per 16 k)
enum class Prec : int { TF32 = 0, TF32X3 = 1, BF16 = 2 };

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Wait until at most N committed MMA groups of this warpgroup are still pending.  The pipelined main loops commit one group
// per k-chunk (or half chunk) and wait with N = 1: the previous group has retired (the shared-memory stages of a chunk whose
// groups have all retired may be handed back) while the newest one runs.
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_keep(float (&d)[N]) {   // accumulators are live across the asynchronous MMAs
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// The same for register-A fragments: placed after the wait that retires the MMAs reading them, it keeps them live (and
// unmodified) until then, so ptxas neither reuses their registers early nor serialises the MMAs.
template <int P, int K>
__device__ __forceinline__ void wgmma_keep(uint32_t (&a)[P][K][4]) {
#pragma unroll
  for (int p = 0; p < P; ++p)
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
      for (int e = 0; e < 4; ++e) asm volatile("" : "+r"(a[p][k][e])::"memory");
}

// Warpgroup register reallocation (setmaxnreg): every warp of the warpgroup executes the same value.  Warpgroups that only
// issue TMA give registers back, the MMA warpgroups take them, within the CTA's launch allocation.
template <int R>
__device__ __forceinline__ void regs_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void regs_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Host check, once per device before a launch: the sum of the warpgroups' setmaxnreg targets (`regs_sum`, registers per
// thread summed over the CTA's warpgroups) must fit in what the CTA is launched with, or an increase would wait forever.
inline int check_reg_budget(const void* kern, int threads, int regs_sum, const char* who) {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, kern);
  if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "%s: cudaFuncGetAttributes: %s", who, cudaGetErrorString(e));
  const int launched = ((a.numRegs + 7) / 8) * 8 * (threads / 128);
  if (launched < regs_sum)
    return fail(SMAAT_E_CUDA, "%s: built with %d registers per thread, the warpgroups' register split needs %d per 128 threads > %d",
                who, a.numRegs, regs_sum, launched);
  return SMAAT_OK;
}

// Shared-memory matrix descriptor (sm_90 GMMA layout): addr>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64)
// with 1 = SWIZZLE_128B.  K-major SW128 operand: rows of 128 B (32 tf32), 8-row atoms 1 KB apart (SBO); one k8 step is 32 B
// along the row = +2 in the address field.  The tile base must be 1 KB aligned.
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fffu);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// The same for a K-major bf16 operand with 64-byte rows (32 bf16 of k) and the 64-byte swizzle (layout type 2): 8-row atoms
// 512 B apart; one k16 step is 32 B along the row = +2 in the address field.  The tile base must be 512-byte aligned.
__device__ __forceinline__ uint64_t make_kmajor_desc_sw64(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fffu);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(512 >> 4) << 32;
  d |= (uint64_t)2 << 62;
  return d;
}
// B descriptor of a K-major weight tile in precision P: fp32 rows with the 128-byte swizzle, or bf16 rows with the 64-byte one
template <Prec P>
__device__ __forceinline__ uint64_t make_b_desc(uint32_t saddr) {
  return P == Prec::BF16 ? make_kmajor_desc_sw64(saddr) : make_kmajor_desc(saddr);
}

// Byte offset of activation element (k-row kr, pixel m) inside one A tile stored as 4 blocks of [32 k-rows][32 px] with the
// 128-byte swizzle (16-byte chunk index XOR k-row % 8) -- the layout TMA SWIZZLE_128B writes for a 32 px x 32 k box.
__device__ __forceinline__ uint32_t a_tile_offset(int kr, int m) {
  const int j = m >> 5, col = m & 31;
  return (uint32_t)(j * (TC_BK * 128) + kr * 128 + ((((col >> 2) ^ (kr & 7)) << 4) | ((col & 3) << 2)));
}

// Byte offset of element (row, k) of a K-major operand tile with 128-byte rows (32 tf32 of k) and the 128-byte swizzle
// (16-byte chunk index XOR row % 8): the layout make_kmajor_desc describes.
__device__ __forceinline__ uint32_t kmajor_offset(int row, int k) {
  return (uint32_t)(row * 128 + ((((k >> 2) ^ (row & 7)) << 4) | ((k & 3) << 2)));
}

// Pixel (0..127 of the tile) of accumulator row g + 8e of warp wq in consumer warpgroup wg.  A warp's 16 rows are half of a
// 32-pixel block; the 8 rows a fragment register covers are pixels {c..c+3, c+16..c+19}: with the swizzle above, the 32
// lanes of one fragment load (4 k-rows x those 8 pixels) then fall on 32 different banks.
__device__ __forceinline__ int tc_row_pixel(int wg, int wq, int e, int g) {
  return 64 * wg + 32 * (wq >> 1) + 4 * (2 * (wq & 1) + e) + (g & 3) + 16 * (g >> 2);
}

// The thread's A fragment of k-step kk (8 k-rows) from an A tile at `at`: rows m0 / m1 (its two pixels), k-rows 8kk + t, + 4.
__device__ __forceinline__ void load_a_frag(const unsigned char* at, int kk, int t, int m0, int m1, float (&v)[4]) {
  const int k0 = 8 * kk + t;
  v[0] = *reinterpret_cast<const float*>(at + a_tile_offset(k0, m0));
  v[1] = *reinterpret_cast<const float*>(at + a_tile_offset(k0, m1));
  v[2] = *reinterpret_cast<const float*>(at + a_tile_offset(k0 + 4, m0));
  v[3] = *reinterpret_cast<const float*>(at + a_tile_offset(k0 + 4, m1));
}

__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }

// Two fp32 -> one bf16x2 register, round to nearest even: `lo` in the low half (the lower k), `hi` in the high half
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// The bf16 register-A fragment of one k16 step from the tf32 fragments v0 / v1 of k-steps 2s / 2s + 1 (load_a_frag's layout).
// The MMA then sees logical k l of the 16 at physical k-row (l & 8) | ((l & 1) << 2) | ((l >> 1) & 3) of the step;
// smaat_pack_bf16 gives B the same permutation, so the sum over k is the same sum
__device__ __forceinline__ void bf16_frag(const float (&v0)[4], const float (&v1)[4], uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(v0[0], v0[2]);
  a[1] = pack_bf16x2(v0[1], v0[3]);
  a[2] = pack_bf16x2(v1[0], v1[2]);
  a[3] = pack_bf16x2(v1[1], v1[3]);
}

// Register-A fragments of KS tf32 k-steps (one commit group; TC_BK / 8 = 4 k-steps make a k-chunk): f[0][kk] = the values
// (tf32) or their tf32 hi parts (TF32X3), f[1][kk] = the lo remainders v - hi (TF32X3 only); in BF16 the KS / 2 k16
// fragments.  MMAs in flight read them until their group retires.
template <Prec P, int KS = TC_BK / 8>
using AFrags = uint32_t[P == Prec::TF32X3 ? 2 : 1][P == Prec::BF16 ? KS / 2 : KS][4];

// Loads k-steps kk0 .. kk0 + KS - 1 from an fp32 A tile at `at` and splits (TF32X3) or rounds (BF16) them in registers.
template <Prec P, int KS>
__device__ __forceinline__ void load_a_frags(const unsigned char* at, int kk0, int t, int m0, int m1, AFrags<P, KS>& f) {
  constexpr bool X3 = P == Prec::TF32X3;
  if constexpr (P == Prec::BF16) {
#pragma unroll
    for (int s = 0; s < KS / 2; ++s) {
      float v0[4], v1[4];
      load_a_frag(at, kk0 + 2 * s, t, m0, m1, v0);
      load_a_frag(at, kk0 + 2 * s + 1, t, m0, m1, v1);
      bf16_frag(v0, v1, f[0][s]);
    }
  } else {
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      float v[4];
      load_a_frag(at, kk0 + kk, t, m0, m1, v);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float h = X3 ? tf32_hi(v[e]) : v[e];
        f[0][kk][e] = __float_as_uint(h);
        if (X3) f[X3 ? 1 : 0][kk][e] = __float_as_uint(v[e] - h);
      }
    }
  }
}

// Step s of one commit group's MMAs, without fence or commit: tf32 k-step kk0 + s (TF32X3: A_hi B_hi + A_lo B_hi + A_hi B_lo),
// or the BF16 k16 step of k-steps kk0 + 2s, kk0 + 2s + 1.  bd / bl: descriptors of the chunk's B (hi) / lo tiles.  A k8 step of
// fp32 B and a k16 step of bf16 B are both 32 B along the row: + 2 in the descriptor's address field
template <int N_TILE, Prec P, int KS>
__device__ __forceinline__ void mma_a_step(float (&acc)[N_TILE / 2], const AFrags<P, KS>& f, uint64_t bd, uint64_t bl, int kk0,
                                           int s) {
  constexpr bool X3 = P == Prec::TF32X3;
  if constexpr (P == Prec::BF16) {
    Wgmma<N_TILE>::rs_bf16(acc, f[0][s], bd + (uint64_t)(2 * (kk0 / 2 + s)), 1u);
  } else {
    const uint64_t k2 = (uint64_t)(2 * (kk0 + s));
    Wgmma<N_TILE>::rs(acc, f[0][s], bd + k2, 1u);
    if (X3) {
      Wgmma<N_TILE>::rs(acc, f[X3 ? 1 : 0][s], bd + k2, 1u);
      Wgmma<N_TILE>::rs(acc, f[0][s], bl + k2, 1u);
    }
  }
}

// One fence, the MMAs of k-steps kk0 .. kk0 + KS - 1 for NH accumulator sets (the halves of the fused DS conv's paired tile,
// each with its own fragments) and one commit.  Step by step, each set's MMAs in turn against the same B: every accumulator
// sees the sequence of a single set
template <int N_TILE, Prec P, int KS, int NH>
__device__ __forceinline__ void mma_a_frags(float (&acc)[NH][N_TILE / 2], const AFrags<P, KS> (&f)[NH], uint64_t bd, uint64_t bl,
                                            int kk0) {
  wgmma_fence();
#pragma unroll
  for (int s = 0; s < (P == Prec::BF16 ? KS / 2 : KS); ++s)
#pragma unroll
    for (int h = 0; h < NH; ++h) mma_a_step<N_TILE, P, KS>(acc[h], f[h], bd, bl, kk0, s);
  wgmma_commit();
}
// The same for one accumulator set
template <int N_TILE, Prec P, int KS>
__device__ __forceinline__ void mma_a_frags(float (&acc)[N_TILE / 2], const AFrags<P, KS>& f, uint64_t bd, uint64_t bl, int kk0) {
  wgmma_fence();
#pragma unroll
  for (int s = 0; s < (P == Prec::BF16 ? KS / 2 : KS); ++s) mma_a_step<N_TILE, P, KS>(acc, f, bd, bl, kk0, s);
  wgmma_commit();
}

// Sums over the 8 lanes of a fragment column group (lanes with equal t): afterwards lanes 0..3 hold the totals.
__device__ __forceinline__ float frag_colsum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}

// Named barrier over the two consumer warpgroups (256 threads); id 0 is __syncthreads.
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

}  // namespace smaat
