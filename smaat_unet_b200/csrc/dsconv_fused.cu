// dsconv_fused.cu -- DepthwiseSeparableConv forward as ONE kernel: depthwise 3x3 on the CUDA
// cores feeding the pointwise 1x1 on the Hopper tensor cores (wgmma), with the BN-affine/ReLU epilogue.
//
// Replaces DepthwiseSeparableConv.forward (reference models/layers.py:47-50: depthwise then
// pointwise, nothing in between) + eval BatchNorm2d + ReLU (parts_ds.py:25-26,34-35) [+ OutConv,
// unet_parts.py:67-73, for the network's last conv].  The k x -expanded depthwise result never reaches
// HBM: per B=32 forward the DS blocks move 4*B*S^2*(Cin + Cout) bytes instead of
// 4*B*S^2*(Cin + 2*k*Cin + Cout).
//
// One persistent CTA per SM; a tile is a PH x PW = 128-pixel patch of one image and one pass of N_TILE <= 128 output
// channels (Cout <= 128: one pass, so the depthwise work is done exactly once; Cout in {256, 384, 512}: passes of 128).
// At Cout <= 64 a tile can instead be two such patches one above the other, sharing each chunk (DsCfg PAIR, dsconv_pair_kernel);
// at 128 < Cout <= 256 one patch and both 128-channel halves, fed by each chunk once (DsCfg WIDE, dsconv_wide_kernel).
// K = k*Cin is walked in chunks of 32 depthwise channels (CC = 32/k input channels):
//   warp 0      TMA: (PH+2) x (PW+8) x CC input halo box per chunk (OOB zero fill = padding=1; box
//               starts at x0-4, x0-8 for bf16 input: the inner TMA coordinate must be 16-byte aligned) into an IS-deep ring;
//               input may be the virtual concat [x0, x1] of UpDS (parts_ds.py:85).  An L2 prefetch of the next tile's boxes
//               (cp.async.bulk.prefetch.tensor) made bench.py's B = 32 forward slower: 2 220 vs 2 346-2 369 frames/s (H100
//               80GB HBM3 SXM, 700 W; two runs with, six without), so there is none
//   warp 1      prefetches the weight chunks (K-major SW128, [hi rows | lo rows]; BF16: the smaat_pack_bf16 pack, K-major SW64)
//               into their own ring
//               (warpgroup 0 runs on 24 registers per thread: setmaxnreg hands the rest to the consumers)
//   warps 4-11  two consumer warpgroups (64 pixels each): wgmma (TF32X3: A_hi B_hi + A_lo B_hi + A_hi B_lo per k-step) into
//               register accumulators, with the A operand either read by the tensor core from the A ring (A_SMEM) or
//               loaded into registers from it first (and split into tf32 hi / lo there in TF32X3 mode), then the epilogue:
//               scale/shift/ReLU -> NCHW (staged per 32-channel slice in shared memory and written by TMA tensor stores),
//               or the fused 1-class OutConv dot product; [+ BatchNorm batch statistics].
//               The main loop is pipelined: a chunk's MMAs are committed as one group (two half-chunk groups in the
//               register form at N_TILE 64 in TF32X3, where registers are short), the wait leaves the newest group in
//               flight, and the previous chunk's A and B stages are released once it retires.  The register form
//               alternates two fragment sets so that the set a group in flight reads is never overwritten
//   warps 12..  NG depthwise producer groups (128 threads each; group g takes every NG-th chunk): 3x3 stencil
//               from the staged tile with a sliding register window (one LDS.128 per row, edge columns from the
//               neighbouring quads by shuffle), then write the result into an AS-stage A ring in one of two layouts:
//                 A_SMEM   [pixel][k] 128B-swizzled K-major tiles, the layout wgmma reads through a descriptor (one scalar
//                          store per value: a thread's 4 pixels are 4 rows), as hi and lo tf32 parts in TF32X3 mode;
//                 !A_SMEM  [k][pixel] 128B-swizzled fp32 tiles (one 16-byte store per 4 pixels), which the consumers load
//                          into registers conflict-free (tc_common.cuh) and feed to wgmma's register-A form.  Storing fp32
//                          once instead of hi and lo halves the A ring's shared-memory traffic in TF32X3 mode; the split
//                          in the consumer is the same tf32_hi / v - hi on the same value, so results are unchanged
// Which A form a request runs in is smaat_set_dsconv_impl's choice.  ds_select (below) picks the whole instance that runs it
// (A form, single, paired or wide tile, precision, N_TILE, PW), and the eligibility entry points ask it, so they answer for
// that instance; ds_visit maps the choice to its DsCfg.
// BF16 (SMAAT_PW_BF16, dsconv_bf16_kernel): the register form only; the consumers round the fp32 A tiles to bf16 as they load
// them (two k8 fragments make one k16 fragment, tc_common.cuh bf16_frag), so the producers, the A ring and its layout are
// those of TF32, and the B stages are half as large.
#include <stdlib.h>

#include <type_traits>

#include "tc_common.cuh"

namespace smaat {

struct DsParams {
  const float* dw_w;
  const float* dw_b;
  const float* scale;
  const float* shift;
  float* y;
  int64_t y_bstride;
  double* stats;
  const float* oc_w;   // fused OutConv (1 class): logits = sum_c oc_w[c] * act[c] + oc_b, written instead of y
  const float* oc_b;
  float* oc_y;
  // CBAM fusions of the serving forward (smaat_dsconv_cbam_fwd).  gate_sc (B, C0): x0 is read as the CBAM output
  // (x0 * gate_sc[b, c]) * gate_sa[b, p], gate_sa coming in by its own TMA map.  pool_sum / pool_max (B, npart, Cout): per
  // half-patch partial sums / maxima of the output for the channel gate's pools; pooled (B, Cout, H / 2, W / 2): its 2x2 max-pool,
  // also without the pools (smaat_dsconv_maxpool_fwd), and from bf16 maps as bf16 (pooled_bf16) or fp32
  const float* gate_sc;
  float* pool_sum;
  float* pool_max;
  float* pooled;
  int pooled_bf16;
  int npart;
  // K-class OutConv + argmax (smaat_dsconv_classify_fwd): ncls > 0 classes, oc_w (ncls, Cout), oc_b (ncls) or null, oc_y the
  // (B, ncls, H, W) logits or null, cls the (B, H, W) class map or null
  int ncls;
  int64_t* cls;
  int C0, C1, H, W, Cout, relu, K;
  int tiles_x, tiles_y, npass, total_tiles, nchunks;
};

constexpr int DS_MAX_CLASSES = 32;   // classes of the fused K-class OutConv + argmax (smaat_dsconv_classify_fwd)
constexpr int DS_MIN_CLASSES = 21;   // ... that every instance keeps beside its rings (a 21-class model)

// TA: the storage type of the input (x0, x1) and of the output (y or the logits): float, or uint16_t for the bf16 activations
// of the serving forward's bf16 route (dsconv_bf16act_kernel)
// PAIR (dsconv_pair_kernel: N_TILE 64, register form, tf32 / 3xTF32, k = 2 and 4): a tile is two vertically adjacent patches
// (2 PH rows x PW, 256 pixels) that share each chunk's input box, weight chunk and barrier hand-offs; each half keeps the
// single tile's A layout, accumulator rows and epilogue
// WIDE (dsconv_wide_kernel: 128 < Cout <= 256, N_TILE 128 per channel half, register form, tf32 / 3xTF32, fp32 maps, k = 2): a tile is
// one patch and both 128-channel halves, so each chunk's input box and depthwise stencil feed 256 channels instead of being
// computed once per pass; each consumer warpgroup holds one accumulator set per half and feeds both from the same A fragments
template <int N_TILE, int KPL, int PW, Prec P, bool A_SMEM, typename TA = float, bool PAIR = false, bool WIDE = false>
struct DsCfg {
  static constexpr bool X3 = P == Prec::TF32X3;
  static constexpr int ESZ = (int)sizeof(TA);
  static_assert(ESZ == 4 || (P == Prec::BF16 && KPL != 4), "bf16 activations: the bf16 register-form instances, k = 1, 2");
  static_assert(P != Prec::BF16 || !A_SMEM, "BF16: register A form only");
  static_assert(!PAIR || (N_TILE == 64 && !A_SMEM && P != Prec::BF16 && ESZ == 4 && KPL != 1),
                "paired tiles: N_TILE 64, register form, tf32 / 3xTF32, fp32 maps, k = 2, 4");
  static_assert(!WIDE || (N_TILE == 128 && !PAIR && !A_SMEM && P != Prec::BF16 && ESZ == 4 && KPL == 2),
                "wide tiles: two N_TILE 128 halves, register form, tf32 / 3xTF32, fp32 maps, k = 2");
  static constexpr int PH = TC_BM / PW;
  static constexpr int NH = PAIR ? 2 : 1;                      // patches (halves) per tile
  static constexpr int NW = WIDE ? 2 : 1;                      // N_TILE channel halves per tile
  static constexpr int NA = NH * NW;                           // accumulator sets per consumer thread
  static constexpr int TH = NH * PH;                           // tile rows
  // input boxes start XM columns left of the patch: 16 bytes, the alignment TMA takes for the inner coordinate (4 fp32, 8 bf16)
  static constexpr int XM = 16 / ESZ;
  static constexpr int BW = PW + 2 * XM, BH = TH + 2;
  static constexpr int CC = TC_BK / KPL;                       // input channels per chunk
  static constexpr int IN_BYTES = CC * BH * BW * ESZ;          // multiple of 128 for PW in {16,32}
  static constexpr int A_BYTES = TC_BM * TC_BK * 4;            // 16 KB
  static constexpr int B_BYTES = N_TILE * TC_BK * (P == Prec::BF16 ? 2 : 4);   // 128-byte rows (bf16: 64-byte rows)
  // A ring stage: fp32 (register form: the consumers split hi / lo after loading; one 16 KB tile per half), or hi [+ lo]
  // (A_SMEM: the tensor core reads the parts)
  static constexpr int AST_BYTES = (X3 && A_SMEM ? 2 : 1) * NH * A_BYTES;
  static constexpr int BST_BYTES = (X3 ? 2 : 1) * B_BYTES;     // B ring stage: hi [+ lo] of N_TILE rows (wide: one channel half)
  static constexpr int OFF_ALO = A_BYTES;
  static constexpr int OFF_BLO = B_BYTES;
  // depthwise producer groups (128 threads each), sized by the register file: the consumers hold N_TILE / 2 accumulators
  // per thread (two sets in a paired tile).  NG <= AS always: the per-stage a_empty barriers are tested by phase parity, which
  // is only unambiguous while a group can never be two hand-backs of a stage behind
  static constexpr int NG = N_TILE > 64 || PAIR ? 1 : 2;
  // A ring and weight ring (prefetched by its own warp).  The consumers hold two stages of each (chunk i in flight, chunk i - 1
  // retiring); the producers write NG more, the weight loader runs one ahead.  The input ring gets the rest (it must stay deep
  // enough to cover HBM latency).  TF32X3 in the A_SMEM form (32 KB A stages) keeps two-deep rings at N_TILE 128: deeper ones
  // leave too little for the input ring.  BF16 takes TF32's depths: its A stages are TF32's and the four B stages cover the
  // same two in use, NG producing and one loading; the 16 / 32 KB its half-size B stages free go to the input ring and the
  // staging buffers (the table in DESIGN §6).  A paired tile's 32 KB A stages keep the register form's 2 + NG in both modes;
  // in 3xTF32 at PW 16 with k = 2 (27 KB boxes of 18 rows) the B ring is 2 deep, so that the input ring keeps 2 stages
  // Wide tiles: the B ring holds half-stages (one per chunk and channel half, 32 KB in 3xTF32), committed and released one by
  // one, so the consumers hold two of them (the newest MMA group and the one retiring) and the loader fills a third.  Four
  // would leave no room for the staging buffers beside a 2-deep input ring (the table in DESIGN §6).  Both modes take 2 + NG
  // A stages and 3 half-stages
  static constexpr int AS = WIDE ? 2 + NG : X3 ? (A_SMEM ? (N_TILE > 64 ? 2 : 3) : 2 + NG) : (PAIR ? 2 + NG : 4);
  static constexpr int BS = WIDE ? 3 : X3 ? (A_SMEM && N_TILE > 64 ? 2 : (PAIR && PW == 16 && KPL == 2 ? 2 : 3)) : 4;
  static constexpr int AFF_N = WIDE ? 256 : 512;               // scale | shift | OutConv weights of up to 512 (wide: 256) channels
  static constexpr int BAR_BYTES = 512;
  static constexpr int FREE = 224 * 1024 - 1024 - BAR_BYTES - 3 * AFF_N * 4 - AS * AST_BYTES - BS * BST_BYTES;
  // Output staging: per consumer warpgroup ST_BUFS buffers of one 32-channel x 64-pixel TMA store box (8 KB), taken from the
  // input ring.  Two, so that a slice's store overlaps the staging of the next: in 3xTF32 with k = 2 the input ring goes
  // 6 -> 4 at N_TILE 64 and 4 -> 2 at N_TILE 128 (one buffer there, with a 3-deep input ring, measured 1-6 % slower per
  // layer: DESIGN §6).  Where two would leave the input ring under 2 stages one is used, and where even one would (k = 1 at
  // N_TILE 128 in 3xTF32: 30 KB boxes), the instance keeps the direct-store epilogue (ST_BUFS = 0).  Paired tiles take one:
  // their 25-27 KB boxes would leave the input ring under 2 stages beside two
  static constexpr int ST_BOX = 32 * 64 * ESZ;
  static constexpr int ST_WANT = PAIR ? 1 : 2;
  static constexpr int ST_BUFS = (FREE - 2 * ST_WANT * ST_BOX) / IN_BYTES >= 2 ? ST_WANT
                                 : (FREE - 2 * ST_BOX) / IN_BYTES >= 2     ? 1
                                                                           : 0;
  static constexpr int ST_BYTES = 2 * ST_BUFS * ST_BOX;
  static_assert(ST_BUFS > 0 || (FREE - 2 * ST_BOX) / IN_BYTES < 2, "staging falls back only where one buffer does not fit");
  // beside each input stage, the CBAM spatial gate's one-channel halo box (gated chunks only)
  static constexpr int SA_TX = BH * BW * 4;
  static constexpr int SA_BYTES = (SA_TX + 127) / 128 * 128;
  // Input ring: as deep as shared memory allows, up to 8 stages, with a gate box per stage and, past the ring's end (rounded up
  // to 1 KB: OFF_A), room for the class weights of a 21-class model (MAX_CLASSES, below).  The k <= 2 instances meet both
  // with whole input boxes to spare; the 7 680 B boxes of k = 4 would not
  static constexpr int CLS_MIN = DS_MIN_CLASSES * (N_TILE + 1) * 4;
  static constexpr int RING_CLS = (FREE - ST_BYTES + 3 * 1024 - CLS_MIN) / 1024 * 1024;
  static constexpr int IS_FIT = (RING_CLS < FREE - ST_BYTES ? RING_CLS : FREE - ST_BYTES) / (IN_BYTES + SA_BYTES);
  static constexpr int IS = IS_FIT > 8 ? 8 : IS_FIT;
  static_assert(IS * (IN_BYTES + SA_BYTES) + ST_BYTES <= FREE, "gate boxes fit beside the input ring");
  static constexpr int OFF_SA = IS * IN_BYTES;
  static constexpr int OFF_A = ((OFF_SA + IS * SA_BYTES + 1023) / 1024) * 1024;
  static constexpr int OFF_BR = OFF_A + AS * AST_BYTES;
  static constexpr int OFF_ST = OFF_BR + BS * BST_BYTES;       // 1 KB aligned: the 128-byte swizzle repeats every 1 KB
  static constexpr int OFF_BAR = OFF_ST + ST_BYTES;
  static_assert((IS * NG + IS + 2 * AS + 2 * BS) * 8 <= BAR_BYTES, "barrier block");
  static constexpr int TOTAL = OFF_BAR + BAR_BYTES + 3 * AFF_N * 4 + 1024;
  // The K-class OutConv of smaat_dsconv_classify_fwd keeps its weights ([class][N_TILE], zero past Cout) and biases in the shared
  // memory the rings leave under the 227 KB limit (11.5-29.5 KB), appended after the affine block and requested only by class
  // launches: as many classes as fit, at most DS_MAX_CLASSES (22 to 32 by instance, pinned per instance in
  // tests/test_dsconv_dispatch_abi.py).  Read through the L1 the weights were a cache miss per class (the carveout leaves
  // little L1 beside 213 KB of shared memory)
  static constexpr int OFF_CLS = OFF_BAR + BAR_BYTES + 3 * AFF_N * 4;
  static constexpr int CLS_FIT = (227 * 1024 - TOTAL) / ((N_TILE + 1) * 4);
  static constexpr int MAX_CLASSES = CLS_FIT < DS_MAX_CLASSES ? CLS_FIT : DS_MAX_CLASSES;
  static constexpr int CLS_SMEM = MAX_CLASSES * (N_TILE + 1) * 4;
  static_assert(MAX_CLASSES >= DS_MIN_CLASSES, "the class weights of a 21-class model fit beside the rings");
  static_assert(TOTAL + CLS_SMEM <= 227 * 1024, "the class weights take no shared memory from the rings");
  static constexpr uint32_t B_TX = BST_BYTES;
  static constexpr int PROD_WARP = 12;                         // first producer warp
  static constexpr int THREADS = 384 + 128 * NG;               // TMA, loader, 2 idle | 2 consumer warpgroups | producers
  // setmaxnreg split of the registers a CTA launches with (__launch_bounds__(THREADS, 1), 128 or 96 per thread): warpgroup 0
  // gives up all but REGS_TMA, the producer group gives some back at N_TILE 128 (its stencil fits in 104 without spills), the
  // consumers (accumulators + two register-A fragment sets) take the rest: 192 at N_TILE 128 and in paired tiles (two
  // accumulator sets, two fragment sets per half), 128 at N_TILE 64
  static constexpr int REGS_LAUNCH = (65536 / THREADS) / 8 * 8;
  static constexpr int REGS_TMA = 24;
  static constexpr int REGS_PROD = N_TILE > 64 || PAIR ? 104 : REGS_LAUNCH;
  static constexpr int REGS_MMA = ((THREADS / 128 * REGS_LAUNCH - REGS_TMA - NG * REGS_PROD) / 2) / 8 * 8;
  static constexpr int REGS_SUM = REGS_TMA + 2 * REGS_MMA + NG * REGS_PROD;
  static_assert(REGS_SUM <= THREADS / 128 * REGS_LAUNCH && REGS_MMA >= REGS_LAUNCH, "register budget");
  // k-steps per MMA commit group in the register form.  A whole chunk (4) holds 2 x 32 fragment registers in TF32X3; at
  // N_TILE 64 the consumers' 128 registers cannot (ptxas would serialise the MMAs), so groups are half chunks there
  // Wide tiles hold 2 x 64 accumulators: with two half-chunk sets (2 x 16 registers in TF32X3, 2 x 8 in tf32)
  // beside them ptxas serialised the MMAs, so their groups are single k-steps in TF32X3 and half chunks in tf32
  static constexpr int KS = WIDE ? (X3 ? 1 : 2) : (X3 && N_TILE == 64) ? 2 : TC_BK / 8;
  static_assert(IS >= 2, "input ring");
  static_assert(NG <= AS, "phase-parity barriers");
  static_assert(IN_BYTES % 128 == 0, "TMA destination alignment");
  static_assert(TOTAL <= 227 * 1024, "shared memory budget");
  static_assert(!WIDE || ST_BUFS > 0, "wide tiles keep the staged epilogue: the max-pool and the CBAM pools are taken as at N_TILE 128");
  static_assert(!PAIR || ST_BUFS > 0, "paired tiles keep the staged epilogue: the max-pool and the CBAM pools are taken as at N_TILE 64");
  static_assert(!PAIR || MAX_CLASSES >= DS_MIN_CLASSES, "paired tiles take the class launches of up to DS_MIN_CLASSES classes");
};

// ----- staged output epilogue: TMA tensor stores of 32-channel x 64-pixel boxes from shared memory -----
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's committed bulk stores may still be reading their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// 4 x 4 transpose across the 4 lanes of a fragment group with equal t (lanes 4q + t, q = 0..3; quad lane q = g & 3): on entry
// v[s] is slot s at quad pixel q, on exit v[p] is slot q at quad pixel p.  Two butterfly stages (lanes 8 apart, then 4 apart)
__device__ __forceinline__ void quad_transpose(float (&v)[4], int q) {
  const bool h1 = q & 2, h0 = q & 1;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float r = __shfl_xor_sync(0xffffffffu, h1 ? v[e] : v[e + 2], 8);
    if (h1) v[e] = r; else v[e + 2] = r;
  }
#pragma unroll
  for (int e = 0; e < 4; e += 2) {
    const float r = __shfl_xor_sync(0xffffffffu, h0 ? v[e] : v[e + 1], 4);
    if (h0) v[e] = r; else v[e + 1] = r;
  }
}

// The kernel body, shared by the k = 1 / 2 instances (dsconv_fused_kernel) and the k = 4 ones (dsconv_kpl4_kernel).  The tensor
// maps are the kernels' __grid_constant__ parameters
template <int N_TILE, int KPL, int PW, Prec PREC, bool A_SMEM, typename TA = float, bool PAIR = false, bool WIDE = false>
__device__ __forceinline__ void dsconv_body(const CUtensorMap& map_in0, const CUtensorMap& map_in1, const CUtensorMap& map_w,
                                            const CUtensorMap& map_wlo, const CUtensorMap& map_y, const CUtensorMap& map_sa,
                                            const DsParams& p) {
  using L = DsCfg<N_TILE, KPL, PW, PREC, A_SMEM, TA, PAIR, WIDE>;
  constexpr bool X3 = L::X3;
  constexpr bool BA = L::ESZ == 2;   // bf16 activations
  constexpr int PH = L::PH, NH = L::NH, NW = L::NW, NA = L::NA, TH = L::TH, BW = L::BW, BH = L::BH, CC = L::CC, IS = L::IS, AS = L::AS, BS = L::BS;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  unsigned char* a_base = smem + L::OFF_A;
  unsigned char* b_base = smem + L::OFF_BR;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  // [IS][NG] TMA input box landed, one barrier per (stage, group that reads the fill): a group meets a stage only at every
  // NG-th of its fills (unless NG divides IS), and TMA loads may complete out of order -- a parity test on a per-stage
  // barrier could then be satisfied by the wrong fill
  uint64_t* in_full = bars;
  uint64_t* in_empty = in_full + IS * L::NG;      // [IS] producer group finished reading the box (128 arrivals)
  uint64_t* a_full = in_empty + IS;               // [AS] A operand written (128 arrivals)
  uint64_t* a_empty = a_full + AS;                // [AS] the 8 consumer warps' MMAs reading the A stage retired
  uint64_t* b_full = a_empty + AS;                // [BS] weight chunk (wide: half-chunk) landed (TMA tx)
  uint64_t* b_empty = b_full + BS;                // [BS] the 8 consumer warps' MMAs reading the B stage retired
  float* aff = reinterpret_cast<float*>(smem + L::OFF_BAR + L::BAR_BYTES);

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler too
  const int lane = threadIdx.x & 31;
  const int nch = p.nchunks;
  const int tiles_per_img = p.tiles_x * p.tiles_y * p.npass;
  // tile -> (image b, patch row ty, patch column tx, channel pass np); the passes of a patch are consecutive tiles
  auto decode = [&](int tile, int& b, int& ty, int& tx, int& np) {
    b = tile / tiles_per_img;
    int t2 = tile - b * tiles_per_img;
    np = t2 % p.npass;
    t2 /= p.npass;
    ty = t2 / p.tiles_x;
    tx = t2 - ty * p.tiles_x;
  };

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_in0);
    tma_prefetch_desc(&map_in1);
    tma_prefetch_desc(&map_w);
    if (X3) tma_prefetch_desc(&map_wlo);
    if (L::ST_BUFS && !p.oc_y) tma_prefetch_desc(&map_y);
    if (p.gate_sc) tma_prefetch_desc(&map_sa);
    for (int s = 0; s < IS; ++s) {
      for (int g = 0; g < L::NG; ++g) mbar_init(&in_full[s * L::NG + g], 1);
      mbar_init(&in_empty[s], 128);
    }
    for (int s = 0; s < AS; ++s) {
      mbar_init(&a_full[s], 128);
      mbar_init(&a_empty[s], 8);
    }
    for (int s = 0; s < BS; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], 8);
    }
    fence_barrier_init();
  }
  for (int c = threadIdx.x; c < L::AFF_N; c += blockDim.x) {
    aff[c] = (c < p.Cout && p.scale) ? __ldg(p.scale + c) : 1.f;
    aff[L::AFF_N + c] = (c < p.Cout && p.shift) ? __ldg(p.shift + c) : 0.f;
    aff[2 * L::AFF_N + c] = (c < p.Cout && p.oc_w) ? __ldg(p.oc_w + c) : 0.f;
  }
  float* cls_w = reinterpret_cast<float*>(smem + L::OFF_CLS);   // [ncls][N_TILE] (class launches only), then ncls biases
  float* cls_b = cls_w + L::MAX_CLASSES * N_TILE;
  if (p.ncls) {
    for (int i = threadIdx.x; i < p.ncls * N_TILE; i += blockDim.x) {
      const int cl = i / N_TILE, c = i - cl * N_TILE;
      cls_w[i] = c < p.Cout ? __ldg(p.oc_w + (int64_t)cl * p.Cout + c) : 0.f;
    }
    for (int cl = threadIdx.x; cl < p.ncls; cl += blockDim.x) cls_b[cl] = p.oc_b ? __ldg(p.oc_b + cl) : 0.f;
  }
  __syncthreads();

  if (warp < 4) {
    // warpgroup 0 keeps few registers: the consumers' two register-A fragment sets need them (all four warps reallocate)
    regs_dealloc<L::REGS_TMA>();
    // ===== TMA: input halo boxes, running ahead through the IS-deep ring =====
    if (warp == 0 && lane == 0) {
      uint32_t gc = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int b, ty, tx, np;
        decode(tile, b, ty, tx, np);
        const int x0 = tx * PW, y0 = ty * TH;
        for (int i = 0; i < nch; ++i, ++gc) {
          const int s = gc % IS;
          mbar_wait(&in_empty[s], ((gc / IS) & 1u) ^ 1u);
          uint64_t* full = &in_full[s * L::NG + (int)(gc % (uint32_t)L::NG)];      // the barrier of the group that reads this chunk
          const int cb = i * CC;
          const bool gated = p.gate_sc && cb < p.C0;
          mbar_arrive_expect_tx(full, L::IN_BYTES + (gated ? L::SA_TX : 0));
          // the gate's halo box: same origin and extent as the input box, one channel; zero fill outside the image
          if (gated) tma_load_3d(smem + L::OFF_SA + s * L::SA_BYTES, &map_sa, full, x0 - L::XM, y0 - 1, b);
          const CUtensorMap* m = (cb < p.C0) ? &map_in0 : &map_in1;
          const int cc = (cb < p.C0) ? cb : cb - p.C0;
          asm volatile(
              "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
                  "r"(smem_u32(smem + s * L::IN_BYTES)),
              "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(full)), "r"(x0 - L::XM), "r"(y0 - 1), "r"(cc), "r"(b)
              : "memory");
        }
      }
    }
    // ===== weight-ring loader: K-major SW128 chunks (hi [+lo]) of this tile's channel pass, decoupled from the input ring.  Wide
    // tiles: half-stage hs = NW * chunk + half, each N_TILE rows of the chunk =====
    if (warp == 1 && lane == 0) {
      uint32_t hs = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int b, ty, tx, np;
        decode(tile, b, ty, tx, np);
        for (int i = 0; i < nch; ++i) {
#pragma unroll
          for (int hf = 0; hf < NW; ++hf, ++hs) {
            const int sb = hs % BS, row = (np * NW + hf) * N_TILE;
            mbar_wait(&b_empty[sb], ((hs / BS) & 1u) ^ 1u);
            mbar_arrive_expect_tx(&b_full[sb], L::B_TX);
            tma_load_2d(b_base + sb * L::BST_BYTES, &map_w, &b_full[sb], i * TC_BK, row);
            if (X3) tma_load_2d(b_base + sb * L::BST_BYTES + L::OFF_BLO, &map_wlo, &b_full[sb], i * TC_BK, row);
          }
        }
      }
    }
    return;
  }

  if (warp < L::PROD_WARP) {
    regs_alloc<L::REGS_MMA>();
    // ===== consumer warpgroups: MMAs into register accumulators, then the epilogue =====
    const int wg = (warp >> 2) - 1, wq = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    // patch pixels of accumulator rows g, g + 8: A_SMEM tiles hold pixel m in row m
    const int m0 = A_SMEM ? 64 * wg + 16 * wq + g : tc_row_pixel(wg, wq, 0, g);
    const int m1 = A_SMEM ? m0 + 8 : tc_row_pixel(wg, wq, 1, g);
    const float act_lo = p.relu ? 0.f : -INFINITY;
    const int64_t P = (int64_t)p.H * p.W;
    // Staged epilogue.  This warpgroup's patch pixels 64 wg .. 64 wg + 63 (both A forms) are the PW x PH / 2 half-patch its
    // TMA store box covers, so each warpgroup stages and stores on its own.  The box lies [channel][pixel] in shared memory
    // with the TMA swizzle of its row length (128 B at PW 32, 64 B at PW 16).  A warp holds 16 pixels of every channel, and
    // unswizzled channels are 256 B apart: any store order would be at least 2-way bank-conflicted.  So the 4 lanes of a
    // fragment group with equal t (quad pixels q = 0..3 of two pixel quads and channels 2t, 2t + 1) transpose their values
    // (quad_transpose): each lane then stores 4 consecutive pixels of one channel with one STS.128, slot q ^ (t & 2)
    // (slot s: channel 2t + (s & 1), quad of accumulator row s >> 1).  The t & 2 twist puts the lanes t and t + 2 of one
    // quarter-warp on different swizzle phases.  In the register form that makes every STS.128 conflict-free at PW 32; at
    // PW 16 the 64-byte swizzle spans 4 bank groups and a quarter-warp's pixels only 4, so it stays 2-way there (and in the
    // shared-memory form, whose rows are consecutive pixels, 2-way at PW 32 and 4-way at PW 16).
    constexpr int SW_MASK = PW == 32 ? 7 : 3;      // 16-byte chunk bits [4, 7) / [4, 6) ^= address bits [7, 10) / [7, 9)
    const int quad = g & 3, slot = quad ^ (t & 2);
    const int st_ch = 2 * t + (slot & 1);           // channel of this lane's stores within an 8-channel fragment column
    const int st_px = ((slot & 2) ? m1 : m0) - quad - 64 * wg;   // first of its 4 pixels within the half-patch
    // bf16 boxes (rows of 64 / 32 B) are staged and stored unswizzled: [channel][64 pixels] x 2 B, 8-byte stores
    const uint32_t st_a0 = (uint32_t)(st_ch * 64 * L::ESZ + st_px * L::ESZ);
    const uint32_t st_off = BA ? st_a0 : st_a0 ^ (((st_a0 >> 7) & SW_MASK) << 4);   // + 8 channels per fragment column
    const uint32_t st_base = smem_u32(smem + L::OFF_ST) + (uint32_t)(wg * L::ST_BUFS * L::ST_BOX);
    const bool st_leader = (threadIdx.x & 127) == 0;
    uint32_t st_n = 0;                              // this warpgroup's staged boxes so far (buffer st_n % ST_BUFS)
    uint32_t gc = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int b, ty, tx, np;
      decode(tile, b, ty, tx, np);
      // one accumulator set per half of the tile (its 64 rows of that patch, or of that channel half)
      float acc[NA][N_TILE / 2];
#pragma unroll
      for (int h = 0; h < NA; ++h)
#pragma unroll
        for (int i = 0; i < N_TILE / 2; ++i) acc[h][i] = 0.f;
      // Pipelined k loop: chunk i's MMAs are issued as one group, then the wait leaves that group in flight and retires chunk
      // i - 1, whose A and B stages go back to the producers and the weight loader.
      // release(c): chunk c's A stage and its (last) B stage; wide tiles hand half 0's B stage back on its own (release_b)
      auto release = [&](uint32_t c) {
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&a_empty[c % AS]);
          mbar_arrive(&b_empty[(NW * c + NW - 1) % BS]);
        }
      };
      auto release_b = [&](uint32_t hs) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&b_empty[hs % BS]);
      };
      auto wait_b = [&](uint32_t hs, uint64_t& bd, uint64_t& bl) {
        const int sb = hs % BS;
        mbar_wait(&b_full[sb], (hs / BS) & 1u);
        bd = make_b_desc<PREC>(smem_u32(b_base + sb * L::BST_BYTES));
        bl = make_kmajor_desc(smem_u32(b_base + sb * L::BST_BYTES + L::OFF_BLO));
      };
      auto wait_stages = [&](const unsigned char*& ast, uint64_t& bd, uint64_t& bl) {
        const int sa = gc % AS;
        mbar_wait(&a_full[sa], (gc / AS) & 1u);
        ast = a_base + sa * L::AST_BYTES;
        wait_b(NW * gc, bd, bl);
      };
      if (A_SMEM) {
        for (int i = 0; i < nch; ++i, ++gc) {
          const unsigned char* ast;
          uint64_t bd0, bl0;
          wait_stages(ast, bd0, bl0);
          const uint32_t a_addr = smem_u32(ast) + (uint32_t)(wg * 64 * 128);   // this warpgroup's 64 rows: 8 swizzle atoms
          const uint64_t ad0 = make_kmajor_desc(a_addr), al0 = make_kmajor_desc(a_addr + L::OFF_ALO);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < TC_BK / 8; ++kk) {
            Wgmma<N_TILE>::ss(acc[0], ad0 + (uint64_t)(2 * kk), bd0 + (uint64_t)(2 * kk), 1u);
            if (X3) {
              Wgmma<N_TILE>::ss(acc[0], al0 + (uint64_t)(2 * kk), bd0 + (uint64_t)(2 * kk), 1u);
              Wgmma<N_TILE>::ss(acc[0], ad0 + (uint64_t)(2 * kk), bl0 + (uint64_t)(2 * kk), 1u);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (i > 0) release(gc - 1);
        }
        wgmma_wait0();
      } else if constexpr (WIDE) {
        // A wide tile sweeps each chunk twice, half 0's k-steps and then half 1's, one commit group per KS k-steps, each from
        // fragments it loads from the chunk's A stage (the A stage is read twice, the input box and the stencil were done once).
        // The wait after each group retires the one before: at half 0's first group the previous chunk's A stage and half-1 B
        // stage go back, at half 1's first group this chunk's half-0 B stage.  So the weight loader refills half 0's stage
        // halfway through the chunk, and each half-stage has about a chunk's MMAs to land in the 3-deep ring.  (With the halves
        // interleaved per k-step, a chunk's half-0 stage was freed only as its last group retired, two groups before the next
        // chunk's half 1 needed it.)  Each accumulator set sees the k-steps of a single N_TILE pass in its order, so the sums
        // are those of the two-pass route.  Two fragment sets alternate over the 2 x GPC groups of a chunk
        constexpr int KS = L::KS, GPC = (TC_BK / 8) / KS;
        static_assert(GPC % 2 == 0, "fragment sets alternate within a chunk");
        const unsigned char* ast = nullptr;
        uint64_t bd = 0, bl = 0;
        AFrags<PREC, KS> fa, fb;
        // group `part` of half hf (both constants once unrolled) of chunk i
        auto step = [&](int i, int hf, int part, AFrags<PREC, KS>& cur, AFrags<PREC, KS>& prev) {
          if (part == 0) {
            if (hf == 0) {
              const int sa = gc % AS;
              mbar_wait(&a_full[sa], (gc / AS) & 1u);
              ast = a_base + sa * L::AST_BYTES;
            }
            wait_b(NW * gc + hf, bd, bl);
          }
          load_a_frags<PREC, KS>(ast, part * KS, t, m0, m1, cur);
          if (hf == 0) mma_a_frags<N_TILE, PREC, KS>(acc[0], cur, bd, bl, part * KS);
          else mma_a_frags<N_TILE, PREC, KS>(acc[NA - 1], cur, bd, bl, part * KS);
          wgmma_wait<1>();
          wgmma_keep(prev);
          if (part == 0) {
            if (hf == 1) release_b(NW * gc);
            else if (i > 0) release(gc - 1);
          }
        };
        for (int i = 0; i < nch; ++i, ++gc) {
#pragma unroll
          for (int hf = 0; hf < NW; ++hf) {
#pragma unroll
            for (int part = 0; part < GPC; part += 2) {
              step(i, hf, part, fa, fb);
              step(i, hf, part + 1, fb, fa);
            }
          }
        }
        wgmma_wait0();
        wgmma_keep(fa);
        wgmma_keep(fb);
      } else {
        // Chunk i's fragments must stay untouched until it retires, so two fragment sets alternate (the loop is unrolled by 2;
        // no control-flow path may load a set whose chunk is still in flight, or ptxas serialises the MMAs: the odd tail is
        // outside the loop)
        // A commit group is KS k-steps: GPC groups per chunk.  Chunk i - 1 has retired once the first group of chunk i is
        // issued and the wait leaves only that one in flight.  A paired tile's group loads each half's fragments from that
        // half's A tile (its own sets, alternating the same way) and issues both halves' MMAs against the same B
        constexpr int KS = L::KS, GPC = (TC_BK / 8) / KS;
        const unsigned char* ast = nullptr;
        uint64_t bd0 = 0, bl0 = 0;
        auto group = [&](AFrags<PREC, KS>(&cur)[NH], AFrags<PREC, KS>(&prev)[NH], int q) {
          const int part = q % GPC;
          if (part == 0) wait_stages(ast, bd0, bl0);
#pragma unroll
          for (int h = 0; h < NH; ++h) load_a_frags<PREC, KS>(ast + h * L::A_BYTES, part * KS, t, m0, m1, cur[h]);
          mma_a_frags<N_TILE, PREC, KS, NH>(acc, cur, bd0, bl0, part * KS);
          wgmma_wait<1>();
#pragma unroll
          for (int h = 0; h < NH; ++h) wgmma_keep(prev[h]);
          if (part == 0 && q > 0) release(gc - 1);
          if (part == GPC - 1) ++gc;
        };
        AFrags<PREC, KS> fa[NH], fb[NH];
        const int ngrp = nch * GPC;
        int q = 0;
        for (; q + 1 < ngrp; q += 2) {
          group(fa, fb, q);
          group(fb, fa, q + 1);
        }
        if (q < ngrp) group(fa, fb, q);
        wgmma_wait0();
#pragma unroll
        for (int h = 0; h < NH; ++h) {
          wgmma_keep(fa[h]);
          wgmma_keep(fb[h]);
        }
      }
      // the tile's last chunk has retired; its stages are released before the epilogue, so that TMA, the weight loader and
      // the producers run on through it
#pragma unroll
      for (int h = 0; h < NA; ++h) wgmma_keep(acc[h]);
      release(gc - 1);

      // ----- epilogue, once per half (patch rows y_org .., channels n0 ..): rows g / g + 8 are patch pixels m0 / m1, columns
      // n0 + 8j + 2t + {0, 1}
#pragma unroll
      for (int h = 0; h < NA; ++h) {
        float (&ac)[N_TILE / 2] = acc[h];
        const int hp = WIDE ? 0 : h;                 // the patch half (paired tiles)
        const int n0 = (np * NW + (WIDE ? h : 0)) * N_TILE;
        const int y_org = ty * TH + hp * PH;
        const int gy0 = y_org + m0 / PW, gx0 = tx * PW + m0 % PW;
        const int gy1 = y_org + m1 / PW, gx1 = tx * PW + m1 % PW;
        const bool v0 = gy0 < p.H && gx0 < p.W, v1 = gy1 < p.H && gx1 < p.W;
        const int64_t o0 = (int64_t)gy0 * p.W + gx0, o1 = (int64_t)gy1 * p.W + gx1;
        if (!WIDE && p.stats) {
          // BatchNorm batch statistics from the RAW accumulators (one pass: Cout <= 128, not taken by wide tiles); patch pixels outside the image are
          // masked (their stencil still sees the image edge), channels past Cout are exact zeros (TMA zero fill of the weight
          // rows); the affine is applied to the sums analytically
          const double npix = (double)((__popc(__ballot_sync(0xffffffffu, v0)) + __popc(__ballot_sync(0xffffffffu, v1))) / 4);
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float a = v0 ? ac[4 * j + e] : 0.f, bb = v1 ? ac[4 * j + 2 + e] : 0.f;
              const float s1 = frag_colsum(a + bb), s2 = frag_colsum(fmaf(a, a, bb * bb));
              const int c = 8 * j + 2 * t + e;
              if (lane < 4 && c < p.Cout) {
                const double sc = (double)aff[c], sh = (double)aff[L::AFF_N + c];
                atomicAdd(p.stats + c, sc * (double)s1 + npix * sh);
                atomicAdd(p.stats + p.Cout + c, sc * sc * (double)s2 + 2.0 * sc * sh * (double)s1 + npix * sh * sh);
              }
            }
          }
        }
        if (!WIDE && p.ncls) {
          // K-class OutConv + argmax.  The activations replace the accumulators in place (fmaxf(fmaf(acc, sc, sh), act_lo), as
          // below); then, one class at a time, the one-class dot product below in its order (fmaf over the thread's channels, the
          // two xor shuffles, + bias), so class j's logit is bit for bit what that epilogue writes with OutConv row j.  After the
          // butterfly all 4 lanes of a fragment group hold the same logits; each keeps the same running (max, first index) per
          // pixel -- torch.argmax's rule: a NaN wins and stays -- so the registers hold two logits whatever K is.  A lane's two
          // channels 2t, 2t + 1 of a fragment column are one 8-byte shared-memory load (the 8 fragment groups read the same
          // address: a broadcast, conflict-free).  Logit stores rotate over the 4 lanes
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * j + 2 * t + e;
              const float sc = aff[c], sh = aff[L::AFF_N + c];
              ac[4 * j + e] = fmaxf(fmaf(ac[4 * j + e], sc, sh), act_lo);
              ac[4 * j + 2 + e] = fmaxf(fmaf(ac[4 * j + 2 + e], sc, sh), act_lo);
            }
          }
          float best0 = -INFINITY, best1 = -INFINITY;
          int arg0 = 0, arg1 = 0;
#pragma unroll 1
          for (int cl = 0; cl < p.ncls; ++cl) {
            const float* wr = cls_w + cl * N_TILE + 2 * t;   // zero past Cout, where the activation is 0 too
            float d0 = 0.f, d1 = 0.f;
#pragma unroll
            for (int j = 0; j < N_TILE / 8; ++j) {
              const float2 w = *reinterpret_cast<const float2*>(wr + 8 * j);
              d0 = fmaf(ac[4 * j], w.x, d0);
              d1 = fmaf(ac[4 * j + 2], w.x, d1);
              d0 = fmaf(ac[4 * j + 1], w.y, d0);
              d1 = fmaf(ac[4 * j + 3], w.y, d1);
            }
            d0 += __shfl_xor_sync(0xffffffffu, d0, 1);
            d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
            d1 += __shfl_xor_sync(0xffffffffu, d1, 1);
            d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
            const float ob = cls_b[cl];
            const float l0 = d0 + ob, l1 = d1 + ob;
            if (best0 == best0 && (l0 > best0 || l0 != l0)) { best0 = l0; arg0 = cl; }
            if (best1 == best1 && (l1 > best1 || l1 != l1)) { best1 = l1; arg1 = cl; }
            if (p.oc_y && t == (cl & 3)) {
              TA* yk = reinterpret_cast<TA*>(p.oc_y) + ((int64_t)b * p.ncls + cl) * P;
              if (v0) st_act(yk + o0, l0);
              if (v1) st_act(yk + o1, l1);
            }
          }
          if (p.cls) {
            if (v0 && t == 0) p.cls[(int64_t)b * P + o0] = arg0;
            if (v1 && t == 1) p.cls[(int64_t)b * P + o1] = arg1;
          }
        } else if (!WIDE && p.oc_y) {
          // fused OutConv: each pixel's dot product over all Cout <= N_TILE activations.  Channels past Cout have zero
          // accumulators, identity affine and zero OutConv weight: no mask needed
          float d0 = 0.f, d1 = 0.f;
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * j + 2 * t + e;
              const float sc = aff[c], sh = aff[L::AFF_N + c], w = aff[2 * L::AFF_N + c];
              d0 = fmaf(fmaxf(fmaf(ac[4 * j + e], sc, sh), act_lo), w, d0);
              d1 = fmaf(fmaxf(fmaf(ac[4 * j + 2 + e], sc, sh), act_lo), w, d1);
            }
          }
          d0 += __shfl_xor_sync(0xffffffffu, d0, 1);
          d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
          d1 += __shfl_xor_sync(0xffffffffu, d1, 1);
          d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
          const float ob = p.oc_b ? __ldg(p.oc_b) : 0.f;
          if (t == 0) {
            TA* oy = reinterpret_cast<TA*>(p.oc_y) + (int64_t)b * P;
            if (v0) st_act(oy + o0, d0 + ob);
            if (v1) st_act(oy + o1, d1 + ob);
          }
        } else if (L::ST_BUFS) {
          // One 32-channel slice at a time: wait until the buffer's previous store has been read out, stage the slice (the same
          // fmaxf(fmaf(acc, sc, sh), act_lo) as the direct stores: bit-identical), hand it to the async proxy and store it as
          // one box.  TMA clips what lies outside W, H or Cout; slices wholly past Cout are skipped
          const int y_half = y_org + wg * (PH / 2);
#pragma unroll
          for (int s = 0; s < N_TILE / 32; ++s) {
            if (n0 + 32 * s >= p.Cout) break;
            const uint32_t buf = st_base + (st_n % L::ST_BUFS) * L::ST_BOX;
            if (st_leader) bulk_wait_read<L::ST_BUFS - 1>();
            wg_sync(2 + wg);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * s + jj;
              float v[4];
#pragma unroll
              for (int q = 0; q < 4; ++q) v[q] = (t & 2) ? ac[4 * j + (q ^ 2)] : ac[4 * j + q];
              quad_transpose(v, quad);
              const int c = n0 + 8 * j + st_ch;
              const float sc = aff[c], sh = aff[L::AFF_N + c];
              const float4 o = make_float4(fmaxf(fmaf(v[0], sc, sh), act_lo), fmaxf(fmaf(v[1], sc, sh), act_lo),
                                           fmaxf(fmaf(v[2], sc, sh), act_lo), fmaxf(fmaf(v[3], sc, sh), act_lo));
              if constexpr (BA) {
                asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(buf + st_off + 1024u * jj), "r"(f32x2_bf16x2(o.x, o.y)),
                             "r"(f32x2_bf16x2(o.z, o.w))
                             : "memory");
              } else {
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(buf + st_off + 2048u * jj), "f"(o.x), "f"(o.y),
                             "f"(o.z), "f"(o.w)
                             : "memory");
              }
            }
            fence_proxy_async_smem();
            wg_sync(2 + wg);
            if (st_leader) {
              tma_store_4d(&map_y, buf, tx * PW, y_half, n0 + 32 * s, b);
              bulk_commit();
            }
            if (p.pooled) {
              // The next level's MaxPool2d(2) [and the CBAM channel gate's pools: pool_sum, fp32 maps only], read back from the
              // staged slice (the stored values bit for bit -- bf16 boxes hold the rounded values, and the max of bf16 values is
              // one of them; the store reads the buffer too, and nothing writes it before the next wg_sync).  4 threads per
              // channel, 2 items each: an item is 4 columns of a row pair, i.e. two 2 x 2 windows (the half-patch origin is even
              // and PH / 2 is even, so no window straddles it).  Pixels outside H or W are masked; an odd last row goes into the
              // pools but not the max-pool (floor, as MaxPool2d)
              const bool parts = !BA && p.pool_sum;
              const int pt = threadIdx.x & 127, pch = pt >> 2, pq = pt & 3;
              const int c = n0 + 32 * s + pch;
              float psum = 0.f, pmax = -INFINITY;
#pragma unroll
              for (int it = 0; it < 2; ++it) {
                constexpr int NQ = PW / 4;
                const int item = pq + 4 * it, rp = item / NQ, qd = item % NQ;   // lanes pq = 0..3: 4 adjacent items, 32 B of max-pool
                const int px = 2 * rp * PW + 4 * qd;
                float4 u, v;
                if constexpr (BA) {
                  // unswizzled [channel][64 pixels] x 2 B: 4 pixels are one 8-byte load
                  const uint32_t a0 = (uint32_t)(pch * 128 + px * 2), a1 = a0 + (uint32_t)(PW * 2);
                  uint2 hu, hv;
                  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(hu.x), "=r"(hu.y) : "r"(buf + a0));
                  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(hv.x), "=r"(hv.y) : "r"(buf + a1));
                  u = bf16x4_f32(hu);
                  v = bf16x4_f32(hv);
                } else {
                  const uint32_t a0 = (uint32_t)(pch * 256 + px * 4), a1 = a0 + (uint32_t)(PW * 4);
                  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(u.x), "=f"(u.y), "=f"(u.z), "=f"(u.w)
                               : "r"(buf + (a0 ^ (((a0 >> 7) & SW_MASK) << 4))));
                  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                               : "r"(buf + (a1 ^ (((a1 >> 7) & SW_MASK) << 4))));
                }
                const int gy = y_half + 2 * rp, gx = tx * PW + 4 * qd;      // W % 4 == 0: a quad is all in or all out
                const bool in0 = gx < p.W && gy < p.H, in1 = gx < p.W && gy + 1 < p.H;
                if (parts && in0) {
                  psum += (u.x + u.y) + (u.z + u.w);
                  pmax = fmaxf(pmax, fmaxf(fmaxf(u.x, u.y), fmaxf(u.z, u.w)));
                }
                if (in1) {
                  if (parts) {
                    psum += (v.x + v.y) + (v.z + v.w);
                    pmax = fmaxf(pmax, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
                  }
                  if (c < p.Cout) {
                    const int hw = p.W >> 1;
                    const int64_t o = ((int64_t)b * p.Cout + c) * (int64_t)(p.H >> 1) * hw + (int64_t)(gy >> 1) * hw + (gx >> 1);
                    const float2 m2 = make_float2(fmaxf(fmaxf(u.x, u.y), fmaxf(v.x, v.y)), fmaxf(fmaxf(u.z, u.w), fmaxf(v.z, v.w)));
                    if (BA && p.pooled_bf16)   // exact: both maxima are bf16 values
                      *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.pooled) + o) = f32x2_bf16x2(m2.x, m2.y);
                    else
                      *reinterpret_cast<float2*>(p.pooled + o) = m2;
                  }
                }
              }
              if (parts) {   // uniform over the CTA
                psum += __shfl_xor_sync(0xffffffffu, psum, 1);
                psum += __shfl_xor_sync(0xffffffffu, psum, 2);
                pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, 1));
                pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, 2));
                if (pq == 0 && c < p.Cout) {
                  const int64_t o = ((int64_t)b * p.npart + 2 * ((ty * NH + hp) * p.tiles_x + tx) + wg) * p.Cout + c;
                  p.pool_sum[o] = psum;
                  p.pool_max[o] = pmax;
                }
              }
            }
            ++st_n;
          }
        } else {
          TA* yb = reinterpret_cast<TA*>(p.y) + (int64_t)b * p.y_bstride;
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = n0 + 8 * j + 2 * t + e;
              if (c < p.Cout) {
                const float sc = aff[c], sh = aff[L::AFF_N + c];
                TA* yc = yb + (int64_t)c * P;
                if (v0) st_act(yc + o0, fmaxf(fmaf(ac[4 * j + e], sc, sh), act_lo));
                if (v1) st_act(yc + o1, fmaxf(fmaf(ac[4 * j + 2 + e], sc, sh), act_lo));
              }
            }
          }
        }
      }
    }
    if (L::ST_BUFS && st_leader) bulk_wait_all();   // the stores have read their boxes before the CTA's shared memory goes
    return;
  }

  {
    // ===== depthwise producer groups: NG groups of 4 warps (warps 12 ..), group g takes every NG-th chunk =====
    if (L::REGS_PROD < L::REGS_LAUNCH) regs_dealloc<L::REGS_PROD>();
    const int g = (warp - L::PROD_WARP) >> 2;
    const int t = threadIdx.x - 32 * L::PROD_WARP - 128 * g;  // 0..127
    const int Cin = p.C0 + p.C1;
    // A task is one (input channel, column quad[, row group]) of a chunk: NT = CC * 8 of them.  A thread computes KH of its KPL
    // depthwise outputs: all of them at KPL = 1 / 2; at KPL = 4 (CC = 8: 64 tasks) two threads share each task, threads
    // 64 h .. 64 h + 63 computing k-rows 4 ci + 2 h and 4 ci + 2 h + 1 (kr0 = 2 h), so that all 128 producer threads work and
    // each holds the weight registers of KPL = 2
    constexpr int KH = KPL == 4 ? 2 : KPL, NT = CC * 8;
    const int kr0 = KH == KPL ? 0 : t / NT * KH;
    // this thread's depthwise weights and biases start at k-row kr0 (offset in the pointers: in the per-chunk weight index,
    // ptxas spilled the KPL = 4 producers)
    const float* dw_w = p.dw_w + kr0 * 9;
    const float* dw_b = p.dw_b ? p.dw_b + kr0 : nullptr;
    uint32_t gc = 0, iph = 0;       // iph: phase bit per input stage of this group's fill barriers
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int b = tile / tiles_per_img;
      for (int i = 0; i < nch; ++i, ++gc) {
        if ((int)(gc % (uint32_t)L::NG) != g) continue;
        const int s = gc % IS;
        // chunks of x0 under a CBAM gate: each staged value is read as (x * sc[b, c]) * sa[b, p], the two rounded products of
        // cbam_gate_scale_kernel in its order, so the stencil sees exactly the materialised CBAM output
        const bool gated = p.gate_sc && i * CC < p.C0;
        // (thread t's task at KPL = 4: t % NT, both halves)
        auto task_base = [&](int task) { return KH == KPL ? task : task & (NT - 1); };
        // depthwise weights of this thread's (first) task: issued before the ring waits so that their latency hides there
        float wr[KH][9], br[KH], gsc = 0.f;
        auto task_channel = [&](int task) { return (PW == 32) ? (task >> 3) : (((task >> 4) << 1) | ((task >> 2) & 1)); };
        auto load_weights = [&](int task) {
          const int gch = i * CC + task_channel(task_base(task));
          const bool chv = gch < Cin;
#pragma unroll
          for (int kk = 0; kk < KH; ++kk) {
            const int gk = gch * KPL + kk;
#pragma unroll
            for (int w9 = 0; w9 < 9; ++w9) wr[kk][w9] = chv ? __ldg(dw_w + (int64_t)gk * 9 + w9) : 0.f;
            br[kk] = (chv && dw_b) ? __ldg(dw_b + gk) : 0.f;
          }
          if (gated) gsc = gch < p.C0 ? __ldg(p.gate_sc + (int64_t)b * p.C0 + gch) : 0.f;
        };
        load_weights(t);
        mbar_wait(&in_full[s * L::NG + g], (iph >> s) & 1u);
        iph ^= 1u << s;
        const int sa = gc % AS;
        mbar_wait(&a_empty[sa], ((gc / AS) & 1u) ^ 1u);  // the MMAs that read this A stage AS chunks ago retired
        unsigned char* my_op = a_base + sa * L::AST_BYTES;
        const TA* in_stage = reinterpret_cast<const TA*>(smem + s * L::IN_BYTES);
        const float* sa_stage = reinterpret_cast<const float*>(smem + L::OFF_SA + s * L::SA_BYTES);
        // the gated and the plain stencil are compiled apart, so that chunks without the gate run the plain loop unchanged
        auto stencil = [&](auto gate_c) {
          constexpr bool G = decltype(gate_c)::value;
#pragma unroll 1
          for (int task = t; task < NT * (KPL / KH); task += 128) {
            // task -> (input channel ci, column quad qc, row group rg).  A quarter-warp (8 lanes: one 128-bit shared-memory
            // wavefront) must touch 8 different 16-byte bank groups: PW = 32 -> the 8 quads of one channel row; PW = 16 ->
            // the 4 quads of TWO channels (16 words apart in the input tile, and KPL k-rows apart = a different
            // swizzle phase in the A operand).  Pairing the two row groups of one channel instead (rows 4 apart: 96 words in
            // the input tile, 4 KB in the A operand) put both halves on the same banks: every LDS.128 / STS.128 2-way.
            // At KPL = 4 the two halves of a task are 64 threads apart (warps 0-1 and 2-3 of the group), so every warp maps its
            // lanes as above: the halves read the same input window, and the A ring still takes 16 KB per chunk
            const int tb = task_base(task);
            int ci, qc, rg;
            if (PW == 32) {
              ci = tb >> 3; qc = tb & 7; rg = 0;
            } else {
              qc = tb & 3; ci = ((tb >> 4) << 1) | ((tb >> 2) & 1); rg = (tb >> 3) & 1;
            }
            constexpr int NQ = PW / 4;
            const int c0 = qc << 2, r0 = rg << 2;
            if (task != t) load_weights(task);   // KPL = 1: a second task per chunk (every other KPL: one task per thread)
            // smem column of patch column c (dx = -1..1) is c + XM + dx: the 4 outputs read cols c0+XM-1 .. c0+XM+4
            const TA* trow = in_stage + (ci * BH + r0) * BW + c0 + L::XM - 1;
            const float* srow = sa_stage + r0 * BW + c0 + L::XM - 1;
            float win[3][6];
            // one LDS.128 per row; the two edge values come from the neighbouring quads' registers (lane -1 / +1 hold columns
            // c0-4..c0-1 / c0+4..c0+7 of the same channel row), only the first / last quad of a patch row reads the halo
            // column -- the 32 lanes' scalar loads would all fall on 8 banks (stride 4 words): a 4-way conflict each
            const bool lb = (qc == 0), rb = (qc == NQ - 1);
            const int edge = lb ? 0 : 5;
            auto load_row = [&](float* wl, int r) {
              // bf16 stages: one LDS.64 per row (rows of 96 / 64 B, c0 + 8 a multiple of 4), widened to fp32 before the stencil
              float4 a;
              if constexpr (BA) a = bf16x4_f32(*reinterpret_cast<const uint2*>(trow + r * BW + 1));
              else a = *reinterpret_cast<const float4*>(trow + r * BW + 1);
              if (G) {
                const float4 ga = *reinterpret_cast<const float4*>(srow + r * BW + 1);
                a.x = __fmul_rn(__fmul_rn(a.x, gsc), ga.x);
                a.y = __fmul_rn(__fmul_rn(a.y, gsc), ga.y);
                a.z = __fmul_rn(__fmul_rn(a.z, gsc), ga.z);
                a.w = __fmul_rn(__fmul_rn(a.w, gsc), ga.w);
              }
              float left = __shfl_up_sync(0xffffffffu, a.w, 1), right = __shfl_down_sync(0xffffffffu, a.x, 1);
              if (lb | rb) {
                float e;
                if constexpr (BA) e = bf16_f32(trow[r * BW + edge]);
                else e = trow[r * BW + edge];
                if (G) e = __fmul_rn(__fmul_rn(e, gsc), srow[r * BW + edge]);
                if (lb) left = e; else right = e;
              }
              wl[0] = left; wl[1] = a.x; wl[2] = a.y; wl[3] = a.z; wl[4] = a.w; wl[5] = right;
            };
            // a paired tile's halves: rows h PH .. of the box, into that half's A tile (the same task, weights and window)
#pragma unroll
            for (int h = 0; h < NH; ++h) {
#pragma unroll
              for (int r = 0; r < 2; ++r) load_row(win[r], h * PH + r);
#pragma unroll
              for (int rr = 0; rr < 4; ++rr) {
                load_row(win[(rr + 2) % 3], h * PH + rr + 2);
                const float* w0 = win[rr % 3];
                const float* w1 = win[(rr + 1) % 3];
                const float* w2 = win[(rr + 2) % 3];
                const int m = (r0 + rr) * PW + c0;
#pragma unroll
                for (int kk = 0; kk < KH; ++kk) {
                  float o4[4];
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
                    float a = br[kk];
                    a = fmaf(wr[kk][0], w0[j], a); a = fmaf(wr[kk][1], w0[j + 1], a); a = fmaf(wr[kk][2], w0[j + 2], a);
                    a = fmaf(wr[kk][3], w1[j], a); a = fmaf(wr[kk][4], w1[j + 1], a); a = fmaf(wr[kk][5], w1[j + 2], a);
                    a = fmaf(wr[kk][6], w2[j], a); a = fmaf(wr[kk][7], w2[j + 1], a); a = fmaf(wr[kk][8], w2[j + 2], a);
                    o4[j] = a;
                  }
                  if (A_SMEM) {
                    const int kr = ci * KPL + kr0 + kk;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                      const uint32_t off = kmajor_offset(m + j, kr);
                      const float hi = X3 ? tf32_hi(o4[j]) : o4[j];
                      *reinterpret_cast<float*>(my_op + off) = hi;
                      if (X3) *reinterpret_cast<float*>(my_op + L::OFF_ALO + off) = o4[j] - hi;
                    }
                    continue;
                  }
                  // fp32 in both modes: the consumers split TF32X3's hi / lo parts after loading (one pass through shared memory)
                  *reinterpret_cast<float4*>(my_op + h * L::A_BYTES + a_tile_offset(ci * KPL + kr0 + kk, m)) =
                      make_float4(o4[0], o4[1], o4[2], o4[3]);
                }
              }
            }
          }
        };
        if (gated) stencil(std::true_type{}); else stencil(std::false_type{});
        if (A_SMEM) fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
        mbar_arrive(&a_full[sa]);
        mbar_arrive(&in_empty[s]);
      }
    }
  }
}

__host__ __device__ constexpr Prec tf32_prec(bool x3) { return x3 ? Prec::TF32X3 : Prec::TF32; }

template <int N_TILE, int KPL, int PW, bool X3, bool A_SMEM>
__global__ void __launch_bounds__(DsCfg<N_TILE, KPL, PW, tf32_prec(X3), A_SMEM>::THREADS, 1)
    dsconv_fused_kernel(const __grid_constant__ CUtensorMap map_in0, const __grid_constant__ CUtensorMap map_in1,
                        const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo,
                        const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_sa,
                        const DsParams p) {
  dsconv_body<N_TILE, KPL, PW, tf32_prec(X3), A_SMEM>(map_in0, map_in1, map_w, map_wlo, map_y, map_sa, p);
}

// kernels_per_layer = 4: CC = 8 input channels per chunk (7 680 B input boxes at both patch widths), two producer threads per
// task.  Register form only
template <int N_TILE, int PW, bool X3>
__global__ void __launch_bounds__(DsCfg<N_TILE, 4, PW, tf32_prec(X3), false>::THREADS, 1)
    dsconv_kpl4_kernel(const __grid_constant__ CUtensorMap map_in0, const __grid_constant__ CUtensorMap map_in1,
                       const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo,
                       const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_sa,
                       const DsParams p) {
  dsconv_body<N_TILE, 4, PW, tf32_prec(X3), false>(map_in0, map_in1, map_w, map_wlo, map_y, map_sa, p);
}

// SMAAT_PW_BF16, k = 1, 2 and 4: the register form with bf16 operands.  A kernel of its own, so that the tf32 kernels above
// keep their names and instance sets
template <int N_TILE, int KPL, int PW>
__global__ void __launch_bounds__(DsCfg<N_TILE, KPL, PW, Prec::BF16, false>::THREADS, 1)
    dsconv_bf16_kernel(const __grid_constant__ CUtensorMap map_in0, const __grid_constant__ CUtensorMap map_in1,
                       const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo,
                       const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_sa,
                       const DsParams p) {
  dsconv_body<N_TILE, KPL, PW, Prec::BF16, false>(map_in0, map_in1, map_w, map_wlo, map_y, map_sa, p);
}

// The serving forward's bf16 route (smaat_dsconv_bf16_fwd and its head forms): bf16 input and output in HBM, bf16 operands.
// k = 1, 2
template <int N_TILE, int KPL, int PW>
__global__ void __launch_bounds__(DsCfg<N_TILE, KPL, PW, Prec::BF16, false, uint16_t>::THREADS, 1)
    dsconv_bf16act_kernel(const __grid_constant__ CUtensorMap map_in0, const __grid_constant__ CUtensorMap map_in1,
                          const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo,
                          const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_sa,
                          const DsParams p) {
  dsconv_body<N_TILE, KPL, PW, Prec::BF16, false, uint16_t>(map_in0, map_in1, map_w, map_wlo, map_y, map_sa, p);
}

// Paired tiles (DsCfg PAIR: two patches of PH rows per tile): N_TILE 64, the register form, tf32 / 3xTF32, k = 2 and 4.  A
// kernel of its own, so that the single-tile kernels above keep their names and instance sets
template <int KPL, int PW, bool X3>
__global__ void __launch_bounds__(DsCfg<64, KPL, PW, tf32_prec(X3), false, float, true>::THREADS, 1)
    dsconv_pair_kernel(const __grid_constant__ CUtensorMap map_in0, const __grid_constant__ CUtensorMap map_in1,
                       const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo,
                       const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_sa,
                       const DsParams p) {
  dsconv_body<64, KPL, PW, tf32_prec(X3), false, float, true>(map_in0, map_in1, map_w, map_wlo, map_y, map_sa, p);
}

// Wide tiles (DsCfg WIDE: both 128-channel halves of 128 < Cout <= 256 per tile): the register form, tf32 / 3xTF32, k = 2.  A kernel
// of its own, so that the two-pass kernels keep their names and instance sets
template <int PW, bool X3>
__global__ void __launch_bounds__(DsCfg<128, 2, PW, tf32_prec(X3), false, float, false, true>::THREADS, 1)
    dsconv_wide_kernel(const __grid_constant__ CUtensorMap map_in0, const __grid_constant__ CUtensorMap map_in1,
                       const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_wlo,
                       const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_sa,
                       const DsParams p) {
  dsconv_body<128, 2, PW, tf32_prec(X3), false, float, false, true>(map_in0, map_in1, map_w, map_wlo, map_y, map_sa, p);
}

template <int N_TILE, int KPL, int PW, Prec P, bool A_SMEM, typename TA = float, bool PAIR = false, bool WIDE = false>
static auto ds_kernel() {
  static_assert(KPL == 1 || KPL == 2 || (KPL == 4 && !A_SMEM), "fused DS conv instances: k = 1, 2 (both A forms), 4 (register form)");
  if constexpr (WIDE) return dsconv_wide_kernel<PW, P == Prec::TF32X3>;
  else if constexpr (PAIR) return dsconv_pair_kernel<KPL, PW, P == Prec::TF32X3>;
  else if constexpr (sizeof(TA) == 2) return dsconv_bf16act_kernel<N_TILE, KPL, PW>;
  else if constexpr (P == Prec::BF16) return dsconv_bf16_kernel<N_TILE, KPL, PW>;
  else if constexpr (KPL == 4) return dsconv_kpl4_kernel<N_TILE, PW, P == Prec::TF32X3>;
  else return dsconv_fused_kernel<N_TILE, KPL, PW, P == Prec::TF32X3, A_SMEM>;
}

template <int N_TILE, int KPL, int PW, Prec P, bool A_SMEM, typename TA, bool PAIR, bool WIDE>
static int launch_ds(DsCfg<N_TILE, KPL, PW, P, A_SMEM, TA, PAIR, WIDE>, const CUtensorMap& m0, const CUtensorMap& m1,
                     const CUtensorMap& mw, const CUtensorMap& mwl, const CUtensorMap& my, const CUtensorMap& msa, DsParams p, int B,
                     cudaStream_t st) {
  using L = DsCfg<N_TILE, KPL, PW, P, A_SMEM, TA, PAIR, WIDE>;
  auto kern = ds_kernel<N_TILE, KPL, PW, P, A_SMEM, TA, PAIR, WIDE>();
  static std::atomic<uint64_t> attr_mask{0};   // cudaFuncSetAttribute is per device
  if (first_use_on_device(attr_mask)) {
    // class launches append the class weights (CLS_SMEM); every other launch requests TOTAL, as before
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL + L::CLS_SMEM);
    if (e != cudaSuccess)
      return fail(SMAAT_E_CUDA, "dsconv: smem attribute (%d B): %s", L::TOTAL + L::CLS_SMEM, cudaGetErrorString(e));
    int r = check_reg_budget((const void*)kern, L::THREADS, L::REGS_SUM, "dsconv");
    if (r) return r;
  }
  p.tiles_x = ceil_div(p.W, PW);
  p.tiles_y = ceil_div(p.H, L::TH);
  p.npass = ceil_div(p.Cout, N_TILE * L::NW);
  const int64_t total = (int64_t)B * p.tiles_x * p.tiles_y * p.npass;
  SMAAT_REQUIRE(total < (1ll << 31), "dsconv: too many tiles");
  p.total_tiles = (int)total;
  p.nchunks = ceil_div(p.C0 + p.C1, L::CC);
  p.npart = 2 * p.tiles_x * p.tiles_y * L::NH;   // per half-patch, as smaat_dsconv_pool_parts counts them
  const int grid = p.total_tiles < num_sms() ? p.total_tiles : num_sms();
  kern<<<grid, L::THREADS, L::TOTAL + (p.ncls ? L::CLS_SMEM : 0), st>>>(m0, m1, mw, mwl, my, msa, p);
  SMAAT_LAUNCH_CHECK("smaat_dsconv_fwd");
  return SMAAT_OK;
}

// patch width: 32 (PH = 4) or 16 (PH = 8), whichever wastes fewer MMA rows; 0 = not worth fusing
static int pick_pw(int H, int W) {
  double best = 1e9;
  int pw = 0;
  const int cand[2] = {32, 16};
  for (int i = 0; i < 2; ++i) {
    const int c = cand[i], ph = TC_BM / c;
    const double waste = ((double)ceil_div(W, c) * c / W) * ((double)ceil_div(H, ph) * ph / H);
    if (waste < best - 1e-9) {
      best = waste;
      pw = c;
    }
  }
  return best <= 1.35 ? pw : 0;
}

// Where the A operand (the depthwise result) goes to the tensor core: 0 = auto (the register form), 1 = read by wgmma from
// shared memory through a descriptor, 2 = loaded into registers first.  SMAAT_DS_IMPL presets it.  Auto takes the register
// form: bench.py's B = 32, 12 x 288 x 288 forward ran at 2 365-2 369 frames/s with it and 2 187-2 194 with the shared-memory
// form (H100 80GB HBM3 SXM, 700 W power limit, two alternated runs each); the scalar K-major stores of the shared-memory form
// cost the producers more than the register form's fragment loads cost the consumers.
static std::atomic<int> g_ds_impl{-1};
static int ds_impl() {
  int v = g_ds_impl.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("SMAAT_DS_IMPL");
    v = e ? atoi(e) : 0;
    if (v < 0 || v > 2) v = 0;
    g_ds_impl.store(v, std::memory_order_relaxed);
  }
  return v;
}

// Whether 128 < Cout <= 256 runs as wide tiles (1, the default) or in two 128-channel passes (0).  SMAAT_DSCONV_WIDE presets it
static std::atomic<int> g_ds_wide{-1};
static bool ds_wide_on() {
  int v = g_ds_wide.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("SMAAT_DSCONV_WIDE");
    v = (e && atoi(e) == 0) ? 0 : 1;
    g_ds_wide.store(v, std::memory_order_relaxed);
  }
  return v != 0;
}

// Whether paired tiles run where ds_select takes them (1, the default) or one patch per tile (0).  SMAAT_DSCONV_PAIR presets it
static std::atomic<int> g_ds_pair{-1};
static bool ds_pair_on() {
  int v = g_ds_pair.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("SMAAT_DSCONV_PAIR");
    v = (e && atoi(e) == 0) ? 0 : 1;
    g_ds_pair.store(v, std::memory_order_relaxed);
  }
  return v != 0;
}

// One fused DS conv request, its operands by name.  x0 / x1, y, the logits (oc_y) and the max-pool are fp32, or bf16 bits where
// bact (and pooled_bf16) say so; pw_w is fp32, or the smaat_pack_bf16 pack in SMAAT_PW_BF16.  The fields up to Cout are those
// every entry point takes, initialised in their order there; the eligibility queries then fill the epilogue they ask about,
// with y null (not known yet)
struct DsReq {
  const void* x0; int C0; int64_t x0_bstride;
  const void* x1; int C1; int64_t x1_bstride;
  const void* pw_w; int H, W, k, Cout;
  int B = 0, relu = 0, mode = SMAAT_PW_TF32;
  bool bact = false;   // bf16 activations
  const float* dw_w = nullptr; const float* dw_b = nullptr; const float* pw_w_lo = nullptr;
  const float* scale = nullptr; const float* shift = nullptr;
  void* y = nullptr; int64_t y_bstride = 0;
  // the epilogue
  double* stats = nullptr;                                         // batch statistics
  const float* oc_w = nullptr; const float* oc_b = nullptr;        // a head, an OutConv in place of y: one class into oc_y,
  void* oc_y = nullptr; int ncls = 0; int64_t* cls = nullptr;      // or ncls classes into the logits oc_y and / or the map cls
  const float* gate_sc = nullptr; const float* gate_sa = nullptr;  // the CBAM gate on x0
  float* pool_sum = nullptr; float* pool_max = nullptr;            // the CBAM partial pools
  void* pooled = nullptr; int pooled_bf16 = 0;                     // the max-pool
  bool head() const { return oc_y || ncls > 0; }
};

// An eligibility query asks about batch statistics or a max-pool it has no address for yet by this one; ds_select only tests
// those pointers for null
alignas(16) static char g_ds_asked[16];

// The kernel instance that runs a request, the DsCfg parameters ds_visit maps it to, and why ds_select declines the request if
// it does
enum DsDecline { DS_TAKEN, DS_SHAPE, DS_UNSTAGED, DS_CLASSES };
struct DsInst {
  int n_tile, k, pw;
  Prec prec;
  bool a_smem, bact, pair, wide;
  DsDecline declined;
};

// ds_visit: the DsCfg type of an instance, handed to f.  With ds_kernel, the only list of the instances that are built
template <int N_TILE, int KPL, int PW, Prec P, typename F>
static int ds_visit_inst(const DsInst& c, F& f) {
  if constexpr (P != Prec::BF16 && N_TILE == 128 && KPL == 2) {
    if (c.wide) return f(DsCfg<128, 2, PW, P, false, float, false, true>{});
  }
  if constexpr (P != Prec::BF16 && N_TILE == 64 && KPL != 1) {
    if (c.pair) return f(DsCfg<64, KPL, PW, P, false, float, true>{});
  }
  if constexpr (P == Prec::BF16 && KPL != 4) {
    if (c.bact) return f(DsCfg<N_TILE, KPL, PW, P, false, uint16_t>{});
  }
  if constexpr (P != Prec::BF16 && KPL != 4) {
    if (c.a_smem) return f(DsCfg<N_TILE, KPL, PW, P, true>{});
  }
  return f(DsCfg<N_TILE, KPL, PW, P, false>{});
}
template <int N_TILE, int KPL, int PW, typename F>
static int ds_visit_prec(const DsInst& c, F& f) {
  if (c.prec == Prec::BF16) return ds_visit_inst<N_TILE, KPL, PW, Prec::BF16>(c, f);
  if (c.prec == Prec::TF32X3) return ds_visit_inst<N_TILE, KPL, PW, Prec::TF32X3>(c, f);
  return ds_visit_inst<N_TILE, KPL, PW, Prec::TF32>(c, f);
}
template <typename F>
static int ds_visit(const DsInst& c, F f) {
  if (c.n_tile == 64) {
    if (c.k == 4) return c.pw == 32 ? ds_visit_prec<64, 4, 32>(c, f) : ds_visit_prec<64, 4, 16>(c, f);
    if (c.k == 2) return c.pw == 32 ? ds_visit_prec<64, 2, 32>(c, f) : ds_visit_prec<64, 2, 16>(c, f);
    return c.pw == 32 ? ds_visit_prec<64, 1, 32>(c, f) : ds_visit_prec<64, 1, 16>(c, f);
  }
  if (c.k == 4) return c.pw == 32 ? ds_visit_prec<128, 4, 32>(c, f) : ds_visit_prec<128, 4, 16>(c, f);
  if (c.k == 2) return c.pw == 32 ? ds_visit_prec<128, 2, 32>(c, f) : ds_visit_prec<128, 2, 16>(c, f);
  return c.pw == 32 ? ds_visit_prec<128, 1, 32>(c, f) : ds_visit_prec<128, 1, 16>(c, f);
}

// The most classes whose OutConv weights an instance keeps in shared memory
static int ds_max_classes(const DsInst& c) {
  return ds_visit(c, [](auto cfg) { return (int)decltype(cfg)::MAX_CLASSES; });
}

// The instance that runs a request (wide, else paired, else single tiles), or why none does.  The epilogue's limits are those
// of that instance: the CBAM pools and the max-pool are read back from its staging buffers (ST_BUFS > 0), and the class
// weights must fit beside its rings (MAX_CLASSES)
static DsInst ds_select(const DsReq& r) {
  const bool a_smem = ds_impl() == 1, bf16 = r.mode == SMAAT_PW_BF16, head = r.head(), stats = r.stats;
  const int k = r.k, Cout = r.Cout;
  const Prec prec = bf16 ? Prec::BF16 : r.mode == SMAAT_PW_TF32X3 ? Prec::TF32X3 : Prec::TF32;
  DsInst c{Cout > 64 ? 128 : 64, k, pick_pw(r.H, r.W), prec, a_smem, r.bact, false, false, DS_SHAPE};
  // k = 4 and BF16 have register-form instances only (dsconv_kpl4_kernel, dsconv_bf16_kernel): with the shared-memory A form
  // selected they stay unfused
  if ((k != 1 && k != 2 && k != 4) || (a_smem && (k == 4 || bf16))) return c;
  // bf16 activations (dsconv_bf16act_kernel): bf16 operands, k = 1, 2, no batch statistics; TMA takes 16-byte row and plane
  // strides, so W and the batch strides are multiples of 8 elements
  if (r.bact && (!bf16 || k == 4 || stats || r.W % 8 != 0 || r.x0_bstride % 8 != 0 || (r.C1 > 0 && r.x1_bstride % 8 != 0) ||
                 (r.y && r.y_bstride % 8 != 0)))
    return c;
  // y: the epilogue stores it by TMA, which needs a 16-byte aligned base and 16-byte multiples as strides
  if (r.y && (!aligned16(r.y) || r.y_bstride % 4 != 0)) return c;
  // Wide tiles (dsconv_wide_kernel) where they are built (k = 2, the register form, tf32 / 3xTF32, fp32 maps) and switched on
  // (smaat_set_dsconv_wide): 128 < Cout <= 256 in one pass instead of two, with no OutConv (no network ends in such a conv)
  c.wide = ds_wide_on() && Cout > 128 && Cout <= 256 && k == 2 && !a_smem && !bf16 && !head;
  // Cout > 128: whole passes of 128 channels, or one wide tile for any Cout up to 256; batch statistics and the fused OutConv are
  // taken up to 128 channels
  if (Cout < 8 || Cout > 512 || (Cout > 128 && (stats || head))) return c;
  if (Cout > 128 && Cout % 128 != 0 && !c.wide) return c;
  if (r.W % 4 != 0 || !aligned16(r.x0) || r.x0_bstride % 4 != 0) return c;
  if (r.C1 > 0 && (!aligned16(r.x1) || r.x1_bstride % 4 != 0 || r.C0 % (TC_BK / k) != 0)) return c;
  // fp32 weight rows are K * 4 bytes, which TMA takes in multiples of 16; the bf16 pack's rows are padded to 32 k (bact only, so
  // that the fp32 route keeps its choices)
  if ((k * (r.C0 + r.C1) % 4 != 0 && !r.bact) || !aligned16(r.pw_w) || (r.pw_w_lo && !aligned16(r.pw_w_lo))) return c;
  if (!c.pw) return c;
  // Paired tiles (dsconv_pair_kernel) where they are built (N_TILE 64, k = 2, 4, the register form, tf32 / 3xTF32, fp32 maps)
  // and they cover the image with no more rows than single patches: an even number of patch rows.  The pair then runs the same
  // pixels with half the chunks' fixed costs (input box, weight chunk, hand-offs) per pixel.  Its rings leave room for the
  // weights of DS_MIN_CLASSES classes, not always 32: more classes take the single tile
  c.pair = ds_pair_on() && c.n_tile == 64 && (k == 2 || k == 4) && !a_smem && !bf16 && ceil_div(r.H, TC_BM / c.pw) % 2 == 0 &&
           r.ncls <= DS_MIN_CLASSES;
  const bool staged = ds_visit(c, [](auto cfg) { return (int)decltype(cfg)::ST_BUFS; }) > 0;
  c.declined = r.pooled && !staged ? DS_UNSTAGED : r.ncls > ds_max_classes(c) ? DS_CLASSES : DS_TAKEN;
  return c;
}

// Launches the request on the instance ds_select takes, after the argument checks; a declined request launches nothing
static int ds_launch(const DsReq& r, void* stream) {
  const int B = r.B, C0 = r.C0, C1 = r.C1, H = r.H, W = r.W, k = r.k, Cout = r.Cout;
  const bool head = r.head(), bf16 = r.mode == SMAAT_PW_BF16;
  SMAAT_REQUIRE(r.x0 && r.dw_w && r.pw_w && (r.y || r.oc_y || r.cls), "dsconv: null pointer");
  SMAAT_REQUIRE(!r.gate_sc == !r.gate_sa, "dsconv: the CBAM gate needs both sc and sa");
  SMAAT_REQUIRE(!r.gate_sa || aligned16(r.gate_sa), "dsconv: the CBAM gate map must be 16-byte aligned");
  SMAAT_REQUIRE(!r.pool_sum || (r.pool_max && r.pooled && r.y && !r.oc_y && !r.stats),
                "dsconv: the CBAM pools need sum, max and max-pool outputs and y");
  SMAAT_REQUIRE(!r.pooled || (r.y && !head && !r.stats), "dsconv: the max-pool needs y, and no OutConv or batch statistics");
  SMAAT_REQUIRE(!r.pooled_bf16 || r.bact, "dsconv: a bf16 max-pool needs bf16 activations");
  SMAAT_REQUIRE(!r.pooled || (reinterpret_cast<uintptr_t>(r.pooled) & (r.pooled_bf16 ? 3u : 7u)) == 0,
                "dsconv: the max-pool output must be %d-byte aligned", r.pooled_bf16 ? 4 : 8);
  SMAAT_REQUIRE(B > 0 && C0 > 0 && C1 >= 0 && H > 0 && W > 0 && Cout > 0, "dsconv: bad shape");
  SMAAT_REQUIRE(C1 == 0 || r.x1, "dsconv: C1=%d but x1 is null", C1);
  SMAAT_REQUIRE(r.mode == SMAAT_PW_TF32 || r.mode == SMAAT_PW_TF32X3 || r.mode == SMAAT_PW_BF16,
                "dsconv: mode must be SMAAT_PW_TF32, SMAAT_PW_TF32X3 or SMAAT_PW_BF16");
  SMAAT_REQUIRE(r.mode != SMAAT_PW_TF32X3 || r.pw_w_lo, "dsconv: TF32X3 needs pw_w_lo (see smaat_split_tf32)");
  SMAAT_REQUIRE(head || r.y_bstride >= (int64_t)Cout * H * W, "dsconv: y batch stride too small");
  SMAAT_REQUIRE(!head || (r.oc_w && !r.stats), "dsconv+outconv: needs the OutConv weight and no batch statistics");
  SMAAT_REQUIRE(!r.bact || (bf16 && !r.stats && !r.pool_sum), "dsconv: bf16 activations take bf16 operands, no statistics and no pools");
  const DsInst c = ds_select(r);
  if (c.declined == DS_SHAPE)
    return fail(SMAAT_E_UNSUPPORTED,
                r.bact ? "dsconv_bf16: not taken by the bf16-activation kernel (k=%d Cout=%d H=%d W=%d; needs k = 1 or 2, W and the "
                         "batch strides multiples of 8, 16-byte aligned tensors, the register A form)"
                       : "dsconv: shape or output layout not taken by the fused kernel (k=%d Cout=%d H=%d W=%d, y 16-byte aligned "
                         "with a batch stride that is a multiple of 4); use dw3x3 + pw1x1",
                k, Cout, H, W);
  if (c.declined == DS_UNSTAGED)
    return fail(SMAAT_E_UNSUPPORTED, "dsconv: the CBAM pools and the max-pool need the staged epilogue");
  if (c.declined == DS_CLASSES)
    return fail(SMAAT_E_UNSUPPORTED, "dsconv+classify: %d classes, this instance keeps the weights of at most %d", r.ncls,
                ds_max_classes(c));
  const int pw = c.pw, ph = TC_BM / pw, cc = TC_BK / k, K = k * (C0 + C1);
  const int th = c.pair ? 2 * ph : ph;   // a paired tile's boxes span both patches
  // activation maps: fp32, or bf16 (bact)
  const CUtensorMapDataType adt = r.bact ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const uint64_t esz = r.bact ? 2 : 4;

  CUtensorMap m0, m1, mw, mwl;
  const int xm = 16 / (int)esz;   // DsCfg::XM
  const uint32_t box[4] = {(uint32_t)(pw + 2 * xm), (uint32_t)(th + 2), (uint32_t)cc, 1u};
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C0, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * esz, (uint64_t)H * W * esz, (uint64_t)r.x0_bstride * esz};
    int e = make_tmap(&m0, adt, r.x0, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "dsconv(x0)");
    if (e) return e;
    m1 = m0;
  }
  if (C1 > 0) {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C1, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * esz, (uint64_t)H * W * esz, (uint64_t)r.x1_bstride * esz};
    int e = make_tmap(&m1, adt, r.x1, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, "dsconv(x1)");
    if (e) return e;
  }
  {
    const uint64_t kw = bf16 ? (uint64_t)(K + TC_BK - 1) / TC_BK * TC_BK : (uint64_t)K;   // the bf16 pack's row length
    const uint64_t dims[2] = {kw, (uint64_t)Cout};
    const uint64_t str[2] = {0, kw * (bf16 ? 2 : 4)};
    const uint32_t wbox[2] = {(uint32_t)TC_BK, (uint32_t)c.n_tile};
    int e = bf16 ? make_tmap(&mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, r.pw_w, 2, dims, str, wbox, CU_TENSOR_MAP_SWIZZLE_64B, "dsconv(w bf16)")
                 : make_tmap_f32(&mw, r.pw_w, 2, dims, str, wbox, CU_TENSOR_MAP_SWIZZLE_128B, "dsconv(w)");
    if (e) return e;
    mwl = mw;
    if (r.mode == SMAAT_PW_TF32X3) {
      e = make_tmap_f32(&mwl, r.pw_w_lo, 2, dims, str, wbox, CU_TENSOR_MAP_SWIZZLE_128B, "dsconv(w_lo)");
      if (e) return e;
    }
  }
  // the staged epilogue's store box: one warpgroup's half-patch (PW x PH / 2 pixels) x 32 channels, swizzled by its row length
  CUtensorMap my = m0;
  if (!head) {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)Cout, (uint64_t)B};
    const uint64_t str[4] = {0, (uint64_t)W * esz, (uint64_t)H * W * esz, (uint64_t)r.y_bstride * esz};
    const uint32_t ybox[4] = {(uint32_t)pw, (uint32_t)(ph / 2), 32u, 1u};
    // bf16 boxes are staged unswizzled (the epilogue's bf16 branch)
    const CUtensorMapSwizzle ysw = r.bact ? CU_TENSOR_MAP_SWIZZLE_NONE : pw == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    int e = make_tmap(&my, adt, r.y, 4, dims, str, ybox, ysw, "dsconv(y)");
    if (e) return e;
  }
  // the CBAM spatial gate sa (B, 1, H, W): one-channel halo boxes at the input boxes' origin
  CUtensorMap msa = m0;
  if (r.gate_sa) {
    const uint64_t dims[3] = {(uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t str[3] = {0, (uint64_t)W * 4, (uint64_t)H * W * 4};
    const uint32_t sbox[3] = {(uint32_t)(pw + 2 * xm), (uint32_t)(th + 2), 1u};
    int e = make_tmap_f32(&msa, r.gate_sa, 3, dims, str, sbox, CU_TENSOR_MAP_SWIZZLE_NONE, "dsconv(gate sa)");
    if (e) return e;
  }
  DsParams p{};
  p.dw_w = r.dw_w; p.dw_b = r.dw_b; p.scale = r.scale; p.shift = r.shift; p.y = static_cast<float*>(r.y); p.y_bstride = r.y_bstride;
  p.stats = r.stats; p.oc_w = r.oc_w; p.oc_b = r.oc_b; p.oc_y = static_cast<float*>(r.oc_y); p.ncls = r.ncls; p.cls = r.cls;
  p.gate_sc = r.gate_sc; p.pool_sum = r.pool_sum; p.pool_max = r.pool_max; p.pooled = static_cast<float*>(r.pooled);
  p.pooled_bf16 = r.pooled_bf16; p.C0 = C0; p.C1 = C1; p.H = H; p.W = W; p.Cout = Cout; p.relu = r.relu; p.K = K;
  return ds_visit(c, [&](auto cfg) { return launch_ds(cfg, m0, m1, mw, mwl, my, msa, p, B, (cudaStream_t)stream); });
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_set_dsconv_impl(int impl) {
  SMAAT_REQUIRE(impl >= 0 && impl <= 2, "set_dsconv_impl: 0 = auto, 1 = A operand from shared memory, 2 = A operand from registers");
  g_ds_impl.store(impl, std::memory_order_relaxed);
  return SMAAT_OK;
}

extern "C" int smaat_set_dsconv_wide(int enabled) {
  SMAAT_REQUIRE(enabled == 0 || enabled == 1, "set_dsconv_wide: 1 = wide tiles for 128 < Cout <= 256, 0 = passes of 128 channels");
  g_ds_wide.store(enabled, std::memory_order_relaxed);
  return SMAAT_OK;
}

extern "C" int smaat_set_dsconv_pair(int enabled) {
  SMAAT_REQUIRE(enabled == 0 || enabled == 1, "set_dsconv_pair: 1 = paired tiles where they are built, 0 = one patch per tile");
  g_ds_pair.store(enabled, std::memory_order_relaxed);
  return SMAAT_OK;
}

extern "C" int smaat_dsconv_eligible2(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                      const float* pw_w, int H, int W, int k, int Cout, int with_stats) {
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.stats = with_stats ? reinterpret_cast<double*>(g_ds_asked) : nullptr;
  return ds_select(q).declined == DS_TAKEN;
}

extern "C" int smaat_dsconv_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                     const float* pw_w, int H, int W, int k, int Cout) {
  return smaat_dsconv_eligible2(x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout, 0);
}

extern "C" int smaat_dsconv_cbam_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                          const float* pw_w, int H, int W, int k, int Cout, int mode, int with_gate, int with_pools) {
  if (mode != SMAAT_PW_TF32 && mode != SMAAT_PW_TF32X3 && mode != SMAAT_PW_BF16) return 0;
  (void)with_gate;   // every fused instance takes the gate
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.mode = mode; q.pooled = with_pools ? g_ds_asked : nullptr;
  return ds_select(q).declined == DS_TAKEN;
}

extern "C" int smaat_dsconv_pool_parts(int H, int W) {
  const int pw = (H > 0 && W > 0) ? pick_pw(H, W) : 0;
  return pw ? 2 * ceil_div(W, pw) * ceil_div(H, TC_BM / pw) : 0;
}

extern "C" int smaat_dsconv_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                                const float* scale, const float* shift, float* y, int64_t y_bstride, double* stats, int B, int H,
                                int W, int k, int Cout, int relu, int mode, void* stream) {
  SMAAT_REQUIRE(y, "dsconv: null output");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = mode; q.dw_w = dw_w; q.dw_b = dw_b; q.pw_w_lo = pw_w_lo; q.scale = scale; q.shift = shift;
  q.y = y; q.y_bstride = y_bstride; q.stats = stats;
  return ds_launch(q, stream);
}

/* The network's last two modules in one kernel: DS conv -> BN/ReLU -> OutConv(Cout -> 1) (reference models/SmaAt_UNet.py:55-56,
 * unet_parts.py:67-73).  The Cout-channel activation never reaches HBM: the four lanes of a fragment group hold one pixel's
 * Cout <= 128 accumulators and reduce them against oc_w.  logits: (B, 1, H, W). */
extern "C" int smaat_dsconv_outconv_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                        const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                                        const float* scale, const float* shift, const float* oc_w, const float* oc_b,
                                        float* logits, int B, int H, int W, int k, int Cout, int relu, int mode, void* stream) {
  SMAAT_REQUIRE(oc_w && logits, "dsconv+outconv: null pointer");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = mode; q.dw_w = dw_w; q.dw_b = dw_b; q.pw_w_lo = pw_w_lo; q.scale = scale; q.shift = shift;
  q.oc_w = oc_w; q.oc_b = oc_b; q.oc_y = logits;
  return ds_launch(q, stream);
}

extern "C" int smaat_dsconv_classify_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                              const float* pw_w, int H, int W, int k, int Cout, int K, int mode) {
  if (mode != SMAAT_PW_TF32 && mode != SMAAT_PW_TF32X3 && mode != SMAAT_PW_BF16) return 0;
  if (K < 1 || K > DS_MAX_CLASSES) return 0;
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.mode = mode; q.ncls = K;
  return ds_select(q).declined == DS_TAKEN;
}

/* The network's last two modules for a K-class model, ending in the class map: DS conv -> BN/ReLU -> OutConv(Cout -> K) ->
 * argmax over the K logits of each pixel (the reference's torch.argmax(softmax(y_pred), dim=1), train_SmaAtUNet.py:76; softmax
 * keeps the order).  Neither the Cout-channel activation nor, unless asked for, the K logit planes reach HBM. */
extern "C" int smaat_dsconv_classify_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                         const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                                         const float* scale, const float* shift, const float* oc_w, const float* oc_b, int K,
                                         float* logits, int64_t* classes, int B, int H, int W, int k, int Cout, int relu, int mode,
                                         void* stream) {
  SMAAT_REQUIRE(oc_w && (logits || classes), "dsconv+classify: needs the OutConv weight and a logits or a classes output");
  SMAAT_REQUIRE(K >= 1, "dsconv+classify: K=%d classes", K);
  if (K > DS_MAX_CLASSES)
    return fail(SMAAT_E_UNSUPPORTED, "dsconv+classify: K=%d classes, the fused epilogue takes at most %d; use smaat_dsconv_fwd + "
                                     "smaat_outconv_fwd + smaat_argmax_channels_fwd", K, DS_MAX_CLASSES);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(oc_w) & 3u) == 0 && (reinterpret_cast<uintptr_t>(logits) & 3u) == 0 &&
                    (reinterpret_cast<uintptr_t>(classes) & 7u) == 0,
                "dsconv+classify: weights / logits must be 4-byte and classes 8-byte aligned");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = mode; q.dw_w = dw_w; q.dw_b = dw_b; q.pw_w_lo = pw_w_lo; q.scale = scale; q.shift = shift;
  q.oc_w = oc_w; q.oc_b = oc_b; q.oc_y = logits; q.ncls = K; q.cls = classes;
  return ds_launch(q, stream);
}

/* The fused DS conv of the serving forward with the CBAM fusions around it (models/layers.py:90-141, SmaAt_UNet.py:41-57).
 * gate_sc (B, C0) and gate_sa (B, 1, H, W), both or neither: x0 is read as the CBAM output (x0 * sc) * sa, exactly as
 * smaat_cbam_gate_scale_fwd / smaat_cbam_scale_fwd would have written it.  pool_sum / pool_max (B, npart, Cout) and pooled
 * (B, Cout, H / 2, W / 2), all or none: the epilogue also writes per half-patch partial sums and maxima of y for the channel
 * gate's pools (npart = smaat_dsconv_pool_parts(H, W); smaat_cbam_mlp_partials_fwd finishes them) and MaxPool2d(2)(y). */
extern "C" int smaat_dsconv_cbam_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                     const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                                     const float* scale, const float* shift, float* y, int64_t y_bstride, const float* gate_sc,
                                     const float* gate_sa, float* pool_sum, float* pool_max, float* pooled, int B, int H, int W, int k,
                                     int Cout, int relu, int mode, void* stream) {
  SMAAT_REQUIRE(y, "dsconv_cbam: null output");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = mode; q.dw_w = dw_w; q.dw_b = dw_b; q.pw_w_lo = pw_w_lo; q.scale = scale; q.shift = shift;
  q.y = y; q.y_bstride = y_bstride; q.gate_sc = gate_sc; q.gate_sa = gate_sa; q.pool_sum = pool_sum; q.pool_max = pool_max;
  q.pooled = pooled;
  return ds_launch(q, stream);
}

/* The fused DS conv that also writes MaxPool2d(2) of its output, for the DownDS that reads it next (UNetDS's encoder, which has
 * no CBAM to hand the max-pool over): the staged epilogue reads each stored slice back, so pooled is the max-pool of y bit for
 * bit, without a second read of y.  No partial sums, no atomics.  pooled (B, Cout, H / 2, W / 2), 8-byte aligned; floor for
 * odd H.  Eligibility: smaat_dsconv_cbam_eligible with pools. */
extern "C" int smaat_dsconv_maxpool_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                             const float* pw_w, int H, int W, int k, int Cout, int mode) {
  return smaat_dsconv_cbam_eligible(x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout, mode, 0, 1);
}

extern "C" int smaat_dsconv_maxpool_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                        const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                                        const float* scale, const float* shift, float* y, int64_t y_bstride, float* pooled, int B,
                                        int H, int W, int k, int Cout, int relu, int mode, void* stream) {
  SMAAT_REQUIRE(y && pooled, "dsconv_maxpool: null output");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = mode; q.dw_w = dw_w; q.dw_b = dw_b; q.pw_w_lo = pw_w_lo; q.scale = scale; q.shift = shift;
  q.y = y; q.y_bstride = y_bstride; q.pooled = pooled;
  return ds_launch(q, stream);
}

/* ---- bf16 activations: the serving forward's bf16 route -------------------------------------------------------------------
 * x0 / x1 and the output (y or the logits) are bf16 (raw uint16_t bits) in HBM; the depthwise stencil, the accumulation and
 * the epilogue run in fp32, the GEMM takes bf16 operands (pw_w: the smaat_pack_bf16 pack), and each stored value is rounded
 * to bf16 once.  k = 1 or 2, the register A form, no batch statistics and no CBAM pools.  The CBAM gate (gate_sc, gate_sa:
 * fp32, both or neither) is applied as in smaat_dsconv_cbam_fwd, (x0 * sc) * sa in fp32 from the widened x0. */
extern "C" int smaat_dsconv_bf16_eligible(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                          const void* pw_w, int H, int W, int k, int Cout, int ncls) {
  if (ncls < 0 || ncls > DS_MAX_CLASSES) return 0;
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.mode = SMAAT_PW_BF16; q.bact = true; q.ncls = ncls;
  return ds_select(q).declined == DS_TAKEN;
}

extern "C" int smaat_dsconv_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                     const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale,
                                     const float* shift, void* y, int64_t y_bstride, const float* gate_sc, const float* gate_sa,
                                     int B, int H, int W, int k, int Cout, int relu, void* stream) {
  SMAAT_REQUIRE(y, "dsconv_bf16: null output");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = SMAAT_PW_BF16; q.bact = true; q.dw_w = dw_w; q.dw_b = dw_b; q.scale = scale; q.shift = shift;
  q.y = y; q.y_bstride = y_bstride; q.gate_sc = gate_sc; q.gate_sa = gate_sa;
  return ds_launch(q, stream);
}

/* smaat_dsconv_outconv_fwd from bf16 activations: the (B, 1, H, W) logits, accumulated in fp32 and stored as bf16. */
extern "C" int smaat_dsconv_outconv_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                             const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale,
                                             const float* shift, const float* oc_w, const float* oc_b, void* logits, int B, int H,
                                             int W, int k, int Cout, int relu, void* stream) {
  SMAAT_REQUIRE(oc_w && logits, "dsconv+outconv bf16: null pointer");
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(logits) & 1u) == 0, "dsconv+outconv bf16: logits must be 2-byte aligned");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = SMAAT_PW_BF16; q.bact = true; q.dw_w = dw_w; q.dw_b = dw_b; q.scale = scale; q.shift = shift;
  q.oc_w = oc_w; q.oc_b = oc_b; q.oc_y = logits;
  return ds_launch(q, stream);
}

/* smaat_dsconv_classify_fwd from bf16 activations: the argmax runs on the fp32 logits in registers; the logits, when asked
 * for, are stored as bf16. */
extern "C" int smaat_dsconv_classify_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                              const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale,
                                              const float* shift, const float* oc_w, const float* oc_b, int K, void* logits,
                                              int64_t* classes, int B, int H, int W, int k, int Cout, int relu, void* stream) {
  SMAAT_REQUIRE(oc_w && (logits || classes), "dsconv+classify bf16: needs the OutConv weight and a logits or a classes output");
  SMAAT_REQUIRE(K >= 1, "dsconv+classify bf16: K=%d classes", K);
  if (K > DS_MAX_CLASSES)
    return fail(SMAAT_E_UNSUPPORTED, "dsconv+classify bf16: K=%d classes, the fused epilogue takes at most %d; use smaat_dsconv_bf16_fwd + "
                                     "smaat_outconv_bf16_fwd + smaat_argmax_channels_bf16_fwd", K, DS_MAX_CLASSES);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(oc_w) & 3u) == 0 && (reinterpret_cast<uintptr_t>(logits) & 1u) == 0 &&
                    (reinterpret_cast<uintptr_t>(classes) & 7u) == 0,
                "dsconv+classify bf16: weights must be 4-byte, logits 2-byte and classes 8-byte aligned");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = SMAAT_PW_BF16; q.bact = true; q.dw_w = dw_w; q.dw_b = dw_b; q.scale = scale; q.shift = shift;
  q.oc_w = oc_w; q.oc_b = oc_b; q.oc_y = logits; q.ncls = K; q.cls = classes;
  return ds_launch(q, stream);
}

/* smaat_dsconv_maxpool_fwd from bf16 activations: y bf16, the max-pool written as bf16 (pooled_bf16 = 1, 4-byte aligned) or
 * fp32 (8-byte aligned), the dtype of the level it feeds; either way bit for bit MaxPool2d(2) of the stored y. */
extern "C" int smaat_dsconv_maxpool_bf16_eligible(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1,
                                                  int64_t x1_bstride, const void* pw_w, int H, int W, int k, int Cout) {
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.mode = SMAAT_PW_BF16; q.bact = true; q.pooled = g_ds_asked;
  return ds_select(q).declined == DS_TAKEN;
}

extern "C" int smaat_dsconv_maxpool_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                             const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale,
                                             const float* shift, void* y, int64_t y_bstride, void* pooled, int pooled_bf16, int B,
                                             int H, int W, int k, int Cout, int relu, void* stream) {
  SMAAT_REQUIRE(y && pooled, "dsconv_maxpool_bf16: null output");
  SMAAT_REQUIRE(pooled_bf16 == 0 || pooled_bf16 == 1, "dsconv_maxpool_bf16: pooled_bf16 must be 0 or 1");
  DsReq q{x0, C0, x0_bstride, x1, C1, x1_bstride, pw_w, H, W, k, Cout};
  q.B = B; q.relu = relu; q.mode = SMAAT_PW_BF16; q.bact = true; q.dw_w = dw_w; q.dw_b = dw_b; q.scale = scale; q.shift = shift;
  q.y = y; q.y_bstride = y_bstride; q.pooled = pooled; q.pooled_bf16 = pooled_bf16;
  return ds_launch(q, stream);
}
