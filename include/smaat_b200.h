/*
 * smaat_b200.h -- C ABI of libsmaat_b200.so: the H100 (sm_90a) kernels behind the
 * SmaAt-UNet hot path (depthwise-separable conv blocks + CBAM + their glue): forward for
 * inference, train-mode forward + backward, and the training step's loss/metric pass.
 *
 * The reference (HansBambel/SmaAt-UNet) has no FFI / plugin registry: its boundary is
 * the Python nn.Module interface (SURVEY.md section 8b).  Each entry point below
 * replaces the torch.nn call(s) cited next to it; `smaat_unet_b200/modules.py` is the
 * host-side mirror of the reference classes that binds them through ctypes, and
 * INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - all tensors are fp32, NCHW, dense in (H, W); device pointers owned by the caller
 *     (PyTorch caching allocator).  The library allocates nothing persistent.
 *   - every call only ENQUEUES work on `stream` (a cudaStream_t passed as void*):
 *     no device synchronisation, no allocation -> CUDA-graph capturable.
 *   - return value: 0 on success, negative SMAAT_E_* otherwise; smaat_last_error()
 *     returns a thread-local description.  Nothing throws or exits across the ABI.
 *   - "bstride" arguments are batch strides in ELEMENTS (>= C*H*W) so a kernel can
 *     read from / write into a channel slice of a wider tensor without a copy.
 */
#ifndef SMAAT_B200_H_
#define SMAAT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 2: the tensor-memory kernel's debug hooks and smaat_debug_dsconv_timing are gone
 * 3: the DS conv's softmax epilogue and the dense 3x3 conv's OutConv / argmax / softmax epilogue are gone: each measured
 *    slower than the separate launches it replaced */
#define SMAAT_ABI_VERSION 3

#define SMAAT_OK 0
#define SMAAT_E_BADARG (-1)   /* shape / pointer / alignment rejected by host-side validation */
#define SMAAT_E_CUDA (-2)     /* CUDA runtime or driver error at launch (see smaat_last_error) */
#define SMAAT_E_UNSUPPORTED (-3) /* valid request this build has no kernel for */

/* GEMM arithmetic modes (the `mode` argument of smaat_pw1x1_fwd, smaat_dsconv_*, smaat_conv3x3_fwd) */
#define SMAAT_PW_FP32_SIMT 0  /* CUDA-core FFMA, exact fp32 products                      */
#define SMAAT_PW_TF32 1       /* wgmma tf32, fp32 accumulate (1 pass)                     */
#define SMAAT_PW_TF32X3 2     /* wgmma 3xTF32 split (a_hi*b_hi + a_lo*b_hi + a_hi*b_lo)   */
/* wgmma bf16: each GEMM operand rounded to bf16 (round to nearest even: fp32's exponent range, 8-bit significand), the products
 * accumulated in fp32 registers, the epilogue unchanged.  Activations stay fp32 in memory (the kernels round them in
 * registers); the weight argument is the smaat_pack_bf16 pack of the fp32 weight.  Forward GEMMs only: the weight-gradient
 * entry points (smaat_pw1x1_bwd_weight_tc, smaat_conv3x3_bwd_weight) refuse it. */
#define SMAAT_PW_BF16 3

int smaat_abi_version(void);
const char* smaat_last_error(void);
/* Number of kernel launches enqueued by this library in the calling process so far. */
uint64_t smaat_launch_count(void);

/* ---- depthwise 3x3, padding 1, groups=Cin, k outputs per input channel -------------
 * replaces DepthwiseSeparableConv.depthwise  (models/layers.py:38-44,48)
 * Input is the virtual channel-concat of x0 (C0 channels) and x1 (C1 channels, may be
 * NULL/0): this is torch.cat([x2, x1], dim=1) of UpDS.forward
 * (models/unet_parts_depthwise_separable.py:85) without materialising the concat.
 * y[b, o] = bias[o] + sum_{dy,dx} w[o,dy,dx] * in[b, o / k, i+dy-1, j+dx-1]
 *   w: (k*(C0+C1), 3, 3)   bias: (k*(C0+C1)) or NULL   y: (B, k*(C0+C1), H, W) dense
 * in_scale/in_shift (per INPUT channel, may be NULL): when given the kernel applies
 *   relu(in_scale[c] * x + in_shift[c]) on load -- the train-mode BatchNorm+ReLU of the
 *   producing layer (parts_ds.py:25-26), with zero padding applied AFTER the activation.
 * loader: 0 = auto, 1 = force the LDG loader, 2 = force TMA (error if ineligible). */
int smaat_dw3x3_fwd(const float* x0, int C0, int64_t x0_bstride,
                    const float* x1, int C1, int64_t x1_bstride,
                    const float* w, const float* bias,
                    const float* in_scale, const float* in_shift,
                    float* y, int B, int H, int W, int k, int loader, void* stream);

/* ---- pointwise 1x1 + per-channel affine (+ReLU) epilogue -----------------------------
 * replaces DepthwiseSeparableConv.pointwise (models/layers.py:45,49) fused with the
 * following nn.BatchNorm2d (eval) + nn.ReLU (parts_ds.py:25-26,34-35):
 *   y[b,o,p] = act( scale[o] * sum_c w[o,c] x[b,c,p] + shift[o] )
 *   x: (B, K, P) dense   w: (Cout, K)   scale/shift: (Cout) (scale NULL = 1, shift NULL = 0)
 *   y: (B, Cout, P) with batch stride y_bstride elements.
 * w_lo: (Cout, K) low parts for SMAAT_PW_TF32X3 (w must then hold the tf32-truncated
 *   high parts, see smaat_split_tf32); NULL otherwise.
 * stats: NULL, or (2*Cout) fp64 zero-initialised accumulators receiving per-channel
 *   sum and sum of squares of the PRE-activation value scale*acc+shift (train-mode BN). */
/* mode SMAAT_PW_BF16: w is the smaat_pack_bf16 pack of the (Cout, K) weight ((Cout, K rounded up to 32) bf16), w_lo NULL. */
int smaat_pw1x1_fwd(const float* x, const float* w, const float* w_lo,
                    const float* scale, const float* shift,
                    float* y, int64_t y_bstride, double* stats,
                    int B, int K, int Cout, int P, int relu, int mode, void* stream);

/* ---- fused DepthwiseSeparableConv: depthwise 3x3 -> pointwise 1x1 -> affine (+ReLU) in ONE kernel ----
 * replaces DepthwiseSeparableConv.forward (models/layers.py:47-50) + eval BatchNorm2d + ReLU
 * (parts_ds.py:25-26,34-35); the k*Cin-channel depthwise result stays on chip (CUDA-core stencil writes
 * the wgmma A operand tiles directly).  Arguments as smaat_dw3x3_fwd (input = virtual concat [x0, x1],
 * dw_w: (k*Cin,3,3), dw_b: (k*Cin) or NULL) and smaat_pw1x1_fwd (pw_w: (Cout, k*Cin) -- the tf32 hi
 * parts in TF32X3 mode, pw_w_lo the lo parts; scale/shift/stats/relu as there).
 * mode: SMAAT_PW_TF32, SMAAT_PW_TF32X3 or SMAAT_PW_BF16 (pw_w the smaat_pack_bf16 pack of the (Cout, k*Cin) weight, pw_w_lo
 * NULL; register A form only: with smaat_set_dsconv_impl(1) bf16 requests return SMAAT_E_UNSUPPORTED, as k = 4 does there).
 * The same modes and weight forms apply to smaat_dsconv_outconv_fwd, smaat_dsconv_classify_fwd and smaat_dsconv_cbam_fwd.
 * Returns SMAAT_E_UNSUPPORTED for shapes the fused kernel
 * does not take (k not in {1,2}; Cout < 8, or Cout > 128 unless a multiple of 128 up to 512 without batch
 * statistics or OutConv; W % 4; patch waste > 35 %): callers then run
 * smaat_dw3x3_fwd + smaat_pw1x1_fwd.  smaat_dsconv_eligible returns 1/0 for the same test. */
int smaat_dsconv_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                          const float* pw_w, int H, int W, int k, int Cout);
/* Same test with the batch-statistics request made explicit: `with_stats` != 0 asks for the kernel that accumulates the
 * per-channel sum / sum of squares of its output (train-mode BatchNorm, parts_ds.py:25,34): Cout <= 128 only. */
int smaat_dsconv_eligible2(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                           const float* pw_w, int H, int W, int k, int Cout, int with_stats);
int smaat_dsconv_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                     const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                     const float* scale, const float* shift, float* y, int64_t y_bstride, double* stats,
                     int B, int H, int W, int k, int Cout, int relu, int mode, void* stream);
/* The network's last two modules in one kernel: the fused DS conv above followed by OutConv(Cout -> 1 class)
 * (models/SmaAt_UNet.py:55-56, unet_parts.py:67-73).  oc_w: (Cout), oc_b: (1) or NULL, logits: (B, 1, H, W); the
 * Cout-channel activation is reduced in the epilogue registers and never written.  Same eligibility
 * as smaat_dsconv_fwd, with Cout <= 128. */
int smaat_dsconv_outconv_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                             const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                             const float* scale, const float* shift, const float* oc_w, const float* oc_b, float* logits,
                             int B, int H, int W, int k, int Cout, int relu, int mode, void* stream);
/* The same kernel for a K-class OutConv, ending in the class map the reference's validation loop predicts
 * (pred_class = torch.argmax(softmax(y_pred), dim=1), train_SmaAtUNet.py:76; softmax keeps the order).  oc_w: (K, Cout),
 * oc_b: (K) or NULL; logits: (B, K, H, W) or NULL; classes: (B, H, W) int64 or NULL, not both NULL.  Class j's logit is bit for
 * bit what smaat_dsconv_outconv_fwd writes with oc_w row j and oc_b[j]; classes[b, p] is the argmax of the K logits, ties to
 * the first index, a NaN logit wins (torch.argmax), identical whether or not logits are written.  Neither the Cout-channel
 * activation nor (with logits NULL) the K logit planes reach HBM.  Eligibility: that of smaat_dsconv_outconv_fwd (Cout <= 128,
 * no batch statistics) and 1 <= K <= 32 (K <= 22 for Cout > 64: the class weights live in the shared memory the kernel
 * leaves free); SMAAT_E_UNSUPPORTED otherwise (callers then run smaat_dsconv_fwd or dw3x3 + pw1x1,
 * smaat_outconv_fwd and smaat_argmax_channels_fwd).  smaat_dsconv_classify_eligible returns 1/0 for the same test in `mode`. */
int smaat_dsconv_classify_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                   const float* pw_w, int H, int W, int k, int Cout, int K, int mode);
int smaat_dsconv_classify_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                              const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                              const float* scale, const float* shift, const float* oc_w, const float* oc_b, int K,
                              float* logits, int64_t* classes, int B, int H, int W, int k, int Cout, int relu, int mode, void* stream);

/* The fused DS conv with the CBAM fusions of the serving forward (models/layers.py:90-141 around the DS blocks of
 * models/SmaAt_UNet.py:41-57); arguments as smaat_dsconv_fwd, without batch statistics.
 *   gate_sc (B, C0), gate_sa (B, 1, H, W), both or neither: x0 is read as the CBAM output (x0 * gate_sc) * gate_sa, bit for bit
 *     what smaat_cbam_scale_fwd writes (zero padding stays zero), so the CBAM output of a skip is never materialised.
 *   pool_sum, pool_max (B, npart, Cout) and pooled (B, Cout, H / 2, W / 2), all or none: the epilogue also writes per half-patch
 *     partial sums / maxima of y (npart = smaat_dsconv_pool_parts(H, W); smaat_cbam_mlp_partials_fwd finishes the channel
 *     gate from them) and MaxPool2d(2)(y) (parts_ds.py:48; floor for odd H).  Fixed layout and order: no atomics.
 * smaat_dsconv_cbam_eligible: 1 if smaat_dsconv_cbam_fwd takes this request in `mode` (the pools need an instance with the
 *   staged epilogue), else 0.  Answers for all three tensor-core modes (0 for SMAAT_PW_FP32_SIMT), as
 *   smaat_dsconv_classify_eligible does. */
int smaat_dsconv_cbam_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                               const float* pw_w, int H, int W, int k, int Cout, int mode, int with_gate, int with_pools);
int smaat_dsconv_pool_parts(int H, int W);
int smaat_dsconv_cbam_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                          const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                          const float* scale, const float* shift, float* y, int64_t y_bstride,
                          const float* gate_sc, const float* gate_sa, float* pool_sum, float* pool_max, float* pooled,
                          int B, int H, int W, int k, int Cout, int relu, int mode, void* stream);
/* The fused DS conv that also writes pooled = MaxPool2d(2)(y) (parts_ds.py:48) for the DownDS that reads y next, as the CBAM
 * pools' epilogue does but without the partial sums (no atomics either way): UNetDS's encoder, which has no CBAM to hand the
 * max-pool over (unet_precip_regression_lightning.py:107-112).  pooled (B, Cout, H / 2, W / 2), 8-byte aligned, bit for bit the
 * max-pool of the stored y; floor for odd H.  Arguments otherwise as smaat_dsconv_fwd, without batch statistics.
 * smaat_dsconv_maxpool_eligible: 1 if smaat_dsconv_maxpool_fwd takes the request in `mode` (an instance with the staged
 * epilogue: smaat_dsconv_cbam_eligible with with_pools), else 0. */
int smaat_dsconv_maxpool_eligible(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                                  const float* pw_w, int H, int W, int k, int Cout, int mode);
int smaat_dsconv_maxpool_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                             const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_w_lo,
                             const float* scale, const float* shift, float* y, int64_t y_bstride, float* pooled,
                             int B, int H, int W, int k, int Cout, int relu, int mode, void* stream);

/* How the fused DS conv (smaat_dsconv_fwd / smaat_dsconv_outconv_fwd, same reference lines, models/layers.py:47-50) hands the
 * depthwise result to the tensor core: 0 = auto (default; 2, the faster of the two on an H100), 1 = K-major tiles in shared memory that wgmma reads
 * through a descriptor, 2 = tiles the consumers load into registers for wgmma's register-A form.  Same results up to
 * summation order.  Process-wide; the environment variable SMAAT_DS_IMPL presets it.  For A/B measurements and tests. */
int smaat_set_dsconv_impl(int impl);

/* 1 if this (x, w, K, Cout, P) can take the tensor-core (wgmma) path (P % 4 == 0, K % 4 == 0, 16-byte aligned
 * pointers, Cout >= 8), else 0: the caller then uses SMAAT_PW_FP32_SIMT. */
int smaat_pw1x1_tc_eligible(const float* x, const float* w, int K, int Cout, int P);

/* hi[i] = tf32_truncate(src[i]); lo[i] = src[i] - hi[i]   (weight preparation for TF32X3) */
int smaat_split_tf32(const float* src, float* hi, float* lo, int64_t n, void* stream);
/* Weight preparation for SMAAT_PW_BF16: w (rows, cols) fp32 -> out (rows, cols_out) bf16 (uint16 bit patterns), cols_out = cols
 * rounded up to 32 (else SMAAT_E_BADARG), out 4-byte aligned.  out[r][16 q + l] = bf16_rn(w[r][16 q + (l & 8) | ((l & 1) << 2) |
 * ((l >> 1) & 3)]), zero where that column is >= cols: round to nearest even (NaN stays NaN), and within each group of 16 the k
 * order in which the kernels' bf16 register fragments present the activations, so the GEMM pairs every product as in fp32. */
int smaat_pack_bf16(const float* w, uint16_t* out, int rows, int cols, int cols_out, void* stream);

/* ---- eval-mode BatchNorm folded to the affine the pw epilogue applies -----------------
 * nn.BatchNorm2d.eval (parts_ds.py:25,34):  scale = gamma / sqrt(rv + eps),
 *   shift = beta + (conv_bias - rm) * scale        (conv_bias may be NULL) */
int smaat_bn_fold(const float* gamma, const float* beta, const float* rm, const float* rv,
                  const float* conv_bias, float eps, float* scale, float* shift, int C, void* stream);

/* ---- train-mode BatchNorm2d (parts_ds.py:25,34; layers.py:120 in .train()) ----------------------
 * The producing kernel accumulates per-channel sum / sum of squares in fp64 (`stats`, 2*C doubles,
 * zero-initialised by the caller); smaat_channel_stats does the same for an existing tensor
 * x: (B, C, P) (SpatialAttention's 1-channel BN).
 * bn_finalize: mean = s1/n, var = s2/n - mean^2 (biased), scale = gamma/sqrt(var+eps),
 *   shift = beta - mean*scale; writes mean / inv-std for the backward pass (may be NULL) and updates
 *   running_mean <- (1-m) rm + m mean, running_var <- (1-m) rv + m var*n/(n-1)  (may be NULL).
 *   num_batches_tracked (nullable, device int64) is incremented by one, like nn.BatchNorm2d does in train mode.
 * affine_act: y[b,c,p] = act(scale[c]*x[b,c,p] + shift[c]), act 0 = none, 1 = ReLU, 2 = sigmoid
 *   (scale NULL = 1, shift NULL = 0). */
int smaat_channel_stats(const float* x, double* stats, int B, int C, int P, void* stream);
int smaat_bn_finalize(const double* stats, double count, const float* gamma, const float* beta, float eps, float momentum,
                      float* running_mean, float* running_var, float* scale, float* shift,
                      float* mean_out, float* invstd_out, long long* num_batches_tracked, int C, void* stream);
int smaat_affine_act_fwd(const float* x, const float* scale, const float* shift, float* y,
                         int B, int C, int P, int act, void* stream);

/* ---- nn.MaxPool2d(2) (parts_ds.py:48): stride 2, floor ---------------------------------
 * x: (N, H, W) planes -> y: (N, H/2, W/2) */
int smaat_maxpool2_fwd(const float* x, float* y, int64_t N, int H, int W, void* stream);

/* ---- nn.Upsample(x2, bilinear, align_corners=True) + F.pad to the skip size -----------
 * (parts_ds.py:64,78-81).  x: (B, C, H, W) -> y: (B, C, Ho, Wo) with Ho >= 2H, Wo >= 2W,
 * zero border of (Ho-2H)//2 rows on top, (Wo-2W)//2 columns on the left. */
int smaat_upsample2x_pad_fwd(const float* x, float* y, int64_t y_bstride,
                             int B, int C, int H, int W, int Ho, int Wo, void* stream);

/* ---- CBAM (models/layers.py:90-141) -----------------------------------------------------
 * pool:   avg[n] = mean_p x[n,p], mx[n] = max_p x[n,p] over N = B*C planes of P pixels
 *         (AdaptiveAvgPool2d(1)/AdaptiveMaxPool2d(1), layers.py:107-108)
 * mlp:    sc[b,c] = sigmoid( MLP(avg[b]) + MLP(mx[b]) ), MLP = W2 relu(W1 v + b1) + b2
 *         (layers.py:98-103,109)
 * reduce: pooled[b,0,p] = mean_c x[b,c,p]*sc[b,c]; pooled[b,1,p] = max_c ...  (layers.py:123-125)
 * gate:   a = conv_kxk(pooled, wsp)  (2->1 ch, pad k/2, no bias, layers.py:119,126);
 *         sa[b,p] = sigmoid(bn_affine[0] * a + bn_affine[1])  (BatchNorm2d(1) + sigmoid, :127-128);
 *         bn_affine = 2 floats ON THE DEVICE (smaat_bn_fold with C=1), NULL = identity;
 *         if raw != NULL the pre-BN conv output a is also written (train-mode statistics).
 * scale:  y[b,c,p] = x[b,c,p] * sc[b,c] * sa[b,p]   (layers.py:110,128) */
int smaat_cbam_pool_fwd(const float* x, float* avg, float* mx, int64_t N, int P, void* stream);
/* The same pools plus nn.MaxPool2d(2) of the same planes in ONE read of x (every encoder map of SmaAt-UNet feeds both
 * cbam_l and down_l: models/SmaAt_UNet.py:42-50).  x: (N, H, W) -> avg (N), mx (N), pooled (N, H/2, W/2).
 * SMAAT_E_UNSUPPORTED unless W % 4 == 0 and H % 2 == 0 (then run smaat_cbam_pool_fwd + smaat_maxpool2_fwd). */
int smaat_cbam_pool_maxpool_fwd(const float* x, float* avg, float* mx, float* pooled, int64_t N, int H, int W, void* stream);
int smaat_cbam_mlp_fwd(const float* avg, const float* mx, const float* w1, const float* b1,
                       const float* w2, const float* b2, float* sc, int B, int C, int hidden, void* stream);
int smaat_cbam_reduce_fwd(const float* x, const float* sc, float* pooled, int B, int C, int P, void* stream);
int smaat_cbam_gate_fwd(const float* pooled, const float* wsp, const float* bn_affine, float* sa, float* raw,
                        int B, int H, int W, int ks, void* stream);
int smaat_cbam_scale_fwd(const float* x, const float* sc, const float* sa, float* y, int64_t y_bstride,
                         int B, int C, int P, void* stream);

/* ---- OutConv (models/unet_parts.py:67-73): 1x1 conv Cin -> ncls (small), bias, no activation */
int smaat_outconv_fwd(const float* x, const float* w, const float* bias, float* y,
                      int B, int Cin, int ncls, int P, void* stream);

/* ======================================= backward (training step) =======================================
 * Gradients of the same path (BASELINE configs[2]): what torch autograd runs for these modules when the reference calls
 * loss.backward() (train_SmaAtUNet.py:55; Lightning automatic optimisation over UNetBase.training_step,
 * models/regression_lightning.py:67-78).  Each group names the forward lines it differentiates.  Notation: z = pre-BatchNorm activation,
 * a = act(scale*z+shift), dA = dL/da masked by the activation (act: 0 none, 1 ReLU recomputed from z).
 * Accumulating outputs (dW, db, dgamma, dbeta, d_sc, stats-like sums) are += : the caller zero-initialises.
 *
 * BatchNorm(+ReLU) backward -- nn.BatchNorm2d + nn.ReLU, parts_ds.py:25-26,34-35; BatchNorm2d(1), layers.py:120,127 --
 * = reduce -> coeffs -> apply:
 *   reduce: sums[c] += sum dA, sums[C+c] += sum dA*z                       (fp64)
 *   coeffs: dgamma += invstd*(S2 - mean*S1), dbeta += S1; per-channel a,b,cc with dz = a*dA + b*z + cc
 *           (train: batch-statistics terms; eval (train=0): dz = gamma*invstd*dA); dz_sum (nullable) += sum_{b,p} dz
 *           per channel, i.e. the bias gradient of the conv that produced z, from the sums alone (0 with batch statistics)
 *   apply : dz[b,c,p] = a[c]*dA + b[c]*z + cc[c] */
int smaat_bn_act_bwd_reduce(const float* dy, const float* z, const float* scale, const float* shift, double* sums,
                            int B, int C, int P, int act, void* stream);
int smaat_bn_bwd_coeffs(const double* sums, double count, const float* gamma, const float* mean, const float* invstd, int train,
                        float* a, float* b, float* cc, float* dgamma, float* dbeta, float* dz_sum, int C, void* stream);
int smaat_bn_act_bwd_apply(const float* dy, const float* z, const float* scale, const float* shift,
                           const float* a, const float* b, const float* cc, float* dz, int B, int C, int P, int act, void* stream);

/* depthwise 3x3 backward (DepthwiseSeparableConv.depthwise, models/layers.py:38-44,48): input gradient (split over the virtual concat x0|x1) and weight/bias gradient;
 * in_scale/in_shift: the forward's on-load BN+ReLU prologue (input of the conv was relu(in_scale*x+in_shift)). */
int smaat_dw3x3_bwd_input(const float* dd, const float* w, float* dx0, int C0, int64_t dx0_bstride,
                          float* dx1, int C1, int64_t dx1_bstride, int B, int H, int W, int k, void* stream);
int smaat_dw3x3_bwd_weight(const float* dd, const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                           const float* in_scale, const float* in_shift, float* dw, float* db,
                           int B, int H, int W, int k, void* stream);

/* pointwise 1x1 backward (DepthwiseSeparableConv.pointwise, models/layers.py:45,49): dW[o][c] += sum_{b,p} dz[b,o,p]*d[b,c,p],
 * db[o] += sum dz.  (The input gradient is
 * smaat_pw1x1_fwd(dz, W^T): use smaat_transpose for W^T.) */
int smaat_pw1x1_bwd_weight(const float* dz, const float* d, float* dW, float* db, int B, int K, int Cout, int P, void* stream);
/* tensor-core (wgmma, split over pixels + fp32 atomics) variant; mode SMAAT_PW_TF32 / SMAAT_PW_TF32X3;
 * SMAAT_E_UNSUPPORTED when P % 4 != 0 (use the CUDA-core smaat_pw1x1_bwd_weight). */
int smaat_pw1x1_bwd_weight_tc(const float* dz, const float* d, float* dW, float* db, int B, int K, int Cout, int P,
                              int mode, void* stream);
int smaat_transpose(const float* src, float* dst, int rows, int cols, void* stream);

/* glue backward: nn.MaxPool2d(2) (parts_ds.py:48), nn.Upsample(x2, bilinear, align_corners) + F.pad (parts_ds.py:64,78-81),
 * OutConv (unet_parts.py:67-73) */
int smaat_maxpool2_bwd(const float* x, const float* dy, float* dx, int64_t N, int H, int W, void* stream);
int smaat_upsample2x_pad_bwd(const float* dy, int64_t dy_bstride, float* dx, int B, int C, int H, int W, int Ho, int Wo, void* stream);
int smaat_outconv_bwd(const float* dy, const float* x, const float* w, float* dx, float* dW, float* db,
                      int B, int Cin, int ncls, int P, void* stream);

/* CBAM backward (models/layers.py:90-141 differentiated; see cbam_bwd.cu for the chain): gate_in -> [BN(1) backward] -> gate_bwd -> dsc -> mlp_bwd -> dx.
 * amax: (B, P) int32 channel argmax of x*sc written by gate_in; pkey: (B*C) uint64, zeroed by the caller, receives the
 * packed plane argmax of x in dsc and is consumed by dx; dsc (B, C) is accumulated into (caller zeroes it). */
int smaat_cbam_bwd_gate_in(const float* g, const float* x, const float* sc, const float* sa, float* dpre, int* amax,
                           int B, int C, int P, void* stream);
int smaat_cbam_gate_bwd(const float* draw, const float* pooled, const float* wsp, float* dpooled, float* dW,
                        int B, int H, int W, int ks, void* stream);
int smaat_cbam_bwd_dsc(const float* g, const float* x, const float* sa, const float* dpooled, const int* amax, float* dsc,
                       unsigned long long* pkey, int B, int C, int P, void* stream);
int smaat_cbam_mlp_bwd(const float* avg, const float* mx, const float* w1, const float* b1, const float* w2, const float* sc,
                       const float* dsc, float* dw1, float* db1, float* dw2, float* db2, float* davg, float* dmx,
                       int B, int C, int hidden, void* stream);
int smaat_cbam_bwd_dx(const float* g, const float* sc, const float* sa, const float* dpooled, const int* amax,
                      const float* davg, const float* dmx, const unsigned long long* pkey, float* dx,
                      int B, int C, int P, void* stream);

/* ---- loss + metric bookkeeping of one training/validation step, one pass, no host sync ------------
 * Replaces UNetBase.loss_func (models/regression_lightning.py:57-65) and PrecipitationMetrics.update
 * (metric/precipitation_metrics.py:37-95).  pred/target: n floats.  batch_acc: double[8], overwritten:
 *   [0] sum (p-y)^2  [1] sum (p*f-y*f)^2 (f = factor if denormalize else 1)  [2] number of NaNs in p or y
 *   [3] TN [4] FP [5] FN [6] TP of ((x*f)*12 > threshold)  [7] n
 * dpred (nullable): 2*(p-y)*grad_scale, the gradient of sum((p-y)^2)*grad_scale (grad_scale = 1/B).
 * smaat_metrics_commit adds one batch to totals (double[9]: total_loss, total_loss_denorm, total_samples,
 * total_pixels, TN, FP, FN, TP, skipped batches) on the device, skipping NaN batches like the reference (:46-48). */
int smaat_mse_metrics_fwd(const float* pred, const float* target, int64_t n, float factor, float threshold,
                          int denormalize, double* batch_acc, float* dpred, float grad_scale, void* stream);
int smaat_metrics_commit(const double* batch_acc, double* totals, int batch_size, int denormalize, void* stream);

/* ---- PrecipitationMetrics for several thresholds at once, every image as a batch of one (test-set evaluation) ------
 * smaat_precip_sweep_fwd: B images of P pixels.  Image b of pred starts at pred + b * pred_bstride (pred_bstride >= P
 *   when B > 1: a model's (B, 1, H, W) output has stride P, the last frame x[:, C-1] of a (B, C, H, W) input stride C * P);
 *   target (B, P) dense.  thresholds: T HOST floats, strictly increasing, 1 <= T <= 32 (else SMAAT_E_BADARG before any
 *   launch).  A value's bin is #{i : (v * factor) * 12 > thresholds[i]} in fp32 (v * 12 when denormalize == 0), the
 *   comparison of smaat_mse_metrics_fwd.  Both outputs are overwritten:
 *   per_image (B, 3) double: sum (p-y)^2, sum (p*f-y*f)^2, number of NaNs in p or y;
 *   hist (B, T+1, T+1) uint32: hist[b][a][c] = pixels of image b with target bin a and pred bin c.  At threshold i,
 *   TP = sum_{a>=i, c>=i}, FN = sum_{a>=i, c<i}, FP = sum_{a<i, c>=i}, TN = sum_{a<i, c<i}.
 *   128-bit loads when pred, target, pred_bstride and P allow (16-byte aligned images), a scalar kernel otherwise.
 * smaat_precip_sweep_commit folds the B images into totals (double[5 + (T+1)^2]: total_loss, total_loss_denorm,
 *   total_samples, total_pixels, images skipped, then the summed histogram) as B batches of one: an image with a NaN
 *   adds nothing but one skipped image (metric/precipitation_metrics.py:46-48 at batch size 1); the others add their
 *   sums (the denormalised one only when denormalize != 0), 1 sample, P pixels and their histogram. */
int smaat_precip_sweep_fwd(const float* pred, int64_t pred_bstride, const float* target, int B, int64_t P, float factor,
                           const float* thresholds, int T, int denormalize, double* per_image, unsigned* hist, void* stream);
int smaat_precip_sweep_commit(const double* per_image, const unsigned* hist, int B, int64_t P, int T, int denormalize,
                              double* totals, void* stream);

/* ---- multi-class cross-entropy + confusion matrix of one segmentation step, one pass, no host sync ----------------
 * Replaces nn.CrossEntropyLoss() of train_SmaAtUNet.py:54,182 (log_softmax + nll_loss) and the per-batch host histogram
 * behind metric.iou.IoU.add (metric/iou.py:38-62, metric/confusionmatrix.py:40-69).
 * smaat_ce_fwd: logits (B, K, P) fp32 NCHW dense, target (B, P) int64 class indices, 2 <= K <= 1024 (larger K:
 *   SMAAT_E_UNSUPPORTED).  A pixel whose label equals ignore_index (only when use_ignore != 0) is skipped; a label outside
 *   [0, K) that is not ignored is INVALID: counted, never used as an index, no loss, no gradient, no confusion entry.
 *   batch_acc: double[3], overwritten: [0] sum over counted pixels of logsumexp_c(l) - l_target (fp32 terms, fp64 sum)
 *                                      [1] counted pixels   [2] invalid labels
 *   dlogits (nullable): (B, K, P), softmax(l) - onehot(target), unscaled; exactly 0 on ignored and invalid pixels.
 *   conf (nullable): int64 K x K, ADDED INTO: conf[target][argmax_c l] += 1 per counted pixel; ties go to the first index.
 *   NaN logits: the pixel's loss term and gradient are NaN (so is the loss, as in torch); its argmax is the first NaN
 *   channel, as torch.argmax / np.argmax return, and the pixel is counted in conf under that column.
 *   128-bit loads when P % 4 == 0 and logits / target / dlogits are 16-byte aligned, a scalar kernel otherwise.
 * smaat_confusion_add: conf[target[i]][pred[i]] += 1 over n int64 (pred, target) pairs; a pair with either value outside
 *   [0, K) is skipped and added to *invalid (int64 device counter, nullable). */
int smaat_ce_fwd(const float* logits, const int64_t* target, int B, int K, int64_t P, int64_t ignore_index, int use_ignore,
                 double* batch_acc, float* dlogits, int64_t* conf, void* stream);
int smaat_confusion_add(const int64_t* pred, const int64_t* target, int64_t n, int K, int64_t* conf, int64_t* invalid,
                        void* stream);
/* smaat_cross_entropy_fwd: F.cross_entropy with the options smaat_ce_fwd leaves out, in the same single pass (a separate
 *   kernel, so the plain path keeps its registers).  Logits as smaat_ce_fwd; EXACTLY ONE of
 *     target      (B, P) int64 class indices (ignore_index / use_ignore and invalid labels as smaat_ce_fwd), or
 *     target_prob (B, K, P) fp32 probabilities (use_ignore must be 0: torch rejects ignore_index for them).
 *   weight (nullable): K fp32 class weights on the device (NULL: all ones); label_smoothing eps in [0, 1].
 *   With W = sum_k w_k, lse = logsumexp_c(l), p = softmax(l), the per-pixel loss and its gradient are
 *     class index t:  (1 - eps) w_t (lse - l_t) + (eps / K) (W lse - sum_k w_k l_k)
 *                     d_j = ((1 - eps) w_t + eps W / K) p_j - (1 - eps) w_t [j == t] - (eps / K) w_j
 *     probabilities:  q' = q (1 - eps) + eps / K;  loss = lse sum_k w_k q'_k - sum_k w_k q'_k l_k;  d_j = p_j sum_k w_k q'_k - w_j q'_j
 *   batch_acc: double[4], overwritten: [0] sum of the per-pixel losses of counted pixels (fp32 terms, fp64 sum)
 *     [1] counted pixels (probability targets: every pixel)   [2] invalid labels; with probability targets, rows that
 *     fail the one-hot check below (they do not affect the loss)   [3] D = sum of w_t over counted pixels (probability
 *     targets: the pixel count) -- the divisor of torch's "mean".
 *   loss_map (nullable): (B, P) fp32 per-pixel loss; 0 on ignored pixels, NaN on invalid labels.
 *   dlogits (nullable): (B, K, P) unscaled per-pixel gradient; exactly 0 on ignored and invalid pixels.  With weight NULL
 *     and eps = 0 it is bitwise smaat_ce_fwd's.
 *   conf (nullable): as smaat_ce_fwd.  With probability targets the row is the target's first argmax, counted only when the
 *     target row passes metric/confusionmatrix.py:57-61's checks: every value in [0, 1] and the row sums to 1 (fp32 sum in
 *     class order; numpy's pairwise order can differ by an ulp on rows that are not one-hot).
 *   NaN logits poison their own pixel, as in smaat_ce_fwd.
 * smaat_onehot_classes: one-hot / probability targets (B, K, P) fp32 -> classes (B, P) int64: the row's first argmax, or -1
 *   when the row fails the checks above, so smaat_confusion_add / the score path count it as invalid.  1 <= K <= 1024. */
int smaat_cross_entropy_fwd(const float* logits, const int64_t* target, const float* target_prob, const float* weight, int B, int K,
                            int64_t P, float label_smoothing, int64_t ignore_index, int use_ignore, double* batch_acc,
                            float* loss_map, float* dlogits, int64_t* conf, void* stream);
int smaat_onehot_classes(const float* target, int64_t* classes, int B, int K, int64_t P, void* stream);
/* smaat_argmax_channels_fwd: the class map of any (B, K, P) logits, classes[b, p] = argmax_c x[b, c, p] (int64), in one read:
 *   ties go to the first index and a NaN logit wins, as torch.argmax (and smaat_ce_fwd's confusion column).  1 <= K <= 1024
 *   (larger K: SMAAT_E_UNSUPPORTED).  128-bit loads when P % 4 == 0 and x / classes are 16-byte aligned, a scalar kernel
 *   otherwise.  Serves every class map smaat_dsconv_classify_fwd does not produce, the dense models' among them. */
int smaat_argmax_channels_fwd(const float* x, int64_t* classes, int B, int K, int64_t P, void* stream);
/* smaat_softmax_channels_fwd: the class probabilities of any (B, K, P) logits, probs[b, c, p] = softmax_c x[b, :, p], the
 *   softmax(y_pred) of train_SmaAtUNet.py:76 (torch.softmax(x, 1)).  One thread per pixel (4 with 128-bit loads when P % 4 == 0
 *   and x / probs are 16-byte aligned) keeps a running (max, sum of exp) over the classes in order, then re-reads the logits,
 *   from L2 (the grid is sized so that the lines it reads between its two sweeps fit in half of it), and writes
 *   exp(l - max) / sum.  Non-finite logits give torch's pattern: a NaN or +inf logit makes the pixel's K probabilities NaN, a
 *   pixel of -inf logits is NaN, a -inf logit among finite ones gets 0; K = 1 gives 1.  1 <= K <= 1024 (larger K:
 *   SMAAT_E_UNSUPPORTED).  Serves the probabilities of every model: the softmax of the logits its serving forward returns. */
int smaat_softmax_channels_fwd(const float* x, float* probs, int B, int K, int64_t P, void* stream);

/* CBAM in three launches (reference models/layers.py:90-141).
 * smaat_cbam_pool_mlp_fwd: ChannelAttention's global pools AND its shared MLP + sigmoid (layers.py:98-109): the last pooling
 *   CTA of each image finishes the MLP; pooled != NULL also emits MaxPool2d(2)(x) from the same read (parts_ds.py:48).
 *   counters: B ints, zero on entry and on exit.  C % 8 == 0, C <= 512, hidden <= 64 (else SMAAT_E_UNSUPPORTED).
 * smaat_cbam_reduce_fwd (above): per-pixel channel mean / max of x * sc (layers.py:123-125).
 * smaat_cbam_gate_scale_fwd: conv k x k (2 -> 1) + BatchNorm2d(1) affine + sigmoid AND y = (x * sc) * gate
 *   (layers.py:126-128, :110): the gate map never reaches HBM.  W % 4 == 0, 16-byte aligned x / y (else SMAAT_E_UNSUPPORTED). */
int smaat_cbam_pool_mlp_fwd(const float* x, float* avg, float* mx, float* pooled, const float* w1, const float* b1, const float* w2,
                            const float* b2, float* sc, int* counters, int B, int C, int H, int W, int hidden, void* stream);
int smaat_cbam_gate_scale_fwd(const float* pooled, const float* wsp, const float* bn_affine, const float* x, const float* sc, float* y,
                              int64_t y_bstride, int B, int C, int H, int W, int ks, void* stream);
/* smaat_cbam_mlp_partials_fwd: the channel gate of a map whose producer (smaat_dsconv_cbam_fwd) already pooled it: reduces
 *   psum / pmax (B, npart, C) per (b, c) in a fixed order to avg = sum / (H * W) and mx, then the shared MLP + sigmoid as
 *   smaat_cbam_pool_mlp_fwd (same counters).  C % 16 == 0, C <= 512, hidden <= 64 (else SMAAT_E_UNSUPPORTED). */
int smaat_cbam_mlp_partials_fwd(const float* psum, const float* pmax, int npart, float* avg, float* mx, const float* w1,
                                const float* b1, const float* w2, const float* b2, float* sc, int* counters, int B, int C,
                                int H, int W, int hidden, void* stream);

/* ---- UpDS(bilinear=False): nn.ConvTranspose2d(in, in // 2, 2, stride=2) + F.pad (reference
 * models/unet_parts_depthwise_separable.py:72-73, 76-81).  Kernel = stride = 2: no overlapping taps, so the transposed conv is ONE
 * pointwise GEMM Cin -> 4 Cout packed channels (smaat_pw1x1_fwd on the repacked weight) followed by a 2x2 pixel shuffle.
 *   smaat_convt2x2_pack_weight:  W (Cin, Cout, 2, 2) -> Wp (4 Cout, Cin), row (2 dy + dx) Cout + o
 *   smaat_pixel_shuffle2_pad_fwd: t (B, 4 Cout, H, W) [+ bias (Cout) or NULL] -> y (B, Cout, Ho, Wo), zero pad frame
 *   smaat_pixel_shuffle2_pad_bwd: the gather transpose; smaat_convt2x2_unpack_wgrad ACCUMULATES dWp / dbp into dW / db. */
int smaat_convt2x2_pack_weight(const float* w, float* wp, int Cin, int Cout, void* stream);
int smaat_convt2x2_unpack_wgrad(const float* dwp, const float* dbp, float* dw, float* db, int Cin, int Cout, void* stream);
int smaat_pixel_shuffle2_pad_fwd(const float* t, const float* bias, float* y, int64_t y_bstride, int B, int Cout, int H, int W, int Ho,
                                 int Wo, void* stream);
int smaat_pixel_shuffle2_pad_bwd(const float* g, int64_t g_bstride, float* dt, int B, int Cout, int H, int W, int Ho, int Wo, void* stream);

/* ---- dense 3x3 conv, padding 1: nn.Conv2d(Cin, Cout, 3, padding=1) of DoubleConv (models/unet_parts.py:16,19), with the
 * eval BatchNorm2d + ReLU that follow it (:17-18, 20-21) in the epilogue, over the virtual concat [x0, x1] of Up
 * (unet_parts.py:63, torch.cat never materialised).
 * smaat_conv3x3_pack_weight: w (Cout, C0 + C1, 3, 3) -> wp (Cout, 9, C0p + C1p), Cxp = Cx rounded up to 32, zero padded:
 *   wp[o][3 dy + dx][c] = w[o][c][dy][dx] with x1's channels at offset C0p.  flip_transpose != 0 packs the input-gradient
 *   weight instead: wp (C0 + C1, 9, Coutp), wp[c][3 dy + dx][o] = w[o][c][2 - dy][2 - dx]; run it through smaat_conv3x3_fwd
 *   with x0 = dz (Cout channels, C1 = 0) and Cout = C0 + C1 to get dX (split [dx0 | dx1] by channel).
 * smaat_conv3x3_fwd: y[b,o,p] = act(scale[o] * sum_{c,dy,dx} w[o,c,dy,dx] in[b,c,p+(dy-1,dx-1)] + shift[o]), zero outside the
 *   image; scale/shift/stats/relu/y_bstride as smaat_pw1x1_fwd (affine for Cout <= 1024).  mode: SMAAT_PW_FP32_SIMT (CUDA
 *   cores, any shape), SMAAT_PW_TF32 / SMAAT_PW_TF32X3 (wgmma implicit GEMM; wp_lo = the lo parts of smaat_split_tf32 of wp in
 *   TF32X3, wp the hi parts) / SMAAT_PW_BF16 (wp the smaat_pack_bf16 pack of the packed weight, whose rows are already
 *   multiples of 32 long).  The tensor-core modes return SMAAT_E_UNSUPPORTED unless W % 4 == 0, Cout >= 8, x0 / x1 / wp
 *   16-byte aligned and the batch strides multiples of 4; smaat_conv3x3_tc_eligible answers the same test (1/0).
 * smaat_conv3x3_bwd_weight: dW (Cout, C0 + C1, 3, 3) += sum_{b,p} dz[b,o,p] in[b,c,p+(dy-1,dx-1)], in the nn.Conv2d layout.
 *   dz: (B, Cout, H, W) dense.  mode: SMAAT_PW_FP32_SIMT (CUDA cores, any shape) or SMAAT_PW_TF32 / SMAAT_PW_TF32X3 (wgmma,
 *   split over pixel chunks; SMAAT_E_UNSUPPORTED unless W % 4 == 0, dz / x0 / x1 16-byte aligned and the batch strides
 *   multiples of 4).  The bias gradient is the dz_sum of smaat_bn_bwd_coeffs. */
int smaat_conv3x3_pack_weight(const float* w, float* wp, int Cout, int C0, int C1, int flip_transpose, void* stream);
int smaat_conv3x3_tc_eligible(const float* x0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                              const float* wp, int W, int Cout);
int smaat_conv3x3_fwd(const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1, int64_t x1_bstride,
                      const float* wp, const float* wp_lo, const float* scale, const float* shift, float* y, int64_t y_bstride,
                      double* stats, int B, int H, int W, int Cout, int relu, int mode, void* stream);
int smaat_conv3x3_bwd_weight(const float* dz, const float* x0, int C0, int64_t x0_bstride, const float* x1, int C1,
                             int64_t x1_bstride, float* dW, int B, int H, int W, int Cout, int mode, void* stream);

/* ---- optimizer step (reference models/regression_lightning.py:47-48, train_SmaAtUNet.py:25: torch.optim.Adam with its
 * defaults) over flat fp32 buffers of n floats (n % 4 == 0, 16-byte aligned; parameters, gradients, first and second moment
 * share one layout; padding must carry zero gradients).  lr and step are DEVICE scalars (fp32; step = completed steps,
 * incremented by the call), so a CUDA graph holding this call follows learning-rate changes.  torch's arithmetic:
 *   m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr / (1-b1^t) * m / (sqrt(v) / sqrt(1-b2^t) + eps). */
int smaat_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, const float* lr,
                    float* step, double beta1, double beta2, double eps, void* stream);

/* ---- VOC training input: the per-sample random augmentations, ToTensor, Normalize and the target map of
 * VOCSegmentation.__getitem__ / apply_augmentations (reference utils/dataset_VOC.py:139-168), after the deterministic
 * Resize(256) + CenterCrop(224) (train_SmaAtUNet.py:149) has run offline, in one launch per batch.
 * x_u8 (B, H, W, 3) uint8 RGB and y_u8 (B, H, W) uint8 mask indices, dense.  aug (B, 3) int8 device rows
 * (flip, rot, bright), or NULL for none: flip != 0 -> TF.hflip of image and mask; then rot > 0 / < 0 -> TF.rotate(+10 / -10)
 * of both (PIL NEAREST, expand=False, fill 0, bit for bit: the fixed-point or double coordinate walk PIL takes for H x W);
 * then bright > 0 / < 0 -> TF.adjust_brightness(1.2 / 1.2 - 0.4) of the image.  x (B, 3, H, W) fp32 receives
 * (v / 255 - mean[c]) / std[c] (IEEE fp32 operations, ToTensor + Normalize), y (B, H, W) int64 the mask with 255 -> 0;
 * x_bstride >= 3 H W, y_bstride >= H W (elements).  mean, std: HOST float[3], read at the call (their values are baked into
 * a captured launch).  Any H, W >= 1. */
int smaat_voc_augment_fwd(const uint8_t* x_u8, const uint8_t* y_u8, const int8_t* aug, const float* mean, const float* std,
                          float* x, int64_t x_bstride, int64_t* y, int64_t y_bstride, int B, int H, int W, void* stream);

/* ---- bf16 activations: SmaAt-UNet's serving forward from bf16 input ------------------------------------------------------
 * The serving forward's bf16 storage route keeps the input and the level 1-3 feature maps (and the logits / probabilities) as
 * bf16 in HBM: raw uint16_t bits, round to nearest even, passed as void*.  Arithmetic stays fp32 (the GEMMs take bf16 operands
 * with fp32 accumulation, as SMAAT_PW_BF16); every stored bf16 value is rounded once.  Weights, scales, gates, pools and the
 * class map keep their fp32 / int64 forms.  Each entry point mirrors the fp32 one named beside it.
 *
 * smaat_dsconv_bf16_fwd (smaat_dsconv_fwd / smaat_dsconv_cbam_fwd): x0, x1 and y bf16, pw_w the smaat_pack_bf16 pack; gate_sc /
 *   gate_sa (fp32, both or neither) read x0 as the CBAM output (x0 * sc) * sa, computed in fp32.  k = 1 or 2, the register A
 *   form, W and the batch strides multiples of 8, 16-byte aligned tensors; no batch statistics, no CBAM pools.
 * smaat_dsconv_outconv_bf16_fwd / smaat_dsconv_classify_bf16_fwd (the *_fwd of the same name): the 1-class OutConv, or the
 *   K-class OutConv and the argmax, in the epilogue; logits (optional for classify) stored as bf16, the argmax taken on the fp32
 *   logits in registers.
 * smaat_dsconv_bf16_eligible: 1 if those take the request: ncls = 0 for smaat_dsconv_bf16_fwd, else the classes of the head.
 * smaat_dsconv_maxpool_bf16_fwd (smaat_dsconv_maxpool_fwd): bf16 y and its max-pool, written as bf16 (pooled_bf16 = 1, 4-byte
 *   aligned) or fp32 (8-byte aligned), the dtype of the level it feeds; bit for bit the max-pool of the stored y.
 *   smaat_dsconv_maxpool_bf16_eligible: 1 if it takes the request (smaat_dsconv_bf16_eligible and the staged epilogue).
 * smaat_cbam_pool_mlp_bf16_fwd / smaat_cbam_pool_maxpool_bf16_fwd: the pools (+ MLP) and the 2x2 max-pool of a bf16 x; the max-pool
 *   is written as bf16 (pooled_bf16 = 1) or fp32, the dtype of the level it feeds.  The max-pool is required (even H, W % 4 == 0).
 * smaat_cbam_reduce_bf16_fwd: the per-pixel channel mean / max of x * sc from a bf16 x, fp32 out.
 * smaat_upsample2x_pad_bf16_fwd: bilinear x2 + pad to a bf16 y, from an fp32 (x_bf16 = 0) or bf16 x; Wo % 4 == 0.
 * smaat_outconv_bf16_fwd, smaat_argmax_channels_bf16_fwd, smaat_softmax_channels_bf16_fwd: the unfused heads from bf16
 *   activations / logits; OutConv and the softmax write bf16. */
int smaat_dsconv_bf16_eligible(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                               const void* pw_w, int H, int W, int k, int Cout, int ncls);
int smaat_dsconv_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                          const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale, const float* shift,
                          void* y, int64_t y_bstride, const float* gate_sc, const float* gate_sa, int B, int H, int W, int k,
                          int Cout, int relu, void* stream);
int smaat_dsconv_outconv_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                  const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale,
                                  const float* shift, const float* oc_w, const float* oc_b, void* logits, int B, int H, int W,
                                  int k, int Cout, int relu, void* stream);
int smaat_dsconv_classify_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                   const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale,
                                   const float* shift, const float* oc_w, const float* oc_b, int K, void* logits,
                                   int64_t* classes, int B, int H, int W, int k, int Cout, int relu, void* stream);
int smaat_dsconv_maxpool_bf16_eligible(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                       const void* pw_w, int H, int W, int k, int Cout);
int smaat_dsconv_maxpool_bf16_fwd(const void* x0, int C0, int64_t x0_bstride, const void* x1, int C1, int64_t x1_bstride,
                                  const float* dw_w, const float* dw_b, const uint16_t* pw_w, const float* scale,
                                  const float* shift, void* y, int64_t y_bstride, void* pooled, int pooled_bf16, int B, int H,
                                  int W, int k, int Cout, int relu, void* stream);
int smaat_cbam_pool_mlp_bf16_fwd(const void* x, float* avg, float* mx, void* pooled, int pooled_bf16, const float* w1,
                                 const float* b1, const float* w2, const float* b2, float* sc, int* counters, int B, int C,
                                 int H, int W, int hidden, void* stream);
int smaat_cbam_pool_maxpool_bf16_fwd(const void* x, float* avg, float* mx, void* pooled, int pooled_bf16, int64_t N, int H,
                                     int W, void* stream);
int smaat_cbam_reduce_bf16_fwd(const void* x, const float* sc, float* pooled, int B, int C, int P, void* stream);
int smaat_upsample2x_pad_bf16_fwd(const void* x, int x_bf16, void* y, int64_t y_bstride, int B, int C, int H, int W, int Ho,
                                  int Wo, void* stream);
int smaat_outconv_bf16_fwd(const void* x, const float* w, const float* bias, void* y, int B, int Cin, int ncls, int P,
                           void* stream);
int smaat_argmax_channels_bf16_fwd(const void* x, int64_t* classes, int B, int K, int64_t P, void* stream);
int smaat_softmax_channels_bf16_fwd(const void* x, void* probs, int B, int K, int64_t P, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SMAAT_B200_H_ */
