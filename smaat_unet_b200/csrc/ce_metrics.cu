// ce_metrics.cu -- multi-class cross-entropy, its gradient and the confusion-matrix update in ONE pass, no host sync.
//
// Replaces nn.CrossEntropyLoss()(y_pred, y) of the reference's segmentation loop (train_SmaAtUNet.py:54,182: log_softmax
// + nll_loss over (B, K, H, W) logits, several passes) and the per-batch `.cpu().numpy()` + np.bincount of
// metric/confusionmatrix.py:40-43,66-69 behind IoU.add (metric/iou.py:38-62).
//
// Per pixel (b, p) with label t = target[b, p]:
//   ignored  t == ignore_index (when use_ignore)      -> contributes nothing; dlogits = 0
//   invalid  t outside [0, K) and not ignored         -> batch_acc[2] += 1;   dlogits = 0
//   counted  otherwise                                -> batch_acc[0] += logsumexp_c(l) - l_t, batch_acc[1] += 1,
//                                                        dlogits = softmax(l) - onehot(t), conf[t][argmax_c l] += 1
// The logits are read once from HBM: the first sweep keeps an online (max, sum of exp) per pixel together with the
// first-index argmax and l_t; the gradient sweep re-reads the same lines while they are still in L2 (the grid is sized so
// that the lines in flight fit in about half of the L2) and streams dlogits out with evict-first stores.
// Confusion counts go to a per-CTA shared-memory histogram (K <= CE_SMEM_HIST_MAX_K) flushed with one 64-bit atomic per
// non-zero bin, or for larger K straight to the global matrix; either way lanes holding the same (t, argmax) pair are
// merged with __match_any_sync first, since neighbouring pixels of a segmentation map usually share both.
#include "common.cuh"

namespace smaat {

constexpr int CE_THREADS = 256;
constexpr int CE_SMEM_HIST_MAX_K = 96;       // 96*96 u32 = 36 KB of shared memory: under the 48 KB default

__device__ __forceinline__ double ce_warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ unsigned ce_warp_sum_u32(unsigned v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Add one to bin `key` (key < 0: nothing), merging the lanes of the calling (converged or not) warp that hit the same bin.
// No histogram requested (gl == NULL, uniform over the grid): nothing to do.
template <bool SMEM>
__device__ __forceinline__ void hist_add(int key, unsigned* sh, unsigned long long* gl) {
  if (gl == nullptr) return;
  const unsigned active = __activemask();
  const unsigned peers = __match_any_sync(active, key);
  if (key < 0) return;
  const int lane = threadIdx.x & 31;
  if (lane != __ffs(peers) - 1) return;
  const unsigned n = __popc(peers);
  if (SMEM)
    atomicAdd(sh + key, n);
  else
    atomicAdd(gl + key, (unsigned long long)n);
}

template <bool SMEM>
__device__ __forceinline__ void hist_flush(const unsigned* sh, unsigned long long* gl, int bins) {
  if (!SMEM || gl == nullptr) return;
  __syncthreads();
  for (int i = threadIdx.x; i < bins; i += blockDim.x) {
    const unsigned v = sh[i];
    if (v) atomicAdd(gl + i, (unsigned long long)v);
  }
}

template <int NPX>
__device__ __forceinline__ void load_px(const float* p, float (&v)[NPX]) {
  if constexpr (NPX == 4) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
#pragma unroll
    for (int j = 0; j < NPX; ++j) v[j] = __ldg(p + j);
  }
}
template <int NPX>
__device__ __forceinline__ void load_px_last(const float* p, float (&v)[NPX]) {
  if constexpr (NPX == 4) {
    const float4 q = __ldcs(reinterpret_cast<const float4*>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
#pragma unroll
    for (int j = 0; j < NPX; ++j) v[j] = __ldcs(p + j);
  }
}
template <int NPX>
__device__ __forceinline__ void store_px(float* p, const float (&v)[NPX]) {
  if constexpr (NPX == 4) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
  } else {
#pragma unroll
    for (int j = 0; j < NPX; ++j) __stcs(p + j, v[j]);
  }
}

// NPX consecutive pixels of one image per thread: NPX = 4 takes 128-bit loads (P % 4 == 0, 16-byte aligned logits,
// target and dlogits), NPX = 1 is the scalar path for every other layout.
template <int NPX, bool SMEM>
__global__ void __launch_bounds__(CE_THREADS) ce_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                            int K, int64_t P, int64_t groups, int64_t ignore_index, int use_ignore,
                                                            double* __restrict__ acc, float* __restrict__ dlogits,
                                                            unsigned long long* __restrict__ conf) {
  extern __shared__ unsigned sh_hist[];
  if (SMEM) {
    for (int i = threadIdx.x; i < K * K; i += blockDim.x) sh_hist[i] = 0u;
    __syncthreads();
  }
  const int64_t gpi = P / NPX;                  // pixel groups per image
  double loss = 0.0;
  unsigned counted = 0u, invalid = 0u;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    const int64_t b = g / gpi;
    const int64_t p0 = (g - b * gpi) * NPX;
    const float* base = logits + b * (int64_t)K * P + p0;
    int tl[NPX];
    bool ok[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) {
      const int64_t t = __ldg(target + b * P + p0 + j);
      const bool ign = use_ignore && t == ignore_index;
      ok[j] = !ign && t >= 0 && t < K;
      invalid += (unsigned)(!ign && !ok[j]);
      tl[j] = ok[j] ? (int)t : -1;              // never used as an index unless ok
    }
    float m[NPX], s[NPX], lt[NPX];
    int am[NPX];
    bool nan_seen[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) { m[j] = -INFINITY; s[j] = 0.f; lt[j] = 0.f; am[j] = 0; nan_seen[j] = false; }
    for (int c = 0; c < K; ++c) {
      float v[NPX];
      load_px<NPX>(base + (int64_t)c * P, v);
#pragma unroll
      for (int j = 0; j < NPX; ++j) {
        if (v[j] > m[j]) {                      // online log-sum-exp; first strictly larger value wins the argmax
          s[j] = fmaf(s[j], expf(m[j] - v[j]), 1.f);
          m[j] = v[j];
          if (!nan_seen[j]) am[j] = c;
        } else {
          s[j] += expf(v[j] - m[j]);            // NaN logits poison s, hence the pixel's loss and gradient
          if (v[j] != v[j] && !nan_seen[j]) { nan_seen[j] = true; am[j] = c; }   // torch.argmax: NaN is the maximum
        }
        lt[j] = (c == tl[j]) ? v[j] : lt[j];
      }
    }
    float inv_s[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) {
      inv_s[j] = 1.f / s[j];
      if (ok[j]) {
        loss += (double)((m[j] - lt[j]) + logf(s[j]));
        ++counted;
      }
      hist_add<SMEM>(ok[j] ? tl[j] * K + am[j] : -1, sh_hist, conf);
    }
    if (dlogits) {
      float* gbase = dlogits + b * (int64_t)K * P + p0;
      for (int c = 0; c < K; ++c) {
        float v[NPX], d[NPX];
        load_px_last<NPX>(base + (int64_t)c * P, v);
#pragma unroll
        for (int j = 0; j < NPX; ++j) d[j] = ok[j] ? expf(v[j] - m[j]) * inv_s[j] - (c == tl[j] ? 1.f : 0.f) : 0.f;
        store_px<NPX>(gbase + (int64_t)c * P, d);
      }
    }
  }
  hist_flush<SMEM>(sh_hist, conf, K * K);
  __shared__ double red_l[CE_THREADS / 32];
  __shared__ unsigned red_c[CE_THREADS / 32], red_i[CE_THREADS / 32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  loss = ce_warp_sum_f64(loss);
  counted = ce_warp_sum_u32(counted);
  invalid = ce_warp_sum_u32(invalid);
  if (lane == 0) { red_l[wp] = loss; red_c[wp] = counted; red_i[wp] = invalid; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double l = 0.0, c = 0.0, iv = 0.0;
    for (int i = 0; i < CE_THREADS / 32; ++i) { l += red_l[i]; c += red_c[i]; iv += red_i[i]; }
    if (c != 0.0) { atomicAdd(acc + 0, l); atomicAdd(acc + 1, c); }
    if (iv != 0.0) atomicAdd(acc + 2, iv);
  }
}

// One class of a probability / one-hot target row, in class order: the reference's checks (metric/confusionmatrix.py:57-61:
// every value in [0, 1], the row sums to 1 -- summed here in fp32 in class order) and the row's first argmax.
__device__ __forceinline__ void onehot_step(float q, int c, float& sum, float& qmax, int& qam, bool& bad) {
  sum += q;
  bad |= !(q >= 0.f && q <= 1.f);               // NaN fails too
  if (q > qmax) { qmax = q; qam = c; }
}

// Cross-entropy with the options smaat_ce_fwd leaves out: class weights w, label smoothing eps, probability targets
// (PROB) and a per-pixel loss map.  Same sweep structure as ce_fwd_kernel (logits and, with PROB, targets read once from
// HBM; the gradient sweep re-reads them from L2); the options live here so the plain kernel keeps its registers.
// Per pixel, with lse = logsumexp(l), W = sum_k w_k and the first logit l_0 as the shift of every difference below
// (W * lse - sum_k w_k l_k = W * (lse - l_0) - sum_k w_k (l_k - l_0) cancels far less when the logits are large):
//   class index t:  loss = (1 - eps) w_t (lse - l_t) + (eps / K) (W lse - sum_k w_k l_k),   D += w_t
//                   grad_j = ((1 - eps) w_t + eps W / K) p_j - (1 - eps) w_t [j == t] - (eps / K) w_j
//   probabilities:  q'_k = q_k (1 - eps) + eps / K,  S = sum_k w_k q'_k
//                   loss = S lse - sum_k w_k q'_k l_k,   grad_j = S p_j - w_j q'_j,   D += 1
// With w = 1 and eps = 0 the class-index gradient is computed by the same expression as ce_fwd_kernel's, so it is bitwise
// the same.  With PROB the confusion row is the target's first argmax, and a row that fails the reference's one-hot checks
// is left out and counted in acc[2] (the loss does not validate probability targets, as torch does not).
// Class-index targets are held to 64 registers (4 CTAs of 256 threads per SM, ce_fwd_kernel's occupancy; without the bound
// ptxas takes 75 and the streaming loop runs at 3 CTAs per SM); each thread's share of D is an fp32 sum to stay under it.
template <int NPX, bool SMEM, bool PROB>
__global__ void __launch_bounds__(CE_THREADS, PROB ? 2 : 4) cross_entropy_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target,
                                                                   const float* __restrict__ prob, const float* __restrict__ weight,
                                                                   int K, int64_t P, int64_t groups, float eps, int64_t ignore_index,
                                                                   int use_ignore, double* __restrict__ acc, float* __restrict__ loss_map,
                                                                   float* __restrict__ dlogits, unsigned long long* __restrict__ conf) {
  extern __shared__ unsigned sh_dyn[];
  unsigned* sh_hist = sh_dyn;
  float* sh_w = reinterpret_cast<float*>(sh_dyn + (SMEM ? K * K : 0));
  __shared__ float sh_wsum;
  if (SMEM)
    for (int i = threadIdx.x; i < K * K; i += blockDim.x) sh_hist[i] = 0u;
  for (int i = threadIdx.x; i < K; i += blockDim.x) sh_w[i] = weight ? __ldg(weight + i) : 1.f;
  __syncthreads();
  if (threadIdx.x < 32) {                       // W in a fixed order: every CTA gets the same value
    float s = 0.f;
    for (int i = threadIdx.x; i < K; i += 32) s += sh_w[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) sh_wsum = s;
  }
  __syncthreads();
  const float W = sh_wsum;
  const float keep = 1.f - eps, eps_k = eps / (float)K;
  const bool smooth = eps != 0.f;
  const int64_t gpi = P / NPX;
  double loss = 0.0;
  float dsum = 0.f;                             // a thread's share of D: a few dozen weights, exact enough in fp32
  unsigned counted = 0u, invalid = 0u;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    const int64_t b = g / gpi;
    const int64_t p0 = (g - b * gpi) * NPX;
    const float* base = logits + b * (int64_t)K * P + p0;
    const float* qbase = PROB ? prob + b * (int64_t)K * P + p0 : nullptr;
    int tl[NPX];
    bool ok[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) {
      if (PROB) {
        ok[j] = true;
        tl[j] = -1;
      } else {
        const int64_t t = __ldg(target + b * P + p0 + j);
        const bool ign = use_ignore && t == ignore_index;
        ok[j] = !ign && t >= 0 && t < K;
        invalid += (unsigned)(!ign && !ok[j]);
        tl[j] = ok[j] ? (int)t : (ign ? -1 : -2);   // -2: invalid; never used as an index unless ok
      }
    }
    float m[NPX], s[NPX], lt[NPX], l0[NPX], wd[NPX], sq[NPX], qs[NPX], qmax[NPX];
    int am[NPX], qam[NPX];
    bool nan_seen[NPX], qbad[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) {
      m[j] = -INFINITY; s[j] = 0.f; lt[j] = 0.f; l0[j] = 0.f; wd[j] = 0.f; sq[j] = 0.f; qs[j] = 0.f; qmax[j] = -INFINITY;
      am[j] = 0; qam[j] = 0; nan_seen[j] = false; qbad[j] = false;
    }
    for (int c = 0; c < K; ++c) {
      float v[NPX], q[NPX];
      load_px<NPX>(base + (int64_t)c * P, v);
      if (PROB) load_px<NPX>(qbase + (int64_t)c * P, q);
      const float wc = sh_w[c];
#pragma unroll
      for (int j = 0; j < NPX; ++j) {
        if (v[j] > m[j]) {                      // ce_fwd_kernel's online log-sum-exp and argmax
          s[j] = fmaf(s[j], expf(m[j] - v[j]), 1.f);
          m[j] = v[j];
          if (!nan_seen[j]) am[j] = c;
        } else {
          s[j] += expf(v[j] - m[j]);
          if (v[j] != v[j] && !nan_seen[j]) { nan_seen[j] = true; am[j] = c; }
        }
        l0[j] = c == 0 ? v[j] : l0[j];
        if (PROB) {
          const float wq = wc * fmaf(q[j], keep, eps_k);
          sq[j] += wq;
          wd[j] = fmaf(wq, v[j] - l0[j], wd[j]);
          onehot_step(q[j], c, qs[j], qmax[j], qam[j], qbad[j]);
        } else {
          lt[j] = (c == tl[j]) ? v[j] : lt[j];
          if (smooth) wd[j] = fmaf(wc, v[j] - l0[j], wd[j]);
        }
      }
    }
    float inv_s[NPX], lm[NPX], ga[NPX], gb[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) {
      const float ls = logf(s[j]);
      const float lse0 = (m[j] - l0[j]) + ls;   // lse - l_0
      if (PROB) {
        lm[j] = sq[j] * lse0 - wd[j];
        loss += (double)lm[j];
        dsum += 1.f;
        ++counted;
        inv_s[j] = sq[j] / s[j];
        const bool row_ok = !qbad[j] && qs[j] == 1.f;
        invalid += (unsigned)!row_ok;
        hist_add<SMEM>(row_ok ? qam[j] * K + am[j] : -1, sh_hist, conf);
      } else {
        const float wt = ok[j] ? sh_w[tl[j]] : 0.f;
        gb[j] = keep * wt;
        ga[j] = smooth ? fmaf(eps_k, W, gb[j]) : gb[j];
        inv_s[j] = ga[j] * (1.f / s[j]);        // w = 1, eps = 0: exactly ce_fwd_kernel's 1 / s
        if (ok[j]) {
          float term = gb[j] * ((m[j] - lt[j]) + ls);
          if (smooth) term = fmaf(eps_k, W * lse0 - wd[j], term);
          lm[j] = term;
          loss += (double)term;
          dsum += wt;
          ++counted;
        } else {
          lm[j] = tl[j] == -1 ? 0.f : NAN;      // ignored: 0; invalid label: NaN
        }
        hist_add<SMEM>(ok[j] ? tl[j] * K + am[j] : -1, sh_hist, conf);
      }
    }
    if (loss_map) store_px<NPX>(loss_map + b * P + p0, lm);
    if (dlogits) {
      float* gbase = dlogits + b * (int64_t)K * P + p0;
      for (int c = 0; c < K; ++c) {
        float v[NPX], q[NPX], d[NPX];
        load_px_last<NPX>(base + (int64_t)c * P, v);
        if (PROB) load_px_last<NPX>(qbase + (int64_t)c * P, q);
        const float wc = sh_w[c];
#pragma unroll
        for (int j = 0; j < NPX; ++j) {
          if (PROB) {
            d[j] = expf(v[j] - m[j]) * inv_s[j] - wc * fmaf(q[j], keep, eps_k);
          } else {
            d[j] = ok[j] ? expf(v[j] - m[j]) * inv_s[j] - (c == tl[j] ? gb[j] : 0.f) : 0.f;
            if (smooth && ok[j]) d[j] -= eps_k * wc;
          }
        }
        store_px<NPX>(gbase + (int64_t)c * P, d);
      }
    }
  }
  hist_flush<SMEM>(sh_hist, conf, K * K);
  __shared__ double red_l[CE_THREADS / 32], red_d[CE_THREADS / 32];
  __shared__ unsigned red_c[CE_THREADS / 32], red_i[CE_THREADS / 32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  loss = ce_warp_sum_f64(loss);
  const double dsum_d = ce_warp_sum_f64((double)dsum);
  counted = ce_warp_sum_u32(counted);
  invalid = ce_warp_sum_u32(invalid);
  if (lane == 0) { red_l[wp] = loss; red_d[wp] = dsum_d; red_c[wp] = counted; red_i[wp] = invalid; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double l = 0.0, dd = 0.0, c = 0.0, iv = 0.0;
    for (int i = 0; i < CE_THREADS / 32; ++i) { l += red_l[i]; dd += red_d[i]; c += red_c[i]; iv += red_i[i]; }
    if (c != 0.0) { atomicAdd(acc + 0, l); atomicAdd(acc + 1, c); atomicAdd(acc + 3, dd); }
    if (iv != 0.0) atomicAdd(acc + 2, iv);
  }
}

// One-hot / probability targets (B, K, P) -> int64 class indices (B, P): the row's first argmax, or -1 for a row that fails
// the reference's checks (onehot_step), which smaat_confusion_add and the score path then count as invalid.
template <int NPX>
__global__ void __launch_bounds__(CE_THREADS) onehot_classes_kernel(const float* __restrict__ x, int64_t* __restrict__ classes, int K,
                                                                    int64_t P, int64_t groups) {
  const int64_t gpi = P / NPX;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    const int64_t b = g / gpi;
    const int64_t p0 = (g - b * gpi) * NPX;
    const float* base = x + b * (int64_t)K * P + p0;
    float sum[NPX], qmax[NPX];
    int qam[NPX];
    bool bad[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) { sum[j] = 0.f; qmax[j] = -INFINITY; qam[j] = 0; bad[j] = false; }
    for (int c = 0; c < K; ++c) {
      float v[NPX];
      load_px_last<NPX>(base + (int64_t)c * P, v);
#pragma unroll
      for (int j = 0; j < NPX; ++j) onehot_step(v[j], c, sum[j], qmax[j], qam[j], bad[j]);
    }
    int64_t* out = classes + b * P + p0;
#pragma unroll
    for (int j = 0; j < NPX; ++j) out[j] = (bad[j] || sum[j] != 1.f) ? -1 : qam[j];
  }
}

template <bool SMEM>
__global__ void __launch_bounds__(CE_THREADS) confusion_add_kernel(const int64_t* __restrict__ pred, const int64_t* __restrict__ target,
                                                                   int64_t n, int K, unsigned long long* __restrict__ conf,
                                                                   unsigned long long* __restrict__ invalid_out) {
  extern __shared__ unsigned sh_hist[];
  if (SMEM) {
    for (int i = threadIdx.x; i < K * K; i += blockDim.x) sh_hist[i] = 0u;
    __syncthreads();
  }
  unsigned invalid = 0u;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t p = __ldg(pred + i), t = __ldg(target + i);
    const bool ok = p >= 0 && p < K && t >= 0 && t < K;
    invalid += (unsigned)!ok;
    hist_add<SMEM>(ok ? (int)t * K + (int)p : -1, sh_hist, conf);
  }
  hist_flush<SMEM>(sh_hist, conf, K * K);
  if (invalid_out) {
    invalid = ce_warp_sum_u32(invalid);
    if ((threadIdx.x & 31) == 0 && invalid) atomicAdd(invalid_out, (unsigned long long)invalid);
  }
}

// Channel argmax: the class map of (B, K, P) logits in one read, NPX consecutive pixels of one image per thread (NPX = 4: 128-bit
// loads and two 128-bit stores of the int64 classes).  The first strictly larger value wins, and a NaN wins and stays: the
// answer of torch.argmax, and of ce_fwd_kernel's argmax above.
template <int NPX>
__global__ void __launch_bounds__(CE_THREADS) argmax_channels_kernel(const float* __restrict__ x, int64_t* __restrict__ classes, int K,
                                                                     int64_t P, int64_t groups) {
  const int64_t gpi = P / NPX;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    const int64_t b = g / gpi;
    const int64_t p0 = (g - b * gpi) * NPX;
    const float* base = x + b * (int64_t)K * P + p0;
    float m[NPX];
    int am[NPX];
#pragma unroll
    for (int j = 0; j < NPX; ++j) { m[j] = -INFINITY; am[j] = 0; }
    for (int c = 0; c < K; ++c) {
      float v[NPX];
      load_px_last<NPX>(base + (int64_t)c * P, v);
#pragma unroll
      for (int j = 0; j < NPX; ++j) {
        if (m[j] == m[j] && (v[j] > m[j] || v[j] != v[j])) { m[j] = v[j]; am[j] = c; }
      }
    }
    int64_t* out = classes + b * P + p0;
    if constexpr (NPX == 4) {
      reinterpret_cast<longlong2*>(out)[0] = make_longlong2(am[0], am[1]);
      reinterpret_cast<longlong2*>(out)[1] = make_longlong2(am[2], am[3]);
    } else {
#pragma unroll
      for (int j = 0; j < NPX; ++j) out[j] = am[j];
    }
  }
}

// bf16 logits (the serving forward's bf16 route): one pixel per thread, each logit widened exactly; the same rule
__global__ void __launch_bounds__(CE_THREADS) argmax_channels_bf16_kernel(const uint16_t* __restrict__ x, int64_t* __restrict__ classes,
                                                                          int K, int64_t P, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += stride) {
    const int64_t b = g / P, p = g - b * P;
    const uint16_t* base = x + b * (int64_t)K * P + p;
    float m = -INFINITY;
    int am = 0;
    for (int c = 0; c < K; ++c) {
      const float v = ld_act(base + (int64_t)c * P);
      if (m == m && (v > m || v != v)) { m = v; am = c; }
    }
    classes[g] = am;
  }
}

// Online (max m, sum s) over one pixel's logits, then p = exp(l - m) / s.  Each add() computes
//   s = fmaf(s, exp(m_old - m_new), exp(l - m_new)),  m_new = fmaxf(m_old, l)
// in two branches: a new maximum (l > m) evaluates that formula; otherwise m_new = m_old, exp(m - m) is exactly 1 wherever s is
// still finite, and the fmaf is the single-rounding s + exp(l - m): one exp instead of two, the same bits.  The results match
// torch.softmax on non-finite logits:
//   a NaN logit: it is never a new maximum, exp(NaN - m) makes s NaN, and every class of the pixel is NaN;
//   a +inf logit: exp(inf - inf) = NaN in s, every class NaN;
//   all logits -inf: s stays 0 and exp(-inf + inf) / 0 is NaN for every class;
//   a -inf logit among finite ones: exp(-inf - m) / s = 0 for that class;
//   K = 1, finite: exp(0) / 1 = 1.
// A -inf logit adds exp(-inf) = 0 and leaves the max alone, so add() skips it: fed through the formula as a pixel's first
// logit it would give s = 0 * exp(-inf + inf) + exp(-inf + inf) = NaN and poison the finite classes after it.
struct SoftmaxAcc {
  float m = -INFINITY, s = 0.f;
  __device__ __forceinline__ void add(float l) {
    if (l > m) {
      s = fmaf(s, expf(m - l), expf(l - l));   // l - l: NaN for l = +inf, as the formula
      m = l;
    } else if (l != -INFINITY) {
      s += expf(l - m);
    }
  }
  __device__ __forceinline__ float prob(float l) const { return expf(l - m) / s; }
};

// Channel softmax: the probabilities of (B, K, P) logits, NPX consecutive pixels of one image per thread, as
// argmax_channels_kernel.  The first sweep feeds the classes in order to SoftmaxAcc; the second re-reads the
// same lines, which the grid keeps in L2 (smaat_softmax_channels_fwd), and streams the probabilities out.
template <int NPX>
__global__ void __launch_bounds__(CE_THREADS) softmax_channels_kernel(const float* __restrict__ x, float* __restrict__ probs, int K,
                                                                      int64_t P, int64_t groups) {
  const int64_t gpi = P / NPX;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    const int64_t b = g / gpi;
    const int64_t off = b * (int64_t)K * P + (g - b * gpi) * NPX;
    SoftmaxAcc acc[NPX];
    for (int c = 0; c < K; ++c) {
      float v[NPX];
      load_px<NPX>(x + off + (int64_t)c * P, v);
#pragma unroll
      for (int j = 0; j < NPX; ++j) acc[j].add(v[j]);
    }
    for (int c = 0; c < K; ++c) {
      float v[NPX];
      load_px_last<NPX>(x + off + (int64_t)c * P, v);
#pragma unroll
      for (int j = 0; j < NPX; ++j) v[j] = acc[j].prob(v[j]);
      store_px<NPX>(probs + off + (int64_t)c * P, v);
    }
  }
}

// bf16 logits to bf16 probabilities: softmax_channels_kernel's two sweeps (SoftmaxAcc) on the widened logits, one pixel
// per thread, each probability rounded once
__global__ void __launch_bounds__(CE_THREADS) softmax_channels_bf16_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ probs,
                                                                           int K, int64_t P, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += stride) {
    const int64_t b = g / P;
    const int64_t off = b * (int64_t)K * P + (g - b * P);
    SoftmaxAcc acc;
    for (int c = 0; c < K; ++c) acc.add(ld_act(x + off + (int64_t)c * P));
    for (int c = 0; c < K; ++c) st_act(probs + off + (int64_t)c * P, acc.prob(ld_act(x + off + (int64_t)c * P)));
  }
}

static int64_t l2_bytes() {
  int dev = 0, l2 = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev) != cudaSuccess || l2 <= 0) l2 = 50 << 20;
  return l2;
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_ce_fwd(const float* logits, const int64_t* target, int B, int K, int64_t P, int64_t ignore_index,
                            int use_ignore, double* batch_acc, float* dlogits, int64_t* conf, void* stream) {
  SMAAT_REQUIRE(logits && target && batch_acc && B > 0 && P > 0, "ce_fwd: bad arguments (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE(K >= 2, "ce_fwd: K=%d classes, need at least 2", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "ce_fwd: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(logits) & 3u) == 0 && (reinterpret_cast<uintptr_t>(target) & 7u) == 0 &&
                    (!dlogits || (reinterpret_cast<uintptr_t>(dlogits) & 3u) == 0),
                "ce_fwd: logits / dlogits must be 4-byte and target 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(batch_acc, 0, 3 * sizeof(double), st);
  if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "ce_fwd: memset: %s", cudaGetErrorString(e));
  const bool vec = P % 4 == 0 && aligned16(logits) && aligned16(target) && (!dlogits || aligned16(dlogits));
  const int npx = vec ? 4 : 1;
  const int64_t groups = (int64_t)B * (P / npx);
  // lines a CTA touches between its two sweeps: keep the whole grid's share under half of the L2 so the gradient sweep
  // re-reads from L2, but never fewer than one CTA per SM
  const int64_t per_cta = (int64_t)CE_THREADS * npx * K * 4;
  int64_t cap = l2_bytes() / 2 / per_cta;
  if (cap < num_sms()) cap = num_sms();
  if (cap > (int64_t)num_sms() * 8) cap = (int64_t)num_sms() * 8;
  int64_t blocks = ceil_div64(groups, CE_THREADS);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  const bool smem = conf && K <= CE_SMEM_HIST_MAX_K;
  const size_t shb = smem ? (size_t)K * K * sizeof(unsigned) : 0;
  auto* cf = reinterpret_cast<unsigned long long*>(conf);
  const unsigned g = (unsigned)blocks;
  if (vec) {
    if (smem) ce_fwd_kernel<4, true><<<g, CE_THREADS, shb, st>>>(logits, target, K, P, groups, ignore_index, use_ignore, batch_acc, dlogits, cf);
    else      ce_fwd_kernel<4, false><<<g, CE_THREADS, 0, st>>>(logits, target, K, P, groups, ignore_index, use_ignore, batch_acc, dlogits, cf);
  } else {
    if (smem) ce_fwd_kernel<1, true><<<g, CE_THREADS, shb, st>>>(logits, target, K, P, groups, ignore_index, use_ignore, batch_acc, dlogits, cf);
    else      ce_fwd_kernel<1, false><<<g, CE_THREADS, 0, st>>>(logits, target, K, P, groups, ignore_index, use_ignore, batch_acc, dlogits, cf);
  }
  SMAAT_LAUNCH_CHECK("smaat_ce_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_cross_entropy_fwd(const float* logits, const int64_t* target, const float* target_prob, const float* weight,
                                       int B, int K, int64_t P, float label_smoothing, int64_t ignore_index, int use_ignore,
                                       double* batch_acc, float* loss_map, float* dlogits, int64_t* conf, void* stream) {
  SMAAT_REQUIRE(logits && batch_acc && B > 0 && P > 0, "cross_entropy_fwd: bad arguments (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE((target != nullptr) != (target_prob != nullptr),
                "cross_entropy_fwd: pass exactly one of class-index targets and probability targets");
  SMAAT_REQUIRE(K >= 2, "cross_entropy_fwd: K=%d classes, need at least 2", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "cross_entropy_fwd: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE(label_smoothing >= 0.f && label_smoothing <= 1.f, "cross_entropy_fwd: label_smoothing=%g outside [0, 1]",
                (double)label_smoothing);
  SMAAT_REQUIRE(!(target_prob && use_ignore), "cross_entropy_fwd: ignore_index is not supported for probability targets");
  auto a4 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; };
  SMAAT_REQUIRE(a4(logits) && a4(target_prob) && a4(weight) && a4(loss_map) && a4(dlogits) &&
                    (reinterpret_cast<uintptr_t>(target) & 7u) == 0 && (reinterpret_cast<uintptr_t>(batch_acc) & 7u) == 0 &&
                    (reinterpret_cast<uintptr_t>(conf) & 7u) == 0,
                "cross_entropy_fwd: float arrays must be 4-byte and target / batch_acc / conf 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(batch_acc, 0, 4 * sizeof(double), st);
  if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "cross_entropy_fwd: memset: %s", cudaGetErrorString(e));
  const bool prob = target_prob != nullptr;
  const bool vec = P % 4 == 0 && aligned16(logits) && (prob ? aligned16(target_prob) : aligned16(target)) &&
                   (!dlogits || aligned16(dlogits)) && (!loss_map || aligned16(loss_map));
  const int npx = vec ? 4 : 1;
  const int64_t groups = (int64_t)B * (P / npx);
  // smaat_ce_fwd's grid rule; probability targets are re-read from L2 too, so a CTA holds twice the lines
  const int64_t per_cta = (int64_t)CE_THREADS * npx * K * 4 * (prob ? 2 : 1);
  int64_t cap = l2_bytes() / 2 / per_cta;
  if (cap < num_sms()) cap = num_sms();
  if (cap > (int64_t)num_sms() * 8) cap = (int64_t)num_sms() * 8;
  int64_t blocks = ceil_div64(groups, CE_THREADS);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  const bool smem = conf && K <= CE_SMEM_HIST_MAX_K;
  const size_t shb = ((smem ? (size_t)K * K : 0) + (size_t)K) * sizeof(unsigned);
  auto* cf = reinterpret_cast<unsigned long long*>(conf);
  const unsigned g = (unsigned)blocks;
  const float eps = label_smoothing;
#define SMAAT_XENT(NPX, SMEM, PROB)                                                                                          \
  cross_entropy_kernel<NPX, SMEM, PROB><<<g, CE_THREADS, shb, st>>>(logits, target, target_prob, weight, K, P, groups, eps, \
                                                                     ignore_index, use_ignore, batch_acc, loss_map, dlogits, cf)
  if (prob) {
    if (vec) { if (smem) SMAAT_XENT(4, true, true); else SMAAT_XENT(4, false, true); }
    else     { if (smem) SMAAT_XENT(1, true, true); else SMAAT_XENT(1, false, true); }
  } else {
    if (vec) { if (smem) SMAAT_XENT(4, true, false); else SMAAT_XENT(4, false, false); }
    else     { if (smem) SMAAT_XENT(1, true, false); else SMAAT_XENT(1, false, false); }
  }
#undef SMAAT_XENT
  SMAAT_LAUNCH_CHECK("smaat_cross_entropy_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_onehot_classes(const float* target, int64_t* classes, int B, int K, int64_t P, void* stream) {
  SMAAT_REQUIRE(target && classes && B > 0 && P > 0, "onehot_classes: bad arguments (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE(K >= 1, "onehot_classes: K=%d classes", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "onehot_classes: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(target) & 3u) == 0 && (reinterpret_cast<uintptr_t>(classes) & 7u) == 0,
                "onehot_classes: target must be 4-byte and classes 8-byte aligned");
  const bool vec = P % 4 == 0 && aligned16(target) && aligned16(classes);
  const int npx = vec ? 4 : 1;
  const int64_t groups = (int64_t)B * (P / npx);
  int64_t blocks = ceil_div64(groups, CE_THREADS);
  const int64_t cap = (int64_t)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  cudaStream_t st = (cudaStream_t)stream;
  if (vec) onehot_classes_kernel<4><<<(unsigned)blocks, CE_THREADS, 0, st>>>(target, classes, K, P, groups);
  else     onehot_classes_kernel<1><<<(unsigned)blocks, CE_THREADS, 0, st>>>(target, classes, K, P, groups);
  SMAAT_LAUNCH_CHECK("smaat_onehot_classes");
  return SMAAT_OK;
}

extern "C" int smaat_argmax_channels_fwd(const float* x, int64_t* classes, int B, int K, int64_t P, void* stream) {
  SMAAT_REQUIRE(x && classes && B > 0 && P > 0, "argmax_channels: bad arguments (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE(K >= 1, "argmax_channels: K=%d classes", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "argmax_channels: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3u) == 0 && (reinterpret_cast<uintptr_t>(classes) & 7u) == 0,
                "argmax_channels: logits must be 4-byte and classes 8-byte aligned");
  const bool vec = P % 4 == 0 && aligned16(x) && aligned16(classes);
  const int npx = vec ? 4 : 1;
  const int64_t groups = (int64_t)B * (P / npx);
  int64_t blocks = ceil_div64(groups, CE_THREADS);
  const int64_t cap = (int64_t)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  cudaStream_t st = (cudaStream_t)stream;
  if (vec) argmax_channels_kernel<4><<<(unsigned)blocks, CE_THREADS, 0, st>>>(x, classes, K, P, groups);
  else     argmax_channels_kernel<1><<<(unsigned)blocks, CE_THREADS, 0, st>>>(x, classes, K, P, groups);
  SMAAT_LAUNCH_CHECK("smaat_argmax_channels_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_softmax_channels_fwd(const float* x, float* probs, int B, int K, int64_t P, void* stream) {
  SMAAT_REQUIRE(x && probs && B > 0 && P > 0, "softmax_channels: bad arguments (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE(K >= 1, "softmax_channels: K=%d classes", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "softmax_channels: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3u) == 0 && (reinterpret_cast<uintptr_t>(probs) & 3u) == 0,
                "softmax_channels: logits and probs must be 4-byte aligned");
  const bool vec = P % 4 == 0 && aligned16(x) && aligned16(probs);
  const int npx = vec ? 4 : 1;
  const int64_t groups = (int64_t)B * (P / npx);
  // smaat_ce_fwd's grid rule: the lines the grid reads between its two sweeps fit in half of the L2
  const int64_t per_cta = (int64_t)CE_THREADS * npx * K * 4;
  int64_t cap = l2_bytes() / 2 / per_cta;
  if (cap < num_sms()) cap = num_sms();
  if (cap > (int64_t)num_sms() * 8) cap = (int64_t)num_sms() * 8;
  int64_t blocks = ceil_div64(groups, CE_THREADS);
  if (blocks > cap) blocks = cap;
  cudaStream_t st = (cudaStream_t)stream;
  if (vec) softmax_channels_kernel<4><<<(unsigned)blocks, CE_THREADS, 0, st>>>(x, probs, K, P, groups);
  else     softmax_channels_kernel<1><<<(unsigned)blocks, CE_THREADS, 0, st>>>(x, probs, K, P, groups);
  SMAAT_LAUNCH_CHECK("smaat_softmax_channels_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_confusion_add(const int64_t* pred, const int64_t* target, int64_t n, int K, int64_t* conf,
                                   int64_t* invalid, void* stream) {
  SMAAT_REQUIRE(pred && target && conf && n > 0, "confusion_add: bad arguments (n=%lld)", (long long)n);
  SMAAT_REQUIRE(K >= 2, "confusion_add: K=%d classes, need at least 2", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "confusion_add: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(pred) & 7u) == 0 && (reinterpret_cast<uintptr_t>(target) & 7u) == 0,
                "confusion_add: pred / target must be 8-byte aligned");
  int64_t blocks = ceil_div64(n, CE_THREADS * 8);
  const int64_t cap = (int64_t)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  cudaStream_t st = (cudaStream_t)stream;
  auto* cf = reinterpret_cast<unsigned long long*>(conf);
  auto* iv = reinterpret_cast<unsigned long long*>(invalid);
  if (K <= CE_SMEM_HIST_MAX_K)
    confusion_add_kernel<true><<<(unsigned)blocks, CE_THREADS, (size_t)K * K * sizeof(unsigned), st>>>(pred, target, n, K, cf, iv);
  else
    confusion_add_kernel<false><<<(unsigned)blocks, CE_THREADS, 0, st>>>(pred, target, n, K, cf, iv);
  SMAAT_LAUNCH_CHECK("smaat_confusion_add");
  return SMAAT_OK;
}

extern "C" int smaat_argmax_channels_bf16_fwd(const void* x, int64_t* classes, int B, int K, int64_t P, void* stream) {
  SMAAT_REQUIRE(x && classes && B > 0 && P > 0, "argmax_channels_bf16: bad arguments (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE(K >= 1, "argmax_channels_bf16: K=%d classes", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "argmax_channels_bf16: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE((reinterpret_cast<uintptr_t>(x) & 1u) == 0 && (reinterpret_cast<uintptr_t>(classes) & 7u) == 0,
                "argmax_channels_bf16: logits must be 2-byte and classes 8-byte aligned");
  const int64_t n = (int64_t)B * P;
  int64_t blocks = ceil_div64(n, CE_THREADS);
  const int64_t cap = (int64_t)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  argmax_channels_bf16_kernel<<<(unsigned)blocks, CE_THREADS, 0, (cudaStream_t)stream>>>(static_cast<const uint16_t*>(x), classes, K,
                                                                                        P, n);
  SMAAT_LAUNCH_CHECK("smaat_argmax_channels_bf16_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_softmax_channels_bf16_fwd(const void* x, void* probs, int B, int K, int64_t P, void* stream) {
  SMAAT_REQUIRE(x && probs && B > 0 && P > 0, "softmax_channels_bf16: bad arguments (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE(K >= 1, "softmax_channels_bf16: K=%d classes", K);
  if (K > 1024) return fail(SMAAT_E_UNSUPPORTED, "softmax_channels_bf16: K=%d classes, this build supports at most 1024", K);
  SMAAT_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(probs)) & 1u) == 0,
                "softmax_channels_bf16: logits and probs must be 2-byte aligned");
  const int64_t n = (int64_t)B * P;
  // smaat_softmax_channels_fwd's grid rule: the lines the grid reads between its two sweeps fit in half of the L2
  const int64_t per_cta = (int64_t)CE_THREADS * K * 2;
  int64_t cap = l2_bytes() / 2 / per_cta;
  if (cap < num_sms()) cap = num_sms();
  if (cap > (int64_t)num_sms() * 8) cap = (int64_t)num_sms() * 8;
  int64_t blocks = ceil_div64(n, CE_THREADS);
  if (blocks > cap) blocks = cap;
  softmax_channels_bf16_kernel<<<(unsigned)blocks, CE_THREADS, 0, (cudaStream_t)stream>>>(static_cast<const uint16_t*>(x),
                                                                                         static_cast<uint16_t*>(probs), K, P, n);
  SMAAT_LAUNCH_CHECK("smaat_softmax_channels_bf16_fwd");
  return SMAAT_OK;
}
