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
