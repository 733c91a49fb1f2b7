// loss_metrics.cu -- the training/validation step's loss and metric bookkeeping in ONE pass, no host sync.
//
// Replaces UNetBase.loss_func (reference models/regression_lightning.py:57-65: mse_loss(reduction="sum") / B)
// and PrecipitationMetrics.update (reference metric/precipitation_metrics.py:37-95): the NaN guard (:46, a
// host-syncing `.any()` in the reference), the normalised and de-normalised squared errors (:60-73), and the
// TN/FP/FN/TP confusion counts of `x * factor * 12 > threshold` (:80-93).  HBM-bound: 8 bytes per pixel read
// (+4 written when the loss gradient 2*(p-y)*grad_scale is requested in the same pass).
//
// batch_acc (double[8], zeroed by the call): [0] sum (p-y)^2   [1] sum (p*f - y*f)^2   [2] #NaN in p or y
//                                            [3] TN  [4] FP  [5] FN  [6] TP            [7] n
// smaat_metrics_commit folds one batch into the running totals ON THE DEVICE and skips the batch when [2] != 0,
// which is what the reference's early `return` does -- without the device->host round trip.
// smaat_precip_sweep_fwd / _commit: the same bookkeeping for several thresholds at once, every image a batch of one
// (test-set evaluation, calc_metrics_test_set.py runs batch size 1).
#include "common.cuh"

namespace smaat {

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ unsigned warp_sum_u32(unsigned v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct LmAcc {
  float sse, sse_d;          // per-thread fp32 partials over <= a few hundred elements, merged in fp64
  unsigned nan, cnt[4];
};

// The value the reference thresholds, in its fp32 operation order: (x * factor) * 12 (x * 12 without denormalize),
// precipitation_metrics.py:69-70, :80-81.  lm_one and the threshold sweep both compare this against an fp32 threshold.
__device__ __forceinline__ float lm_denorm(float v, float factor, bool denorm) { return denorm ? __fmul_rn(v, factor) : v; }
__device__ __forceinline__ float lm_hourly(float vu) { return __fmul_rn(vu, 12.f); }

__device__ __forceinline__ void lm_one(float p, float y, float factor, float thr, bool denorm, LmAcc& a, float* g, float gs) {
  const float d = p - y;
  a.sse = fmaf(d, d, a.sse);
  const float pu = lm_denorm(p, factor, denorm), yu = lm_denorm(y, factor, denorm);
  const float dd = pu - yu;
  a.sse_d = fmaf(dd, dd, a.sse_d);
  a.nan += (unsigned)((p != p) | (y != y));
  const int pm = lm_hourly(pu) > thr, tm = lm_hourly(yu) > thr;
  a.cnt[tm * 2 + pm] += 1u;
  if (g) *g = 2.f * d * gs;
}

template <bool VEC>
__global__ void __launch_bounds__(256) mse_metrics_kernel(const float* __restrict__ pred, const float* __restrict__ target, int64_t n,
                                                          float factor, float thr, int denorm, double* __restrict__ acc,
                                                          float* __restrict__ dpred, float gs) {
  double tot[7] = {0, 0, 0, 0, 0, 0, 0};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  LmAcc a;
  a.sse = a.sse_d = 0.f; a.nan = 0u; a.cnt[0] = a.cnt[1] = a.cnt[2] = a.cnt[3] = 0u;
  if (VEC) {
    const int64_t n4 = n >> 2;
    const float4* p4 = reinterpret_cast<const float4*>(pred);
    const float4* y4 = reinterpret_cast<const float4*>(target);
    float4* g4 = reinterpret_cast<float4*>(dpred);
    int it = 0;
    for (int64_t i = tid; i < n4; i += stride) {
      const float4 p = __ldg(p4 + i), y = __ldg(y4 + i);
      float4 g;
      lm_one(p.x, y.x, factor, thr, denorm, a, dpred ? &g.x : nullptr, gs);
      lm_one(p.y, y.y, factor, thr, denorm, a, dpred ? &g.y : nullptr, gs);
      lm_one(p.z, y.z, factor, thr, denorm, a, dpred ? &g.z : nullptr, gs);
      lm_one(p.w, y.w, factor, thr, denorm, a, dpred ? &g.w : nullptr, gs);
      if (dpred) g4[i] = g;
      if (++it == 64) {  // bound the fp32 partial sums to 256 terms
        tot[0] += a.sse; tot[1] += a.sse_d; a.sse = a.sse_d = 0.f; it = 0;
      }
    }
    for (int64_t i = (n4 << 2) + tid; i < n; i += stride)
      lm_one(__ldg(pred + i), __ldg(target + i), factor, thr, denorm, a, dpred ? dpred + i : nullptr, gs);
  } else {
    int it = 0;
    for (int64_t i = tid; i < n; i += stride) {
      lm_one(__ldg(pred + i), __ldg(target + i), factor, thr, denorm, a, dpred ? dpred + i : nullptr, gs);
      if (++it == 256) { tot[0] += a.sse; tot[1] += a.sse_d; a.sse = a.sse_d = 0.f; it = 0; }
    }
  }
  tot[0] += a.sse; tot[1] += a.sse_d; tot[2] = a.nan;
  tot[3] = a.cnt[0]; tot[4] = a.cnt[1]; tot[5] = a.cnt[2]; tot[6] = a.cnt[3];
  __shared__ double red[7][8];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 7; ++q) {
    const double v = warp_sum_f64(tot[q]);
    if (lane == 0) red[q][wp] = v;
  }
  __syncthreads();
  if (threadIdx.x < 7) {
    double v = 0.0;
    for (int i = 0; i < 8; ++i) v += red[threadIdx.x][i];
    if (v != 0.0) atomicAdd(acc + threadIdx.x, v);
  }
  if (blockIdx.x == 0 && threadIdx.x == 7) acc[7] = (double)n;
}

// totals (double[9]): [0] total_loss  [1] total_loss_denorm  [2] total_samples  [3] total_pixels
//                     [4] TN [5] FP [6] FN [7] TP   [8] batches skipped by the NaN guard
__global__ void metrics_commit_kernel(const double* __restrict__ b, double* __restrict__ t, int batch_size, int denorm) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (b[2] != 0.0) { t[8] += 1.0; return; }
  t[0] += b[0] / batch_size;
  if (denorm) t[1] += b[1] / batch_size;
  t[2] += batch_size;
  t[3] += b[7];
  t[4] += b[3]; t[5] += b[4]; t[6] += b[5]; t[7] += b[6];
}

// ---- threshold sweep: per-image sums and one joint (target bin, pred bin) histogram per image --------------------------
// bin(v) = #{i : lm_hourly(lm_denorm(v)) > thr[i]}.  For strictly increasing thresholds (x > t_i) implies (x > t_j) for j < i,
// so the histogram H[a][b] over (target bin a, pred bin b) holds every threshold's confusion matrix:
// TP_i = sum_{a>=i, b>=i} H[a][b], FN_i = sum_{a>=i, b<i}, FP_i = sum_{a<i, b>=i}, TN_i = sum_{a<i, b<i}.
constexpr int kSweepMaxT = 32;
constexpr int kSweepThreads = 256;
constexpr int kSweepUnitsPerBlock = kSweepThreads * 4;   // loads (float4 or float) per block and operand

struct SweepThresholds {
  float t[kSweepMaxT];
};

struct SweepAcc {
  float sse, sse_d;
  unsigned nan;
};

__device__ __forceinline__ int sweep_bin(float v, float factor, bool denorm, const float* thr, int T) {
  const float h = lm_hourly(lm_denorm(v, factor, denorm));
  int b = 0;
  for (int i = 0; i < T; ++i) b += h > thr[i];
  return b;
}

// Called by all 32 lanes of a warp together (valid = this lane has an element): lanes that hit the same cell add to it once.
__device__ __forceinline__ void sweep_one(float p, float y, bool valid, float factor, bool denorm, const float* thr, int T,
                                          SweepAcc& a, unsigned* hist) {
  int cell = -1;
  if (valid) {
    const float d = p - y;
    a.sse = fmaf(d, d, a.sse);
    const float dd = lm_denorm(p, factor, denorm) - lm_denorm(y, factor, denorm);
    a.sse_d = fmaf(dd, dd, a.sse_d);
    a.nan += (unsigned)((p != p) | (y != y));
    cell = sweep_bin(y, factor, denorm, thr, T) * (T + 1) + sweep_bin(p, factor, denorm, thr, T);
  }
  const unsigned peers = __match_any_sync(0xffffffffu, cell);
  if (cell >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(hist + cell, (unsigned)__popc(peers));
}

// grid (slices, B): block (s, b) covers slice s of image b.  pred image b starts at pred + b * pred_bstride, target image b
// at target + b * P.  VEC: both 16-byte aligned at every image (aligned bases, pred_bstride % 4 == 0, P % 4 == 0).
template <bool VEC>
__global__ void __launch_bounds__(kSweepThreads) precip_sweep_kernel(const float* __restrict__ pred, int64_t pred_bstride,
                                                                     const float* __restrict__ target, int64_t P, float factor,
                                                                     const SweepThresholds thresholds, int T, int denorm,
                                                                     double* __restrict__ per_image, unsigned* __restrict__ hist) {
  __shared__ unsigned s_hist[(kSweepMaxT + 1) * (kSweepMaxT + 1)];
  __shared__ float s_thr[kSweepMaxT];
  __shared__ double red[3][kSweepThreads / 32];
  const int cells = (T + 1) * (T + 1);
  for (int c = threadIdx.x; c < cells; c += kSweepThreads) s_hist[c] = 0u;
  if (threadIdx.x < T) s_thr[threadIdx.x] = thresholds.t[threadIdx.x];
  __syncthreads();

  const int64_t img = blockIdx.y;
  const float* p_img = pred + img * pred_bstride;
  const float* y_img = target + img * P;
  const int64_t units = VEC ? (P >> 2) : P;
  const int64_t start = (int64_t)blockIdx.x * kSweepUnitsPerBlock;
  const int64_t end = min(units, start + kSweepUnitsPerBlock);
  SweepAcc a;
  a.sse = a.sse_d = 0.f; a.nan = 0u;
  // kSweepUnitsPerBlock / kSweepThreads = 4 loads per thread: at most 16 fp32 terms per partial sum
  for (int64_t base = start; base < end; base += kSweepThreads) {
    const int64_t i = base + threadIdx.x;
    const bool ok = i < end;
    if (VEC) {
      float4 p = make_float4(0.f, 0.f, 0.f, 0.f), y = p;
      if (ok) {
        p = __ldg(reinterpret_cast<const float4*>(p_img) + i);
        y = __ldg(reinterpret_cast<const float4*>(y_img) + i);
      }
      sweep_one(p.x, y.x, ok, factor, denorm, s_thr, T, a, s_hist);
      sweep_one(p.y, y.y, ok, factor, denorm, s_thr, T, a, s_hist);
      sweep_one(p.z, y.z, ok, factor, denorm, s_thr, T, a, s_hist);
      sweep_one(p.w, y.w, ok, factor, denorm, s_thr, T, a, s_hist);
    } else {
      sweep_one(ok ? __ldg(p_img + i) : 0.f, ok ? __ldg(y_img + i) : 0.f, ok, factor, denorm, s_thr, T, a, s_hist);
    }
  }

  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const double v0 = warp_sum_f64((double)a.sse), v1 = warp_sum_f64((double)a.sse_d);
  const unsigned v2 = warp_sum_u32(a.nan);
  if (lane == 0) { red[0][wp] = v0; red[1][wp] = v1; red[2][wp] = (double)v2; }
  __syncthreads();
  if (threadIdx.x < 3) {
    double v = 0.0;
    for (int w = 0; w < kSweepThreads / 32; ++w) v += red[threadIdx.x][w];
    if (v != 0.0) atomicAdd(per_image + img * 3 + threadIdx.x, v);
  }
  unsigned* h = hist + img * cells;
  for (int c = threadIdx.x; c < cells; c += kSweepThreads) {
    const unsigned v = s_hist[c];
    if (v) atomicAdd(h + c, v);
  }
}

// totals (double[5 + (T+1)^2]): [0] total_loss  [1] total_loss_denorm  [2] total_samples  [3] total_pixels
//                               [4] images skipped for NaN  [5 + a*(T+1) + b] joint histogram summed over the counted images
// Images in index order, each as a batch of one: what T batch-1 PrecipitationMetrics runs add.
__global__ void precip_sweep_commit_kernel(const double* __restrict__ per_image, const unsigned* __restrict__ hist, int B,
                                           int64_t P, int T, int denorm, double* __restrict__ totals) {
  const int cells = (T + 1) * (T + 1);
  for (int c = threadIdx.x; c < cells; c += blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < B; ++b)
      if (per_image[3 * b + 2] == 0.0) s += (double)hist[(int64_t)b * cells + c];
    totals[5 + c] += s;
  }
  if (threadIdx.x == 0) {
    for (int b = 0; b < B; ++b) {
      const double* r = per_image + 3 * b;
      if (r[2] != 0.0) { totals[4] += 1.0; continue; }
      totals[0] += r[0];
      if (denorm) totals[1] += r[1];
      totals[2] += 1.0;
      totals[3] += (double)P;
    }
  }
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_mse_metrics_fwd(const float* pred, const float* target, int64_t n, float factor, float threshold,
                                     int denormalize, double* batch_acc, float* dpred, float grad_scale, void* stream) {
  SMAAT_REQUIRE(pred && target && batch_acc && n > 0, "mse_metrics: bad arguments (n=%lld)", (long long)n);
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(batch_acc, 0, 8 * sizeof(double), st);
  if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "mse_metrics: memset: %s", cudaGetErrorString(e));
  const bool vec = aligned16(pred) && aligned16(target) && (!dpred || aligned16(dpred));
  int64_t blocks = ceil_div64(n, 256 * 16);
  const int64_t cap = (int64_t)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (vec)
    mse_metrics_kernel<true><<<(unsigned)blocks, 256, 0, st>>>(pred, target, n, factor, threshold, denormalize, batch_acc, dpred, grad_scale);
  else
    mse_metrics_kernel<false><<<(unsigned)blocks, 256, 0, st>>>(pred, target, n, factor, threshold, denormalize, batch_acc, dpred, grad_scale);
  SMAAT_LAUNCH_CHECK("smaat_mse_metrics_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_metrics_commit(const double* batch_acc, double* totals, int batch_size, int denormalize, void* stream) {
  SMAAT_REQUIRE(batch_acc && totals && batch_size > 0, "metrics_commit: bad arguments");
  metrics_commit_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(batch_acc, totals, batch_size, denormalize);
  SMAAT_LAUNCH_CHECK("smaat_metrics_commit");
  return SMAAT_OK;
}

extern "C" int smaat_precip_sweep_fwd(const float* pred, int64_t pred_bstride, const float* target, int B, int64_t P,
                                      float factor, const float* thresholds, int T, int denormalize, double* per_image,
                                      unsigned* hist, void* stream) {
  SMAAT_REQUIRE(pred && target && thresholds && per_image && hist, "precip_sweep: null pointer");
  SMAAT_REQUIRE(B >= 1 && B <= 65535 && P >= 1, "precip_sweep: bad shape (B=%d, P=%lld)", B, (long long)P);
  SMAAT_REQUIRE(B == 1 || pred_bstride >= P, "precip_sweep: pred batch stride %lld < P=%lld", (long long)pred_bstride,
                (long long)P);
  SMAAT_REQUIRE(T >= 1 && T <= kSweepMaxT, "precip_sweep: T=%d thresholds, need 1..%d", T, kSweepMaxT);
  SweepThresholds th;
  for (int i = 0; i < T; ++i) {
    SMAAT_REQUIRE(thresholds[i] == thresholds[i], "precip_sweep: threshold %d is NaN", i);
    SMAAT_REQUIRE(i == 0 || thresholds[i - 1] < thresholds[i], "precip_sweep: thresholds must be strictly increasing "
                  "(thresholds[%d]=%g, thresholds[%d]=%g)", i - 1, (double)thresholds[i > 0 ? i - 1 : 0], i, (double)thresholds[i]);
    th.t[i] = thresholds[i];
  }
  for (int i = T; i < kSweepMaxT; ++i) th.t[i] = 0.f;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t cells = (int64_t)(T + 1) * (T + 1);
  cudaError_t e = cudaMemsetAsync(per_image, 0, (size_t)B * 3 * sizeof(double), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(hist, 0, (size_t)B * cells * sizeof(unsigned), st);
  if (e != cudaSuccess) return fail(SMAAT_E_CUDA, "precip_sweep: memset: %s", cudaGetErrorString(e));
  const bool vec = aligned16(pred) && aligned16(target) && P % 4 == 0 && (B == 1 || pred_bstride % 4 == 0);
  const int64_t slices = ceil_div64(vec ? P / 4 : P, kSweepUnitsPerBlock);
  SMAAT_REQUIRE(slices <= 0x7fffffff, "precip_sweep: P=%lld too large", (long long)P);
  const dim3 grid((unsigned)slices, (unsigned)B);
  if (vec)
    precip_sweep_kernel<true><<<grid, kSweepThreads, 0, st>>>(pred, pred_bstride, target, P, factor, th, T, denormalize,
                                                              per_image, hist);
  else
    precip_sweep_kernel<false><<<grid, kSweepThreads, 0, st>>>(pred, pred_bstride, target, P, factor, th, T, denormalize,
                                                               per_image, hist);
  SMAAT_LAUNCH_CHECK("smaat_precip_sweep_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_precip_sweep_commit(const double* per_image, const unsigned* hist, int B, int64_t P, int T,
                                         int denormalize, double* totals, void* stream) {
  SMAAT_REQUIRE(per_image && hist && totals, "precip_sweep_commit: null pointer");
  SMAAT_REQUIRE(B >= 1 && P >= 1 && T >= 1 && T <= kSweepMaxT, "precip_sweep_commit: bad arguments (B=%d, P=%lld, T=%d)",
                B, (long long)P, T);
  precip_sweep_commit_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(per_image, hist, B, P, T, denormalize, totals);
  SMAAT_LAUNCH_CHECK("smaat_precip_sweep_commit");
  return SMAAT_OK;
}
