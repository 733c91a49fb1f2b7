// cbam.cu -- CBAM channel + spatial attention, forward (reference models/layers.py:90-141).
//
// Op-level traffic: the HW-global pool forces two reads of x before anything can be scaled,
// so the practical minimum is pool (1R) + channel-reduce (1R) + scale (1R+1W) = 4 |x|
// (SURVEY 8d).  Kernels:
//   pool    per-(b,c) plane mean+max           -- 128-bit loads, warp-shuffle + smem tree
//   mlp     shared 2-layer MLP + sigmoid       -- tiny, one CTA per image
//   reduce  per-pixel mean/max over channels of x*sc -> [B,2,H,W]
//   gate    k x k conv (2->1) + BN(1) affine + sigmoid on the small map
//   scale   y = (x*sc)*sa                      -- 128-bit streaming
#include "common.cuh"

namespace smaat {

__device__ __forceinline__ float sigmoidf_acc(float v) { return 1.f / (1.f + expf(-v)); }

// ---- shared MLP finished by the LAST pooling CTA of an image (SURVEY 7 step 5-i) ------------------------------------
// Every pooling CTA publishes its planes' (avg, max), fences, and bumps the image's counter; the CTA that completes the
// count owns the finished (avg, max) vectors of that image and runs the two-layer MLP + sigmoid right there -- no
// separate launch.  The counter is handed back at zero.  C <= 512, hidden <= 64 (host-checked).
struct MlpTail {
  const float* w1; const float* b1; const float* w2; const float* b2;   // MLP.1 (hidden x C), MLP.3 (C x hidden)
  float* sc;            // (B, C) out
  int* counters;        // (B) zero on entry, zero on exit
  int C, hidden;
};

__device__ void cbam_mlp_tail(const MlpTail& t, int b, const float* avg, const float* mx) {
  __shared__ float sa[512], sm[512], ha[64], hm[64];
  for (int c = threadIdx.x; c < t.C; c += blockDim.x) {
    sa[c] = __ldcg(avg + (int64_t)b * t.C + c);      // written by other CTAs: read at L2
    sm[c] = __ldcg(mx + (int64_t)b * t.C + c);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = warp; j < t.hidden; j += nw) {
    float da = 0.f, dm = 0.f;
    for (int c = lane; c < t.C; c += 32) {
      const float wv = __ldg(t.w1 + (int64_t)j * t.C + c);
      da = fmaf(wv, sa[c], da);
      dm = fmaf(wv, sm[c], dm);
    }
    da = warp_sum(da);
    dm = warp_sum(dm);
    if (lane == 0) {
      ha[j] = fmaxf(da + t.b1[j], 0.f);
      hm[j] = fmaxf(dm + t.b1[j], 0.f);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < t.C; c += blockDim.x) {
    float oa = t.b2[c], om = t.b2[c];  // second-layer bias is counted twice (layers.py:109)
    for (int j = 0; j < t.hidden; ++j) {
      const float wv = __ldg(t.w2 + (int64_t)c * t.hidden + j);
      oa = fmaf(wv, ha[j], oa);
      om = fmaf(wv, hm[j], om);
    }
    t.sc[(int64_t)b * t.C + c] = sigmoidf_acc(oa + om);
  }
}

// Called by ALL threads of a pooling CTA after its planes' results are in global memory; `planes` of image b were done here.
__device__ __forceinline__ void cbam_pool_finish(const MlpTail& t, int b, int planes, const float* avg, const float* mx) {
  __shared__ int last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int prev = atomicAdd(t.counters + b, planes);
    last = (prev + planes == t.C);
    if (last) t.counters[b] = 0;
  }
  __syncthreads();
  if (last) {
    __threadfence();
    cbam_mlp_tail(t, b, avg, mx);
  }
}

// ---- pool ----------------------------------------------------------------------------------------
// TPP threads cooperate on one plane; blockDim.x / TPP planes per CTA.
template <int TPP, bool VEC>
__global__ void __launch_bounds__(256) cbam_pool_kernel(const float* __restrict__ x, float* __restrict__ avg,
                                                        float* __restrict__ mx, int64_t N, int P, const MlpTail tail) {
  constexpr int PPB = 256 / TPP;
  const int sub = threadIdx.x / TPP;
  const int lane = threadIdx.x % TPP;
  const int64_t n = (int64_t)blockIdx.x * PPB + sub;
  float s = 0.f, m = -INFINITY;
  if (n < N) {
    const float* src = x + n * (int64_t)P;
    if (VEC) {
      const float4* s4 = reinterpret_cast<const float4*>(src);
      const int n4 = P >> 2;
      int i = lane;
      // 4 independent 128-bit loads in flight per thread
      for (; i + 3 * TPP < n4; i += 4 * TPP) {
        const float4 a = __ldg(s4 + i), b = __ldg(s4 + i + TPP), c = __ldg(s4 + i + 2 * TPP), d = __ldg(s4 + i + 3 * TPP);
        s += ((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w)) + ((c.x + c.y) + (c.z + c.w)) + ((d.x + d.y) + (d.z + d.w));
        m = fmaxf(m, fmaxf(fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)), fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w))));
        m = fmaxf(m, fmaxf(fmaxf(fmaxf(c.x, c.y), fmaxf(c.z, c.w)), fmaxf(fmaxf(d.x, d.y), fmaxf(d.z, d.w))));
      }
      for (; i < n4; i += TPP) {
        const float4 a = __ldg(s4 + i);
        s += (a.x + a.y) + (a.z + a.w);
        m = fmaxf(m, fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)));
      }
    } else {
      for (int i = lane; i < P; i += TPP) {
        const float v = __ldg(src + i);
        s += v;
        m = fmaxf(m, v);
      }
    }
  }
  s = warp_sum(s);
  m = warp_max(m);
  if (TPP == 32) {
    if (lane == 0 && n < N) {
      avg[n] = s / (float)P;
      mx[n] = m;
    }
  } else {
    __shared__ float ss[8], sm[8];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
      ss[w] = s;
      sm[w] = m;
    }
    __syncthreads();
    if (threadIdx.x == 0 && n < N) {
      float S = 0.f, M = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        S += ss[i];
        M = fmaxf(M, sm[i]);
      }
      avg[n] = S / (float)P;
      mx[n] = M;
    }
  }
  if (tail.sc) {   // planes of one CTA belong to one image (C % PPB == 0, host-checked)
    const int64_t n0 = (int64_t)blockIdx.x * PPB;
    const int planes = (int)((N - n0) < PPB ? (N - n0) : PPB);
    cbam_pool_finish(tail, (int)(n0 / tail.C), planes, avg, mx);
  }
}

// ---- shared MLP + sigmoid ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cbam_mlp_kernel(const float* __restrict__ avg, const float* __restrict__ mx,
                                                       const float* __restrict__ w1, const float* __restrict__ b1,
                                                       const float* __restrict__ w2, const float* __restrict__ b2,
                                                       float* __restrict__ sc, int C, int hidden) {
  extern __shared__ float sh[];  // avg[C] mx[C] ha[hidden] hm[hidden]
  float* sa = sh;
  float* sm = sh + C;
  float* ha = sm + C;
  float* hm = ha + hidden;
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    sa[c] = avg[(int64_t)b * C + c];
    sm[c] = mx[(int64_t)b * C + c];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = warp; j < hidden; j += nw) {
    float da = 0.f, dm = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float wv = __ldg(w1 + (int64_t)j * C + c);
      da = fmaf(wv, sa[c], da);
      dm = fmaf(wv, sm[c], dm);
    }
    da = warp_sum(da);
    dm = warp_sum(dm);
    if (lane == 0) {
      ha[j] = fmaxf(da + b1[j], 0.f);
      hm[j] = fmaxf(dm + b1[j], 0.f);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float oa = b2[c], om = b2[c];  // second-layer bias is counted twice (layers.py:109)
    for (int j = 0; j < hidden; ++j) {
      const float wv = __ldg(w2 + (int64_t)c * hidden + j);
      oa = fmaf(wv, ha[j], oa);
      om = fmaf(wv, hm[j], om);
    }
    sc[(int64_t)b * C + c] = sigmoidf_acc(oa + om);
  }
}

// ---- per-pixel channel mean / max of x*sc --------------------------------------------------------------
// Large planes: a thread owns 4 pixels and walks every channel with 8 independent 128-bit loads in flight -- no
// cross-thread reduction, no barrier; s_c of the image is staged in shared memory.
// TI: the storage type of x (float, or uint16_t bf16 in the serving forward's bf16 route); pooled is fp32 either way
template <typename TI>
__global__ void __launch_bounds__(256) cbam_reduce_v4_kernel(const TI* __restrict__ x, const float* __restrict__ sc,
                                                             float* __restrict__ pooled, int C, int P4) {
  extern __shared__ float scs[];
  const int b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) scs[c] = __ldg(sc + (int64_t)b * C + c);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P4) return;
  const TI* x4 = x + ((int64_t)b * C * P4 + i) * 4;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  int c = 0;
  for (; c + 8 <= C; c += 8) {
    float4 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = ld_act4(x4 + (int64_t)(c + u) * P4 * 4);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float g = scs[c + u];
      const float a0 = v[u].x * g, a1 = v[u].y * g, a2 = v[u].z * g, a3 = v[u].w * g;
      s.x += a0; s.y += a1; s.z += a2; s.w += a3;
      m.x = fmaxf(m.x, a0); m.y = fmaxf(m.y, a1); m.z = fmaxf(m.z, a2); m.w = fmaxf(m.w, a3);
    }
  }
  for (; c < C; ++c) {
    const float4 v = ld_act4(x4 + (int64_t)c * P4 * 4);
    const float g = scs[c];
    const float a0 = v.x * g, a1 = v.y * g, a2 = v.z * g, a3 = v.w * g;
    s.x += a0; s.y += a1; s.z += a2; s.w += a3;
    m.x = fmaxf(m.x, a0); m.y = fmaxf(m.y, a1); m.z = fmaxf(m.z, a2); m.w = fmaxf(m.w, a3);
  }
  const float inv = 1.f / (float)C;
  float4* pa = reinterpret_cast<float4*>(pooled) + (int64_t)b * 2 * P4 + i;
  pa[0] = make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv);
  pa[P4] = m;
}

// blockDim = (32 pixel-quads, 8 channel groups); smem tree over the 8 groups.
template <bool VEC, typename TI = float>
__global__ void __launch_bounds__(256) cbam_reduce_kernel(const TI* __restrict__ x, const float* __restrict__ sc,
                                                          float* __restrict__ pooled, int C, int P) {
  __shared__ float4 rs[8][32];
  __shared__ float4 rm[8][32];
  const int tx = threadIdx.x, cg = threadIdx.y;
  const int b = blockIdx.y;
  const int pp = (blockIdx.x * 32 + tx) * 4;
  const TI* xb = x + (int64_t)b * C * P;
  const float* scb = sc + (int64_t)b * C;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  if (pp < P) {
#pragma unroll 4
    for (int c = cg; c < C; c += 8) {
      const float g = __ldg(scb + c);
      float4 v;
      const TI* src = xb + (int64_t)c * P + pp;
      if (VEC) {
        v = ld_act4(src);
      } else {
        v.x = ld_act(src);
        v.y = (pp + 1 < P) ? ld_act(src + 1) : 0.f;
        v.z = (pp + 2 < P) ? ld_act(src + 2) : 0.f;
        v.w = (pp + 3 < P) ? ld_act(src + 3) : 0.f;
      }
      v.x *= g; v.y *= g; v.z *= g; v.w *= g;
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
    }
  }
  rs[cg][tx] = s;
  rm[cg][tx] = m;
  __syncthreads();
  if (cg == 0 && pp < P) {
#pragma unroll
    for (int i = 1; i < 8; ++i) {
      const float4 a = rs[i][tx], q = rm[i][tx];
      s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
      m.x = fmaxf(m.x, q.x); m.y = fmaxf(m.y, q.y); m.z = fmaxf(m.z, q.z); m.w = fmaxf(m.w, q.w);
    }
    const float inv = 1.f / (float)C;
    float* pa = pooled + (int64_t)b * 2 * P + pp;
    float* pm = pa + P;
    const float4 mean = make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv);
    if (VEC) {
      *reinterpret_cast<float4*>(pa) = mean;
      *reinterpret_cast<float4*>(pm) = m;
    } else {
      const float me[4] = {mean.x, mean.y, mean.z, mean.w};
      const float ma[4] = {m.x, m.y, m.z, m.w};
      for (int q = 0; q < 4; ++q)
        if (pp + q < P) {
          pa[q] = me[q];
          pm[q] = ma[q];
        }
    }
  }
}

// ---- spatial gate: conv kxk (2->1) + affine + sigmoid ------------------------------------------------
// 32 x 32 output tile per CTA; one thread -> 4 consecutive pixels of one row.  Each (channel, tap row) needs a
// 10-float segment of the staged tile: 2 LDS.128 + 1 LDS.64 feed 28 FMAs (10.5 shared loads per output
// instead of 98); row pitch 40 floats keeps the 128-bit loads aligned and conflict-free per quarter-warp.
constexpr int GT_W = 32, GT_H = 32, GT_P = 40;
template <int KS>
__global__ void __launch_bounds__(256) cbam_gate_kernel(const float* __restrict__ pooled, const float* __restrict__ wsp,
                                                        const float* __restrict__ bn_affine, float* __restrict__ sa,
                                                        float* __restrict__ raw, int H, int W) {
  constexpr int R = KS / 2;
  constexpr int SH = GT_H + 2 * R;
  __shared__ __align__(16) float t[2][SH][GT_P];  // column c holds global x = x0 - 4 + c (4-float left margin >= R)
  __shared__ float wk[2 * KS * KS];
  const int b = blockIdx.z;
  const int x0 = blockIdx.x * GT_W, y0 = blockIdx.y * GT_H;
  const int tid = threadIdx.x;
  if (tid < 2 * KS * KS) wk[tid] = __ldg(wsp + tid);
  const float* pb = pooled + (int64_t)b * 2 * H * W;
  for (int i = tid; i < 2 * SH * GT_P; i += 256) {
    const int ch = i / (SH * GT_P);
    const int r = (i / GT_P) % SH, c = i % GT_P;
    const int gy = y0 - R + r, gx = x0 - 4 + c;
    float v = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(pb + ((int64_t)ch * H + gy) * W + gx);
    t[ch][r][c] = v;
  }
  __syncthreads();
  const int tx = tid & 7, ty = tid >> 3;  // 8 quads x 32 rows
  const float a_s = bn_affine ? __ldg(bn_affine) : 1.f;
  const float a_t = bn_affine ? __ldg(bn_affine + 1) : 0.f;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int ch = 0; ch < 2; ++ch)
#pragma unroll
    for (int dy = 0; dy < KS; ++dy) {
      // outputs x0+4tx+j (j<4) with taps dx read smem columns 4tx + 4 - R + j + dx: a 4+KS-1 <= 10 float window
      const float* rowp = &t[ch][ty + dy][4 * tx];
      const float4 v0 = *reinterpret_cast<const float4*>(rowp);
      const float4 v1 = *reinterpret_cast<const float4*>(rowp + 4);
      const float4 v2 = *reinterpret_cast<const float4*>(rowp + 8);
      const float seg[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
#pragma unroll
      for (int dx = 0; dx < KS; ++dx) {
        const float wv = wk[(ch * KS + dy) * KS + dx];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = fmaf(wv, seg[4 - R + j + dx], acc[j]);
      }
    }
  const int gy = y0 + ty;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int gx = x0 + 4 * tx + j;
    if (gy < H && gx < W) {
      const int64_t o = ((int64_t)b * H + gy) * W + gx;
      if (raw) raw[o] = acc[j];
      sa[o] = sigmoidf_acc(fmaf(acc[j], a_s, a_t));
    }
  }
}

// ---- y = (x * sc) * sa -------------------------------------------------------------------------------------
constexpr int SC_CH = 8;  // channels per thread (sa quad reused from registers)
template <bool VEC>
__global__ void __launch_bounds__(256) cbam_scale_kernel(const float* __restrict__ x, const float* __restrict__ sc,
                                                         const float* __restrict__ sa, float* __restrict__ y,
                                                         int64_t y_bstride, int C, int P) {
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * SC_CH;
  const int pp = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (pp >= P) return;
  float4 g;
  const float* sab = sa + (int64_t)b * P + pp;
  if (VEC) {
    g = __ldg(reinterpret_cast<const float4*>(sab));
  } else {
    g.x = __ldg(sab);
    g.y = (pp + 1 < P) ? __ldg(sab + 1) : 0.f;
    g.z = (pp + 2 < P) ? __ldg(sab + 2) : 0.f;
    g.w = (pp + 3 < P) ? __ldg(sab + 3) : 0.f;
  }
  const float* xb = x + ((int64_t)b * C + c0) * P + pp;
  float* yb = y + (int64_t)b * y_bstride + (int64_t)c0 * P + pp;
  const float* scb = sc + (int64_t)b * C + c0;
  const int nc = min(SC_CH, C - c0);
  if (VEC && nc == SC_CH) {
    float4 v[SC_CH];
#pragma unroll
    for (int i = 0; i < SC_CH; ++i) v[i] = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)i * P));
#pragma unroll
    for (int i = 0; i < SC_CH; ++i) {
      const float s = __ldg(scb + i);
      float4 o;
      o.x = (v[i].x * s) * g.x; o.y = (v[i].y * s) * g.y; o.z = (v[i].z * s) * g.z; o.w = (v[i].w * s) * g.w;
      *reinterpret_cast<float4*>(yb + (int64_t)i * P) = o;
    }
  } else {
    const float gg[4] = {g.x, g.y, g.z, g.w};
    for (int i = 0; i < nc; ++i) {
      const float s = __ldg(scb + i);
      for (int q = 0; q < 4; ++q)
        if (pp + q < P) yb[(int64_t)i * P + q] = (__ldg(xb + (int64_t)i * P + q) * s) * gg[q];
    }
  }
}

// Global avg/max pool of a plane AND its 2x2 max-pool in the same read: in SmaAt-UNet every encoder map feeds both
// cbam_l (ChannelAttention pools, layers.py:107-108) and down_l (MaxPool2d(2), parts_ds.py:48) -- models/SmaAt_UNet.py:42-50.
// A thread takes the same 4 columns of rows 2i and 2i+1 (two 128-bit loads), emits 2 pooled outputs (64-bit store) and
// folds all 8 values into the plane's sum / max.  TPP threads per plane (256: one plane per CTA; 32: 8 planes per CTA).
// TI / TO: the storage types of x and of pooled (float, or uint16_t bf16 in the serving forward's bf16 route; the max of bf16
// values is a bf16 value, so a bf16 max-pool is exact in either type)
template <int TPP, typename TI = float, typename TO = float>
__global__ void __launch_bounds__(256) cbam_pool_maxpool_kernel(const TI* __restrict__ x, float* __restrict__ avg,
                                                                float* __restrict__ mx, TO* __restrict__ pooled, int64_t N,
                                                                int H, int W, const MlpTail tail) {
  constexpr int PPB = 256 / TPP;
  const int sub = threadIdx.x / TPP, lane = threadIdx.x % TPP;
  const int64_t n = (int64_t)blockIdx.x * PPB + sub;
  const int wq = W >> 2, hp = H >> 1;
  const int items = wq * hp;
  float s = 0.f, m = -INFINITY;
  if (n < N) {
    const TI* src = x + n * (int64_t)H * W;
    TO* dst = pooled + n * (int64_t)hp * (W >> 1);
#pragma unroll 2
    for (int i = lane; i < items; i += TPP) {
      const int rp = i / wq, q = i - rp * wq;
      const float4 a = ld_act4(src + ((int64_t)(2 * rp) * wq + q) * 4), b = ld_act4(src + ((int64_t)(2 * rp + 1) * wq + q) * 4);
      const float m0 = fmaxf(fmaxf(a.x, a.y), fmaxf(b.x, b.y)), m1 = fmaxf(fmaxf(a.z, a.w), fmaxf(b.z, b.w));
      if constexpr (sizeof(TO) == 4) reinterpret_cast<float2*>(dst)[(int64_t)rp * wq + q] = make_float2(m0, m1);
      else reinterpret_cast<uint32_t*>(dst)[(int64_t)rp * wq + q] = f32x2_bf16x2(m0, m1);
      s += ((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w));
      m = fmaxf(m, fmaxf(m0, m1));
    }
  }
  s = warp_sum(s);
  m = warp_max(m);
  if (TPP == 32) {
    if (lane == 0 && n < N) {
      avg[n] = s / (float)(H * W);
      mx[n] = m;
    }
  } else {
    __shared__ float ss[8], sm[8];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { ss[w] = s; sm[w] = m; }
    __syncthreads();
    if (threadIdx.x == 0 && n < N) {
      float S = 0.f, M = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) { S += ss[i]; M = fmaxf(M, sm[i]); }
      avg[n] = S / (float)(H * W);
      mx[n] = M;
    }
  }
  if (tail.sc) {
    const int64_t n0 = (int64_t)blockIdx.x * PPB;
    const int planes = (int)((N - n0) < PPB ? (N - n0) : PPB);
    cbam_pool_finish(tail, (int)(n0 / tail.C), planes, avg, mx);
  }
}

// ---- channel gate from the partial pools the producing DS conv wrote in its epilogue (smaat_dsconv_cbam_fwd) ---------------
// psum / pmax: (B, npart, C).  CTA (channel block, image) reduces MP_CB channels: thread (group j, channel quad q) folds parts
// j, j + MP_NJ, ... with 128-bit loads, then one thread per quad folds the groups in order -- a fixed order, so the result
// does not depend on timing.  The last CTA of an image runs the MLP (cbam_pool_finish), as in cbam_pool_kernel.
constexpr int MP_CB = 16, MP_NQ = MP_CB / 4, MP_NJ = 256 / MP_NQ;
__global__ void __launch_bounds__(256) cbam_mlp_partials_kernel(const float* __restrict__ psum, const float* __restrict__ pmax,
                                                                int npart, float* __restrict__ avg, float* __restrict__ mx, int P,
                                                                const MlpTail tail) {
  __shared__ float4 rs[MP_NJ][MP_NQ], rm[MP_NJ][MP_NQ];
  const int b = blockIdx.y, c0 = blockIdx.x * MP_CB;
  const int q = threadIdx.x % MP_NQ, j = threadIdx.x / MP_NQ;
  const int64_t step = tail.C / 4;                               // float4s per part
  const int64_t base = ((int64_t)b * npart * tail.C + c0) / 4 + q;
  const float4* s4 = reinterpret_cast<const float4*>(psum) + base;
  const float4* m4 = reinterpret_cast<const float4*>(pmax) + base;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f), m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll 4
  for (int i = j; i < npart; i += MP_NJ) {
    const float4 a = __ldg(s4 + i * step), e = __ldg(m4 + i * step);
    s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
    m.x = fmaxf(m.x, e.x); m.y = fmaxf(m.y, e.y); m.z = fmaxf(m.z, e.z); m.w = fmaxf(m.w, e.w);
  }
  rs[j][q] = s;
  rm[j][q] = m;
  __syncthreads();
  if (threadIdx.x < MP_NQ) {
    for (int jj = 1; jj < MP_NJ; ++jj) {
      const float4 a = rs[jj][q], e = rm[jj][q];
      s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
      m.x = fmaxf(m.x, e.x); m.y = fmaxf(m.y, e.y); m.z = fmaxf(m.z, e.z); m.w = fmaxf(m.w, e.w);
    }
    const int64_t o = (int64_t)b * tail.C + c0 + 4 * q;
    avg[o] = s.x / (float)P; avg[o + 1] = s.y / (float)P; avg[o + 2] = s.z / (float)P; avg[o + 3] = s.w / (float)P;
    mx[o] = m.x; mx[o + 1] = m.y; mx[o + 2] = m.z; mx[o + 3] = m.w;
  }
  cbam_pool_finish(tail, b, MP_CB, avg, mx);
}

// ---- spatial gate + scale in one kernel: y = (x * sc) * sigmoid(BN(conv kxk(pooled))) --------------------------------------
// The gate of a 32 x 32 pixel tile is computed exactly as cbam_gate_kernel does (staged 2-channel tile with halo), then the
// same thread walks its 4 pixels through the CTA's slice of the channels: the 1-channel gate map never reaches HBM and
// one launch disappears.  grid.z = B * csplit (channel slices: small planes need the parallelism).
template <int KS>
__global__ void __launch_bounds__(256, 4) cbam_gate_scale_kernel(const float* __restrict__ pooled, const float* __restrict__ wsp,
                                                              const float* __restrict__ bn_affine, const float* __restrict__ x,
                                                              const float* __restrict__ sc, float* __restrict__ y, int64_t y_bstride,
                                                              int C, int H, int W, int csplit) {
  constexpr int R = KS / 2;
  constexpr int SH = GT_H + 2 * R;
  __shared__ __align__(16) float t[2][SH][GT_P];
  __shared__ float wk[2 * KS * KS];
  const int b = blockIdx.z / csplit, cs = blockIdx.z - b * csplit;
  const int x0 = blockIdx.x * GT_W, y0 = blockIdx.y * GT_H;
  const int tid = threadIdx.x;
  if (tid < 2 * KS * KS) wk[tid] = __ldg(wsp + tid);
  const float* pb = pooled + (int64_t)b * 2 * H * W;
  for (int i = tid; i < 2 * SH * GT_P; i += 256) {
    const int ch = i / (SH * GT_P);
    const int r = (i / GT_P) % SH, c = i % GT_P;
    const int gy = y0 - R + r, gx = x0 - 4 + c;
    float v = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(pb + ((int64_t)ch * H + gy) * W + gx);
    t[ch][r][c] = v;
  }
  __syncthreads();
  const int tx = tid & 7, ty = tid >> 3;
  const float a_s = bn_affine ? __ldg(bn_affine) : 1.f;
  const float a_t = bn_affine ? __ldg(bn_affine + 1) : 0.f;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
  for (int ch = 0; ch < 2; ++ch)
#pragma unroll 1
    for (int dy = 0; dy < KS; ++dy) {
      const float* rowp = &t[ch][ty + dy][4 * tx];
      const float4 v0 = *reinterpret_cast<const float4*>(rowp);
      const float4 v1 = *reinterpret_cast<const float4*>(rowp + 4);
      const float4 v2 = *reinterpret_cast<const float4*>(rowp + 8);
      const float seg[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
#pragma unroll
      for (int dx = 0; dx < KS; ++dx) {
        const float wv = wk[(ch * KS + dy) * KS + dx];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = fmaf(wv, seg[4 - R + j + dx], acc[j]);
      }
    }
  const int gy = y0 + ty, gx = x0 + 4 * tx;
  if (gy >= H || gx >= W) return;
  float4 g;
  g.x = sigmoidf_acc(fmaf(acc[0], a_s, a_t)); g.y = sigmoidf_acc(fmaf(acc[1], a_s, a_t));
  g.z = sigmoidf_acc(fmaf(acc[2], a_s, a_t)); g.w = sigmoidf_acc(fmaf(acc[3], a_s, a_t));
  const int cper = (C + csplit - 1) / csplit;
  const int c_lo = cs * cper, c_hi = min(C, c_lo + cper);
  const int64_t P = (int64_t)H * W;
  const float* xb = x + ((int64_t)b * C + c_lo) * P + (int64_t)gy * W + gx;      // W % 4 == 0 (host-checked): quads never straddle
  float* yb = y + (int64_t)b * y_bstride + (int64_t)c_lo * P + (int64_t)gy * W + gx;
  const float* scb = sc + (int64_t)b * C;
  int c = c_lo;
  for (; c + 8 <= c_hi; c += 8) {
    float4 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)u * P));
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float s = __ldg(scb + c + u);
      *reinterpret_cast<float4*>(yb + (int64_t)u * P) = make_float4((v[u].x * s) * g.x, (v[u].y * s) * g.y, (v[u].z * s) * g.z, (v[u].w * s) * g.w);
    }
    xb += 8 * P;
    yb += 8 * P;
  }
  for (; c < c_hi; ++c) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(xb));
    const float s = __ldg(scb + c);
    *reinterpret_cast<float4*>(yb) = make_float4((v.x * s) * g.x, (v.y * s) * g.y, (v.z * s) * g.z, (v.w * s) * g.w);
    xb += P;
    yb += P;
  }
}

}  // namespace smaat

using namespace smaat;

/* x: (N, H, W) planes -> avg (N), mx (N), pooled (N, H/2, W/2).  Needs W % 4 == 0, H % 2 == 0 and 16-byte aligned x,
 * 8-byte aligned pooled; SMAAT_E_UNSUPPORTED otherwise (run smaat_cbam_pool_fwd and smaat_maxpool2_fwd). */
extern "C" int smaat_cbam_pool_maxpool_fwd(const float* x, float* avg, float* mx, float* pooled, int64_t N, int H, int W,
                                           void* stream) {
  SMAAT_REQUIRE(x && avg && mx && pooled && N > 0 && H > 0 && W > 0, "cbam_pool_maxpool: bad arguments");
  if (W % 4 != 0 || H % 2 != 0 || !aligned16(x) || (reinterpret_cast<uintptr_t>(pooled) & 7u))
    return fail(SMAAT_E_UNSUPPORTED, "cbam_pool_maxpool: needs W %% 4 == 0, even H and aligned pointers (H=%d W=%d)", H, W);
  cudaStream_t st = (cudaStream_t)stream;
  if ((int64_t)H * W >= 2048) {
    SMAAT_REQUIRE(N < (1ll << 31), "cbam_pool_maxpool: too many planes");
    cbam_pool_maxpool_kernel<256><<<(unsigned)N, 256, 0, st>>>(x, avg, mx, pooled, N, H, W, MlpTail{});
  } else {
    cbam_pool_maxpool_kernel<32><<<(unsigned)ceil_div64(N, 8), 256, 0, st>>>(x, avg, mx, pooled, N, H, W, MlpTail{});
  }
  SMAAT_LAUNCH_CHECK("smaat_cbam_pool_maxpool_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_cbam_pool_fwd(const float* x, float* avg, float* mx, int64_t N, int P, void* stream) {
  SMAAT_REQUIRE(x && avg && mx && N > 0 && P > 0, "cbam_pool: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = (P % 4 == 0) && aligned16(x);
  if (P >= 2048) {
    SMAAT_REQUIRE(N < (1ll << 31), "cbam_pool: too many planes");
    if (vec) cbam_pool_kernel<256, true><<<(unsigned)N, 256, 0, st>>>(x, avg, mx, N, P, MlpTail{});
    else cbam_pool_kernel<256, false><<<(unsigned)N, 256, 0, st>>>(x, avg, mx, N, P, MlpTail{});
  } else {
    const unsigned grid = (unsigned)ceil_div64(N, 8);
    if (vec) cbam_pool_kernel<32, true><<<grid, 256, 0, st>>>(x, avg, mx, N, P, MlpTail{});
    else cbam_pool_kernel<32, false><<<grid, 256, 0, st>>>(x, avg, mx, N, P, MlpTail{});
  }
  SMAAT_LAUNCH_CHECK("smaat_cbam_pool_fwd");
  return SMAAT_OK;
}

/* ChannelAttention's pools AND its shared MLP + sigmoid in one launch (layers.py:98-109): x (B, C, H, W) -> avg, mx (B, C),
 * sc (B, C) = sigmoid(MLP(avg) + MLP(max)); pooled (B, C, H/2, W/2) = MaxPool2d(2)(x) when non-NULL (needs even H).  The MLP
 * is run by the last pooling CTA of each image; `counters`: B ints, zero on entry, zero again on exit.  Needs C % 8 == 0,
 * C <= 512, hidden <= 64; pooled additionally W % 4 == 0: SMAAT_E_UNSUPPORTED otherwise (use the separate entry points). */
extern "C" int smaat_cbam_pool_mlp_fwd(const float* x, float* avg, float* mx, float* pooled, const float* w1, const float* b1,
                                       const float* w2, const float* b2, float* sc, int* counters, int B, int C, int H, int W,
                                       int hidden, void* stream) {
  SMAAT_REQUIRE(x && avg && mx && w1 && b1 && w2 && b2 && sc && counters && B > 0 && C > 0 && H > 0 && W > 0 && hidden > 0,
                "cbam_pool_mlp: bad arguments");
  if (C % 8 != 0 || C > 512 || hidden > 64) return fail(SMAAT_E_UNSUPPORTED, "cbam_pool_mlp: needs C %% 8 == 0, C <= 512, hidden <= 64");
  if (pooled && (W % 4 != 0 || H % 2 != 0 || !aligned16(x) || (reinterpret_cast<uintptr_t>(pooled) & 7u)))
    return fail(SMAAT_E_UNSUPPORTED, "cbam_pool_mlp: the fused max-pool needs W %% 4 == 0, even H and aligned pointers (H=%d W=%d)", H, W);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t N = (int64_t)B * C;
  const int P = H * W;
  SMAAT_REQUIRE(N < (1ll << 31), "cbam_pool_mlp: too many planes");
  MlpTail t{w1, b1, w2, b2, sc, counters, C, hidden};
  if (pooled) {
    if (P >= 2048) cbam_pool_maxpool_kernel<256><<<(unsigned)N, 256, 0, st>>>(x, avg, mx, pooled, N, H, W, t);
    else cbam_pool_maxpool_kernel<32><<<(unsigned)ceil_div64(N, 8), 256, 0, st>>>(x, avg, mx, pooled, N, H, W, t);
  } else {
    const bool vec = (P % 4 == 0) && aligned16(x);
    if (P >= 2048) {
      if (vec) cbam_pool_kernel<256, true><<<(unsigned)N, 256, 0, st>>>(x, avg, mx, N, P, t);
      else cbam_pool_kernel<256, false><<<(unsigned)N, 256, 0, st>>>(x, avg, mx, N, P, t);
    } else {
      const unsigned grid = (unsigned)ceil_div64(N, 8);
      if (vec) cbam_pool_kernel<32, true><<<grid, 256, 0, st>>>(x, avg, mx, N, P, t);
      else cbam_pool_kernel<32, false><<<grid, 256, 0, st>>>(x, avg, mx, N, P, t);
    }
  }
  SMAAT_LAUNCH_CHECK("smaat_cbam_pool_mlp_fwd");
  return SMAAT_OK;
}

/* ChannelAttention's pools finished from the partial sums / maxima smaat_dsconv_cbam_fwd wrote for the map x (B, C, H, W), and its
 * shared MLP + sigmoid (layers.py:98-109): avg, mx, sc (B, C).  psum / pmax: (B, npart, C).  counters as smaat_cbam_pool_mlp_fwd.
 * Needs C % 16 == 0, C <= 512, hidden <= 64 and 16-byte aligned psum / pmax: SMAAT_E_UNSUPPORTED otherwise. */
extern "C" int smaat_cbam_mlp_partials_fwd(const float* psum, const float* pmax, int npart, float* avg, float* mx, const float* w1,
                                           const float* b1, const float* w2, const float* b2, float* sc, int* counters, int B, int C,
                                           int H, int W, int hidden, void* stream) {
  SMAAT_REQUIRE(psum && pmax && avg && mx && w1 && b1 && w2 && b2 && sc && counters && npart > 0 && B > 0 && C > 0 && H > 0 && W > 0 &&
                    hidden > 0,
                "cbam_mlp_partials: bad arguments");
  SMAAT_REQUIRE(B <= 65535, "cbam_mlp_partials: batch too large for grid.y");
  if (C % MP_CB != 0 || C > 512 || hidden > 64 || !aligned16(psum) || !aligned16(pmax))
    return fail(SMAAT_E_UNSUPPORTED, "cbam_mlp_partials: needs C %% %d == 0, C <= 512, hidden <= 64, aligned partials", MP_CB);
  MlpTail t{w1, b1, w2, b2, sc, counters, C, hidden};
  cbam_mlp_partials_kernel<<<dim3(C / MP_CB, B), 256, 0, (cudaStream_t)stream>>>(psum, pmax, npart, avg, mx, H * W, t);
  SMAAT_LAUNCH_CHECK("smaat_cbam_mlp_partials_fwd");
  return SMAAT_OK;
}

/* SpatialAttention's conv k x k (2 -> 1) + BatchNorm2d(1) affine + sigmoid AND the final scaling in one launch
 * (layers.py:126-128 + :110): y = (x * sc[b, c]) * sigmoid(bn(conv(pooled))).  pooled: (B, 2, H, W) from smaat_cbam_reduce_fwd,
 * bn_affine: device [scale, shift] or NULL.  Needs W % 4 == 0 and 16-byte aligned x / y: SMAAT_E_UNSUPPORTED otherwise
 * (use smaat_cbam_gate_fwd + smaat_cbam_scale_fwd). */
extern "C" int smaat_cbam_gate_scale_fwd(const float* pooled, const float* wsp, const float* bn_affine, const float* x, const float* sc,
                                         float* y, int64_t y_bstride, int B, int C, int H, int W, int ks, void* stream) {
  SMAAT_REQUIRE(pooled && wsp && x && sc && y && B > 0 && C > 0 && H > 0 && W > 0, "cbam_gate_scale: bad arguments");
  SMAAT_REQUIRE(ks == 3 || ks == 7, "cbam_gate_scale: kernel size must be 3 or 7 (layers.py:117), got %d", ks);
  SMAAT_REQUIRE(y_bstride >= (int64_t)C * H * W, "cbam_gate_scale: y batch stride too small");
  if (W % 4 != 0 || !aligned16(x) || !aligned16(y) || y_bstride % 4 != 0)
    return fail(SMAAT_E_UNSUPPORTED, "cbam_gate_scale: needs W %% 4 == 0 and 16-byte aligned x / y");
  const int tiles = ceil_div(W, GT_W) * ceil_div(H, GT_H);
  // channel slices so that small planes still fill the machine (~4 CTAs per SM), at least 8 channels per slice
  int csplit = ceil_div(4 * num_sms(), tiles * B);
  if (csplit < 1) csplit = 1;
  if (csplit > ceil_div(C, 8)) csplit = ceil_div(C, 8);
  SMAAT_REQUIRE((int64_t)B * csplit <= 65535, "cbam_gate_scale: grid.z too large");
  dim3 grid(ceil_div(W, GT_W), ceil_div(H, GT_H), B * csplit);
  if (ks == 7) cbam_gate_scale_kernel<7><<<grid, 256, 0, (cudaStream_t)stream>>>(pooled, wsp, bn_affine, x, sc, y, y_bstride, C, H, W, csplit);
  else cbam_gate_scale_kernel<3><<<grid, 256, 0, (cudaStream_t)stream>>>(pooled, wsp, bn_affine, x, sc, y, y_bstride, C, H, W, csplit);
  SMAAT_LAUNCH_CHECK("smaat_cbam_gate_scale_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_cbam_mlp_fwd(const float* avg, const float* mx, const float* w1, const float* b1, const float* w2,
                                  const float* b2, float* sc, int B, int C, int hidden, void* stream) {
  SMAAT_REQUIRE(avg && mx && w1 && b1 && w2 && b2 && sc && B > 0 && C > 0 && hidden > 0, "cbam_mlp: bad arguments (hidden=%d)",
                hidden);
  const size_t smem = (size_t)(2 * C + 2 * hidden) * sizeof(float);
  SMAAT_REQUIRE(smem <= 48 * 1024, "cbam_mlp: C=%d too large", C);
  cbam_mlp_kernel<<<B, 256, smem, (cudaStream_t)stream>>>(avg, mx, w1, b1, w2, b2, sc, C, hidden);
  SMAAT_LAUNCH_CHECK("smaat_cbam_mlp_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_cbam_reduce_fwd(const float* x, const float* sc, float* pooled, int B, int C, int P, void* stream) {
  SMAAT_REQUIRE(x && sc && pooled && B > 0 && C > 0 && P > 0, "cbam_reduce: bad arguments");
  SMAAT_REQUIRE(B <= 65535, "cbam_reduce: batch too large for grid.y");
  const bool vec = (P % 4 == 0) && aligned16(x) && aligned16(pooled);
  if (vec && P >= 8192 && (size_t)C * sizeof(float) <= 48 * 1024) {
    cbam_reduce_v4_kernel<float><<<dim3(ceil_div(P / 4, 256), B), 256, (size_t)C * sizeof(float), (cudaStream_t)stream>>>(x, sc, pooled, C,
                                                                                                              P / 4);
    SMAAT_LAUNCH_CHECK("smaat_cbam_reduce_fwd");
    return SMAAT_OK;
  }
  dim3 grid(ceil_div(P, 128), B), block(32, 8);
  if (vec) cbam_reduce_kernel<true><<<grid, block, 0, (cudaStream_t)stream>>>(x, sc, pooled, C, P);
  else cbam_reduce_kernel<false><<<grid, block, 0, (cudaStream_t)stream>>>(x, sc, pooled, C, P);
  SMAAT_LAUNCH_CHECK("smaat_cbam_reduce_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_cbam_gate_fwd(const float* pooled, const float* wsp, const float* bn_affine, float* sa, float* raw, int B,
                                   int H, int W, int ks, void* stream) {
  SMAAT_REQUIRE(pooled && wsp && sa && B > 0 && H > 0 && W > 0, "cbam_gate: bad arguments");
  SMAAT_REQUIRE(ks == 3 || ks == 7, "cbam_gate: kernel size must be 3 or 7 (layers.py:117), got %d", ks);
  SMAAT_REQUIRE(B <= 65535, "cbam_gate: batch too large for grid.z");
  dim3 grid(ceil_div(W, GT_W), ceil_div(H, GT_H), B);
  if (ks == 7) cbam_gate_kernel<7><<<grid, 256, 0, (cudaStream_t)stream>>>(pooled, wsp, bn_affine, sa, raw, H, W);
  else cbam_gate_kernel<3><<<grid, 256, 0, (cudaStream_t)stream>>>(pooled, wsp, bn_affine, sa, raw, H, W);
  SMAAT_LAUNCH_CHECK("smaat_cbam_gate_fwd");
  return SMAAT_OK;
}

extern "C" int smaat_cbam_scale_fwd(const float* x, const float* sc, const float* sa, float* y, int64_t y_bstride, int B, int C,
                                    int P, void* stream) {
  SMAAT_REQUIRE(x && sc && sa && y && B > 0 && C > 0 && P > 0, "cbam_scale: bad arguments");
  SMAAT_REQUIRE(y_bstride >= (int64_t)C * P, "cbam_scale: y batch stride too small");
  SMAAT_REQUIRE(B <= 65535 && ceil_div(C, SC_CH) <= 65535, "cbam_scale: grid too large");
  const bool vec = (P % 4 == 0) && aligned16(x) && aligned16(y) && aligned16(sa) && (y_bstride % 4 == 0);
  const int threads = 128;
  dim3 grid(ceil_div(ceil_div(P, 4), threads), ceil_div(C, SC_CH), B);
  if (vec) cbam_scale_kernel<true><<<grid, threads, 0, (cudaStream_t)stream>>>(x, sc, sa, y, y_bstride, C, P);
  else cbam_scale_kernel<false><<<grid, threads, 0, (cudaStream_t)stream>>>(x, sc, sa, y, y_bstride, C, P);
  SMAAT_LAUNCH_CHECK("smaat_cbam_scale_fwd");
  return SMAAT_OK;
}

/* ---- bf16 input: the serving forward's bf16 route ----------------------------------------------------------------------------
 * x is bf16 (raw uint16_t bits); the pools, the MLP, the gates and the channel reduce run and are stored in fp32.  The 2x2 max-pool
 * is written in the storage type of the level it feeds: bf16 (pooled_bf16 = 1) or fp32. */
template <typename TO>
static int cbam_pool_maxpool_bf16_launch(const uint16_t* x, float* avg, float* mx, void* pooled, int64_t N, int H, int W,
                                         const MlpTail& t, cudaStream_t st) {
  TO* po = static_cast<TO*>(pooled);
  if ((int64_t)H * W >= 2048) {
    SMAAT_REQUIRE(N < (1ll << 31), "cbam_pool_maxpool_bf16: too many planes");
    cbam_pool_maxpool_kernel<256, uint16_t, TO><<<(unsigned)N, 256, 0, st>>>(x, avg, mx, po, N, H, W, t);
  } else {
    cbam_pool_maxpool_kernel<32, uint16_t, TO><<<(unsigned)ceil_div64(N, 8), 256, 0, st>>>(x, avg, mx, po, N, H, W, t);
  }
  return SMAAT_OK;
}

static int cbam_pool_maxpool_bf16_check(const void* x, void* pooled, int pooled_bf16, int H, int W) {
  // 4 bf16 columns of a row are one 8-byte load; the two pooled values one 4-byte (bf16) or 8-byte (fp32) store
  if (W % 4 != 0 || H % 2 != 0 || (reinterpret_cast<uintptr_t>(x) & 7u) ||
      (reinterpret_cast<uintptr_t>(pooled) & (pooled_bf16 ? 3u : 7u)))
    return fail(SMAAT_E_UNSUPPORTED, "cbam_pool_maxpool_bf16: needs W %% 4 == 0, even H and aligned pointers (H=%d W=%d)", H, W);
  return SMAAT_OK;
}

extern "C" int smaat_cbam_pool_maxpool_bf16_fwd(const void* x, float* avg, float* mx, void* pooled, int pooled_bf16, int64_t N, int H,
                                                int W, void* stream) {
  SMAAT_REQUIRE(x && avg && mx && pooled && N > 0 && H > 0 && W > 0, "cbam_pool_maxpool_bf16: bad arguments");
  if (int r = cbam_pool_maxpool_bf16_check(x, pooled, pooled_bf16, H, W)) return r;
  const uint16_t* xb = static_cast<const uint16_t*>(x);
  cudaStream_t st = (cudaStream_t)stream;
  int r = pooled_bf16 ? cbam_pool_maxpool_bf16_launch<uint16_t>(xb, avg, mx, pooled, N, H, W, MlpTail{}, st)
                      : cbam_pool_maxpool_bf16_launch<float>(xb, avg, mx, pooled, N, H, W, MlpTail{}, st);
  if (r) return r;
  SMAAT_LAUNCH_CHECK("smaat_cbam_pool_maxpool_bf16_fwd");
  return SMAAT_OK;
}

/* smaat_cbam_pool_mlp_fwd with the max-pool (required here) from a bf16 x. */
extern "C" int smaat_cbam_pool_mlp_bf16_fwd(const void* x, float* avg, float* mx, void* pooled, int pooled_bf16, const float* w1,
                                            const float* b1, const float* w2, const float* b2, float* sc, int* counters, int B, int C,
                                            int H, int W, int hidden, void* stream) {
  SMAAT_REQUIRE(x && avg && mx && pooled && w1 && b1 && w2 && b2 && sc && counters && B > 0 && C > 0 && H > 0 && W > 0 && hidden > 0,
                "cbam_pool_mlp_bf16: bad arguments");
  if (C % 8 != 0 || C > 512 || hidden > 64)
    return fail(SMAAT_E_UNSUPPORTED, "cbam_pool_mlp_bf16: needs C %% 8 == 0, C <= 512, hidden <= 64");
  if (int r = cbam_pool_maxpool_bf16_check(x, pooled, pooled_bf16, H, W)) return r;
  MlpTail t{w1, b1, w2, b2, sc, counters, C, hidden};
  const uint16_t* xb = static_cast<const uint16_t*>(x);
  const int64_t N = (int64_t)B * C;
  cudaStream_t st = (cudaStream_t)stream;
  int r = pooled_bf16 ? cbam_pool_maxpool_bf16_launch<uint16_t>(xb, avg, mx, pooled, N, H, W, t, st)
                      : cbam_pool_maxpool_bf16_launch<float>(xb, avg, mx, pooled, N, H, W, t, st);
  if (r) return r;
  SMAAT_LAUNCH_CHECK("smaat_cbam_pool_mlp_bf16_fwd");
  return SMAAT_OK;
}

/* smaat_cbam_reduce_fwd from a bf16 x: pooled (B, 2, H, W) fp32. */
extern "C" int smaat_cbam_reduce_bf16_fwd(const void* x, const float* sc, float* pooled, int B, int C, int P, void* stream) {
  SMAAT_REQUIRE(x && sc && pooled && B > 0 && C > 0 && P > 0, "cbam_reduce_bf16: bad arguments");
  SMAAT_REQUIRE(B <= 65535, "cbam_reduce_bf16: batch too large for grid.y");
  const uint16_t* xb = static_cast<const uint16_t*>(x);
  const bool vec = (P % 4 == 0) && (reinterpret_cast<uintptr_t>(x) & 7u) == 0 && aligned16(pooled);
  if (vec && P >= 8192 && (size_t)C * sizeof(float) <= 48 * 1024) {
    cbam_reduce_v4_kernel<uint16_t><<<dim3(ceil_div(P / 4, 256), B), 256, (size_t)C * sizeof(float), (cudaStream_t)stream>>>(
        xb, sc, pooled, C, P / 4);
  } else {
    dim3 grid(ceil_div(P, 128), B), block(32, 8);
    if (vec) cbam_reduce_kernel<true, uint16_t><<<grid, block, 0, (cudaStream_t)stream>>>(xb, sc, pooled, C, P);
    else cbam_reduce_kernel<false, uint16_t><<<grid, block, 0, (cudaStream_t)stream>>>(xb, sc, pooled, C, P);
  }
  SMAAT_LAUNCH_CHECK("smaat_cbam_reduce_bf16_fwd");
  return SMAAT_OK;
}
