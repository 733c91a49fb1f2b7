// voc_augment.cu -- the VOC training input pipeline's per-sample random part and normalisation in one pass over uint8 data.
//
// Replaces, per sample, VOCSegmentation.apply_augmentations + ToTensor + Normalize + `target[target == 255] = 0`
// (reference utils/dataset_VOC.py:139-168): hflip, a +-10 degree NEAREST rotation of image and mask, a x1.2 / x0.8
// brightness blend of the image, v / 255, (v - mean) / std and the 255 -> 0 target map.  The random choices are drawn on the
// host (aug row per sample); the arithmetic reproduces PIL's bit for bit:
//   - Image.rotate(angle, NEAREST, expand=False, center=(w/2, h/2), fillcolor=0) builds a 6-coefficient affine matrix in
//     Python doubles (cos / sin rounded to 15 decimals) and hands it to ImagingTransformAffine, which walks each output row
//     with 16.16 fixed-point increments when the four corners map inside +-32768, and with double increments otherwise.
//     Both walks are restated exactly: the fixed-point one in closed form (integer sums are exact), the double one as the
//     same sequence of additions (rounding depends on the order), which only images wider or taller than ~32k ever take.
//   - ImageEnhance.Brightness blends with black: out = (uint8)(alpha * v) with alpha converted to fp32 and clamped to
//     [0, 255] when alpha > 1; the darkening factor is the reference's 1.2 - 0.4 in doubles, then fp32.
//   - ToTensor / Normalize: fp32 v / 255, then (v - mean) / std, each an IEEE-rounded fp32 operation.
// One thread per output pixel; reads 3 + 1 bytes (gathered through the rotation), writes 12 + 8.
#include <math.h>
#include <stdlib.h>

#include "common.cuh"

namespace smaat {

struct VocRotation {
  int fixed;                       // 1: 16.16 fixed-point walk, 0: double walk
  long long f0, f1, f2, f3, f4, f5;  // fixed-point coefficients (xx = f2 + y f1 + x f0, yy = f5 + y f4 + x f3)
  double a0, a1, a3, a4, xo, yo;   // double walk: row start (xo, yo) += (a1, a4) per row, += (a0, a3) per pixel
};

struct VocParams {
  VocRotation rot[2];              // [0]: TF.rotate(img, -10), [1]: TF.rotate(img, +10)
  float alpha[2];                  // [0]: brightness 1.2 - 0.4, [1]: 1.2 (as PIL's ImagingBlend takes them: fp32)
  float mean[3], std[3];
};

// Python's round(v, 15): the correctly rounded 15-decimal string, read back correctly rounded (glibc printf / strtod are
// exact, as CPython's dtoa is)
static double round15(double v) {
  char buf[64];
  snprintf(buf, sizeof(buf), "%.15f", v);
  return strtod(buf, nullptr);
}

// PIL's Image.rotate(deg, expand=False) matrix (Image.py) and ImagingTransformAffine's choice of walk (Geometry.c)
static void pil_rotation(double deg, int w, int h, VocRotation* r) {
  double angle = fmod(deg, 360.0);                 // Python's float %: the result takes the divisor's sign
  if (angle < 0.0) angle += 360.0;
  angle = -(angle * (M_PI / 180.0));               // -math.radians(angle)
  const double a = round15(cos(angle)), b = round15(sin(angle)), d = round15(-sin(angle)), e = round15(cos(angle));
  const double cx = w / 2.0, cy = h / 2.0;
  double c = a * -cx + b * -cy + 0.0;
  double f = d * -cx + e * -cy + 0.0;
  c += cx;
  f += cy;
  const double m[6] = {a, b, c, d, e, f};
  auto in_range = [&](int x, int y) {
    return fabs(x * m[0] + y * m[1] + m[2]) < 32768.0 && fabs(x * m[3] + y * m[4] + m[5]) < 32768.0;
  };
  r->fixed = in_range(0, 0) && in_range(w, h) && in_range(0, h) && in_range(w, 0);
  auto fix = [](double v) { return (long long)floor(v * 65536.0 + 0.5); };
  r->f0 = fix(m[0]);
  r->f1 = fix(m[1]);
  r->f3 = fix(m[3]);
  r->f4 = fix(m[4]);
  r->f2 = fix(m[2] + m[0] * 0.5 + m[1] * 0.5);
  r->f5 = fix(m[5] + m[3] * 0.5 + m[4] * 0.5);
  r->a0 = m[0];
  r->a1 = m[1];
  r->a3 = m[3];
  r->a4 = m[4];
  r->xo = m[2] + m[1] * 0.5 + m[0] * 0.5;
  r->yo = m[5] + m[4] * 0.5 + m[3] * 0.5;
}

__host__ __device__ __forceinline__ float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float sub_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ float div_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// PIL's COORD(v) of the double walk: -1 below zero, else truncation
__host__ __device__ __forceinline__ long long pil_coord(double v) { return v < 0.0 ? -1 : (long long)v; }

// source pixel of output (x, y) under the rotation; false where PIL leaves the fill
__host__ __device__ __forceinline__ bool rotate_source(const VocRotation& r, int x, int y, int W, int H, int& xs, int& ys) {
  long long xi, yi;
  if (r.fixed) {
    xi = (r.f2 + (long long)y * r.f1 + (long long)x * r.f0) >> 16;
    yi = (r.f5 + (long long)y * r.f4 + (long long)x * r.f3) >> 16;
  } else {
    double xo = r.xo, yo = r.yo;
    for (int i = 0; i < y; ++i) {
      xo = add_rn(xo, r.a1);
      yo = add_rn(yo, r.a4);
    }
    for (int i = 0; i < x; ++i) {
      xo = add_rn(xo, r.a0);
      yo = add_rn(yo, r.a3);
    }
    xi = pil_coord(xo);
    yi = pil_coord(yo);
  }
  xs = (int)xi;
  ys = (int)yi;
  return xi >= 0 && xi < W && yi >= 0 && yi < H;
}

// one output pixel of sample b: 3 normalised channels and the class index
__host__ __device__ __forceinline__ void voc_pixel(const VocParams& P, const uint8_t* __restrict__ xb, const uint8_t* __restrict__ yb,
                                                   int flip, int rot, int bright, int x, int y, int W, int H, float v[3],
                                                   int64_t& t) {
  int xs = x, ys = y;
  bool in = true;
  if (rot != 0) in = rotate_source(P.rot[rot > 0], x, y, W, H, xs, ys);
  if (flip) xs = W - 1 - xs;                       // the rotation reads the flipped image
  uint8_t u[3] = {0, 0, 0}, m = 0;
  if (in) {
    const int64_t s = (int64_t)ys * W + xs;
    u[0] = xb[3 * s];
    u[1] = xb[3 * s + 1];
    u[2] = xb[3 * s + 2];
    m = yb[s];
  }
  for (int c = 0; c < 3; ++c) {
    int q = u[c];
    if (bright != 0) {
      const float p = mul_rn(P.alpha[bright > 0], (float)q);
      q = p >= 255.f ? 255 : (int)p;               // the blend clamps above only when extrapolating (alpha > 1)
    }
    v[c] = div_rn(sub_rn(div_rn((float)q, 255.f), P.mean[c]), P.std[c]);
  }
  t = m == 255 ? 0 : (int64_t)m;
}

__global__ void __launch_bounds__(256) voc_augment_kernel(const uint8_t* __restrict__ x_u8, const uint8_t* __restrict__ y_u8,
                                                          const int8_t* __restrict__ aug, const VocParams P, float* __restrict__ out_x,
                                                          int64_t x_bstride, int64_t* __restrict__ out_y, int64_t y_bstride,
                                                          int B, int H, int W) {
  const int64_t HW = (int64_t)H * W, n = (int64_t)B * HW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / HW);
    const int64_t p = i - (int64_t)b * HW;
    const int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
    int flip = 0, rot = 0, bright = 0;
    if (aug) {
      flip = aug[3 * b];
      rot = aug[3 * b + 1];
      bright = aug[3 * b + 2];
    }
    float v[3];
    int64_t t;
    voc_pixel(P, x_u8 + (int64_t)b * HW * 3, y_u8 + (int64_t)b * HW, flip, rot, bright, x, y, W, H, v, t);
    float* o = out_x + (int64_t)b * x_bstride + p;
    o[0] = v[0];
    o[HW] = v[1];
    o[2 * HW] = v[2];
    out_y[(int64_t)b * y_bstride + p] = t;
  }
}

int voc_params(const float* mean, const float* std, int H, int W, VocParams* P) {
  SMAAT_REQUIRE(mean && std, "voc_augment: mean and std are required (host float[3] each)");
  pil_rotation(-10.0, W, H, &P->rot[0]);
  pil_rotation(10.0, W, H, &P->rot[1]);
  P->alpha[0] = (float)(1.2 - 0.4);
  P->alpha[1] = (float)1.2;
  for (int c = 0; c < 3; ++c) {
    P->mean[c] = mean[c];
    P->std[c] = std[c];
  }
  return SMAAT_OK;
}

}  // namespace smaat

using namespace smaat;

extern "C" int smaat_voc_augment_fwd(const uint8_t* x_u8, const uint8_t* y_u8, const int8_t* aug, const float* mean,
                                     const float* std, float* x, int64_t x_bstride, int64_t* y, int64_t y_bstride, int B, int H,
                                     int W, void* stream) {
  SMAAT_REQUIRE(x_u8 && y_u8 && x && y && B >= 1 && H >= 1 && W >= 1, "voc_augment: bad arguments (B=%d H=%d W=%d)", B, H, W);
  const int64_t HW = (int64_t)H * W;
  SMAAT_REQUIRE(x_bstride >= 3 * HW && y_bstride >= HW, "voc_augment: batch strides (%lld, %lld) below (3*H*W, H*W) = (%lld, %lld)",
                (long long)x_bstride, (long long)y_bstride, (long long)(3 * HW), (long long)HW);
  VocParams P;
  const int rc = voc_params(mean, std, H, W, &P);
  if (rc != SMAAT_OK) return rc;
  int64_t blocks = ceil_div64((int64_t)B * HW, 256);
  const int64_t cap = (int64_t)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  voc_augment_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x_u8, y_u8, aug, P, x, x_bstride, y, y_bstride, B, H, W);
  SMAAT_LAUNCH_CHECK("smaat_voc_augment_fwd");
  return SMAAT_OK;
}
