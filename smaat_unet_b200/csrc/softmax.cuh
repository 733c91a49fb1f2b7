// softmax.cuh -- the per-pixel channel softmax of smaat_softmax_channels_fwd (csrc/ce_metrics.cu) and of the probability
// epilogue of smaat_dsconv_probs_fwd (csrc/dsconv_fused.cu).  Both routes feed a pixel's logits through add() in class order
// and normalise each with prob(), so equal logits give bit-identical probabilities on either route.
#pragma once
#include <math.h>

namespace smaat {

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

}  // namespace smaat
