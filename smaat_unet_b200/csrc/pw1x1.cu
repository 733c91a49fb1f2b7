// pw1x1.cu -- C-ABI entry for the pointwise 1x1 conv: validates, then routes to the exact
// CUDA-core GEMM (pw1x1_simt.cu) or the wgmma tensor-core GEMM (pw1x1_tc.cu).
#include "common.cuh"

namespace smaat {
int pw1x1_simt_launch(const float* x, const float* w, const float* scale, const float* shift, float* y, int64_t y_bstride,
                      double* stats, int B, int K, int Cout, int P, int relu, cudaStream_t st);
int pw1x1_tc_launch(const float* x, const float* w, const float* w_lo, const float* scale, const float* shift, float* y,
                    int64_t y_bstride, double* stats, int B, int K, int Cout, int P, int relu, int mode, cudaStream_t st);
bool pw1x1_tc_eligible(const float* x, const float* w, const float* w_lo, int K, int Cout, int P);
}  // namespace smaat

using namespace smaat;

extern "C" int smaat_pw1x1_fwd(const float* x, const float* w, const float* w_lo, const float* scale, const float* shift,
                               float* y, int64_t y_bstride, double* stats, int B, int K, int Cout, int P, int relu, int mode,
                               void* stream) {
  SMAAT_REQUIRE(x && w && y, "pw1x1: null pointer");
  SMAAT_REQUIRE(B > 0 && K > 0 && Cout > 0 && P > 0, "pw1x1: bad shape B=%d K=%d Cout=%d P=%d", B, K, Cout, P);
  SMAAT_REQUIRE(y_bstride >= (int64_t)Cout * P, "pw1x1: y batch stride %lld < Cout*P", (long long)y_bstride);
  cudaStream_t st = (cudaStream_t)stream;
  switch (mode) {
    case SMAAT_PW_FP32_SIMT:
      return pw1x1_simt_launch(x, w, scale, shift, y, y_bstride, stats, B, K, Cout, P, relu, st);
    case SMAAT_PW_TF32:
      return pw1x1_tc_launch(x, w, nullptr, scale, shift, y, y_bstride, stats, B, K, Cout, P, relu, mode, st);
    case SMAAT_PW_TF32X3:
      return pw1x1_tc_launch(x, w, w_lo, scale, shift, y, y_bstride, stats, B, K, Cout, P, relu, mode, st);
    case SMAAT_PW_BF16:
      return pw1x1_tc_launch(x, w, nullptr, scale, shift, y, y_bstride, stats, B, K, Cout, P, relu, mode, st);
    default:
      return fail(SMAAT_E_BADARG, "pw1x1: unknown mode %d", mode);
  }
}

/* 1 if (x, w, K, Cout, P) can take the tensor-core path, else 0 (caller then uses SMAAT_PW_FP32_SIMT). */
extern "C" int smaat_pw1x1_tc_eligible(const float* x, const float* w, int K, int Cout, int P) {
  return pw1x1_tc_eligible(x, w, nullptr, K, Cout, P) ? 1 : 0;
}
