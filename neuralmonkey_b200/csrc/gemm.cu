// nm_gemm: dense projections.  Dispatches between the wgmma/TMA kernel
// (gemm_tc.cu) and the fp32 CUDA-core tile (gemm_simt.cuh).
#include "gemm_simt.cuh"
#include "gemm_tc.h"

namespace nm {

struct DenseEpi {
  float* C;
  int64_t ldc;
  const float* bias;
  int act;
  float beta;
  __device__ void operator()(int64_t m, int64_t n, float acc) const {
    float x = acc + (bias ? bias[n] : 0.f);
    x = apply_act(x, act);
    float* c = C + m * ldc + n;
    *c = (beta != 0.f) ? (x + beta * *c) : x;
  }
};

}  // namespace nm

using namespace nm;

extern "C" {

int nm_gemm_uses_tc(int transA, int transB, int64_t M, int64_t N, int64_t K, int64_t lda,
                    int64_t ldb, int64_t ldc) {
  return tc_gemm_supported(M, N, K, lda, ldb, nullptr, nullptr) ? 1 : 0;
}

int nm_gemm_tc_plan(int64_t M, int64_t N, int64_t K, int act, int sms, int* bn, int* splits, int* kb_per_split) {
  NM_REQUIRE(bn && splits && kb_per_split, NM_E_INVALID, "nm_gemm_tc_plan: null output");
  NM_REQUIRE(M >= 1 && N >= 1 && K >= 1 && M <= 0x7fffffffLL && N <= 0x7fffffffLL && K <= 0x7fffffffLL,
             NM_E_INVALID, "nm_gemm_tc_plan: bad shape %lld x %lld x %lld", (long long)M, (long long)N,
             (long long)K);
  NM_REQUIRE(act >= NM_ACT_NONE && act <= NM_ACT_SIGMOID, NM_E_INVALID, "nm_gemm_tc_plan: unknown act %d", act);
  const TcPlan p = tc_dense_plan(M, N, K, act, sms > 0 ? sms : sm_count());
  *bn = p.bn;
  *splits = p.splits;
  *kb_per_split = p.kb_per;
  return NM_OK;
}

int nm_gemm(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda,
            const float* B, int64_t ldb, float* C, int64_t ldc, const float* bias, int act,
            float beta, int backend, void* stream) {
  NM_REQUIRE(A && B && C, NM_E_INVALID, "nm_gemm: null pointer");
  NM_REQUIRE(M >= 0 && N >= 0 && K >= 0, NM_E_INVALID, "nm_gemm: negative size");
  NM_REQUIRE(lda >= (transA ? M : K) && ldb >= (transB ? K : N) && ldc >= N, NM_E_INVALID,
             "nm_gemm: leading dimension too small (lda=%lld ldb=%lld ldc=%lld)", (long long)lda,
             (long long)ldb, (long long)ldc);
  NM_REQUIRE(beta == 0.f || beta == 1.f, NM_E_UNSUPPORTED, "nm_gemm: beta must be 0 or 1");
  NM_REQUIRE(act >= NM_ACT_NONE && act <= NM_ACT_SIGMOID, NM_E_INVALID, "nm_gemm: unknown act %d", act);
  NM_REQUIRE(backend >= NM_GEMM_AUTO && backend <= NM_GEMM_TC, NM_E_INVALID, "nm_gemm: bad backend");
  if (M == 0 || N == 0) return NM_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const bool tc_ok = K > 0 && tc_gemm_supported(M, N, K, lda, ldb, A, B);
  if (backend == NM_GEMM_TC)
    NM_REQUIRE(tc_ok, NM_E_UNSUPPORTED,
               "nm_gemm: shape not addressable by TMA (needs 16-byte aligned rows/pointers)");
  if (tc_ok && backend != NM_GEMM_SIMT) {
    TcEpilogue epi{};
    epi.mode = TC_EPI_DENSE;
    epi.C = C;
    epi.ldc = ldc;
    epi.bias = bias;
    epi.act = act;
    epi.beta = beta;
    return tc_gemm_launch(transA, transB, M, N, K, A, lda, B, ldb, epi, s);
  }
  DenseEpi epi{C, ldc, bias, act, beta};
  const int64_t sAm = transA ? 1 : lda, sAk = transA ? lda : 1;
  const int64_t sBk = transB ? 1 : ldb, sBn = transB ? ldb : 1;
  simt_gemm_launch(A, sAm, sAk, B, sBk, sBn, M, N, K, epi, s);
  NM_LAUNCH_CHECK("nm_gemm(simt)");
  return NM_OK;
}

}  // extern "C"
