// K5/K6 fused on the tensor cores: vocabulary projection + softmax cross-entropy
// statistics without a second pass over fp32 logits
// (decoders/autoregressive.py:288-316,446-459 of the reference).
#include "common.cuh"
#include "gemm_tc.h"

namespace nm {

// One warp per row: merge the per-N-tile (max, sumexp, argmax, target) partials.
__global__ void xent_combine_kernel(const float4* __restrict__ part, int64_t M, int64_t tiles_n,
                                    const int64_t* __restrict__ targets,
                                    const float* __restrict__ weights, float* __restrict__ lse,
                                    float* __restrict__ xent, int64_t* __restrict__ argmax) {
  const int lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  float mx = -INFINITY, tgt = -INFINITY;
  int32_t arg = 0x7fffffff;
  for (int64_t t = lane; t < tiles_n; t += 32) {
    const float4 p = part[row * tiles_n + t];
    const int32_t a = __float_as_int(p.z);
    if (p.x > mx || (p.x == mx && a < arg)) { mx = p.x; arg = a; }
    tgt = fmaxf(tgt, p.w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float omx = __shfl_xor_sync(0xffffffffu, mx, o);
    const int32_t oarg = __shfl_xor_sync(0xffffffffu, arg, o);
    if (omx > mx || (omx == mx && oarg < arg)) { mx = omx; arg = oarg; }
    tgt = fmaxf(tgt, __shfl_xor_sync(0xffffffffu, tgt, o));
  }
  float s = 0.f;
  for (int64_t t = lane; t < tiles_n; t += 32) {
    const float4 p = part[row * tiles_n + t];
    s += p.y * expf(p.x - mx);
  }
  s = warp_sum(s);
  if (lane == 0) {
    const float l = mx + logf(s);
    lse[row] = l;
    if (argmax) argmax[row] = (int64_t)arg;
    if (targets && xent) xent[row] = (l - tgt) * (weights ? weights[row] : 1.f);
  }
}

}  // namespace nm

using namespace nm;

extern "C" {

int64_t nm_logits_xent_scratch(int64_t M, int64_t V) {
  if (M <= 0 || V <= 0) return 0;
  return M * ceil_div(V, TC_XENT_BN) * 2 * 4;  // two epilogue halves per (row, n-tile)
}

int nm_logits_xent_fwd(const float* X, int64_t ldx, const float* W, int64_t ldw, int transW,
                       const float* b, int64_t unk_index, const int64_t* targets, const float* weights, float* lse,
                       float* xent, int64_t* argmax, float* part, float* logits_out, int64_t ldl,
                       int64_t M, int64_t V, int64_t K, void* stream) {
  NM_REQUIRE(X && W && lse && part, NM_E_INVALID, "nm_logits_xent_fwd: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= (transW ? K : V), NM_E_INVALID,
             "nm_logits_xent_fwd: bad sizes");
  NM_REQUIRE(!logits_out || ldl >= V, NM_E_INVALID, "nm_logits_xent_fwd: ldl < V");
  NM_REQUIRE((reinterpret_cast<uintptr_t>(part) & 15) == 0, NM_E_INVALID,
             "nm_logits_xent_fwd: part must be 16-byte aligned");
  NM_REQUIRE(tc_gemm_supported(M, V, K, ldx, ldw, X, W), NM_E_UNSUPPORTED,
             "nm_logits_xent_fwd: operands not TMA-addressable (use nm_gemm + nm_xent_fwd)");
  cudaStream_t s = (cudaStream_t)stream;
  TcEpilogue epi{};
  epi.mode = TC_EPI_XENT_FWD;
  epi.C = logits_out;
  epi.ldc = ldl;
  epi.bias = b;
  epi.unk_index = unk_index;
  epi.targets = targets;
  epi.part = reinterpret_cast<float4*>(part);
  const int rc = tc_gemm_launch(0, transW, M, V, K, X, ldx, W, ldw, epi, s);
  if (rc) return rc;
  const int64_t tiles_n = 2 * ceil_div(V, TC_XENT_BN);  // partials per row
  xent_combine_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, s>>>(reinterpret_cast<const float4*>(part), M,
                                                              tiles_n, targets, weights, lse, xent,
                                                              argmax);
  NM_LAUNCH_CHECK("nm_logits_xent_fwd(combine)");
  return NM_OK;
}

int nm_logits_xent_bwd(const float* X, int64_t ldx, const float* W, int64_t ldw, int transW,
                       const float* b, int64_t unk_index, const int64_t* targets, const float* weights,
                       const float* lse, const float* scale, float* dlogits, int64_t ldd, int64_t M,
                       int64_t V, int64_t K, void* stream) {
  NM_REQUIRE(X && W && targets && lse && scale && dlogits, NM_E_INVALID,
             "nm_logits_xent_bwd: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= (transW ? K : V) && ldd >= V, NM_E_INVALID,
             "nm_logits_xent_bwd: bad sizes");
  NM_REQUIRE(tc_gemm_supported(M, V, K, ldx, ldw, X, W), NM_E_UNSUPPORTED,
             "nm_logits_xent_bwd: operands not TMA-addressable (use nm_gemm + nm_xent_bwd)");
  TcEpilogue epi{};
  epi.mode = TC_EPI_XENT_BWD;
  epi.C = dlogits;
  epi.ldc = ldd;
  epi.bias = b;
  epi.unk_index = unk_index;
  epi.targets = targets;
  epi.weights = weights;
  epi.lse = lse;
  epi.scale = scale;
  return tc_gemm_launch(0, transW, M, V, K, X, ldx, W, ldw, epi, (cudaStream_t)stream);
}

// fp16 operands (X16 [M,K], WT16 [V,K], both K-major): see xent16.cu
int nm_logits_xent_fwd16(const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                         int64_t unk_index, const int64_t* targets, const float* weights, float* lse,
                         float* xent, int64_t* argmax, float* part, float* logits_out, int64_t ldl,
                         int64_t M, int64_t V, int64_t K, void* stream) {
  NM_REQUIRE(X16 && WT16 && lse && part, NM_E_INVALID, "nm_logits_xent_fwd16: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= K, NM_E_INVALID, "nm_logits_xent_fwd16: bad sizes");
  NM_REQUIRE(!logits_out || ldl >= V, NM_E_INVALID, "nm_logits_xent_fwd16: ldl < V");
  NM_REQUIRE((reinterpret_cast<uintptr_t>(part) & 15) == 0, NM_E_INVALID,
             "nm_logits_xent_fwd16: part must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if (K <= XENT16_MAX_K) {
    rc = xent16_launch(false, X16, ldx, WT16, ldw, b, unk_index, targets, nullptr, nullptr,
                       reinterpret_cast<float4*>(part), logits_out, ldl, nullptr, 0, M, V, K, s);
  } else {
    TcEpilogue epi{};
    epi.mode = TC_EPI_XENT_FWD;
    epi.C = logits_out;
    epi.ldc = ldl;
    epi.bias = b;
    epi.unk_index = unk_index;
    epi.targets = targets;
    epi.part = reinterpret_cast<float4*>(part);
    rc = tc_gemm16_launch(M, V, K, X16, ldx, WT16, ldw, epi, TcExt{}, s);
  }
  if (rc) return rc;
  const int64_t tiles_n = 2 * ceil_div(V, TC_XENT_BN);
  xent_combine_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, s>>>(reinterpret_cast<const float4*>(part), M,
                                                              tiles_n, targets, weights, lse, xent, argmax);
  NM_LAUNCH_CHECK("nm_logits_xent_fwd16(combine)");
  return NM_OK;
}

}  // extern "C"
