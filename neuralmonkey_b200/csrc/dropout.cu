// K15: dropout (tf.nn.dropout as nn/utils.py:6-22 of the reference selects it in training mode) in ONE pass:
// the keep decisions come from Philox4x32-10 evaluated in the kernel, so no random tensor, no comparison, no cast
// and no mask ever exists in HBM - the backward pass evaluates the same counters again.  (As five element-wise
// library kernels a dropout of a [4096, 512] activation cost 40 us; 56 of them run in a Transformer step.)
//
// Random stream: key = seed, counter = (element index / 4, call site, step).  `state` is a device array
// {seed, step}: the host bumps `step` once per training step (outside any captured graph), `site` numbers the
// dropout calls of a step in program order - a CUDA graph that replays the step draws new masks each replay.
// Sites stay below 2^31: the sampler of rl.cu owns the counters whose third word has its top bit set.
#include "common.cuh"

namespace nm {

__device__ __forceinline__ uint4 keep_bits(const int64_t* __restrict__ state, int64_t quad, uint32_t site) {
  return philox4x32_10(make_uint4((uint32_t)quad, (uint32_t)((uint64_t)quad >> 32), site, (uint32_t)state[1]),
                       philox_step_key(state));
}

// MODE 0: y = keep ? x * scale : 0 (+ residual);  MODE 1: y = keep ? scale : 0 (the mask itself)
template <int MODE>
__global__ void __launch_bounds__(256)
dropout_kernel(const float* __restrict__ x, const float* __restrict__ residual, float* __restrict__ y, int64_t n,
               uint32_t threshold, float scale, const int64_t* __restrict__ state, uint32_t site, int vec) {
  const int64_t nquad = (n + 3) >> 2;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nquad; q += (int64_t)gridDim.x * blockDim.x) {
    const uint4 r = keep_bits(state, q, site);
    const float m0 = r.x < threshold ? scale : 0.f, m1 = r.y < threshold ? scale : 0.f;
    const float m2 = r.z < threshold ? scale : 0.f, m3 = r.w < threshold ? scale : 0.f;
    const int64_t i = q << 2;
    if (vec && i + 3 < n) {
      float4 v = make_float4(m0, m1, m2, m3);
      if (MODE == 0) {
        const float4 a = *reinterpret_cast<const float4*>(x + i);
        v = make_float4(a.x * m0, a.y * m1, a.z * m2, a.w * m3);
        if (residual) {
          const float4 b = *reinterpret_cast<const float4*>(residual + i);
          v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
        }
      }
      *reinterpret_cast<float4*>(y + i) = v;
    } else {
      const float m[4] = {m0, m1, m2, m3};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (i + j < n) {
          float v = m[j];
          if (MODE == 0) v = x[i + j] * m[j] + (residual ? residual[i + j] : 0.f);
          y[i + j] = v;
        }
      }
    }
  }
}

static uint32_t keep_threshold(float keep_prob) {
  const double t = (double)keep_prob * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
}

template <int MODE>
static int launch_dropout(const float* x, const float* residual, float* y, int64_t n, float keep_prob,
                          const int64_t* state, int64_t site, cudaStream_t s, const char* name) {
  const int64_t nquad = (n + 3) >> 2;
  int64_t blocks = ceil_div(nquad, 256);
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  const bool aligned = ((reinterpret_cast<uintptr_t>(y) & 15) == 0) &&
                       (MODE == 1 || (((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                                      (!residual || (reinterpret_cast<uintptr_t>(residual) & 15) == 0)));
  dropout_kernel<MODE><<<(unsigned)blocks, 256, 0, s>>>(x, residual, y, n, keep_threshold(keep_prob),
                                                       1.0f / keep_prob, state, (uint32_t)site, aligned ? 1 : 0);
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_dropout_apply(const float* x, const float* residual, float* y, int64_t n, float keep_prob,
                     const int64_t* state, int64_t site, void* stream) {
  NM_REQUIRE(x && y && state, NM_E_INVALID, "nm_dropout_apply: null pointer");
  NM_REQUIRE(n >= 0 && keep_prob > 0.f && keep_prob <= 1.f, NM_E_INVALID,
             "nm_dropout_apply: n >= 0 and 0 < keep_prob <= 1 expected (n=%lld keep_prob=%g)", (long long)n,
             (double)keep_prob);
  NM_REQUIRE(site >= 0 && site <= 0xFFFFFFFFLL, NM_E_INVALID, "nm_dropout_apply: call-site id out of range");
  if (n == 0) return NM_OK;
  return launch_dropout<0>(x, residual, y, n, keep_prob, state, site, (cudaStream_t)stream, "nm_dropout_apply");
}

int nm_dropout_mask(float* mask, int64_t n, float keep_prob, const int64_t* state, int64_t site, void* stream) {
  NM_REQUIRE(mask && state, NM_E_INVALID, "nm_dropout_mask: null pointer");
  NM_REQUIRE(n >= 0 && keep_prob > 0.f && keep_prob <= 1.f, NM_E_INVALID,
             "nm_dropout_mask: n >= 0 and 0 < keep_prob <= 1 expected (n=%lld keep_prob=%g)", (long long)n,
             (double)keep_prob);
  NM_REQUIRE(site >= 0 && site <= 0xFFFFFFFFLL, NM_E_INVALID, "nm_dropout_mask: call-site id out of range");
  if (n == 0) return NM_OK;
  return launch_dropout<1>(nullptr, nullptr, mask, n, keep_prob, state, site, (cudaStream_t)stream,
                           "nm_dropout_mask");
}

}  // extern "C"
