// Shared helpers for libnmb200 (sm_90a).  Error convention of include/nmb200.h:
// 0 ok, <0 invalid argument, >0 cudaError_t; message via nm_last_error().
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/nmb200.h"

namespace nm {

void set_error(const char* fmt, ...);
// process-wide count of kernel launches issued by this library (bench.py's gpu_launches)
void count_launches(int64_t n);

#define NM_REQUIRE(cond, code, ...)   \
  do {                                \
    if (!(cond)) {                    \
      nm::set_error(__VA_ARGS__);     \
      return (code);                  \
    }                                 \
  } while (0)

#define NM_LAUNCH_CHECK(name)                                                  \
  do {                                                                         \
    nm::count_launches(1);                                                     \
    cudaError_t e__ = cudaGetLastError();                                      \
    if (e__ != cudaSuccess) {                                                  \
      nm::set_error("%s: %s", name, cudaGetErrorString(e__));                  \
      return (int)e__;                                                         \
    }                                                                          \
  } while (0)

#define NM_CUDA_TRY(expr)                                                      \
  do {                                                                         \
    cudaError_t e__ = (expr);                                                  \
    if (e__ != cudaSuccess) {                                                  \
      nm::set_error("%s: %s", #expr, cudaGetErrorString(e__));                 \
      return (int)e__;                                                         \
    }                                                                          \
  } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Number of SMs of the current device (cached per process; 132 on an H100 SXM).
int sm_count();

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum; `red` is >= 32 floats of shared memory. All threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (w == 0) r = warp_sum(r);
  if (threadIdx.x == 0) red[0] = r;
  __syncthreads();
  return red[0];
}
__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : -INFINITY;
  if (w == 0) r = warp_max(r);
  if (threadIdx.x == 0) red[0] = r;
  __syncthreads();
  return red[0];
}

// Philox4x32-10 (Salmon et al., SC'11): counter-based random bits, shared by dropout (dropout.cu) and the
// sampler of rl.cu.  Their counters occupy disjoint ranges of the third word (see the two files).
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += W0;
    k.y += W1;
  }
  return c;
}

// The Philox key of a training step from the device state {seed, step} the runtime keeps.
__device__ __forceinline__ uint2 philox_step_key(const int64_t* __restrict__ state) {
  const uint64_t seed = (uint64_t)state[0], step = (uint64_t)state[1];
  return make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32));
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case NM_ACT_TANH: return tanhf(x);
    case NM_ACT_RELU: return fmaxf(x, 0.f);
    case NM_ACT_SIGMOID: return sigmoidf_(x);
    default: return x;
  }
}

}  // namespace nm
