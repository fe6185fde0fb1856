// Sentence classification and regression (reference: encoders/pooling.py, encoders/attentive.py,
// encoders/sequence_cnn_encoder.py, decoders/sequence_regressor.py): pooling over time, the self-attentive
// pooling of Lin et al. (2017) and the squared-error loss.  The Kim-CNN convolution itself is nm_gemm over
// row-shifted views of the embeddings (ops.conv1d_valid); only its max over time lives here.
//
// Every reduction runs in a fixed order (one thread per output column walking the time axis, or one warp with
// a fixed shuffle tree), so repeat calls give identical bits.
#include <math.h>

#include "common.cuh"

namespace nm {

constexpr int ATT_THREADS = 256;
constexpr int ATT_MAX_HEADS = 32;
constexpr int64_t ATT_MAX_TR = 16384;  // T*R floats per shared-memory plane (three planes in the backward)

static unsigned cls_grid(int64_t total, int threads) {
  const int64_t blocks = ceil_div(total, threads), cap = (int64_t)sm_count() * 16;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// reduce_max(x*m + 1e-15*(1-m)) reads this value at every position; products are kept apart from the sum, as
// TF evaluates them as separate ops.
__device__ __forceinline__ float padded_value(const float* __restrict__ x, const float* __restrict__ mask,
                                              int64_t row, int64_t D, int64_t d) {
  const float v = __ldg(x + row * D + d);
  if (!mask) return v;
  const float m = __ldg(mask + row);
  return __fadd_rn(__fmul_rn(v, m), __fmul_rn(1e-15f, 1.f - m));
}

// y[b,d] = max_{t<L} value(b*T+t, d), then max(., 0) with relu
__global__ void __launch_bounds__(256) seq_max_fwd_kernel(const float* __restrict__ x, const float* __restrict__ mask,
                                                          float* __restrict__ y, int64_t B, int64_t L, int64_t T,
                                                          int64_t D, int relu) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B * D; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / D, d = i - b * D;
    float best = -INFINITY;
    for (int64_t t = 0; t < L; ++t) best = fmaxf(best, padded_value(x, mask, b * T + t, D, d));
    y[i] = relu ? fmaxf(best, 0.f) : best;
  }
}

// TF's _MaxGrad: dy split equally among all positions equal to the maximum, times the mask (the gradient of
// x*m); with relu, zero unless the maximum is positive (ReluGrad at the tied positions).  Rows b*T+t with
// t >= L (windows across a sentence boundary) get zero; rows >= `rows` do not exist.
__global__ void __launch_bounds__(256) seq_max_bwd_kernel(const float* __restrict__ x, const float* __restrict__ mask,
                                                          const float* __restrict__ dy, float* __restrict__ dx,
                                                          int64_t B, int64_t L, int64_t T, int64_t D, int64_t rows,
                                                          int relu) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B * D; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / D, d = i - b * D;
    float best = -INFINITY, count = 0.f;
    for (int64_t t = 0; t < L; ++t) {
      const float v = padded_value(x, mask, b * T + t, D, d);
      if (v > best) {
        best = v;
        count = 1.f;
      } else if (v == best) {
        count += 1.f;
      }
    }
    const float g = (relu && !(best > 0.f)) ? 0.f : __fmul_rn(__fdiv_rn(1.f, count), __ldg(dy + i));
    for (int64_t t = 0; t < T; ++t) {
      const int64_t row = b * T + t;
      if (row >= rows) break;
      float out = 0.f;
      if (t < L && padded_value(x, mask, row, D, d) == best) out = mask ? __fmul_rn(g, __ldg(mask + row)) : g;
      dx[row * D + d] = out;
    }
  }
}

// y[b,d] = sum_t x*m / (sum_t m + 1e-8)
__global__ void __launch_bounds__(256) seq_mean_fwd_kernel(const float* __restrict__ x, const float* __restrict__ mask,
                                                           float* __restrict__ y, int64_t B, int64_t T, int64_t D) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B * D; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / D, d = i - b * D;
    float s = 0.f, ms = 0.f;
    for (int64_t t = 0; t < T; ++t) {
      const float m = mask ? __ldg(mask + b * T + t) : 1.f;
      s = __fadd_rn(s, __fmul_rn(__ldg(x + (b * T + t) * D + d), m));
      ms += m;
    }
    y[i] = __fdiv_rn(s, ms + 1e-8f);
  }
}

__global__ void __launch_bounds__(256) seq_mean_bwd_kernel(const float* __restrict__ mask, const float* __restrict__ dy,
                                                           float* __restrict__ dx, int64_t B, int64_t T, int64_t D) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B * D; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / D, d = i - b * D;
    float ms = 0.f;
    if (mask)
      for (int64_t t = 0; t < T; ++t) ms += __ldg(mask + b * T + t);
    else
      ms = (float)T;
    const float g = __fdiv_rn(__ldg(dy + i), ms + 1e-8f);
    for (int64_t t = 0; t < T; ++t)
      dx[(b * T + t) * D + d] = mask ? __fmul_rn(g, __ldg(mask + b * T + t)) : g;
  }
}

// Column r of the [T,R] plane p: softmax over all T positions (in place); with a mask the result is multiplied
// by it and renormalised with +1e-8 (attentive.py, attention_weights).  Returns the renormaliser (1 without
// mask); `keep_softmax` leaves the plain softmax in p.
__device__ float att_column_softmax(float* p, const float* __restrict__ mask, int T, int R, int r, bool keep_softmax) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int t = lane; t < T; t += 32) mx = fmaxf(mx, p[t * R + r]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int t = lane; t < T; t += 32) {
    const float e = expf(p[t * R + r] - mx);
    p[t * R + r] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  float asum = 0.f;
  for (int t = lane; t < T; t += 32) {
    const float s = __fdiv_rn(p[t * R + r], sum);
    p[t * R + r] = s;
    if (mask) asum += __fmul_rn(s, __ldg(mask + t));
  }
  if (!mask) return 1.f;
  const float z = warp_sum(asum) + 1e-8f;
  if (!keep_softmax)
    for (int t = lane; t < T; t += 32) p[t * R + r] = __fdiv_rn(__fmul_rn(p[t * R + r], __ldg(mask + t)), z);
  return z;
}

// One CTA per sentence.  weights[b] = the renormalised softmaxes [T,R]; out[b] = weights[b]^T . states[b].
__global__ void __launch_bounds__(ATT_THREADS) attentive_fwd_kernel(const float* __restrict__ energies,
                                                                    const float* __restrict__ mask,
                                                                    const float* __restrict__ states,
                                                                    float* __restrict__ weights,
                                                                    float* __restrict__ out, int T, int R, int D) {
  extern __shared__ float sw[];
  const int64_t b = blockIdx.x;
  const int TR = T * R;
  const float* mrow = mask ? mask + b * T : nullptr;
  for (int i = threadIdx.x; i < TR; i += blockDim.x) sw[i] = __ldg(energies + b * TR + i);
  __syncthreads();
  for (int r = threadIdx.x >> 5; r < R; r += blockDim.x >> 5) att_column_softmax(sw, mrow, T, R, r, false);
  __syncthreads();
  for (int i = threadIdx.x; i < TR; i += blockDim.x) weights[b * TR + i] = sw[i];
  const float* v = states + b * T * (int64_t)D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc[ATT_MAX_HEADS];
#pragma unroll
    for (int r = 0; r < ATT_MAX_HEADS; ++r) acc[r] = 0.f;
    for (int t = 0; t < T; ++t) {
      const float x = __ldg(v + (int64_t)t * D + d);
#pragma unroll
      for (int r = 0; r < ATT_MAX_HEADS; ++r)
        if (r < R) acc[r] = fmaf(sw[t * R + r], x, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < ATT_MAX_HEADS; ++r)
      if (r < R) out[(b * R + r) * D + d] = acc[r];
  }
}

// One CTA per sentence: dstates = weights . dout, dW = dout . states^T (+ dweights), then through the
// renormalisation and the softmax to denergies.  Shared memory: softmax, weights, dW planes and R renormalisers.
__global__ void __launch_bounds__(ATT_THREADS) attentive_bwd_kernel(
    const float* __restrict__ energies, const float* __restrict__ mask, const float* __restrict__ states,
    const float* __restrict__ weights, const float* __restrict__ dout, const float* __restrict__ dweights,
    float* __restrict__ denergies, float* __restrict__ dstates, int T, int R, int D) {
  extern __shared__ float smem[];
  const int TR = T * R;
  float* ss = smem;           // softmax
  float* sw = smem + TR;      // weights
  float* sd = smem + 2 * TR;  // dW, then dE
  float* sz = smem + 3 * TR;  // renormalisers [R]
  const int64_t b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const float* mrow = mask ? mask + b * T : nullptr;
  const float* v = states + b * T * (int64_t)D;
  const float* g = dout + b * R * (int64_t)D;
  for (int i = threadIdx.x; i < TR; i += blockDim.x) {
    ss[i] = __ldg(energies + b * TR + i);
    sw[i] = __ldg(weights + b * TR + i);
  }
  __syncthreads();
  for (int r = warp; r < R; r += nwarps) {
    const float z = att_column_softmax(ss, mrow, T, R, r, true);
    if (lane == 0) sz[r] = z;
  }
  // dW[t,r] = <dout[r,:], states[t,:]>, one warp per (t, r)
  for (int p = warp; p < TR; p += nwarps) {
    const int t = p / R, r = p - t * R;
    float acc = 0.f;
    for (int d = lane; d < D; d += 32) acc = fmaf(__ldg(g + (int64_t)r * D + d), __ldg(v + (int64_t)t * D + d), acc);
    acc = warp_sum(acc);
    if (lane == 0) sd[p] = dweights ? acc + __ldg(dweights + b * TR + p) : acc;
  }
  // dstates[t,d] = sum_r W[t,r] dout[r,d]
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float gr[ATT_MAX_HEADS];
#pragma unroll
    for (int r = 0; r < ATT_MAX_HEADS; ++r) gr[r] = r < R ? __ldg(g + (int64_t)r * D + d) : 0.f;
    for (int t = 0; t < T; ++t) {
      float acc = 0.f;
#pragma unroll
      for (int r = 0; r < ATT_MAX_HEADS; ++r)
        if (r < R) acc = fmaf(sw[t * R + r], gr[r], acc);
      dstates[(b * T + t) * (int64_t)D + d] = acc;
    }
  }
  __syncthreads();
  for (int r = warp; r < R; r += nwarps) {
    // through w = s*m / z:  ds_t = m_t (dW_t - sum_u dW_u w_u) / z
    float c = 0.f;
    if (mrow) {
      for (int t = lane; t < T; t += 32) c = fmaf(sd[t * R + r], sw[t * R + r], c);
      c = warp_sum(c);
    }
    float q = 0.f;
    for (int t = lane; t < T; t += 32) {
      float ds = sd[t * R + r];
      if (mrow) ds = __fmul_rn(__fdiv_rn(ds - c, sz[r]), __ldg(mrow + t));
      sd[t * R + r] = ds;
      q = fmaf(ds, ss[t * R + r], q);
    }
    q = warp_sum(q);
    // through the softmax: dE_t = s_t (ds_t - sum_u ds_u s_u)
    for (int t = lane; t < T; t += 32) sd[t * R + r] = __fmul_rn(ss[t * R + r], sd[t * R + r] - q);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < TR; i += blockDim.x) denergies[b * TR + i] = sd[i];
}

// loss = mean over [B,dim] of (pred - target[b])^2; one CTA, fixed-order block sum
__global__ void __launch_bounds__(1024) sq_err_fwd_kernel(const float* __restrict__ pred,
                                                          const float* __restrict__ target, float* __restrict__ loss,
                                                          int64_t B, int64_t dim) {
  __shared__ float red[32];
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < B * dim; i += blockDim.x) {
    const float e = __ldg(pred + i) - __ldg(target + i / dim);
    s = fmaf(e, e, s);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) loss[0] = __fdiv_rn(s, (float)(B * dim));
}

// dpred = dloss / (B*dim) * 2 (pred - target[b])  (the gradients of reduce_mean and tf.square)
__global__ void __launch_bounds__(256) sq_err_bwd_kernel(const float* __restrict__ pred,
                                                         const float* __restrict__ target,
                                                         const float* __restrict__ dloss, float* __restrict__ dpred,
                                                         int64_t B, int64_t dim) {
  const float g = __fdiv_rn(__ldg(dloss), (float)(B * dim));
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B * dim; i += (int64_t)gridDim.x * blockDim.x)
    dpred[i] = __fmul_rn(g, 2.f * (__ldg(pred + i) - __ldg(target + i / dim)));
}

static int att_check(const char* name, int64_t B, int64_t T, int64_t R, int64_t D) {
  NM_REQUIRE(B > 0 && T > 0 && R > 0 && D > 0, NM_E_INVALID, "%s: bad sizes", name);
  NM_REQUIRE(R <= ATT_MAX_HEADS && T * R <= ATT_MAX_TR && D < (1 << 24) && B <= 0x7fffffffLL, NM_E_UNSUPPORTED,
             "%s: needs R <= %d and T*R <= %lld", name, ATT_MAX_HEADS, (long long)ATT_MAX_TR);
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_seq_max_pool_fwd(const float* x, const float* mask, float* y, int64_t B, int64_t L, int64_t T, int64_t D,
                        int relu, void* stream) {
  NM_REQUIRE(x && y, NM_E_INVALID, "nm_seq_max_pool_fwd: null pointer");
  NM_REQUIRE(B > 0 && D > 0 && L > 0 && L <= T, NM_E_INVALID, "nm_seq_max_pool_fwd: bad sizes");
  seq_max_fwd_kernel<<<cls_grid(B * D, 256), 256, 0, (cudaStream_t)stream>>>(x, mask, y, B, L, T, D, relu);
  NM_LAUNCH_CHECK("nm_seq_max_pool_fwd");
  return NM_OK;
}

int nm_seq_max_pool_bwd(const float* x, const float* mask, const float* dy, float* dx, int64_t B, int64_t L,
                        int64_t T, int64_t D, int64_t rows, int relu, void* stream) {
  NM_REQUIRE(x && dy && dx, NM_E_INVALID, "nm_seq_max_pool_bwd: null pointer");
  NM_REQUIRE(B > 0 && D > 0 && L > 0 && L <= T && rows >= (B - 1) * T + L && rows <= B * T, NM_E_INVALID,
             "nm_seq_max_pool_bwd: bad sizes");
  seq_max_bwd_kernel<<<cls_grid(B * D, 256), 256, 0, (cudaStream_t)stream>>>(x, mask, dy, dx, B, L, T, D, rows, relu);
  NM_LAUNCH_CHECK("nm_seq_max_pool_bwd");
  return NM_OK;
}

int nm_seq_mean_pool_fwd(const float* x, const float* mask, float* y, int64_t B, int64_t T, int64_t D, void* stream) {
  NM_REQUIRE(x && y, NM_E_INVALID, "nm_seq_mean_pool_fwd: null pointer");
  NM_REQUIRE(B > 0 && T > 0 && D > 0, NM_E_INVALID, "nm_seq_mean_pool_fwd: bad sizes");
  seq_mean_fwd_kernel<<<cls_grid(B * D, 256), 256, 0, (cudaStream_t)stream>>>(x, mask, y, B, T, D);
  NM_LAUNCH_CHECK("nm_seq_mean_pool_fwd");
  return NM_OK;
}

int nm_seq_mean_pool_bwd(const float* mask, const float* dy, float* dx, int64_t B, int64_t T, int64_t D,
                         void* stream) {
  NM_REQUIRE(dy && dx, NM_E_INVALID, "nm_seq_mean_pool_bwd: null pointer");
  NM_REQUIRE(B > 0 && T > 0 && D > 0, NM_E_INVALID, "nm_seq_mean_pool_bwd: bad sizes");
  seq_mean_bwd_kernel<<<cls_grid(B * D, 256), 256, 0, (cudaStream_t)stream>>>(mask, dy, dx, B, T, D);
  NM_LAUNCH_CHECK("nm_seq_mean_pool_bwd");
  return NM_OK;
}

int nm_attentive_pool_fwd(const float* energies, const float* mask, const float* states, float* weights, float* out,
                          int64_t B, int64_t T, int64_t R, int64_t D, void* stream) {
  NM_REQUIRE(energies && states && weights && out, NM_E_INVALID, "nm_attentive_pool_fwd: null pointer");
  int rc = att_check("nm_attentive_pool_fwd", B, T, R, D);
  if (rc) return rc;
  const size_t smem = (size_t)(T * R) * sizeof(float);
  static bool attr_done = false;
  if (!attr_done) {
    NM_CUDA_TRY(cudaFuncSetAttribute(attentive_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(ATT_MAX_TR * sizeof(float))));
    attr_done = true;
  }
  attentive_fwd_kernel<<<(unsigned)B, ATT_THREADS, smem, (cudaStream_t)stream>>>(energies, mask, states, weights, out,
                                                                                  (int)T, (int)R, (int)D);
  NM_LAUNCH_CHECK("nm_attentive_pool_fwd");
  return NM_OK;
}

int nm_attentive_pool_bwd(const float* energies, const float* mask, const float* states, const float* weights,
                          const float* dout, const float* dweights, float* denergies, float* dstates, int64_t B,
                          int64_t T, int64_t R, int64_t D, void* stream) {
  NM_REQUIRE(energies && states && weights && dout && denergies && dstates, NM_E_INVALID,
             "nm_attentive_pool_bwd: null pointer");
  int rc = att_check("nm_attentive_pool_bwd", B, T, R, D);
  if (rc) return rc;
  const size_t smem = (size_t)(3 * T * R + R) * sizeof(float);
  static bool attr_done = false;
  if (!attr_done) {
    NM_CUDA_TRY(cudaFuncSetAttribute(attentive_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)((3 * ATT_MAX_TR + ATT_MAX_HEADS) * sizeof(float))));
    attr_done = true;
  }
  attentive_bwd_kernel<<<(unsigned)B, ATT_THREADS, smem, (cudaStream_t)stream>>>(
      energies, mask, states, weights, dout, dweights, denergies, dstates, (int)T, (int)R, (int)D);
  NM_LAUNCH_CHECK("nm_attentive_pool_bwd");
  return NM_OK;
}

int nm_squared_error_fwd(const float* pred, const float* target, float* loss, int64_t B, int64_t dim, void* stream) {
  NM_REQUIRE(pred && target && loss, NM_E_INVALID, "nm_squared_error_fwd: null pointer");
  NM_REQUIRE(B > 0 && dim > 0, NM_E_INVALID, "nm_squared_error_fwd: bad sizes");
  sq_err_fwd_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(pred, target, loss, B, dim);
  NM_LAUNCH_CHECK("nm_squared_error_fwd");
  return NM_OK;
}

int nm_squared_error_bwd(const float* pred, const float* target, const float* dloss, float* dpred, int64_t B,
                         int64_t dim, void* stream) {
  NM_REQUIRE(pred && target && dloss && dpred, NM_E_INVALID, "nm_squared_error_bwd: null pointer");
  NM_REQUIRE(B > 0 && dim > 0, NM_E_INVALID, "nm_squared_error_bwd: bad sizes");
  sq_err_bwd_kernel<<<cls_grid(B * dim, 256), 256, 0, (cudaStream_t)stream>>>(pred, target, dloss, dpred, B, dim);
  NM_LAUNCH_CHECK("nm_squared_error_bwd");
  return NM_OK;
}

}  // extern "C"
