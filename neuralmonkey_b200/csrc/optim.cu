// K13: regularisation gradients, per-tensor clip_by_norm and TF-Adam over one flat
// fp32 parameter arena (trainers/generic_trainer.py:84-195 of the reference).
// Two HBM-bound passes over the arena: (1) g = scale*g + 2*l2*p + l1*sign(p) and
// per-tensor sum of squares, (2) clip + Adam.  A CTA owns a fixed chunk of the
// arena and walks the (1-2) tensors that overlap it, so the per-tensor reduction is
// one atomicAdd per CTA per tensor.
#include "common.cuh"

namespace nm {

constexpr int OPT_THREADS = 256;
constexpr int64_t OPT_CHUNK = 8192;  // elements per CTA

__device__ __forceinline__ int64_t find_segment(const int64_t* __restrict__ seg_off, int64_t nseg,
                                                int64_t pos) {
  // largest s with seg_off[s] <= pos
  int64_t lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (seg_off[mid] <= pos) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(OPT_THREADS)
reg_norm_kernel(const float* __restrict__ params, float* __restrict__ grads,
                const int64_t* __restrict__ seg_off, const uint8_t* __restrict__ seg_reg,
                float* __restrict__ norms, int64_t n, int64_t nseg, float grad_scale,
                const float* __restrict__ grad_denominator, float l1, float l2,
                float* __restrict__ l1l2_out) {
  __shared__ float red[32];
  if (grad_denominator) grad_scale /= grad_denominator[0];
  const int64_t c0 = (int64_t)blockIdx.x * OPT_CHUNK;
  const int64_t c1 = min(n, c0 + OPT_CHUNK);
  int64_t seg = find_segment(seg_off, nseg, c0);
  float l1_acc = 0.f, l2_acc = 0.f;
  while (seg < nseg && seg_off[seg] < c1) {
    const int64_t a = max(c0, seg_off[seg]), b = min(c1, seg_off[seg + 1]);
    const bool reg = (seg_reg[seg] & 1) != 0;
    float ss = 0.f;
    // segments start on 64-float boundaries and chunks on 8192: [a, b) is 16-byte aligned, so the bulk goes
    // through 128-bit accesses (four times fewer memory instructions in flight for the same bytes)
    const bool vec_ok = ((a & 3) == 0) &&
                        (((reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(params)) & 15) == 0);
    const int64_t nvec = vec_ok ? (b - a) / 4 : 0;     // arbitrary segment tables (tests) take the scalar loop
    float4* g4 = reinterpret_cast<float4*>(grads + a);
    const float4* p4 = reinterpret_cast<const float4*>(params + a);
    for (int64_t i = threadIdx.x; i < nvec; i += OPT_THREADS) {
      float4 g = g4[i];
      float gv[4] = {g.x * grad_scale, g.y * grad_scale, g.z * grad_scale, g.w * grad_scale};
      if (reg) {
        const float4 p = p4[i];
        const float pv[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          gv[j] += 2.f * l2 * pv[j] + l1 * (pv[j] > 0.f ? 1.f : (pv[j] < 0.f ? -1.f : 0.f));
          l1_acc += fabsf(pv[j]);
          l2_acc += pv[j] * pv[j];
        }
      }
      g4[i] = make_float4(gv[0], gv[1], gv[2], gv[3]);
      ss += gv[0] * gv[0] + gv[1] * gv[1] + gv[2] * gv[2] + gv[3] * gv[3];
    }
    for (int64_t i = a + nvec * 4 + threadIdx.x; i < b; i += OPT_THREADS) {
      float g = grads[i] * grad_scale;
      if (reg) {
        const float p = params[i];
        g += 2.f * l2 * p + l1 * (p > 0.f ? 1.f : (p < 0.f ? -1.f : 0.f));
        l1_acc += fabsf(p);
        l2_acc += p * p;
      }
      grads[i] = g;
      ss += g * g;
    }
    ss = block_sum(ss, red);
    if (threadIdx.x == 0 && b > a) atomicAdd(norms + seg, ss);
    ++seg;
  }
  if (l1l2_out) {
    l1_acc = block_sum(l1_acc, red);
    l2_acc = block_sum(l2_acc, red);
    if (threadIdx.x == 0) {
      if (l1_acc != 0.f) atomicAdd(l1l2_out, l1_acc);
      if (l2_acc != 0.f) atomicAdd(l1l2_out + 1, l2_acc);
    }
  }
}

__global__ void __launch_bounds__(OPT_THREADS)
clip_adam_kernel(float* __restrict__ params, const float* __restrict__ grads, float* __restrict__ m,
                 float* __restrict__ v, const int64_t* __restrict__ seg_off,
                 const uint8_t* __restrict__ seg_reg,
                 const float* __restrict__ norms, int64_t n, int64_t nseg, float lr_t, float beta1,
                 float beta2, float eps, float clip_norm, const float* __restrict__ lr_t_dev) {
  if (lr_t_dev) lr_t = lr_t_dev[0];
  const int64_t c0 = (int64_t)blockIdx.x * OPT_CHUNK;
  const int64_t c1 = min(n, c0 + OPT_CHUNK);
  int64_t seg = find_segment(seg_off, nseg, c0);
  while (seg < nseg && seg_off[seg] < c1) {
    const int64_t a = max(c0, seg_off[seg]), b = min(c1, seg_off[seg + 1]);
    float scale = 1.f;
    if (clip_norm > 0.f) {
      // tf.clip_by_norm: t * clip / max(||t||, clip)
      const float nrm = sqrtf(norms[seg]);
      scale = clip_norm / fmaxf(nrm, clip_norm);
    }
    // flag bit 1: tf.contrib.opt.LazyAdamOptimizer semantics for a sparsely updated table -
    // entries that received no gradient (embedding rows absent from the batch) keep their
    // moments and value instead of decaying
    const bool lazy = (seg_reg[seg] & 2) != 0;
    const bool vec_ok = ((a & 3) == 0) &&
                        (((reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(params) |
                           reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0);
    const int64_t nvec = vec_ok ? (b - a) / 4 : 0;
    const float4* g4 = reinterpret_cast<const float4*>(grads + a);
    float4* m4 = reinterpret_cast<float4*>(m + a);
    float4* v4 = reinterpret_cast<float4*>(v + a);
    float4* p4 = reinterpret_cast<float4*>(params + a);
    for (int64_t i = threadIdx.x; i < nvec; i += OPT_THREADS) {
      const float4 gq = g4[i];
      const float gv[4] = {gq.x * scale, gq.y * scale, gq.z * scale, gq.w * scale};
      if (lazy && gv[0] == 0.f && gv[1] == 0.f && gv[2] == 0.f && gv[3] == 0.f) continue;
      float4 mq = m4[i], vq = v4[i], pq = p4[i];
      float mv[4] = {mq.x, mq.y, mq.z, mq.w}, vv[4] = {vq.x, vq.y, vq.z, vq.w}, pv[4] = {pq.x, pq.y, pq.z, pq.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (lazy && gv[j] == 0.f) continue;
        mv[j] = beta1 * mv[j] + (1.f - beta1) * gv[j];
        vv[j] = beta2 * vv[j] + (1.f - beta2) * gv[j] * gv[j];
        pv[j] -= lr_t * mv[j] / (sqrtf(vv[j]) + eps);
      }
      m4[i] = make_float4(mv[0], mv[1], mv[2], mv[3]);
      v4[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
      p4[i] = make_float4(pv[0], pv[1], pv[2], pv[3]);
    }
    for (int64_t i = a + nvec * 4 + threadIdx.x; i < b; i += OPT_THREADS) {
      const float g = grads[i] * scale;
      if (lazy && g == 0.f) continue;
      const float mi = beta1 * m[i] + (1.f - beta1) * g;
      const float vi = beta2 * v[i] + (1.f - beta2) * g * g;
      m[i] = mi;
      v[i] = vi;
      params[i] -= lr_t * mi / (sqrtf(vi) + eps);
    }
    ++seg;
  }
}


// tf.train.AdadeltaOptimizer after the same clip_by_norm as clip_adam_kernel:
//   accum = rho*accum + (1-rho)*g^2;  update = sqrt(accum_update + eps) / sqrt(accum + eps) * g;
//   accum_update = rho*accum_update + (1-rho)*update^2;  p -= lr*update
__global__ void __launch_bounds__(OPT_THREADS)
clip_adadelta_kernel(float* __restrict__ params, const float* __restrict__ grads, float* __restrict__ accum,
                     float* __restrict__ accum_update, const int64_t* __restrict__ seg_off,
                     const uint8_t* __restrict__ seg_reg, const float* __restrict__ norms, int64_t n, int64_t nseg, float lr, float rho, float eps,
                     float clip_norm, const float* __restrict__ lr_dev) {
  if (lr_dev) lr = lr_dev[0];
  const int64_t c0 = (int64_t)blockIdx.x * OPT_CHUNK;
  const int64_t c1 = min(n, c0 + OPT_CHUNK);
  int64_t seg = find_segment(seg_off, nseg, c0);
  while (seg < nseg && seg_off[seg] < c1) {
    const int64_t a = max(c0, seg_off[seg]), b = min(c1, seg_off[seg + 1]);
    const float scale = clip_norm > 0.f ? clip_norm / fmaxf(sqrtf(norms[seg]), clip_norm) : 1.f;
    const bool lazy = (seg_reg[seg] & 2) != 0;     // (segments outside a trainer's var_scopes)
#pragma unroll 1
    for (int64_t i = a + threadIdx.x; i < b; i += OPT_THREADS) {
      const float g = grads[i] * scale;
      if (lazy && g == 0.f) continue;
      const float acc = rho * accum[i] + (1.f - rho) * g * g;
      const float upd = sqrtf(accum_update[i] + eps) / sqrtf(acc + eps) * g;
      accum[i] = acc;
      accum_update[i] = rho * accum_update[i] + (1.f - rho) * upd * upd;
      params[i] -= lr * upd;
    }
    ++seg;
  }
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_clip_adam_step(float* params, float* grads, float* m, float* v, const int64_t* seg_off,
                      const uint8_t* seg_reg, float* norms, int64_t n, int64_t nseg, float grad_scale,
                      const float* grad_denominator, float lr_t, float beta1, float beta2, float eps, float clip_norm, float l1,
                      float l2, float* l1l2_out, const float* lr_t_dev, void* stream) {
  NM_REQUIRE(params && grads && m && v && seg_off && seg_reg && norms, NM_E_INVALID,
             "nm_clip_adam_step: null pointer");
  NM_REQUIRE(n > 0 && nseg > 0, NM_E_INVALID, "nm_clip_adam_step: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)ceil_div(n, OPT_CHUNK);
  const bool need_pass1 =
      clip_norm > 0.f || l1 != 0.f || l2 != 0.f || grad_scale != 1.f || grad_denominator != nullptr ||
      l1l2_out != nullptr;
  if (need_pass1) {
    NM_CUDA_TRY(cudaMemsetAsync(norms, 0, sizeof(float) * nseg, s));
    if (l1l2_out) NM_CUDA_TRY(cudaMemsetAsync(l1l2_out, 0, sizeof(float) * 2, s));
    reg_norm_kernel<<<blocks, OPT_THREADS, 0, s>>>(params, grads, seg_off, seg_reg, norms, n, nseg,
                                                   grad_scale, grad_denominator, l1, l2, l1l2_out);
    NM_LAUNCH_CHECK("nm_clip_adam_step(reg_norm)");
  }
  clip_adam_kernel<<<blocks, OPT_THREADS, 0, s>>>(params, grads, m, v, seg_off, seg_reg, norms, n, nseg, lr_t,
                                                  beta1, beta2, eps, clip_norm, lr_t_dev);
  NM_LAUNCH_CHECK("nm_clip_adam_step(adam)");
  return NM_OK;
}

int nm_clip_adadelta_step(float* params, float* grads, float* accum, float* accum_update, const int64_t* seg_off,
                          const uint8_t* seg_reg, float* norms, int64_t n, int64_t nseg, float grad_scale,
                          const float* grad_denominator, float lr, float rho, float eps, float clip_norm, float l1,
                          float l2, float* l1l2_out, const float* lr_dev, void* stream) {
  NM_REQUIRE(params && grads && accum && accum_update && seg_off && seg_reg && norms, NM_E_INVALID,
             "nm_clip_adadelta_step: null pointer");
  NM_REQUIRE(n > 0 && nseg > 0, NM_E_INVALID, "nm_clip_adadelta_step: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)ceil_div(n, OPT_CHUNK);
  const bool need_pass1 =
      clip_norm > 0.f || l1 != 0.f || l2 != 0.f || grad_scale != 1.f || grad_denominator != nullptr ||
      l1l2_out != nullptr;
  if (need_pass1) {
    NM_CUDA_TRY(cudaMemsetAsync(norms, 0, sizeof(float) * nseg, s));
    if (l1l2_out) NM_CUDA_TRY(cudaMemsetAsync(l1l2_out, 0, sizeof(float) * 2, s));
    reg_norm_kernel<<<blocks, OPT_THREADS, 0, s>>>(params, grads, seg_off, seg_reg, norms, n, nseg,
                                                   grad_scale, grad_denominator, l1, l2, l1l2_out);
    NM_LAUNCH_CHECK("nm_clip_adadelta_step(reg_norm)");
  }
  clip_adadelta_kernel<<<blocks, OPT_THREADS, 0, s>>>(params, grads, accum, accum_update, seg_off, seg_reg, norms, n, nseg, lr,
                                                      rho, eps, clip_norm, lr_dev);
  NM_LAUNCH_CHECK("nm_clip_adadelta_step(adadelta)");
  return NM_OK;
}

}  // extern "C"
