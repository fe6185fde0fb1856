// K4: Bahdanau (MLP) attention, attention/feed_forward.py:120-166 of the reference,
// for NQ query steps at once.
//
//   e[b,q,t] = sum_a v[a] * tanh(keys[b,t,a] + qproj[b,q,a]) + bias
//   p        = softmax_t(e)                       (over ALL Tx, padding included)
//   w        = p*mask / (sum_t p*mask + 1e-8)     (reference :139-144)
//   ctx[b,q] = sum_t w[b,q,t] * values[b,t,:]
//
// The forward and the key-gradient kernel are bound by the tanh count B*NQ*Tx*A on the SFU.  They use
//
//   tanh(k+q) = 1 - 2r,   r = 1 / (1 + e^{2k} e^{2q}),   1 - tanh^2 = 4r(1-r)
//
// with e^{2k} and e^{2q} taken once per staged key or query element, so each (q,t,a) element costs one
// FFMA and one MUFU.RCP.  A forward CTA handles the queries of one chunk of one sentence so every key
// loaded is reused across the chunk from registers; lanes walk the contiguous A (or C) axis for coalesced
// 128-byte requests, and the softmax over Tx is a warp-shuffle reduction.
#include "attention_common.cuh"

namespace nm {

// grid (nch, B): queries att_chunk(blockIdx.x) of sentence blockIdx.y.
// dynamic smem: es[Tx][QMAX] | v2s[A] | qs[QMAX][A]
__global__ void __launch_bounds__(ATT_THREADS)
bahdanau_fwd_kernel(const float* __restrict__ keys, const float* __restrict__ values,
                    const float* __restrict__ mask, const float* __restrict__ qproj,
                    const float* __restrict__ v, const float* __restrict__ bias,
                    float* __restrict__ energies, float* __restrict__ weights,
                    float* __restrict__ ctx, int Tx, int NQ, int A, int C) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  float* es = smem;
  float* v2s = es + Tx * ATT_QMAX;
  float* qs = v2s + A;
  const int b = blockIdx.y;
  int q0, nq;
  att_chunk(blockIdx.x, gridDim.x, NQ, q0, nq);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = ATT_THREADS / 32;
  const float* kb = keys + (int64_t)b * Tx * A;

  // e = sum_a v tanh = sum_a v + sum_a (-2v) r
  float vsum = 0.f, kq_max = 0.f;
  for (int a = threadIdx.x; a < A; a += ATT_THREADS) {
    const float vv = v[a];
    v2s[a] = -2.f * vv;
    vsum += vv;
  }
  const float* qb = qproj + ((int64_t)b * NQ + q0) * A;
  for (int i = threadIdx.x; i < nq * A; i += ATT_THREADS) {
    const float q = qb[i];
    qs[i] = q;
    kq_max = fmaxf(kq_max, fabsf(q));
  }
  for (int i = threadIdx.x; i < Tx * A; i += ATT_THREADS) kq_max = fmaxf(kq_max, fabsf(kb[i]));
  const float ebase = block_sum(vsum, red) + bias[0];
  const bool fast = __syncthreads_and(kq_max <= ATT_FAST_RANGE);
  if (fast) {
    for (int i = threadIdx.x; i < nq * A; i += ATT_THREADS) qs[i] = expf(2.f * qs[i]);
    __syncthreads();
    fwd_energies_n<true>(nq, kb, v2s, qs, es, ebase, Tx, A);
  } else {
    fwd_energies_n<false>(nq, kb, v2s, qs, es, ebase, Tx, A);
  }
  __syncthreads();

  // softmax over Tx, then mask + renormalise: one warp per query
  for (int j = warp; j < nq; j += nwarps) {
    const int64_t orow = ((int64_t)b * NQ + q0 + j) * Tx;
    float mx = -INFINITY;
    for (int t = lane; t < Tx; t += 32) mx = fmaxf(mx, es[t * ATT_QMAX + j]);
    mx = warp_max(mx);
    float s = 0.f;
    for (int t = lane; t < Tx; t += 32) s += expf(es[t * ATT_QMAX + j] - mx);
    s = warp_sum(s);
    float ws = 0.f;
    for (int t = lane; t < Tx; t += 32) {
      const float e = es[t * ATT_QMAX + j];
      if (energies) energies[orow + t] = e;
      float p = expf(e - mx) / s;
      if (mask) p *= mask[(int64_t)b * Tx + t];
      es[t * ATT_QMAX + j] = p;
      ws += p;
    }
    if (mask) {
      const float norm = warp_sum(ws) + 1e-8f;
      for (int t = lane; t < Tx; t += 32) es[t * ATT_QMAX + j] = es[t * ATT_QMAX + j] / norm;
    }
    __syncwarp();
    for (int t = lane; t < Tx; t += 32) weights[orow + t] = es[t * ATT_QMAX + j];
  }
  __syncthreads();

  // ctx[b,q,c] = sum_t w[q,t] * values[b,t,c]; the weights of one t are two broadcast float4 loads
  for (int c = threadIdx.x; c < C; c += ATT_THREADS) {
    float acc[ATT_QMAX];
#pragma unroll
    for (int j = 0; j < ATT_QMAX; ++j) acc[j] = 0.f;
    const float* vc = values + (int64_t)b * Tx * C + c;
    for (int t = 0; t < Tx; ++t) {
      const float val = vc[(int64_t)t * C];
      const float4 w0 = *reinterpret_cast<const float4*>(es + t * ATT_QMAX);
      const float4 w1 = *reinterpret_cast<const float4*>(es + t * ATT_QMAX + 4);
      const float w[ATT_QMAX] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int j = 0; j < ATT_QMAX; ++j)
        if (j < nq) acc[j] = fmaf(w[j], val, acc[j]);
    }
#pragma unroll
    for (int j = 0; j < ATT_QMAX; ++j)
      if (j < nq) ctx[((int64_t)b * NQ + q0 + j) * C + c] = acc[j];
  }
}

// Backward A: de[b,q,t] from dctx, plus de_in (a loss on the energies themselves) when given.  grid (nch, B) as
// the forward.  DE_IN is whether de_in is given: without it the kernel is the plain dctx path.
// dynamic smem: dcs[QMAX][C] (the chunk's dctx rows, zero beyond nq) | dws[QMAX][Tx]
template <bool DE_IN>
__global__ void __launch_bounds__(ATT_THREADS)
bahdanau_bwd_energy_kernel(const float* __restrict__ values, const float* __restrict__ mask,
                           const float* __restrict__ energies, const float* __restrict__ weights,
                           const float* __restrict__ dctx, const float* __restrict__ de_in,
                           float* __restrict__ de, float* __restrict__ dbias, int Tx, int NQ, int C) {
  extern __shared__ float smem[];
  float* dcs = smem;
  float* dws = dcs + ATT_QMAX * C;
  __shared__ float red[32];
  const int b = blockIdx.y;
  int q0, nq;
  att_chunk(blockIdx.x, gridDim.x, NQ, q0, nq);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = ATT_THREADS / 32;

  const float* dcb = dctx + ((int64_t)b * NQ + q0) * C;
  for (int i = threadIdx.x; i < ATT_QMAX * C; i += ATT_THREADS) dcs[i] = i < nq * C ? dcb[i] : 0.f;
  __syncthreads();

  // dw[q,t] = sum_c dctx[b,q,c] * values[b,t,c]: one warp per t, lanes over C
  for (int t = warp; t < Tx; t += nwarps) {
    const float* vr = values + ((int64_t)b * Tx + t) * C;
    float acc[ATT_QMAX];
#pragma unroll
    for (int j = 0; j < ATT_QMAX; ++j) acc[j] = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float val = vr[c];
#pragma unroll
      for (int j = 0; j < ATT_QMAX; ++j) acc[j] = fmaf(val, dcs[j * C + c], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < ATT_QMAX; ++j) {
      const float s = warp_sum(acc[j]);
      if (lane == 0) dws[j * Tx + t] = s;
    }
  }
  __syncthreads();

  float dbias_local = 0.f;
  for (int j = warp; j < nq; j += nwarps) {
    const int64_t row = ((int64_t)b * NQ + q0 + j) * Tx;
    const float* er = energies + row;
    const float* wr = weights + row;
    float* dwr = dws + j * Tx;
    // recompute p and the renormaliser N
    float mx = -INFINITY;
    for (int t = lane; t < Tx; t += 32) mx = fmaxf(mx, er[t]);
    mx = warp_max(mx);
    float s = 0.f;
    for (int t = lane; t < Tx; t += 32) s += expf(er[t] - mx);
    s = warp_sum(s);
    float norm = 1.f;
    float dot_dw_w = 0.f;
    if (mask) {
      float ws = 0.f;
      for (int t = lane; t < Tx; t += 32) {
        ws += expf(er[t] - mx) / s * mask[(int64_t)b * Tx + t];
        dot_dw_w += dwr[t] * wr[t];
      }
      norm = warp_sum(ws) + 1e-8f;
      dot_dw_w = warp_sum(dot_dw_w);
    }
    // dp_t = mask_t * (dw_t - sum dw.w) / N   (no mask: dp = dw)
    float pdp = 0.f;
    for (int t = lane; t < Tx; t += 32) {
      const float p = expf(er[t] - mx) / s;
      float dp = dwr[t];
      if (mask) dp = mask[(int64_t)b * Tx + t] * (dp - dot_dw_w) / norm;
      dwr[t] = dp;
      pdp += p * dp;
    }
    pdp = warp_sum(pdp);
    for (int t = lane; t < Tx; t += 32) {
      const float p = expf(er[t] - mx) / s;
      float g = p * (dwr[t] - pdp);
      if (DE_IN) g += de_in[row + t];
      de[row + t] = g;
      dbias_local += g;
    }
  }
  dbias_local = block_sum(dbias_local, red);
  if (threadIdx.x == 0 && dbias) atomicAdd(dbias, dbias_local);
}

// Backward B: dkeys, dqproj, dv.  grid (ceil(A/128), B), block 128: one a-column per thread.  The NQ
// queries are walked in register chunks of 32, 16, 8, 4, 2 and 1 (NQ's binary digits), so exactly NQ
// query slots are computed.  Per (t, q), with g = de * v * (1 - tanh^2) = 4v * s(1-r), s = de * r:
//   dkeys[t] = 4v sum_q s(1-r),  dqproj[q] = 4v sum_t s(1-r),  dv = sum de * tanh = sum de - 2 sum s.

// dynamic smem: des[Tx][NQ4], NQ4 = NQ rounded up to 4 (q contiguous for broadcast float4 loads)
__global__ void __launch_bounds__(ATT_ACH)
bahdanau_bwd_keys_kernel(const float* __restrict__ keys, const float* __restrict__ qproj,
                         const float* __restrict__ v, const float* __restrict__ de,
                         float* __restrict__ dkeys, float* __restrict__ dqproj,
                         float* __restrict__ dv, int Tx, int NQ, int A) {
  extern __shared__ float des[];
  __shared__ float red[32];
  const int NQ4 = (NQ + 3) & ~3;
  const int b = blockIdx.y;
  const int a = blockIdx.x * ATT_ACH + threadIdx.x;
  const bool ok = a < A;
  float dsum = 0.f;
  for (int i = threadIdx.x; i < Tx * NQ4; i += ATT_ACH) {
    const int t = i / NQ4, q = i - t * NQ4;
    const float d = q < NQ ? de[((int64_t)b * NQ + q) * Tx + t] : 0.f;
    des[i] = d;
    dsum += d;
  }
  const float* kp = keys + (int64_t)b * Tx * A + a;
  const float* qp = qproj + (int64_t)b * NQ * A + a;
  float mx = 0.f;
  if (ok) {
    for (int t = 0; t < Tx; ++t) mx = fmaxf(mx, fabsf(kp[(int64_t)t * A]));
    for (int q = 0; q < NQ; ++q) mx = fmaxf(mx, fabsf(qp[(int64_t)q * A]));
  }
  dsum = block_sum(dsum, red);
  const bool fast = __syncthreads_and(mx <= ATT_FAST_RANGE);
  if (!ok) return;
  const float va4 = 4.f * v[a];
  float* dkp = dkeys + (int64_t)b * Tx * A + a;
  float* dqp = dqproj + (int64_t)b * NQ * A + a;
  float dvs = 0.f;
  if (fast)
    bwd_keys_all<true>(kp, qp, des, dkp, dqp, Tx, NQ, NQ4, A, va4, dvs);
  else
    bwd_keys_all<false>(kp, qp, des, dkp, dqp, Tx, NQ, NQ4, A, va4, dvs);
  atomicAdd(dv + a, fmaf(-2.f, dvs, dsum));
}

// Backward C: dvalues[b,t,c] = sum_q w[b,q,t] * dctx[b,q,c].  grid (ceil(C/128), B).  A thread computes 8
// t rows of its column at a time: per q one dctx load and two broadcast float4 loads of w for 8 FMAs.
// dynamic smem: ws[NQ][Tx8] (Tx8 = Tx rounded up to 8, zero beyond Tx) | dcs[NQ][128]
__global__ void __launch_bounds__(ATT_ACH)
bahdanau_bwd_values_kernel(const float* __restrict__ weights, const float* __restrict__ dctx,
                           float* __restrict__ dvalues, int Tx, int NQ, int C) {
  extern __shared__ float smem[];
  const int Tx8 = (Tx + ATT_VT - 1) / ATT_VT * ATT_VT;
  float* ws = smem;
  float* dcs = ws + NQ * Tx8;
  const int b = blockIdx.y;
  const int c = blockIdx.x * ATT_ACH + threadIdx.x;
  const bool ok = c < C;
  for (int i = threadIdx.x; i < NQ * Tx8; i += ATT_ACH) {
    const int q = i / Tx8, t = i - q * Tx8;
    ws[i] = t < Tx ? weights[((int64_t)b * NQ + q) * Tx + t] : 0.f;
  }
  for (int q = 0; q < NQ; ++q)
    dcs[q * ATT_ACH + threadIdx.x] = ok ? dctx[((int64_t)b * NQ + q) * C + c] : 0.f;
  __syncthreads();
  if (!ok) return;
  for (int t0 = 0; t0 < Tx; t0 += ATT_VT) {
    float acc[ATT_VT];
#pragma unroll
    for (int i = 0; i < ATT_VT; ++i) acc[i] = 0.f;
    for (int q = 0; q < NQ; ++q) {
      const float d = dcs[q * ATT_ACH + threadIdx.x];
      const float4 w0 = *reinterpret_cast<const float4*>(ws + q * Tx8 + t0);
      const float4 w1 = *reinterpret_cast<const float4*>(ws + q * Tx8 + t0 + 4);
      const float w[ATT_VT] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int i = 0; i < ATT_VT; ++i) acc[i] = fmaf(w[i], d, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < ATT_VT; ++i)
      if (t0 + i < Tx) dvalues[((int64_t)b * Tx + t0 + i) * C + c] = acc[i];
  }
}

// The caller has checked att_values_smem(Tx, NQ) against ATT_SMEM_LIMIT and B <= 65535.
int att_values_grad(const float* weights, const float* dctx, float* dvalues, int64_t B, int64_t Tx, int64_t NQ,
                    int64_t C, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    NM_CUDA_TRY(cudaFuncSetAttribute(bahdanau_bwd_values_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    attr_set = true;
  }
  dim3 grid((unsigned)ceil_div(C, ATT_ACH), (unsigned)B);
  bahdanau_bwd_values_kernel<<<grid, ATT_ACH, att_values_smem(Tx, NQ), s>>>(weights, dctx, dvalues, (int)Tx,
                                                                           (int)NQ, (int)C);
  NM_LAUNCH_CHECK("att_values_grad");
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_bahdanau_fwd(const float* keys, const float* values, const float* mask, const float* qproj,
                    const float* v, const float* bias, float* energies, float* weights, float* ctx,
                    int64_t B, int64_t Tx, int64_t NQ, int64_t A, int64_t C, void* stream) {
  NM_REQUIRE(keys && values && qproj && v && bias && weights && ctx, NM_E_INVALID,
             "nm_bahdanau_fwd: null pointer");
  NM_REQUIRE(B > 0 && Tx > 0 && NQ > 0 && A > 0 && C > 0, NM_E_INVALID, "nm_bahdanau_fwd: bad sizes");
  NM_REQUIRE(B <= 65535, NM_E_UNSUPPORTED, "nm_bahdanau_fwd: B > 65535");
  const size_t smem = sizeof(float) * (size_t)(A + ATT_QMAX * A + ATT_QMAX * Tx);
  NM_REQUIRE(smem <= ATT_SMEM_LIMIT, NM_E_UNSUPPORTED,
             "nm_bahdanau_fwd: A=%lld Tx=%lld need %zu B of shared memory", (long long)A,
             (long long)Tx, smem);
  static bool attr_set = false;
  if (!attr_set) {
    NM_CUDA_TRY(cudaFuncSetAttribute(bahdanau_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    attr_set = true;
  }
  dim3 grid((unsigned)att_chunks(B, NQ), (unsigned)B);
  bahdanau_fwd_kernel<<<grid, ATT_THREADS, smem, (cudaStream_t)stream>>>(
      keys, values, mask, qproj, v, bias, energies, weights, ctx, (int)Tx, (int)NQ, (int)A, (int)C);
  NM_LAUNCH_CHECK("nm_bahdanau_fwd");
  return NM_OK;
}

int nm_bahdanau_bwd(const float* keys, const float* values, const float* mask, const float* qproj,
                    const float* v, const float* energies, const float* weights, const float* dctx,
                    const float* de_in, float* dkeys, float* dvalues, float* dqproj, float* dv, float* dbias,
                    float* de_work,
                    int64_t B, int64_t Tx, int64_t NQ, int64_t A, int64_t C, void* stream) {
  NM_REQUIRE(keys && values && qproj && v && energies && weights && dctx && dkeys && dvalues &&
                 dqproj && dv && dbias && de_work,
             NM_E_INVALID, "nm_bahdanau_bwd: null pointer");
  NM_REQUIRE(B > 0 && Tx > 0 && NQ > 0 && A > 0 && C > 0, NM_E_INVALID, "nm_bahdanau_bwd: bad sizes");
  NM_REQUIRE(B <= 65535, NM_E_UNSUPPORTED, "nm_bahdanau_bwd: B > 65535");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem_a = sizeof(float) * (size_t)(ATT_QMAX * C + ATT_QMAX * Tx);
  const size_t smem_b = sizeof(float) * (size_t)(Tx * ((NQ + 3) & ~3));
  const size_t smem_c = sizeof(float) * (size_t)(NQ * ceil_div(Tx, ATT_VT) * ATT_VT + NQ * ATT_ACH);
  NM_REQUIRE(smem_a <= ATT_SMEM_LIMIT && smem_b <= ATT_SMEM_LIMIT && smem_c <= ATT_SMEM_LIMIT,
             NM_E_UNSUPPORTED, "nm_bahdanau_bwd: NQ=%lld Tx=%lld C=%lld need %zu/%zu/%zu B of shared memory",
             (long long)NQ, (long long)Tx, (long long)C, smem_a, smem_b, smem_c);
  static bool attr_set = false;
  if (!attr_set) {
    NM_CUDA_TRY(cudaFuncSetAttribute(bahdanau_bwd_energy_kernel<false>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM_LIMIT));
    NM_CUDA_TRY(cudaFuncSetAttribute(bahdanau_bwd_energy_kernel<true>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM_LIMIT));
    NM_CUDA_TRY(cudaFuncSetAttribute(bahdanau_bwd_keys_kernel,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM_LIMIT));
    NM_CUDA_TRY(cudaFuncSetAttribute(bahdanau_bwd_values_kernel,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM_LIMIT));
    attr_set = true;
  }
  dim3 grid_a((unsigned)att_chunks(B, NQ), (unsigned)B);
  if (de_in)
    bahdanau_bwd_energy_kernel<true><<<grid_a, ATT_THREADS, smem_a, s>>>(values, mask, energies, weights, dctx, de_in,
                                                                        de_work, dbias, (int)Tx, (int)NQ, (int)C);
  else
    bahdanau_bwd_energy_kernel<false><<<grid_a, ATT_THREADS, smem_a, s>>>(values, mask, energies, weights, dctx,
                                                                         nullptr, de_work, dbias, (int)Tx, (int)NQ,
                                                                         (int)C);
  NM_LAUNCH_CHECK("nm_bahdanau_bwd(energy)");
  dim3 grid_b((unsigned)ceil_div(A, ATT_ACH), (unsigned)B);
  bahdanau_bwd_keys_kernel<<<grid_b, ATT_ACH, smem_b, s>>>(keys, qproj, v, de_work, dkeys, dqproj, dv,
                                                          (int)Tx, (int)NQ, (int)A);
  NM_LAUNCH_CHECK("nm_bahdanau_bwd(keys)");
  dim3 grid_c((unsigned)ceil_div(C, ATT_ACH), (unsigned)B);
  bahdanau_bwd_values_kernel<<<grid_c, ATT_ACH, smem_c, s>>>(weights, dctx, dvalues, (int)Tx, (int)NQ,
                                                            (int)C);
  NM_LAUNCH_CHECK("nm_bahdanau_bwd(values)");
  return NM_OK;
}

}  // extern "C"
