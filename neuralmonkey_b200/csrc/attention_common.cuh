// Device helpers shared by the Bahdanau attention kernels (attention.cu, K4) and the joint multi-source
// attention kernels (joint_attention.cu): the factorised tanh, the query chunking, the shared-key energy
// loop and the key / query gradient loop over shared keys.
#pragma once
#include "common.cuh"

namespace nm {

constexpr int ATT_QMAX = 8;      // most queries per CTA (forward / energy-gradient kernels)
constexpr int ATT_THREADS = 256;
// The factorised tanh is exact in form while neither e^{2k} nor e^{2q} is inf or subnormal in fp32, which
// holds for |k|, |q| <= 40 (e^{80} = 5.5e34).  Within that range a product that overflows or underflows
// means tanh is saturated, and r becomes 0 or 1 as it should.  A CTA whose keys or queries leave the range
// (k = 50, q = -49.5 would give inf * 0) takes the two-SFU form instead; the branch is uniform per CTA.
constexpr float ATT_FAST_RANGE = 40.f;

// r = 1 / (1 + e^{2x}) with SFU ex2 and rcp, tanh x = 1 - 2r: |abs err| <= ~2e-7; saturates correctly.
__device__ __forceinline__ float tanh_r(float x) { return __fdividef(1.f, 1.f + __expf(2.f * x)); }

__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// r for x = k + q from ek = e^{2k} and eq = e^{2q} (FAST), or from k and q (the two-SFU form).  The
// exponentials are taken with the accurate expf, so the fast form's error stays at tanh_r's.
template <bool FAST>
__device__ __forceinline__ float att_r(float k_or_ek, float q_or_eq) {
  return FAST ? rcp_approx(fmaf(k_or_ek, q_or_eq, 1.f)) : tanh_r(k_or_ek + q_or_eq);
}
template <bool FAST>
__device__ __forceinline__ float att_stage(float x) { return FAST ? expf(2.f * x) : x; }

// Queries of forward / energy-gradient CTA `chunk` of `nch`: balanced chunks of at most ATT_QMAX, so no
// CTA computes a padded query slot.
__device__ __forceinline__ void att_chunk(int chunk, int nch, int NQ, int& q0, int& nq) {
  q0 = (int)((int64_t)chunk * NQ / nch);
  nq = (int)((int64_t)(chunk + 1) * NQ / nch) - q0;
}

// es[t][QMAX] = sum_a (-2 v[a]) r(k[t,a], q[j,a]) + ebase for the CTA's NQC queries; one warp per t.
template <bool FAST, int NQC>
__device__ __forceinline__ void fwd_energies(const float* __restrict__ kb, const float* __restrict__ v2s,
                                             const float* __restrict__ qs, float* __restrict__ es,
                                             float ebase, int Tx, int A) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = warp; t < Tx; t += ATT_THREADS / 32) {
    const float* kr = kb + (int64_t)t * A;
    float acc[NQC];
#pragma unroll
    for (int j = 0; j < NQC; ++j) acc[j] = 0.f;
    for (int a = lane; a < A; a += 32) {
      const float k = att_stage<FAST>(kr[a]), v2 = v2s[a];
#pragma unroll
      for (int j = 0; j < NQC; ++j) acc[j] = fmaf(v2, att_r<FAST>(k, qs[j * A + a]), acc[j]);
    }
#pragma unroll
    for (int j = 0; j < NQC; ++j) {
      const float e = warp_sum(acc[j]) + ebase;
      if (lane == 0) es[t * ATT_QMAX + j] = e;
    }
  }
}

template <bool FAST>
__device__ __forceinline__ void fwd_energies_n(int nq, const float* kb, const float* v2s, const float* qs,
                                               float* es, float ebase, int Tx, int A) {
  switch (nq) {
    case 1: fwd_energies<FAST, 1>(kb, v2s, qs, es, ebase, Tx, A); break;
    case 2: fwd_energies<FAST, 2>(kb, v2s, qs, es, ebase, Tx, A); break;
    case 3: fwd_energies<FAST, 3>(kb, v2s, qs, es, ebase, Tx, A); break;
    case 4: fwd_energies<FAST, 4>(kb, v2s, qs, es, ebase, Tx, A); break;
    case 5: fwd_energies<FAST, 5>(kb, v2s, qs, es, ebase, Tx, A); break;
    case 6: fwd_energies<FAST, 6>(kb, v2s, qs, es, ebase, Tx, A); break;
    case 7: fwd_energies<FAST, 7>(kb, v2s, qs, es, ebase, Tx, A); break;
    default: fwd_energies<FAST, 8>(kb, v2s, qs, es, ebase, Tx, A); break;
  }
}

// Key / query gradients over shared keys: one a-column per thread (K4's backward kernel B).
constexpr int ATT_ACH = 128;

template <int NQC>
__device__ __forceinline__ void load_de(const float* __restrict__ p, float (&d)[NQC]) {
  if constexpr (NQC % 4 == 0) {
#pragma unroll
    for (int j = 0; j < NQC; j += 4) {
      const float4 x = *reinterpret_cast<const float4*>(p + j);
      d[j] = x.x, d[j + 1] = x.y, d[j + 2] = x.z, d[j + 3] = x.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < NQC; ++j) d[j] = p[j];
  }
}

// kp/dkp: this column of keys/dkeys (row stride A); qp/dqp: this column of qproj/dqproj rows q0...;
// des: [Tx][NQ4] from query q0.  `first` chunk stores dkeys, later ones add to it.
template <bool FAST, int NQC>
__device__ __forceinline__ void bwd_keys_chunk(const float* __restrict__ kp, const float* __restrict__ qp,
                                               const float* __restrict__ des, float* __restrict__ dkp,
                                               float* __restrict__ dqp, int Tx, int NQ4, int A, float va4,
                                               bool first, float& dvs) {
  float qv[NQC], dq[NQC];
#pragma unroll
  for (int j = 0; j < NQC; ++j) {
    qv[j] = att_stage<FAST>(qp[(int64_t)j * A]);
    dq[j] = 0.f;
  }
  float k_next = kp[0];
  for (int t = 0; t < Tx; ++t) {
    const float k = att_stage<FAST>(k_next);
    if (t + 1 < Tx) k_next = kp[(int64_t)(t + 1) * A];
    float d[NQC];
    load_de<NQC>(des + t * NQ4, d);
    float dk = 0.f;
#pragma unroll
    for (int j = 0; j < NQC; ++j) {
      const float r = att_r<FAST>(k, qv[j]);
      const float s = d[j] * r;
      const float g = fmaf(-s, r, s);
      dk += g;
      dq[j] += g;
      dvs += s;
    }
    float* o = dkp + (int64_t)t * A;
    *o = first ? va4 * dk : fmaf(va4, dk, *o);
  }
#pragma unroll
  for (int j = 0; j < NQC; ++j) dqp[(int64_t)j * A] = va4 * dq[j];
}

template <bool FAST>
__device__ __forceinline__ void bwd_keys_all(const float* kp, const float* qp, const float* des, float* dkp,
                                             float* dqp, int Tx, int NQ, int NQ4, int A, float va4, float& dvs) {
  int q0 = 0;
  for (; NQ - q0 >= 32; q0 += 32)
    bwd_keys_chunk<FAST, 32>(kp, qp + (int64_t)q0 * A, des + q0, dkp, dqp + (int64_t)q0 * A, Tx, NQ4, A,
                             va4, q0 == 0, dvs);
#define ATT_KEYS_CHUNK(N)                                                                                   \
  if (NQ - q0 >= N) {                                                                                       \
    bwd_keys_chunk<FAST, N>(kp, qp + (int64_t)q0 * A, des + q0, dkp, dqp + (int64_t)q0 * A, Tx, NQ4, A, va4, \
                            q0 == 0, dvs);                                                                  \
    q0 += N;                                                                                                \
  }
  ATT_KEYS_CHUNK(16)
  ATT_KEYS_CHUNK(8)
  ATT_KEYS_CHUNK(4)
  ATT_KEYS_CHUNK(2)
  ATT_KEYS_CHUNK(1)
#undef ATT_KEYS_CHUNK
}

constexpr int ATT_VT = 8;        // shared positions per thread pass of the value-gradient kernels

constexpr size_t ATT_SMEM_LIMIT = 200 * 1024;

// Query chunks per sentence for the forward and energy-gradient kernels: at most ATT_QMAX queries each, and
// enough CTAs for about two waves on the device when the batch alone does not give them.
inline int att_chunks(int64_t B, int64_t NQ) {
  const int64_t want = ceil_div(2 * (int64_t)sm_count(), B);
  return (int)std::min(NQ, std::max(ceil_div(NQ, ATT_QMAX), want));
}

// Shared memory of K4's value-gradient kernel, and the kernel itself (attention.cu) for other attentions whose
// values enter only through ctx = w . values: dvalues[b,t,c] = sum_q weights[b,q,t] dctx[b,q,c].
inline size_t att_values_smem(int64_t Tx, int64_t NQ) {
  return sizeof(float) * (size_t)(NQ * ceil_div(Tx, ATT_VT) * ATT_VT + NQ * ATT_ACH);
}
int att_values_grad(const float* weights, const float* dctx, float* dvalues, int64_t B, int64_t Tx, int64_t NQ,
                    int64_t C, cudaStream_t s);

}  // namespace nm
