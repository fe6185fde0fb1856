// Joint-softmax attention for multi-source decoders: attention/combination.py:240-296 (flat) and :394-463
// (hierarchical) of the reference, for NQ query steps at once.
//
//   e[b,q,t]    = sum_a v[a] tanh(keys[b,t,a] + qproj[b,q,a]) + seg_bias[seg(t)]     t < Tx (shared, in segments)
//   e[b,q,Tx+j] = sum_a v[a] tanh(ckeys[b,q,j,a] + qproj[b,q,a]) + cand_bias[j]     j < J  (per-query candidates)
//   p           = softmax over all L = Tx + J positions
//   w           = p*m / (sum p*m + 1e-8), m = mask[b,t] for t < Tx and 1 for candidates   (mask given)
//   w           = p                                                                       (mask NULL)
//   ctx[b,q,:]  = sum_t w[b,q,t] values[b,t,:] + sum_j w[b,q,Tx+j] cvalues[b,q,j,:]
//
// The flat combination is Tx = sum of the encoders' lengths with one segment per encoder and the sentinel as
// the one candidate; the hierarchical one has no shared keys and one candidate per child context (and the
// sentinel).  The decomposition is K4's (attention.cu): a forward CTA per chunk of at most ATT_QMAX queries of
// one sentence reuses every shared key across the chunk from registers with the one-SFU factorised tanh.
// Candidates belong to one query each, so there is no reuse to exploit; they take the same loops one
// (query, candidate) pair per warp.  The backward writes every per-element gradient without atomics and
// reduces the bias and v gradients in a fixed order, so repeated calls give identical bits.
#include "attention_common.cuh"

namespace nm {

constexpr int JA_MAX_SEG = 8;
struct JointSegs {
  int end[JA_MAX_SEG];   // cumulative ends, end[n-1] = Tx
  int n;
};

// end[s] read with constant indices only, so the table stays in the parameter bank (no local-memory copy).
__device__ __forceinline__ int seg_end(const JointSegs& sg, int s) {
  int e = 0;
#pragma unroll
  for (int k = 0; k < JA_MAX_SEG; ++k) e = k == s ? sg.end[k] : e;
  return e;
}

// es[(Tx+i)][QMAX] for candidate i of the chunk's query j: one warp per (j, i).
template <bool FAST>
__device__ __forceinline__ void cand_energies(const float* __restrict__ ckb, const float* __restrict__ v2s,
                                              const float* __restrict__ qs, const float* __restrict__ cand_bias,
                                              float* __restrict__ es, float ebase, int Tx, int J, int nq, int A) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int p = warp; p < nq * J; p += ATT_THREADS / 32) {
    const int j = p / J, i = p - j * J;
    const float* kr = ckb + (int64_t)p * A;   // ckeys rows of the chunk are (j, i)-ordered
    float acc = 0.f;
    for (int a = lane; a < A; a += 32) acc = fmaf(v2s[a], att_r<FAST>(att_stage<FAST>(kr[a]), qs[j * A + a]), acc);
    acc = warp_sum(acc);
    if (lane == 0) es[(Tx + i) * ATT_QMAX + j] = acc + ebase + cand_bias[i];
  }
}

// grid (nch, B): queries att_chunk(blockIdx.x) of sentence blockIdx.y.
// dynamic smem: es[L][QMAX] | v2s[A] | qs[QMAX][A]
__global__ void __launch_bounds__(ATT_THREADS)
joint_fwd_kernel(const float* __restrict__ keys, const float* __restrict__ values, const float* __restrict__ mask,
                 JointSegs segs, const float* __restrict__ seg_bias, const float* __restrict__ ckeys,
                 const float* __restrict__ cvalues, const float* __restrict__ cand_bias,
                 const float* __restrict__ qproj, const float* __restrict__ v, float* __restrict__ energies,
                 float* __restrict__ weights, float* __restrict__ ctx, int Tx, int J, int NQ, int A, int C) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  __shared__ int send[JA_MAX_SEG];
  __shared__ float sbias[JA_MAX_SEG];
  const int L = Tx + J;
  float* es = smem;
  float* v2s = es + L * ATT_QMAX;
  if (threadIdx.x < segs.n) {
    send[threadIdx.x] = seg_end(segs, threadIdx.x);
    sbias[threadIdx.x] = seg_bias[threadIdx.x];
  }
  float* qs = v2s + A;
  const int b = blockIdx.y;
  int q0, nq;
  att_chunk(blockIdx.x, gridDim.x, NQ, q0, nq);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = ATT_THREADS / 32;
  const float* kb = Tx > 0 ? keys + (int64_t)b * Tx * A : nullptr;
  const float* ckb = J > 0 ? ckeys + ((int64_t)b * NQ + q0) * J * A : nullptr;

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
  for (int i = threadIdx.x; i < nq * J * A; i += ATT_THREADS) kq_max = fmaxf(kq_max, fabsf(ckb[i]));
  const float ebase = block_sum(vsum, red);
  const bool fast = __syncthreads_and(kq_max <= ATT_FAST_RANGE);
  if (fast) {
    for (int i = threadIdx.x; i < nq * A; i += ATT_THREADS) qs[i] = expf(2.f * qs[i]);
    __syncthreads();
    cand_energies<true>(ckb, v2s, qs, cand_bias, es, ebase, Tx, J, nq, A);
    fwd_energies_n<true>(nq, kb, v2s, qs, es, ebase, Tx, A);
  } else {
    cand_energies<false>(ckb, v2s, qs, cand_bias, es, ebase, Tx, J, nq, A);
    fwd_energies_n<false>(nq, kb, v2s, qs, es, ebase, Tx, A);
  }
  __syncthreads();

  // segment biases, softmax over L, then mask + renormalise: one warp per query
  for (int j = warp; j < nq; j += nwarps) {
    const int64_t orow = ((int64_t)b * NQ + q0 + j) * L;
    float mx = -INFINITY;
    int sg = 0;
    for (int t = lane; t < L; t += 32) {
      float e = es[t * ATT_QMAX + j];
      if (t < Tx) {
        while (t >= send[sg]) ++sg;
        e += sbias[sg];
        es[t * ATT_QMAX + j] = e;
      }
      mx = fmaxf(mx, e);
    }
    mx = warp_max(mx);
    float s = 0.f;
    for (int t = lane; t < L; t += 32) s += expf(es[t * ATT_QMAX + j] - mx);
    s = warp_sum(s);
    float ws = 0.f;
    for (int t = lane; t < L; t += 32) {
      const float e = es[t * ATT_QMAX + j];
      if (energies) energies[orow + t] = e;
      float p = expf(e - mx) / s;
      if (mask && t < Tx) p *= mask[(int64_t)b * Tx + t];
      es[t * ATT_QMAX + j] = p;
      ws += p;
    }
    if (mask) {
      const float norm = warp_sum(ws) + 1e-8f;
      for (int t = lane; t < L; t += 32) es[t * ATT_QMAX + j] = es[t * ATT_QMAX + j] / norm;
    }
    __syncwarp();
    for (int t = lane; t < L; t += 32) weights[orow + t] = es[t * ATT_QMAX + j];
  }
  __syncthreads();

  // ctx[b,q,c]: shared values as K4 (two broadcast float4 loads of the weights of one t), then the candidates
  for (int c = threadIdx.x; c < C; c += ATT_THREADS) {
    float acc[ATT_QMAX];
#pragma unroll
    for (int j = 0; j < ATT_QMAX; ++j) acc[j] = 0.f;
    if (Tx > 0) {
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
    }
#pragma unroll
    for (int j = 0; j < ATT_QMAX; ++j)
      if (j < nq) ctx[((int64_t)b * NQ + q0 + j) * C + c] = acc[j];
    // the thread adds its own candidates' share to what it just stored (keeps acc[] in registers)
    for (int j = 0; j < nq && J > 0; ++j) {
      const float* cv = cvalues + ((int64_t)b * NQ + q0 + j) * J * C + c;
      float o = ctx[((int64_t)b * NQ + q0 + j) * C + c];
      for (int i = 0; i < J; ++i) o = fmaf(es[(Tx + i) * ATT_QMAX + j], cv[(int64_t)i * C], o);
      ctx[((int64_t)b * NQ + q0 + j) * C + c] = o;
    }
  }
}

// Backward A: de[b,q,:] from dctx, and dcvalues.  grid (nch, B) as the forward.
// dynamic smem: dcs[QMAX][C] (the chunk's dctx rows, zero beyond nq) | dws[QMAX][L]
__global__ void __launch_bounds__(ATT_THREADS)
joint_bwd_energy_kernel(const float* __restrict__ values, const float* __restrict__ mask,
                        const float* __restrict__ cvalues, const float* __restrict__ energies,
                        const float* __restrict__ weights, const float* __restrict__ dctx, float* __restrict__ de,
                        float* __restrict__ dcvalues, int Tx, int J, int NQ, int C) {
  extern __shared__ float smem[];
  const int L = Tx + J;
  float* dcs = smem;
  float* dws = dcs + ATT_QMAX * C;
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
      if (lane == 0) dws[j * L + t] = s;
    }
  }
  // dw[q,Tx+i] = sum_c dctx[b,q,c] * cvalues[b,q,i,c]: one warp per (q, i)
  const float* cvb = cvalues + ((int64_t)b * NQ + q0) * J * C;
  for (int p = warp; p < nq * J; p += nwarps) {
    const int j = p / J, i = p - j * J;
    const float* vr = cvb + (int64_t)p * C;
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) acc = fmaf(vr[c], dcs[j * C + c], acc);
    acc = warp_sum(acc);
    if (lane == 0) dws[j * L + Tx + i] = acc;
  }
  // dcvalues[b,q,i,c] = w[b,q,Tx+i] * dctx[b,q,c]
  float* dcvb = dcvalues + ((int64_t)b * NQ + q0) * J * C;
  for (int64_t k = threadIdx.x; k < (int64_t)nq * J * C; k += ATT_THREADS) {
    const int p = (int)(k / C), c = (int)(k - (int64_t)p * C);
    const int j = p / J, i = p - j * J;
    dcvb[k] = weights[((int64_t)b * NQ + q0 + j) * L + Tx + i] * dcs[j * C + c];
  }
  __syncthreads();

  for (int j = warp; j < nq; j += nwarps) {
    const int64_t row = ((int64_t)b * NQ + q0 + j) * L;
    const float* er = energies + row;
    const float* wr = weights + row;
    float* dwr = dws + j * L;
    float mx = -INFINITY;
    for (int t = lane; t < L; t += 32) mx = fmaxf(mx, er[t]);
    mx = warp_max(mx);
    float s = 0.f;
    for (int t = lane; t < L; t += 32) s += expf(er[t] - mx);
    s = warp_sum(s);
    float norm = 1.f;
    float dot_dw_w = 0.f;
    if (mask) {
      float ws = 0.f;
      for (int t = lane; t < L; t += 32) {
        ws += expf(er[t] - mx) / s * (t < Tx ? mask[(int64_t)b * Tx + t] : 1.f);
        dot_dw_w += dwr[t] * wr[t];
      }
      norm = warp_sum(ws) + 1e-8f;
      dot_dw_w = warp_sum(dot_dw_w);
    }
    // dp_t = m_t * (dw_t - sum dw.w) / N   (no mask: dp = dw)
    float pdp = 0.f;
    for (int t = lane; t < L; t += 32) {
      const float p = expf(er[t] - mx) / s;
      float dp = dwr[t];
      if (mask) dp = (t < Tx ? mask[(int64_t)b * Tx + t] : 1.f) * (dp - dot_dw_w) / norm;
      dwr[t] = dp;
      pdp += p * dp;
    }
    pdp = warp_sum(pdp);
    for (int t = lane; t < L; t += 32) {
      const float p = expf(er[t] - mx) / s;
      de[row + t] = p * (dwr[t] - pdp);
    }
  }
}

// Backward B: dkeys, dckeys, dqproj and the per-sentence partial of dv.  grid (ceil(A/128), B), block 128:
// one a-column per thread.  The shared keys take K4's loops (bwd_keys_all); the candidates of each query
// follow with the two-SFU tanh.  dv_part[b,a] = sum de - 2 sum de*r over the sentence's rows.
// dynamic smem: des[Tx][NQ4], NQ4 = NQ rounded up to 4
__global__ void __launch_bounds__(ATT_ACH)
joint_bwd_keys_kernel(const float* __restrict__ keys, const float* __restrict__ ckeys,
                      const float* __restrict__ qproj, const float* __restrict__ v, const float* __restrict__ de,
                      float* __restrict__ dkeys, float* __restrict__ dckeys, float* __restrict__ dqproj,
                      float* __restrict__ dv_part, JointSegs segs, float* __restrict__ bias_part, int Tx, int J,
                      int NQ, int A) {
  extern __shared__ float des[];
  __shared__ float red[32];
  const int L = Tx + J;
  const int NQ4 = (NQ + 3) & ~3;
  const int b = blockIdx.y;
  const int a = blockIdx.x * ATT_ACH + threadIdx.x;
  const bool ok = a < A;
  float dsum = 0.f;
  for (int i = threadIdx.x; i < Tx * NQ4; i += ATT_ACH) {
    const int t = i / NQ4, q = i - t * NQ4;
    const float d = q < NQ ? de[((int64_t)b * NQ + q) * L + t] : 0.f;
    des[i] = d;
    dsum += d;
  }
  for (int i = threadIdx.x; i < NQ * J; i += ATT_ACH) {
    const int q = i / J, j = i - q * J;
    dsum += de[((int64_t)b * NQ + q) * L + Tx + j];
  }
  const float* qp = qproj + (int64_t)b * NQ * A + a;
  const float* kp = Tx > 0 ? keys + (int64_t)b * Tx * A + a : nullptr;
  float mx = 0.f;
  if (ok && Tx > 0) {
    for (int t = 0; t < Tx; ++t) mx = fmaxf(mx, fabsf(kp[(int64_t)t * A]));
    for (int q = 0; q < NQ; ++q) mx = fmaxf(mx, fabsf(qp[(int64_t)q * A]));
  }
  dsum = block_sum(dsum, red);
  // the sentence's share of each segment and candidate bias gradient (the first column block only)
  if (blockIdx.x == 0) {
    const int nb = segs.n + J;
    for (int k = 0; k < nb; ++k) {
      float acc = 0.f;
      if (k < segs.n) {
        const int lo = k == 0 ? 0 : seg_end(segs, k - 1), hi = seg_end(segs, k);
        for (int i = threadIdx.x; i < (hi - lo) * NQ4; i += ATT_ACH) acc += des[lo * NQ4 + i];   // zero beyond NQ
      } else {
        for (int q = threadIdx.x; q < NQ; q += ATT_ACH) acc += de[((int64_t)b * NQ + q) * L + Tx + k - segs.n];
      }
      acc = block_sum(acc, red);
      if (threadIdx.x == 0) bias_part[(int64_t)b * nb + k] = acc;
    }
  }
  const bool fast = __syncthreads_and(mx <= ATT_FAST_RANGE);
  if (!ok) return;
  const float va4 = 4.f * v[a];
  float* dqp = dqproj + (int64_t)b * NQ * A + a;
  float dvs = 0.f;
  if (Tx > 0) {
    float* dkp = dkeys + (int64_t)b * Tx * A + a;
    if (fast)
      bwd_keys_all<true>(kp, qp, des, dkp, dqp, Tx, NQ, NQ4, A, va4, dvs);
    else
      bwd_keys_all<false>(kp, qp, des, dkp, dqp, Tx, NQ, NQ4, A, va4, dvs);
  }
  if (J > 0) {
    for (int q = 0; q < NQ; ++q) {
      const float qv = qp[(int64_t)q * A];
      const int64_t crow = ((int64_t)b * NQ + q) * J;
      const float* dr = de + ((int64_t)b * NQ + q) * L + Tx;
      float dq = 0.f;
      for (int j = 0; j < J; ++j) {
        const float r = tanh_r(ckeys[(crow + j) * A + a] + qv);
        const float s = dr[j] * r;
        const float g = fmaf(-s, r, s);
        dvs += s;
        dq += g;
        dckeys[(crow + j) * A + a] = va4 * g;
      }
      dqp[(int64_t)q * A] = Tx > 0 ? fmaf(va4, dq, dqp[(int64_t)q * A]) : va4 * dq;
    }
  } else if (Tx == 0) {
    for (int q = 0; q < NQ; ++q) dqp[(int64_t)q * A] = 0.f;
  }
  dv_part[(int64_t)b * A + a] = fmaf(-2.f, dvs, dsum);
}

// Backward C: dvalues[b,t,c] = sum_q w[b,q,t] * dctx[b,q,c] over the shared positions, as K4's kernel C with
// weight rows of L.  grid (ceil(C/128), B).  dynamic smem: ws[NQ][Tx8] | dcs[NQ][128]
__global__ void __launch_bounds__(ATT_ACH)
joint_bwd_values_kernel(const float* __restrict__ weights, const float* __restrict__ dctx,
                        float* __restrict__ dvalues, int Tx, int L, int NQ, int C) {
  extern __shared__ float smem[];
  const int Tx8 = (Tx + ATT_VT - 1) / ATT_VT * ATT_VT;
  float* ws = smem;
  float* dcs = ws + NQ * Tx8;
  const int b = blockIdx.y;
  const int c = blockIdx.x * ATT_ACH + threadIdx.x;
  const bool ok = c < C;
  for (int i = threadIdx.x; i < NQ * Tx8; i += ATT_ACH) {
    const int q = i / Tx8, t = i - q * Tx8;
    ws[i] = t < Tx ? weights[((int64_t)b * NQ + q) * L + t] : 0.f;
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

// Backward D, the fixed-order reductions over the sentences: blocks [0, S) add the per-sentence partials of
// segment s to dseg_bias[s], blocks [S, S+J) those of candidate j to dcand_bias[j], the rest dv_part to dv.
constexpr int JA_RED = 256;
__global__ void __launch_bounds__(JA_RED)
joint_bwd_reduce_kernel(const float* __restrict__ bias_part, const float* __restrict__ dv_part, int S,
                        float* __restrict__ dv, float* __restrict__ dseg_bias, float* __restrict__ dcand_bias,
                        int B, int J, int A) {
  __shared__ float red[32];
  const int k = blockIdx.x, nb = S + J;
  if (k < nb) {
    float acc = 0.f;
    for (int b = threadIdx.x; b < B; b += JA_RED) acc += bias_part[(int64_t)b * nb + k];
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) {
      if (k < S)
        dseg_bias[k] += acc;
      else
        dcand_bias[k - S] += acc;
    }
    return;
  }
  const int a = (k - nb) * JA_RED + threadIdx.x;
  if (a >= A) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += dv_part[(int64_t)b * A + a];
  dv[a] += acc;
}

}  // namespace nm

using namespace nm;

namespace {

int joint_segs(const int64_t* seg_ends, int64_t S, int64_t Tx, const char* who, JointSegs& sg) {
  NM_REQUIRE((Tx == 0) == (S == 0), NM_E_INVALID, "%s: S=%lld segments over Tx=%lld", who, (long long)S,
             (long long)Tx);
  NM_REQUIRE(S <= JA_MAX_SEG, NM_E_UNSUPPORTED, "%s: S=%lld > %d segments", who, (long long)S, JA_MAX_SEG);
  NM_REQUIRE(S == 0 || seg_ends, NM_E_INVALID, "%s: null seg_ends", who);
  sg.n = (int)S;
  int64_t prev = 0;
  for (int s = 0; s < S; ++s) {
    NM_REQUIRE(seg_ends[s] > prev, NM_E_INVALID, "%s: segment %d is empty or out of order", who, s);
    prev = seg_ends[s];
    sg.end[s] = (int)prev;
  }
  for (int s = (int)S; s < JA_MAX_SEG; ++s) sg.end[s] = (int)Tx;
  NM_REQUIRE(prev == Tx, NM_E_INVALID, "%s: segments end at %lld, Tx=%lld", who, (long long)prev, (long long)Tx);
  return NM_OK;
}

}  // namespace

extern "C" {

int nm_joint_attention_fwd(const float* keys, const float* values, const float* mask, const int64_t* seg_ends,
                           const float* seg_bias, const float* ckeys, const float* cvalues, const float* cand_bias,
                           const float* qproj, const float* v, float* energies, float* weights, float* ctx,
                           int64_t B, int64_t Tx, int64_t S, int64_t J, int64_t NQ, int64_t A, int64_t C,
                           void* stream) {
  NM_REQUIRE(qproj && v && weights && ctx, NM_E_INVALID, "nm_joint_attention_fwd: null pointer");
  NM_REQUIRE(Tx == 0 || (keys && values && seg_bias), NM_E_INVALID,
             "nm_joint_attention_fwd: null shared-key pointer");
  NM_REQUIRE(J == 0 || (ckeys && cvalues && cand_bias), NM_E_INVALID,
             "nm_joint_attention_fwd: null candidate pointer");
  NM_REQUIRE(B > 0 && Tx >= 0 && J >= 0 && Tx + J > 0 && NQ > 0 && A > 0 && C > 0, NM_E_INVALID,
             "nm_joint_attention_fwd: bad sizes");
  NM_REQUIRE(B <= 65535, NM_E_UNSUPPORTED, "nm_joint_attention_fwd: B > 65535");
  JointSegs sg;
  const int rc = joint_segs(seg_ends, S, Tx, "nm_joint_attention_fwd", sg);
  if (rc != NM_OK) return rc;
  const size_t smem = sizeof(float) * (size_t)(A + ATT_QMAX * A + ATT_QMAX * (Tx + J));
  NM_REQUIRE(smem <= ATT_SMEM_LIMIT, NM_E_UNSUPPORTED,
             "nm_joint_attention_fwd: A=%lld Tx+J=%lld need %zu B of shared memory", (long long)A,
             (long long)(Tx + J), smem);
  static bool attr_set = false;
  if (!attr_set) {
    NM_CUDA_TRY(cudaFuncSetAttribute(joint_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    attr_set = true;
  }
  dim3 grid((unsigned)att_chunks(B, NQ), (unsigned)B);
  joint_fwd_kernel<<<grid, ATT_THREADS, smem, (cudaStream_t)stream>>>(
      keys, values, mask, sg, seg_bias, ckeys, cvalues, cand_bias, qproj, v, energies, weights, ctx, (int)Tx,
      (int)J, (int)NQ, (int)A, (int)C);
  NM_LAUNCH_CHECK("nm_joint_attention_fwd");
  return NM_OK;
}

int nm_joint_attention_bwd(const float* keys, const float* values, const float* mask, const int64_t* seg_ends,
                           const float* ckeys, const float* cvalues, const float* qproj, const float* v,
                           const float* energies, const float* weights, const float* dctx, float* dkeys,
                           float* dvalues, float* dqproj, float* dckeys, float* dcvalues, float* dv,
                           float* dseg_bias, float* dcand_bias, float* work, int64_t B, int64_t Tx, int64_t S,
                           int64_t J, int64_t NQ, int64_t A, int64_t C, void* stream) {
  NM_REQUIRE(qproj && v && energies && weights && dctx && dqproj && dv && work, NM_E_INVALID,
             "nm_joint_attention_bwd: null pointer");
  NM_REQUIRE(Tx == 0 || (keys && values && dkeys && dvalues && dseg_bias), NM_E_INVALID,
             "nm_joint_attention_bwd: null shared-key pointer");
  NM_REQUIRE(J == 0 || (ckeys && cvalues && dckeys && dcvalues && dcand_bias), NM_E_INVALID,
             "nm_joint_attention_bwd: null candidate pointer");
  NM_REQUIRE(B > 0 && Tx >= 0 && J >= 0 && Tx + J > 0 && NQ > 0 && A > 0 && C > 0, NM_E_INVALID,
             "nm_joint_attention_bwd: bad sizes");
  NM_REQUIRE(B <= 65535, NM_E_UNSUPPORTED, "nm_joint_attention_bwd: B > 65535");
  JointSegs sg;
  const int rc = joint_segs(seg_ends, S, Tx, "nm_joint_attention_bwd", sg);
  if (rc != NM_OK) return rc;
  const int64_t L = Tx + J;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem_a = sizeof(float) * (size_t)(ATT_QMAX * C + ATT_QMAX * L);
  const size_t smem_b = sizeof(float) * (size_t)(Tx * ((NQ + 3) & ~3));
  const size_t smem_c = sizeof(float) * (size_t)(NQ * ceil_div(Tx, ATT_VT) * ATT_VT + NQ * ATT_ACH);
  NM_REQUIRE(smem_a <= ATT_SMEM_LIMIT && smem_b <= ATT_SMEM_LIMIT && (Tx == 0 || smem_c <= ATT_SMEM_LIMIT),
             NM_E_UNSUPPORTED,
             "nm_joint_attention_bwd: NQ=%lld Tx=%lld J=%lld C=%lld need %zu/%zu/%zu B of shared memory",
             (long long)NQ, (long long)Tx, (long long)J, (long long)C, smem_a, smem_b, smem_c);
  static bool attr_set = false;
  if (!attr_set) {
    NM_CUDA_TRY(cudaFuncSetAttribute(joint_bwd_energy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    NM_CUDA_TRY(cudaFuncSetAttribute(joint_bwd_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    NM_CUDA_TRY(cudaFuncSetAttribute(joint_bwd_values_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    attr_set = true;
  }
  float* de = work;
  float* dv_part = de + B * NQ * L;
  float* bias_part = dv_part + B * A;
  dim3 grid_a((unsigned)att_chunks(B, NQ), (unsigned)B);
  joint_bwd_energy_kernel<<<grid_a, ATT_THREADS, smem_a, s>>>(values, mask, cvalues, energies, weights, dctx, de,
                                                             dcvalues, (int)Tx, (int)J, (int)NQ, (int)C);
  NM_LAUNCH_CHECK("nm_joint_attention_bwd(energy)");
  dim3 grid_b((unsigned)ceil_div(A, ATT_ACH), (unsigned)B);
  joint_bwd_keys_kernel<<<grid_b, ATT_ACH, smem_b, s>>>(keys, ckeys, qproj, v, de, dkeys, dckeys, dqproj, dv_part,
                                                       sg, bias_part, (int)Tx, (int)J, (int)NQ, (int)A);
  NM_LAUNCH_CHECK("nm_joint_attention_bwd(keys)");
  if (Tx > 0) {
    dim3 grid_c((unsigned)ceil_div(C, ATT_ACH), (unsigned)B);
    joint_bwd_values_kernel<<<grid_c, ATT_ACH, smem_c, s>>>(weights, dctx, dvalues, (int)Tx, (int)L, (int)NQ,
                                                           (int)C);
    NM_LAUNCH_CHECK("nm_joint_attention_bwd(values)");
  }
  const unsigned nred = (unsigned)(S + J + ceil_div(A, JA_RED));
  joint_bwd_reduce_kernel<<<nred, JA_RED, 0, s>>>(bias_part, dv_part, (int)S, dv, dseg_bias, dcand_bias, (int)B,
                                                  (int)J, (int)A);
  NM_LAUNCH_CHECK("nm_joint_attention_bwd(reduce)");
  return NM_OK;
}

}  // extern "C"
