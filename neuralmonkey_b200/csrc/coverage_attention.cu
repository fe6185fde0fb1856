// Coverage attention (Tu et al. 2016), attention/coverage.py:37-61 of the reference on top of the feed-forward
// attention step (attention/feed_forward.py:125-166), for NQ query steps of a decoder at once.
//
//   fert[b,t]  = 1e-8 + N * sigmoid(sum_c fw[c] S[b,t,c])
//   sum[b,0,t] = cov_in[b,t] (0 when absent),   sum[b,q+1,t] = sum[b,q,t] + w[b,q,t]
//   cov[b,q,t] = sum[b,q,t] / fert[b,t] * m[b,t]
//   e[b,q,t]   = sum_a v[a] tanh(keys[b,t,a] + qproj[b,q,a] + cw[a] cov[b,q,t])          (no energy bias)
//   p          = softmax_t(e);   w = p*m / (sum_t p*m + 1e-8)   (w = p without a mask)
//   ctx[b,q]   = sum_t w[b,q,t] S[b,t,:];   cov_out[b,t] = sum[b,NQ,t]
//
// Step q's energies depend on the weights of the steps before it, so the queries are a scan: one CTA walks a
// sentence's NQ steps in order with the running sum on chip, and the backward walks them in reverse, carrying
// R[t], the gradient that reaches the running sum.  Every step does the same arithmetic in the same order
// whatever NQ is, and cov_out is the running sum itself, so T calls of one step each chained through
// cov_in / cov_out give the bits of one call over T steps.
//
// K4's one-SFU tanh (e^{2k} e^{2q} staged once per element) does not carry over: the coverage term varies per
// (q, t, a), so factoring it costs one EX2 per element, as the plain form does.  Both kernels use the plain
// two-SFU form 1 - 2/(1 + e^{2x}), which saturates correctly for any x and needs no range check.
//
// The backward uses no float atomics: per-element gradients have one owner, and dv, dcw and the fertility
// weight gradient are summed per sentence and then over the sentences in a fixed order.
#include "attention_common.cuh"

namespace nm {

constexpr int COV_THREADS = 512;
constexpr int COV_WARPS = COV_THREADS / 32;
constexpr int FERT_THREADS = 256;

// grid (B).  dynamic smem: vs[A] | cws[A] | ys[A] | sum[Tx] | covs[Tx] | es[Tx] | ws[Tx]
__global__ void __launch_bounds__(COV_THREADS)
coverage_fwd_kernel(const float* __restrict__ keys, const float* __restrict__ values,
                    const float* __restrict__ mask, const float* __restrict__ fert,
                    const float* __restrict__ qproj, const float* __restrict__ v, const float* __restrict__ cw,
                    const float* __restrict__ cov_in, float* __restrict__ energies, float* __restrict__ weights,
                    float* __restrict__ coverage, float* __restrict__ ctx, float* __restrict__ cov_out,
                    int Tx, int NQ, int A, int C) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  float* v2s = smem;
  float* cws = v2s + A;
  float* ys = cws + A;
  float* sum = ys + A;
  float* covs = sum + Tx;
  float* es = covs + Tx;
  float* ws = es + Tx;
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* kb = keys + (int64_t)b * Tx * A;
  const float* fb = fert + (int64_t)b * Tx;
  const float* mb = mask ? mask + (int64_t)b * Tx : nullptr;

  // e = sum_a v tanh = sum_a v + sum_a (-2v) r
  float vsum = 0.f;
  for (int a = threadIdx.x; a < A; a += COV_THREADS) {
    v2s[a] = -2.f * v[a];
    cws[a] = cw[a];
    vsum += v[a];
  }
  for (int t = threadIdx.x; t < Tx; t += COV_THREADS) sum[t] = cov_in ? cov_in[(int64_t)b * Tx + t] : 0.f;
  vsum = block_sum(vsum, red);

  for (int q = 0; q < NQ; ++q) {
    const int64_t row = ((int64_t)b * NQ + q) * Tx;
    for (int a = threadIdx.x; a < A; a += COV_THREADS) ys[a] = qproj[((int64_t)b * NQ + q) * A + a];
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
      const float c = sum[t] / fb[t] * (mb ? mb[t] : 1.f);
      covs[t] = c;
      coverage[row + t] = c;
    }
    __syncthreads();

    for (int t = warp; t < Tx; t += COV_WARPS) {
      const float* kr = kb + (int64_t)t * A;
      const float c = covs[t];
      float acc = 0.f;
      for (int a = lane; a < A; a += 32) acc = fmaf(v2s[a], tanh_r(fmaf(cws[a], c, kr[a] + ys[a])), acc);
      acc = warp_sum(acc);
      if (lane == 0) es[t] = acc + vsum;
    }
    __syncthreads();

    // softmax over Tx, mask and renormalise
    float mx = -INFINITY;
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) mx = fmaxf(mx, es[t]);
    mx = block_max(mx, red);
    float s = 0.f;
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) s += expf(es[t] - mx);
    s = block_sum(s, red);
    float pm = 0.f;
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
      const float e = es[t];
      energies[row + t] = e;
      float p = expf(e - mx) / s;
      if (mb) p *= mb[t];
      ws[t] = p;
      pm += p;
    }
    if (mb) {
      const float norm = block_sum(pm, red) + 1e-8f;
      for (int t = threadIdx.x; t < Tx; t += COV_THREADS) ws[t] = ws[t] / norm;
    }
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
      const float w = ws[t];
      weights[row + t] = w;
      sum[t] += w;
    }
    __syncthreads();

    // ctx[b,q,c] = sum_t w[t] values[b,t,c]
    const float* vb = values + (int64_t)b * Tx * C;
    for (int c = threadIdx.x; c < C; c += COV_THREADS) {
      float acc = 0.f;
      for (int t = 0; t < Tx; ++t) acc = fmaf(ws[t], vb[(int64_t)t * C + c], acc);
      ctx[((int64_t)b * NQ + q) * C + c] = acc;
    }
  }
  for (int t = threadIdx.x; t < Tx; t += COV_THREADS) cov_out[(int64_t)b * Tx + t] = sum[t];
}

// Reverse scan.  grid (B).  Per step q, from NQ-1 down to 0:
//   dw[t]  = dctx[q] . S[t] + R[t];   de = the softmax / mask / renormalisation backward of dw (K4's)
//   g      = de[t] v[a] (1 - tanh^2) = 4 de v r (1-r)
//   dkeys[t,a] += g,  dqproj[q,a] = sum_t g,  dv[a] += de tanh,  dcw[a] += g cov[q,t]
//   dcov[t] = sum_a g cw[a];   R[t] += dcov m / fert;   dfert[t] -= dcov cov[q,t] / fert
// Warp w owns the rows t = w (mod COV_WARPS) for the whole scan, so its dkeys rows are read-modify-written by
// the same lanes every step, and it keeps its share of dqproj / dv / dcw in its own shared-memory row.
// dynamic smem: vs[A] | cws[A] | ys[A] | dcs[C] | R[Tx] | dws[Tx] | des[Tx] | covs[Tx] | dfs[Tx] | dcv[Tx] |
//               pdy[W][A] | pdv[W][A] | pdc[W][A]
__global__ void __launch_bounds__(COV_THREADS)
coverage_bwd_kernel(const float* __restrict__ keys, const float* __restrict__ values,
                    const float* __restrict__ mask, const float* __restrict__ fert,
                    const float* __restrict__ qproj, const float* __restrict__ v, const float* __restrict__ cw,
                    const float* __restrict__ energies, const float* __restrict__ weights,
                    const float* __restrict__ coverage, const float* __restrict__ dctx,
                    const float* __restrict__ dcov_out, float* __restrict__ dkeys, float* __restrict__ dqproj,
                    float* __restrict__ dfert, float* __restrict__ dcov_in, float* __restrict__ dv_part,
                    float* __restrict__ dcw_part, int Tx, int NQ, int A, int C) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  float* vs = smem;
  float* cws = vs + A;
  float* ys = cws + A;
  float* dcs = ys + A;
  float* R = dcs + C;
  float* dws = R + Tx;
  float* des = dws + Tx;
  float* covs = des + Tx;
  float* dfs = covs + Tx;
  float* dcv = dfs + Tx;
  float* pdy = dcv + Tx;
  float* pdv = pdy + COV_WARPS * A;
  float* pdc = pdv + COV_WARPS * A;
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* kb = keys + (int64_t)b * Tx * A;
  const float* vb = values + (int64_t)b * Tx * C;
  const float* fb = fert + (int64_t)b * Tx;
  const float* mb = mask ? mask + (int64_t)b * Tx : nullptr;
  float* dkb = dkeys + (int64_t)b * Tx * A;

  for (int a = threadIdx.x; a < A; a += COV_THREADS) {
    vs[a] = v[a];
    cws[a] = cw[a];
  }
  for (int i = threadIdx.x; i < 3 * COV_WARPS * A; i += COV_THREADS) pdy[i] = 0.f;
  for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
    R[t] = dcov_out ? dcov_out[(int64_t)b * Tx + t] : 0.f;
    dfs[t] = 0.f;
  }

  for (int q = NQ - 1; q >= 0; --q) {
    const int64_t row = ((int64_t)b * NQ + q) * Tx;
    for (int a = threadIdx.x; a < A; a += COV_THREADS) ys[a] = qproj[((int64_t)b * NQ + q) * A + a];
    for (int c = threadIdx.x; c < C; c += COV_THREADS) dcs[c] = dctx[((int64_t)b * NQ + q) * C + c];
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) covs[t] = coverage[row + t];
    __syncthreads();

    for (int t = warp; t < Tx; t += COV_WARPS) {
      const float* vr = vb + (int64_t)t * C;
      float acc = 0.f;
      for (int c = lane; c < C; c += 32) acc = fmaf(vr[c], dcs[c], acc);
      acc = warp_sum(acc);
      if (lane == 0) dws[t] = acc + R[t];
    }
    __syncthreads();

    // de from dw: recompute p and the renormaliser
    const float* er = energies + row;
    const float* wr = weights + row;
    float mx = -INFINITY;
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) mx = fmaxf(mx, er[t]);
    mx = block_max(mx, red);
    float s = 0.f;
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) s += expf(er[t] - mx);
    s = block_sum(s, red);
    float norm = 1.f, dot_dw_w = 0.f;
    if (mb) {
      float pm = 0.f;
      for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
        pm += expf(er[t] - mx) / s * mb[t];
        dot_dw_w += dws[t] * wr[t];
      }
      norm = block_sum(pm, red) + 1e-8f;
      dot_dw_w = block_sum(dot_dw_w, red);
    }
    // dp_t = m_t (dw_t - sum dw.w) / N   (no mask: dp = dw)
    float pdp = 0.f;
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
      const float p = expf(er[t] - mx) / s;
      float dp = dws[t];
      if (mb) dp = mb[t] * (dp - dot_dw_w) / norm;
      dws[t] = dp;
      pdp += p * dp;
    }
    pdp = block_sum(pdp, red);
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) des[t] = expf(er[t] - mx) / s * (dws[t] - pdp);
    __syncthreads();

    float* py = pdy + warp * A;
    float* pv = pdv + warp * A;
    float* pc = pdc + warp * A;
    const bool first = q == NQ - 1;
    for (int t = warp; t < Tx; t += COV_WARPS) {
      const float* kr = kb + (int64_t)t * A;
      float* dkr = dkb + (int64_t)t * A;
      const float c = covs[t], d = des[t];
      float dcov = 0.f;
      for (int a = lane; a < A; a += 32) {
        const float r = tanh_r(fmaf(cws[a], c, kr[a] + ys[a]));
        const float sr = d * r;
        const float g = 4.f * vs[a] * fmaf(-sr, r, sr);
        dkr[a] = first ? g : dkr[a] + g;
        dcov = fmaf(g, cws[a], dcov);
        py[a] += g;
        pv[a] = fmaf(-2.f, sr, pv[a] + d);
        pc[a] = fmaf(g, c, pc[a]);
      }
      dcov = warp_sum(dcov);
      if (lane == 0) dcv[t] = dcov;
    }
    __syncthreads();

    for (int a = threadIdx.x; a < A; a += COV_THREADS) {
      float acc = 0.f;
      for (int w = 0; w < COV_WARPS; ++w) {
        acc += pdy[w * A + a];
        pdy[w * A + a] = 0.f;
      }
      dqproj[((int64_t)b * NQ + q) * A + a] = acc;
    }
    for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
      const float f = fb[t], dc = dcv[t];
      R[t] = fmaf(dc, (mb ? mb[t] : 1.f) / f, R[t]);
      dfs[t] = fmaf(-dc, covs[t] / f, dfs[t]);
    }
    __syncthreads();
  }

  for (int t = threadIdx.x; t < Tx; t += COV_THREADS) {
    if (dcov_in) dcov_in[(int64_t)b * Tx + t] = R[t];
    dfert[(int64_t)b * Tx + t] = dfs[t];
  }
  for (int a = threadIdx.x; a < A; a += COV_THREADS) {
    float sv = 0.f, sc = 0.f;
    for (int w = 0; w < COV_WARPS; ++w) {
      sv += pdv[w * A + a];
      sc += pdc[w * A + a];
    }
    dv_part[(int64_t)b * A + a] = sv;
    dcw_part[(int64_t)b * A + a] = sc;
  }
}

// fert[row] = 1e-8 + N sigmoid(fw . S[row]): one warp per row of [B*Tx, C].
__global__ void __launch_bounds__(FERT_THREADS)
fertility_fwd_kernel(const float* __restrict__ states, const float* __restrict__ fw, float max_fert,
                     float* __restrict__ fert, int64_t rows, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (FERT_THREADS / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* sr = states + row * C;
  float z = 0.f;
  for (int c = lane; c < C; c += 32) z = fmaf(fw[c], sr[c], z);
  z = warp_sum(z);
  if (lane == 0) fert[row] = 1e-8f + max_fert * sigmoidf_(z);
}

// grid (B): dz[t] = dfert N sig (1 - sig), dstates[b,t,:] = dz fw, part[b,c] = sum_t dz[t] S[b,t,c].
// dynamic smem: dzs[Tx]
__global__ void __launch_bounds__(FERT_THREADS)
fertility_bwd_kernel(const float* __restrict__ states, const float* __restrict__ fw, float max_fert,
                     const float* __restrict__ dfert, float* __restrict__ dstates, float* __restrict__ part,
                     int Tx, int C) {
  extern __shared__ float dzs[];
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* sb = states + (int64_t)b * Tx * C;
  for (int t = warp; t < Tx; t += FERT_THREADS / 32) {
    const float* sr = sb + (int64_t)t * C;
    float z = 0.f;
    for (int c = lane; c < C; c += 32) z = fmaf(fw[c], sr[c], z);
    z = warp_sum(z);
    const float sg = sigmoidf_(z);
    const float dz = dfert[(int64_t)b * Tx + t] * max_fert * sg * (1.f - sg);
    float* dr = dstates + ((int64_t)b * Tx + t) * C;
    for (int c = lane; c < C; c += 32) dr[c] = dz * fw[c];
    if (lane == 0) dzs[t] = dz;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += FERT_THREADS) {
    float acc = 0.f;
    for (int t = 0; t < Tx; ++t) acc = fmaf(dzs[t], sb[(int64_t)t * C + c], acc);
    part[(int64_t)b * C + c] = acc;
  }
}

// out[n] += sum_b part[b,n], b in order.
__global__ void rows_sum_kernel(const float* __restrict__ part, float* __restrict__ out, int B, int N) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) acc += part[(int64_t)b * N + n];
  out[n] += acc;
}

static size_t cov_fwd_smem(int64_t Tx, int64_t A) { return sizeof(float) * (size_t)(3 * A + 4 * Tx); }
static size_t cov_bwd_smem(int64_t Tx, int64_t A, int64_t C) {
  return sizeof(float) * (size_t)(3 * A + C + 6 * Tx + 3 * COV_WARPS * A);
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_coverage_fertility_fwd(const float* states, const float* fertility_w, float max_fertility, float* fert,
                              int64_t B, int64_t Tx, int64_t C, void* stream) {
  NM_REQUIRE(states && fertility_w && fert, NM_E_INVALID, "nm_coverage_fertility_fwd: null pointer");
  NM_REQUIRE(B > 0 && Tx > 0 && C > 0, NM_E_INVALID, "nm_coverage_fertility_fwd: bad sizes");
  const int64_t rows = B * Tx, per = FERT_THREADS / 32;
  NM_REQUIRE(ceil_div(rows, per) <= INT32_MAX, NM_E_UNSUPPORTED, "nm_coverage_fertility_fwd: B*Tx too large");
  fertility_fwd_kernel<<<(unsigned)ceil_div(rows, per), FERT_THREADS, 0, (cudaStream_t)stream>>>(
      states, fertility_w, max_fertility, fert, rows, (int)C);
  NM_LAUNCH_CHECK("nm_coverage_fertility_fwd");
  return NM_OK;
}

int nm_coverage_fertility_bwd(const float* states, const float* fertility_w, float max_fertility,
                              const float* dfert, float* dstates, float* dfertility_w, float* work, int64_t B,
                              int64_t Tx, int64_t C, void* stream) {
  NM_REQUIRE(states && fertility_w && dfert && dstates && dfertility_w && work, NM_E_INVALID,
             "nm_coverage_fertility_bwd: null pointer");
  NM_REQUIRE(B > 0 && Tx > 0 && C > 0, NM_E_INVALID, "nm_coverage_fertility_bwd: bad sizes");
  NM_REQUIRE(B <= INT32_MAX && sizeof(float) * Tx <= 48 * 1024, NM_E_UNSUPPORTED,
             "nm_coverage_fertility_bwd: Tx=%lld exceeds the limit of 12288", (long long)Tx);
  cudaStream_t s = (cudaStream_t)stream;
  fertility_bwd_kernel<<<(unsigned)B, FERT_THREADS, sizeof(float) * Tx, s>>>(
      states, fertility_w, max_fertility, dfert, dstates, work, (int)Tx, (int)C);
  NM_LAUNCH_CHECK("nm_coverage_fertility_bwd");
  rows_sum_kernel<<<(unsigned)ceil_div(C, 128), 128, 0, s>>>(work, dfertility_w, (int)B, (int)C);
  NM_LAUNCH_CHECK("nm_coverage_fertility_bwd(reduce)");
  return NM_OK;
}

int nm_coverage_attention_fwd(const float* keys, const float* values, const float* mask, const float* fert,
                              const float* qproj, const float* v, const float* coverage_w, const float* cov_in,
                              float* energies, float* weights, float* coverage, float* ctx, float* cov_out,
                              int64_t B, int64_t Tx, int64_t NQ, int64_t A, int64_t C, void* stream) {
  NM_REQUIRE(keys && values && fert && qproj && v && coverage_w && energies && weights && coverage && ctx &&
                 cov_out,
             NM_E_INVALID, "nm_coverage_attention_fwd: null pointer");
  NM_REQUIRE(B > 0 && Tx > 0 && NQ > 0 && A > 0 && C > 0, NM_E_INVALID, "nm_coverage_attention_fwd: bad sizes");
  NM_REQUIRE(B <= INT32_MAX, NM_E_UNSUPPORTED, "nm_coverage_attention_fwd: B too large");
  const size_t smem = cov_fwd_smem(Tx, A);
  NM_REQUIRE(smem <= ATT_SMEM_LIMIT, NM_E_UNSUPPORTED,
             "nm_coverage_attention_fwd: A=%lld Tx=%lld need %zu B of shared memory, the limit is %zu",
             (long long)A, (long long)Tx, smem, ATT_SMEM_LIMIT);
  static bool attr_set = false;
  if (!attr_set) {
    NM_CUDA_TRY(cudaFuncSetAttribute(coverage_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    attr_set = true;
  }
  coverage_fwd_kernel<<<(unsigned)B, COV_THREADS, smem, (cudaStream_t)stream>>>(
      keys, values, mask, fert, qproj, v, coverage_w, cov_in, energies, weights, coverage, ctx, cov_out, (int)Tx,
      (int)NQ, (int)A, (int)C);
  NM_LAUNCH_CHECK("nm_coverage_attention_fwd");
  return NM_OK;
}

int nm_coverage_attention_bwd(const float* keys, const float* values, const float* mask, const float* fert,
                              const float* qproj, const float* v, const float* coverage_w, const float* energies,
                              const float* weights, const float* coverage, const float* dctx,
                              const float* dcov_out, float* dkeys, float* dvalues, float* dqproj, float* dfert,
                              float* dcov_in, float* dv, float* dcoverage_w, float* work, int64_t B, int64_t Tx,
                              int64_t NQ, int64_t A, int64_t C, void* stream) {
  NM_REQUIRE(keys && values && fert && qproj && v && coverage_w && energies && weights && coverage && dctx &&
                 dkeys && dvalues && dqproj && dfert && dv && dcoverage_w && work,
             NM_E_INVALID, "nm_coverage_attention_bwd: null pointer");
  NM_REQUIRE(B > 0 && Tx > 0 && NQ > 0 && A > 0 && C > 0, NM_E_INVALID, "nm_coverage_attention_bwd: bad sizes");
  NM_REQUIRE(B <= 65535, NM_E_UNSUPPORTED, "nm_coverage_attention_bwd: B > 65535");
  const size_t smem = cov_bwd_smem(Tx, A, C);
  NM_REQUIRE(smem <= ATT_SMEM_LIMIT, NM_E_UNSUPPORTED,
             "nm_coverage_attention_bwd: A=%lld Tx=%lld C=%lld need %zu B of shared memory, the limit is %zu",
             (long long)A, (long long)Tx, (long long)C, smem, ATT_SMEM_LIMIT);
  const size_t smem_values = att_values_smem(Tx, NQ);
  NM_REQUIRE(smem_values <= ATT_SMEM_LIMIT, NM_E_UNSUPPORTED,
             "nm_coverage_attention_bwd: NQ=%lld Tx=%lld need %zu B of shared memory, the limit is %zu",
             (long long)NQ, (long long)Tx, smem_values, ATT_SMEM_LIMIT);
  cudaStream_t s = (cudaStream_t)stream;
  static bool attr_set = false;
  if (!attr_set) {
    NM_CUDA_TRY(cudaFuncSetAttribute(coverage_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)ATT_SMEM_LIMIT));
    attr_set = true;
  }
  float* dv_part = work;
  float* dcw_part = work + B * A;
  coverage_bwd_kernel<<<(unsigned)B, COV_THREADS, smem, s>>>(
      keys, values, mask, fert, qproj, v, coverage_w, energies, weights, coverage, dctx, dcov_out, dkeys, dqproj,
      dfert, dcov_in, dv_part, dcw_part, (int)Tx, (int)NQ, (int)A, (int)C);
  NM_LAUNCH_CHECK("nm_coverage_attention_bwd");
  rows_sum_kernel<<<(unsigned)ceil_div(A, 128), 128, 0, s>>>(dv_part, dv, (int)B, (int)A);
  NM_LAUNCH_CHECK("nm_coverage_attention_bwd(dv)");
  rows_sum_kernel<<<(unsigned)ceil_div(A, 128), 128, 0, s>>>(dcw_part, dcoverage_w, (int)B, (int)A);
  NM_LAUNCH_CHECK("nm_coverage_attention_bwd(dcw)");
  return att_values_grad(weights, dctx, dvalues, B, Tx, NQ, C, s);
}

}  // extern "C"
