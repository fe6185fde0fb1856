// One layer of the convolutional seq2seq encoder (encoders/facebook_conv.py, Gehring et al. 2017): a 1-D convolution
// over time with 2F output channels, the gated linear unit and the residual add,
//   z = conv1d_same(x, W) + b            x [B,T,F], W [k,F,2F], b [2F], z [B,T,2F]
//   y = z[..., :F] * sigmoid(z[..., F:]) + x
// TF's SAME padding at stride 1: pb = (k-1)/2 zeros before, k-1-pb after, and zeros only outside [0, T) of each
// sequence (padded positions inside the batch take part).
//
// Implicit GEMM over the M = B*T positions, K = k*Cin, no patch matrix:
//   A(m, (j, c)) = x[b, t + j - pb, c]  = x[(m - pb)*Cin + (j*Cin + c)] when 0 <= t + j - pb < T, else 0
// so row m of A is one contiguous span of x cut at the sequence ends.  The forward's tile holds output column o and
// its gate column o + F together, so the bias, the GLU and the residual run in the epilogue.  The data gradient is
// the same product over dZ with W's taps reversed and its channel axes swapped (pads k-1-pb before), plus dY in the
// epilogue; the weight gradient is the transposed product dW[(j, c), o] = sum_m A(m, (j, c)) dZ(m, o), split over
// CTAs along m into a caller-owned workspace and summed in a fixed order, with one extra row of ones in A for the
// bias gradient.
//
// Two engines, selected like nm_conv2d_*'s: wgmma with TF32 operands (cvt.rna, 128-byte swizzled K-major tiles,
// fp32 accumulators) and exact fp32 FMA tiles on the CUDA cores (NM_GEMM_SIMT).
#include "gemm_simt.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace nm {

struct GluGeom {
  int T, Cin, Cout;   // input [M/T, T, Cin], output [M/T, T, Cout]
  int k, pb;          // window and the zeros before each sequence
  int F;              // GLU width: the forward's Cout is 2F; the data gradient's Cin is 2F
  int Kd;             // k * Cin
  int flip;           // 0: w is [k, Cin, Cout]; 1: w is the forward filter [k, Cout, Cin], taps reversed
  int64_t M;          // B * T
};

// A(m, gk) of position m (t = m mod T); gk < Kd
__device__ __forceinline__ float glu_a(const float* __restrict__ x, const GluGeom& g, int64_t m, int t, int gk) {
  const int ts = t + gk / g.Cin - g.pb;
  return (ts >= 0 && ts < g.T) ? __ldg(x + (m - g.pb) * g.Cin + gk) : 0.f;
}

// B(gk, o); gk < Kd, o < Cout
__device__ __forceinline__ float glu_b(const float* __restrict__ w, const GluGeom& g, int gk, int o) {
  if (g.flip) {
    const int j = gk / g.Cin, c = gk - j * g.Cin;
    return __ldg(w + ((int64_t)(g.k - 1 - j) * g.Cout + o) * g.Cin + c);
  }
  return __ldg(w + (int64_t)gk * g.Cout + o);
}

// ------------------------------------------------------------------------------------------------------------
// wgmma engine: 128 x 128 output tile, 2 consumer warpgroups of 64 rows, 32-wide k-blocks in a 2-stage ring.
// All 256 threads gather the next k-block while the tensor cores work on the current one.  In the forward the
// tile's columns [0, 64) are the linear halves o0 + n and [64, 128) their gates F + o0 + n, so each thread holds a
// column and its gate in accumulators i and i + 8.
// ------------------------------------------------------------------------------------------------------------
constexpr int GT_BM = 128, GT_BN = 128, GT_BK = 32, GT_THREADS = 256;
constexpr int GT_A_BYTES = GT_BM * 128, GT_B_BYTES = GT_BN * 128;
constexpr int GT_STAGE = GT_A_BYTES + GT_B_BYTES;
constexpr int GT_SMEM = 2 * GT_STAGE + 1024;   // + slack for the 1 KB alignment of the swizzled tiles

__device__ __forceinline__ void gt_mma(float (&acc)[64], uint32_t stage_addr, int wg) {
  const uint32_t a = stage_addr + wg * 64 * 128, b = stage_addr + GT_A_BYTES;
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) Wgmma<128, 4>::mma(acc, gmma_desc_sw128(a + k * 32), gmma_desc_sw128(b + k * 32));
  wgmma_commit();
}

enum { GLU_FWD = 0, GLU_DGRAD = 1 };

// GLU_FWD:   y[m, f] = z_lin * sigmoid(z_gate) + res[m, f], z = A.B + bias (z stored when non-null)
// GLU_DGRAD: y[m, o] = (A.B)[m, o] + res[m, o]
template <int MODE>
__global__ void __launch_bounds__(GT_THREADS)
glu_conv_tc_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                   const float* __restrict__ res, float* __restrict__ y, float* __restrict__ z, GluGeom g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * GT_BM;
  const int c0 = blockIdx.y * (MODE == GLU_FWD ? GT_BN / 2 : GT_BN);
  const int num_kb = (g.Kd + GT_BK - 1) / GT_BK;
  const bool avec = (g.Cin & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const bool bvec = (g.Cin & 3) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0;

  // A: thread owns row tid/2 and the 16 k values of half tid&1
  const int arow = tid >> 1, ahalf = tid & 1;
  const int64_t am = m0 + arow;
  const bool arow_ok = am < g.M;
  const int at = arow_ok ? (int)(am % g.T) : 0;
  const int64_t abase = (am - g.pb) * g.Cin;

  auto gather = [&](int kb, uint8_t* st) {
    const int gk0 = kb * GT_BK + ahalf * 16;
    if (avec) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gk = gk0 + 4 * j;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (arow_ok && gk < g.Kd) {
          const int ts = at + gk / g.Cin - g.pb;
          if (ts >= 0 && ts < g.T) v = __ldg(reinterpret_cast<const float4*>(x + abase + gk));
        }
        sw128_store4(st, arow, ahalf * 4 + j, v);
      }
    } else {
#pragma unroll 4
      for (int j = 0; j < 16; ++j) {
        const int gk = gk0 + j;
        sw128_store1(st, arow, ahalf * 16 + j, (arow_ok && gk < g.Kd) ? glu_a(x, g, am, at, gk) : 0.f);
      }
    }
    uint8_t* bt = st + GT_A_BYTES;
    if (MODE == GLU_FWD) {
      // B: 128 tile columns x 32 k values; consecutive threads take consecutive columns (w is [Kd, 2F])
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int it = tid + GT_THREADS * j;
        const int n = it & 127, word = it >> 7;
        const int gk = kb * GT_BK + word, f = c0 + (n & 63);
        sw128_store1(bt, n, word, (gk < g.Kd && f < g.F) ? glu_b(w, g, gk, n < 64 ? f : g.F + f) : 0.f);
      }
    } else {
      // B: thread owns column tid/2 and 16 k values, contiguous in the flipped filter within a tap
      const int o = c0 + arow;
      if (bvec) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int gk = gk0 + 4 * j;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (o < g.Cout && gk < g.Kd) {
            const int tap = gk / g.Cin, c = gk - tap * g.Cin;
            v = __ldg(reinterpret_cast<const float4*>(w + ((int64_t)(g.k - 1 - tap) * g.Cout + o) * g.Cin + c));
          }
          sw128_store4(bt, arow, ahalf * 4 + j, v);
        }
      } else {
#pragma unroll 4
        for (int j = 0; j < 16; ++j) {
          const int gk = gk0 + j;
          sw128_store1(bt, arow, ahalf * 16 + j, (o < g.Cout && gk < g.Kd) ? glu_b(w, g, gk, o) : 0.f);
        }
      }
    }
  };

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  const int wg = tid >> 7;

  gather(0, smem);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb & 1;
    gt_mma(acc, sbase + s * GT_STAGE, wg);
    // the other stage was last read by the products of kb-1, which completed before the barrier below
    if (kb + 1 < num_kb) gather(kb + 1, smem + (s ^ 1) * GT_STAGE);
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  }

  const int lane = tid & 31, wq = (tid >> 5) & 3;
  const int64_t r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
  if (MODE == GLU_FWD) {
    const int64_t F = g.F;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t m = r0 + 8 * h;
        if (m >= g.M) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int f = c0 + 8 * i + 2 * (lane & 3) + e;
          if (f >= g.F) continue;
          const float zl = acc[4 * i + 2 * h + e] + __ldg(bias + f);
          const float zg = acc[4 * (i + 8) + 2 * h + e] + __ldg(bias + F + f);
          if (z) {
            z[m * 2 * F + f] = zl;
            z[m * 2 * F + F + f] = zg;
          }
          y[m * F + f] = zl * sigmoidf_(zg) + __ldg(res + m * F + f);
        }
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t m = r0 + 8 * h;
        if (m >= g.M) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int o = c0 + 8 * i + 2 * (lane & 3) + e;
          if (o < g.Cout) y[m * g.Cout + o] = acc[4 * i + 2 * h + e] + __ldg(res + m * g.Cout + o);
        }
      }
    }
  }
}

// Weight gradient partials: ws[split][r][o] = sum over this split's positions of A'(r, m) dZ(m, o), where
// A'(r, m) = A(m, r) for r < Kd and A'(Kd, m) = 1 (the bias row).  128 rows x 128 columns per CTA.
__global__ void __launch_bounds__(GT_THREADS)
glu_wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ dz, float* __restrict__ ws, GluGeom g,
                    int kb_per_split) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ int tpos[2][GT_BK];      // t of each position of a k-block, -1 past M
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;
  const int rows = g.Kd + 1;
  const int r0 = blockIdx.y * GT_BM;
  const int o0 = blockIdx.x * GT_BN;
  const int total_kb = (int)((g.M + GT_BK - 1) / GT_BK);
  const int kb0 = blockIdx.z * kb_per_split;
  const int num_kb = min(total_kb, kb0 + kb_per_split) - kb0;

  // A': thread owns row tid & 127 and the words (tid >> 7) + 2j
  const int arow = tid & 127, aw = tid >> 7;
  const int gr = r0 + arow;
  const bool is_bias = gr == g.Kd, row_ok = gr < g.Kd;
  const int shift = row_ok ? gr / g.Cin - g.pb : 0;      // tap offset of this row
  const int c = row_ok ? gr - (gr / g.Cin) * g.Cin : 0;

  auto decode = [&](int kb, int buf) {
    if (tid < GT_BK) {
      const int64_t m = (int64_t)(kb0 + kb) * GT_BK + tid;
      tpos[buf][tid] = m < g.M ? (int)(m % g.T) : -1;
    }
  };
  auto gather = [&](int kb, int buf, uint8_t* st) {
    const int64_t mb = (int64_t)(kb0 + kb) * GT_BK;
#pragma unroll 4
    for (int j = 0; j < 16; ++j) {
      const int word = aw + 2 * j;
      const int t = tpos[buf][word];
      float v = 0.f;
      if (t >= 0) {
        if (is_bias) {
          v = 1.f;
        } else if (row_ok) {
          const int ts = t + shift;
          if (ts >= 0 && ts < g.T) v = __ldg(x + (mb + word + shift) * g.Cin + c);
        }
      }
      sw128_store1(st, arow, word, v);
    }
    uint8_t* bt = st + GT_A_BYTES;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int it = tid + GT_THREADS * j;
      const int o = it & 127, word = it >> 7;
      const int64_t m = mb + word;
      const int go = o0 + o;
      sw128_store1(bt, o, word, (m < g.M && go < g.Cout) ? __ldg(dz + m * g.Cout + go) : 0.f);
    }
  };

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  const int wg = tid >> 7;

  if (num_kb > 0) {
    decode(0, 0);
    __syncthreads();
    gather(0, 0, smem);
    if (num_kb > 1) decode(1, 1);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  }
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb & 1;
    gt_mma(acc, sbase + s * GT_STAGE, wg);
    if (kb + 1 < num_kb) gather(kb + 1, s ^ 1, smem + (s ^ 1) * GT_STAGE);
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // the position table of kb+1 has been read; refill that slot for kb+2
    if (kb + 2 < num_kb) decode(kb + 2, s);
    __syncthreads();
  }

  float* out = ws + (int64_t)blockIdx.z * rows * g.Cout;
  const int lane = tid & 31, wq = (tid >> 5) & 3;
  const int rr = r0 + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 16; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rr + 8 * h;
      if (r >= rows) continue;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int o = o0 + 8 * i + 2 * (lane & 3) + e;
        if (o < g.Cout) out[(int64_t)r * g.Cout + o] = acc[4 * i + 2 * h + e];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Exact fp32 engine (NM_GEMM_SIMT): 64 x 64 tiles of gemm_simt.cuh.  In the forward, tile column n is feature
// c0 + 2*(n/4) + (n & 1), its linear half when (n/2) is even and its gate otherwise, so the 4 columns of a thread
// are two features and their two gates.
// ------------------------------------------------------------------------------------------------------------
constexpr int GS_BM = 64, GS_BN = 64, GS_TM = 4, GS_TN = 4;

template <int MODE>
__global__ void __launch_bounds__(SIMT_THREADS)
glu_conv_simt_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                     const float* __restrict__ res, float* __restrict__ y, float* __restrict__ z, GluGeom g) {
  __shared__ SimtSmem<GS_BM, GS_BN, GS_TM, GS_TN> sm;
  const int64_t m0 = (int64_t)blockIdx.x * GS_BM;
  const int c0 = blockIdx.y * (MODE == GLU_FWD ? GS_BN / 2 : GS_BN);
  const int t = threadIdx.x;
  const int tx = t % (GS_BN / GS_TN), ty = t / (GS_BN / GS_TN);
  // the A rows this thread loads: (t + 256 i) / SIMT_BK = t / SIMT_BK + 16 i
  int arow_t[(GS_BM * SIMT_BK) / SIMT_THREADS];
#pragma unroll
  for (int i = 0; i < (GS_BM * SIMT_BK) / SIMT_THREADS; ++i) {
    const int64_t gm = m0 + t / SIMT_BK + i * (SIMT_THREADS / SIMT_BK);
    arow_t[i] = gm < g.M ? (int)(gm % g.T) : -1;
  }
  float acc[GS_TM][GS_TN] = {};
  for (int k0 = 0; k0 < g.Kd; k0 += SIMT_BK) {
#pragma unroll
    for (int i = 0; i < (GS_BM * SIMT_BK) / SIMT_THREADS; ++i) {
      const int mm = t / SIMT_BK + i * (SIMT_THREADS / SIMT_BK), kk = t % SIMT_BK;
      const int gk = k0 + kk;
      sm.a[kk][mm] = (arow_t[i] >= 0 && gk < g.Kd) ? glu_a(x, g, m0 + mm, arow_t[i], gk) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < (GS_BN * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int kk = idx / GS_BN, n = idx % GS_BN;
      const int gk = k0 + kk;
      float v = 0.f;
      if (gk < g.Kd) {
        if (MODE == GLU_FWD) {
          const int f = c0 + 2 * (n >> 2) + (n & 1);
          if (f < g.F) v = glu_b(w, g, gk, ((n >> 1) & 1) ? g.F + f : f);
        } else if (c0 + n < g.Cout) {
          v = glu_b(w, g, gk, c0 + n);
        }
      }
      sm.b[kk][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SIMT_BK; ++k) {
      float av[GS_TM], bv[GS_TN];
#pragma unroll
      for (int i = 0; i < GS_TM; ++i) av[i] = sm.a[k][ty * GS_TM + i];
#pragma unroll
      for (int j = 0; j < GS_TN; ++j) bv[j] = sm.b[k][tx * GS_TN + j];
#pragma unroll
      for (int i = 0; i < GS_TM; ++i)
#pragma unroll
        for (int j = 0; j < GS_TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < GS_TM; ++i) {
    const int64_t m = m0 + ty * GS_TM + i;
    if (m >= g.M) continue;
    if (MODE == GLU_FWD) {
      const int64_t F = g.F;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int f = c0 + 2 * tx + j;
        if (f >= g.F) continue;
        const float zl = acc[i][j] + bias[f], zg = acc[i][j + 2] + bias[F + f];
        if (z) {
          z[m * 2 * F + f] = zl;
          z[m * 2 * F + F + f] = zg;
        }
        y[m * F + f] = zl * sigmoidf_(zg) + res[m * F + f];
      }
    } else {
#pragma unroll
      for (int j = 0; j < GS_TN; ++j) {
        const int o = c0 + tx * GS_TN + j;
        if (o < g.Cout) y[m * g.Cout + o] = acc[i][j] + res[m * g.Cout + o];
      }
    }
  }
}

__global__ void __launch_bounds__(SIMT_THREADS)
glu_wgrad_simt_kernel(const float* __restrict__ x, const float* __restrict__ dz, float* __restrict__ ws, GluGeom g,
                      int kb_per_split) {
  __shared__ SimtSmem<GS_BM, GS_BN, GS_TM, GS_TN> sm;
  const int rows = g.Kd + 1;
  const int r0 = blockIdx.y * GS_BM, o0 = blockIdx.x * GS_BN;
  const int64_t p_begin = (int64_t)blockIdx.z * kb_per_split * SIMT_BK;
  const int64_t p_end = min(g.M, p_begin + (int64_t)kb_per_split * SIMT_BK);
  const int t = threadIdx.x;
  const int tx = t % (GS_BN / GS_TN), ty = t / (GS_BN / GS_TN);
  float acc[GS_TM][GS_TN] = {};
  for (int64_t p0 = p_begin; p0 < p_end; p0 += SIMT_BK) {
#pragma unroll
    for (int i = 0; i < (GS_BM * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int k = idx / GS_BM, r = idx % GS_BM;      // consecutive threads: consecutive rows (channels)
      const int64_t m = p0 + k;
      const int gr = r0 + r;
      float v = 0.f;
      if (m < p_end) {
        if (gr == g.Kd) v = 1.f;
        else if (gr < g.Kd) v = glu_a(x, g, m, (int)(m % g.T), gr);
      }
      sm.a[k][r] = v;
    }
#pragma unroll
    for (int i = 0; i < (GS_BN * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int k = idx / GS_BN, n = idx % GS_BN;
      const int64_t m = p0 + k;
      const int go = o0 + n;
      sm.b[k][n] = (m < p_end && go < g.Cout) ? dz[m * g.Cout + go] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SIMT_BK; ++k) {
      float av[GS_TM], bv[GS_TN];
#pragma unroll
      for (int i = 0; i < GS_TM; ++i) av[i] = sm.a[k][ty * GS_TM + i];
#pragma unroll
      for (int j = 0; j < GS_TN; ++j) bv[j] = sm.b[k][tx * GS_TN + j];
#pragma unroll
      for (int i = 0; i < GS_TM; ++i)
#pragma unroll
        for (int j = 0; j < GS_TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* out = ws + (int64_t)blockIdx.z * rows * g.Cout;
#pragma unroll
  for (int i = 0; i < GS_TM; ++i) {
    const int r = r0 + ty * GS_TM + i;
    if (r >= rows) continue;
#pragma unroll
    for (int j = 0; j < GS_TN; ++j) {
      const int o = o0 + tx * GS_TN + j;
      if (o < g.Cout) out[(int64_t)r * g.Cout + o] = acc[i][j];
    }
  }
}

// dw[r, o] += sum_s ws[s][r][o] (r < Kd), db[o] += sum_s ws[s][Kd][o]; the splits are added in index order
__global__ void glu_wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, float* __restrict__ db,
                                        int64_t rows, int64_t cols, int splits) {
  const int64_t total = rows * cols;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < splits; ++j) s += ws[j * total + i];
    if (i < total - cols) dw[i] += s;
    else db[i - (total - cols)] += s;
  }
}

// dZ = [dY * s, dY * a * s * (1 - s)], s = sigmoid(gate), a = the linear half
__global__ void glu_dz_kernel(const float* __restrict__ dy, const float* __restrict__ z, float* __restrict__ dz,
                              int64_t M, int64_t F) {
  const int64_t total = M * F;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / F, f = i - m * F;
    const float a = z[m * 2 * F + f], s = sigmoidf_(z[m * 2 * F + F + f]), d = dy[i];
    dz[m * 2 * F + f] = d * s;
    dz[m * 2 * F + F + f] = d * a * s * (1.f - s);
  }
}

static unsigned glu_grid(int64_t total) {
  const int64_t blocks = ceil_div(total, 256), cap = (int64_t)sm_count() * 16;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// The forward's geometry (flip = 0: x [B,T,F] -> z [B,T,2F]) or the data gradient's (flip = 1: dZ [B,T,2F] ->
// dX [B,T,F], pads k-1-pb before).
static int glu_geom(GluGeom& g, int64_t B, int64_t T, int64_t F, int64_t k, int flip, const char* name) {
  NM_REQUIRE(B > 0 && T > 0 && F > 0 && k > 0, NM_E_INVALID, "%s: bad sizes", name);
  NM_REQUIRE(k * 2 * F < (1LL << 30) && T < (1LL << 30) && B * T < (1LL << 40) && B * T * 2 * F < (1LL << 46),
             NM_E_UNSUPPORTED, "%s: sizes out of range", name);
  const int64_t pb = (k - 1) / 2;
  g.T = (int)T;
  g.F = (int)F;
  g.k = (int)k;
  g.Cin = (int)(flip ? 2 * F : F);
  g.Cout = (int)(flip ? F : 2 * F);
  g.pb = (int)(flip ? k - 1 - pb : pb);
  g.Kd = (int)(k * g.Cin);
  g.flip = flip;
  g.M = B * T;
  return NM_OK;
}

// The weight-gradient launch: tile counts and how far the position reduction is split - until ~4 CTAs per SM are
// busy, within the workspace (ws_cap floats; < 0 = unbounded).  One place decides it, for the launch and for
// nm_glu_conv1d_wgrad_workspace.
struct GluWgradPlan {
  int64_t rows, part, tiles_r, tiles_o, splits, kb_per;
};

static GluWgradPlan glu_wgrad_plan(const GluGeom& g, bool simt, int64_t ws_cap) {
  GluWgradPlan p;
  p.rows = (int64_t)g.Kd + 1;
  p.part = p.rows * g.Cout;
  const int bm = simt ? GS_BM : GT_BM, bn = simt ? GS_BN : GT_BN, bk = simt ? SIMT_BK : GT_BK;
  p.tiles_r = ceil_div(p.rows, bm);
  p.tiles_o = ceil_div(g.Cout, bn);
  const int64_t total_kb = ceil_div(g.M, bk);
  int64_t splits = ceil_div(4LL * sm_count(), p.tiles_r * p.tiles_o);
  splits = splits < total_kb ? splits : total_kb;
  if (ws_cap >= 0) splits = splits < ws_cap / p.part ? splits : ws_cap / p.part;
  splits = splits < 65535 ? splits : 65535;
  if (splits < 1) splits = 1;
  p.kb_per = ceil_div(total_kb, splits);
  p.splits = ceil_div(total_kb, p.kb_per);
  return p;
}

template <int MODE>
static int glu_conv_launch(const float* x, const float* w, const float* bias, const float* res, float* y, float* z,
                           const GluGeom& g, int backend, cudaStream_t s, const char* name) {
  if (backend == NM_GEMM_SIMT) {
    const int64_t cols = MODE == GLU_FWD ? GS_BN / 2 : GS_BN;
    NM_REQUIRE(ceil_div(g.M, GS_BM) <= 0x7fffffffLL && ceil_div(MODE == GLU_FWD ? g.F : g.Cout, cols) <= 65535,
               NM_E_UNSUPPORTED, "%s: grid too large", name);
    dim3 grid((unsigned)ceil_div(g.M, GS_BM), (unsigned)ceil_div(MODE == GLU_FWD ? g.F : g.Cout, cols));
    glu_conv_simt_kernel<MODE><<<grid, SIMT_THREADS, 0, s>>>(x, w, bias, res, y, z, g);
    NM_LAUNCH_CHECK(name);
    return NM_OK;
  }
  NM_REQUIRE(backend == NM_GEMM_AUTO || backend == NM_GEMM_TC, NM_E_INVALID, "%s: bad backend", name);
  const int64_t cols = MODE == GLU_FWD ? GT_BN / 2 : GT_BN;
  NM_REQUIRE(ceil_div(g.M, GT_BM) <= 0x7fffffffLL && ceil_div(MODE == GLU_FWD ? g.F : g.Cout, cols) <= 65535,
             NM_E_UNSUPPORTED, "%s: grid too large", name);
  static bool attr = false;
  if (!attr) {
    NM_CUDA_TRY(cudaFuncSetAttribute(glu_conv_tc_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, GT_SMEM));
    attr = true;
  }
  dim3 grid((unsigned)ceil_div(g.M, GT_BM), (unsigned)ceil_div(MODE == GLU_FWD ? g.F : g.Cout, cols));
  glu_conv_tc_kernel<MODE><<<grid, GT_THREADS, GT_SMEM, s>>>(x, w, bias, res, y, z, g);
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_glu_conv1d_fwd(const float* x, const float* w, const float* bias, float* y, float* z, int64_t B, int64_t T,
                      int64_t F, int64_t k, int backend, void* stream) {
  NM_REQUIRE(x && w && bias && y, NM_E_INVALID, "nm_glu_conv1d_fwd: null pointer");
  GluGeom g;
  const int rc = glu_geom(g, B, T, F, k, 0, "nm_glu_conv1d_fwd");
  if (rc) return rc;
  return glu_conv_launch<GLU_FWD>(x, w, bias, x, y, z, g, backend, (cudaStream_t)stream, "nm_glu_conv1d_fwd");
}

int nm_glu_conv1d_dz(const float* dy, const float* z, float* dz, int64_t M, int64_t F, void* stream) {
  NM_REQUIRE(dy && z && dz, NM_E_INVALID, "nm_glu_conv1d_dz: null pointer");
  NM_REQUIRE(M > 0 && F > 0 && M * 2 * F < (1LL << 46), NM_E_INVALID, "nm_glu_conv1d_dz: bad sizes");
  glu_dz_kernel<<<glu_grid(M * F), 256, 0, (cudaStream_t)stream>>>(dy, z, dz, M, F);
  NM_LAUNCH_CHECK("nm_glu_conv1d_dz");
  return NM_OK;
}

int nm_glu_conv1d_dgrad(const float* dz, const float* w, const float* dy, float* dx, int64_t B, int64_t T, int64_t F,
                        int64_t k, int backend, void* stream) {
  NM_REQUIRE(dz && w && dy && dx, NM_E_INVALID, "nm_glu_conv1d_dgrad: null pointer");
  GluGeom g;
  const int rc = glu_geom(g, B, T, F, k, 1, "nm_glu_conv1d_dgrad");
  if (rc) return rc;
  return glu_conv_launch<GLU_DGRAD>(dz, w, nullptr, dy, dx, nullptr, g, backend, (cudaStream_t)stream,
                                    "nm_glu_conv1d_dgrad");
}

int64_t nm_glu_conv1d_wgrad_workspace(int64_t B, int64_t T, int64_t F, int64_t k, int backend) {
  GluGeom g;
  if (glu_geom(g, B, T, F, k, 0, "nm_glu_conv1d_wgrad_workspace")) return -1;
  const GluWgradPlan p = glu_wgrad_plan(g, backend == NM_GEMM_SIMT, -1);
  return p.splits * p.part;
}

int nm_glu_conv1d_wgrad(const float* x, const float* dz, float* dw, float* db, float* workspace,
                        int64_t workspace_floats, int64_t B, int64_t T, int64_t F, int64_t k, int backend,
                        void* stream) {
  NM_REQUIRE(x && dz && dw && db && workspace, NM_E_INVALID, "nm_glu_conv1d_wgrad: null pointer");
  GluGeom g;
  const int rc = glu_geom(g, B, T, F, k, 0, "nm_glu_conv1d_wgrad");
  if (rc) return rc;
  const bool simt = backend == NM_GEMM_SIMT;
  NM_REQUIRE(simt || backend == NM_GEMM_AUTO || backend == NM_GEMM_TC, NM_E_INVALID,
             "nm_glu_conv1d_wgrad: bad backend");
  const GluWgradPlan p = glu_wgrad_plan(g, simt, workspace_floats);
  NM_REQUIRE(workspace_floats >= p.part, NM_E_INVALID, "nm_glu_conv1d_wgrad: workspace below (k*F+1)*2F floats");
  NM_REQUIRE(p.tiles_r <= 65535 && p.tiles_o <= 65535, NM_E_UNSUPPORTED, "nm_glu_conv1d_wgrad: filter too large");
  NM_REQUIRE(p.kb_per < (1LL << 31), NM_E_UNSUPPORTED, "nm_glu_conv1d_wgrad: too many positions");
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)p.tiles_o, (unsigned)p.tiles_r, (unsigned)p.splits);
  if (simt) {
    glu_wgrad_simt_kernel<<<grid, SIMT_THREADS, 0, s>>>(x, dz, workspace, g, (int)p.kb_per);
  } else {
    static bool attr = false;
    if (!attr) {
      NM_CUDA_TRY(cudaFuncSetAttribute(glu_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GT_SMEM));
      attr = true;
    }
    glu_wgrad_tc_kernel<<<grid, GT_THREADS, GT_SMEM, s>>>(x, dz, workspace, g, (int)p.kb_per);
  }
  NM_LAUNCH_CHECK("nm_glu_conv1d_wgrad");
  glu_wgrad_reduce_kernel<<<glu_grid(p.part), 256, 0, s>>>(workspace, dw, db, p.rows, g.Cout, (int)p.splits);
  NM_LAUNCH_CHECK("nm_glu_conv1d_wgrad(reduce)");
  return NM_OK;
}

}  // extern "C"
