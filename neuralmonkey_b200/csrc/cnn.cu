// Trainable CNN layers of encoders/cnn_encoder.py (reference :209-320): k x k convolution (stride 1) with its data
// and weight gradients, batch normalization with the ReLU after it, max / average pooling.  NHWC fp32, HWIO filters.
//
// Convolution = implicit GEMM, M = N*Ho*Wo output pixels, N = Cout, K = k*k*Cin:
//   A(m, (tap, c)) = x[n, oy + ky - pad_top, ox + kx - pad_left, c]   (zero outside the image)
//   B((tap, c), o) = w[tap, c, o]                                       (HWIO viewed as [k*k*Cin, Cout])
// No patch matrix is materialised: each CTA gathers its A tile from x straight into shared memory.  The data
// gradient is the same product over dY with the filter turned by 180 degrees and its channel axes swapped
// (`flip`), with pads k-1-pad_fwd on each side.  The weight gradient is the transposed product
// dW[(tap, c), o] = sum_m A(m, (tap, c)) dY(m, o), split over CTAs along m into a caller-owned workspace and
// summed in a fixed order; one extra row of ones in A gives the bias gradient in the same pass.
//
// Two engines, selected like nm_gemm's: wgmma with TF32 operands (cvt.rna, 128-byte swizzled K-major tiles,
// fp32 accumulators) and exact fp32 FMA tiles on the CUDA cores (NM_GEMM_SIMT).
#include "gemm_simt.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace nm {

struct ConvGeom {
  int N, H, W, C, K;       // input [N,H,W,C], output channels K
  int k, pt, pl;           // window and the pads before the image
  int Ho, Wo;
  int flip;                // 0: w is HWIO [k,k,C,K]; 1: w is the forward filter [k,k,K,C], turned by 180 degrees
  int64_t M;               // N*Ho*Wo
  int Kd;                  // k*k*C
};

__device__ __forceinline__ float conv_b(const float* __restrict__ w, const ConvGeom& g, int gk, int o) {
  const int tap = gk / g.C, c = gk - tap * g.C;
  if (g.flip) return __ldg(w + ((int64_t)(g.k * g.k - 1 - tap) * g.K + o) * g.C + c);
  return __ldg(w + (int64_t)gk * g.K + o);
}

// pixel m -> (offset of image n, oy, ox)
struct Pix {
  int64_t base;
  int oy, ox;
};
__device__ __forceinline__ Pix conv_pix(const ConvGeom& g, int64_t m) {
  const int64_t hw = (int64_t)g.Ho * g.Wo;
  const int64_t n = m / hw;
  const int r = (int)(m - n * hw);
  Pix p;
  p.base = n * g.H * g.W;
  p.oy = r / g.Wo;
  p.ox = r - p.oy * g.Wo;
  return p;
}

// A(m, gk) for a decoded pixel; gk < Kd
__device__ __forceinline__ float conv_a(const float* __restrict__ x, const ConvGeom& g, const Pix& p, int gk) {
  const int tap = gk / g.C, c = gk - tap * g.C;
  const int ky = tap / g.k, kx = tap - ky * g.k;
  const int iy = p.oy + ky - g.pt, ix = p.ox + kx - g.pl;
  if (iy < 0 || iy >= g.H || ix < 0 || ix >= g.W) return 0.f;
  return __ldg(x + ((p.base + (int64_t)iy * g.W + ix) * g.C + c));
}

__device__ __forceinline__ float act_apply(float v, int act) { return act == NM_ACT_RELU ? fmaxf(v, 0.f) : v; }

// ------------------------------------------------------------------------------------------------------------
// wgmma engine: 128 x 64 output tile, 2 consumer warpgroups of 64 rows, 32-wide k-blocks in a 2-stage ring.
// All 256 threads gather the next k-block while the tensor cores work on the current one.
// ------------------------------------------------------------------------------------------------------------
constexpr int CT_BM = 128, CT_BN = 64, CT_BK = 32, CT_THREADS = 256;
constexpr int CT_A_BYTES = CT_BM * 128, CT_B_BYTES = CT_BN * 128;
constexpr int CT_STAGE = CT_A_BYTES + CT_B_BYTES;
constexpr int CT_SMEM = 2 * CT_STAGE + 1024;   // + slack for the 1 KB alignment of the swizzled tiles

// Each warpgroup multiplies its 64 rows of the stage's A tile by the B tile (4 instructions of k = 8).
__device__ __forceinline__ void ct_mma(float (&acc)[32], uint32_t stage_addr, int wg) {
  const uint32_t a = stage_addr + wg * 64 * 128, b = stage_addr + CT_A_BYTES;
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) Wgmma<64, 4>::mma(acc, gmma_desc_sw128(a + k * 32), gmma_desc_sw128(b + k * 32));
  wgmma_commit();
}

// Forward / data gradient: y[m, o] = act(sum A(m, :) B(:, o) + bias[o]).
__global__ void __launch_bounds__(CT_THREADS)
conv_fwd_tc_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                   float* __restrict__ y, ConvGeom g, int act) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * CT_BM;
  const int o0 = blockIdx.y * CT_BN;
  const int num_kb = (g.Kd + CT_BK - 1) / CT_BK;
  const bool vec = (g.C & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;

  // A: thread owns row tid/2 and the 16 k values of half tid&1
  const int arow = tid >> 1, ahalf = tid & 1;
  const int64_t am = m0 + arow;
  const bool arow_ok = am < g.M;
  const Pix ap = conv_pix(g, arow_ok ? am : 0);

  auto gather = [&](int kb, uint8_t* st) {
    uint8_t* at = st;
    const int gk0 = kb * CT_BK + ahalf * 16;
    if (vec) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gk = gk0 + 4 * j;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (arow_ok && gk < g.Kd) {
          const int tap = gk / g.C, c = gk - tap * g.C;
          const int ky = tap / g.k, kx = tap - ky * g.k;
          const int iy = ap.oy + ky - g.pt, ix = ap.ox + kx - g.pl;
          if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
            v = __ldg(reinterpret_cast<const float4*>(x + (ap.base + (int64_t)iy * g.W + ix) * g.C + c));
        }
        sw128_store4(at, arow, ahalf * 4 + j, v);
      }
    } else {
#pragma unroll 4
      for (int j = 0; j < 16; ++j) {
        const int gk = gk0 + j;
        const float v = (arow_ok && gk < g.Kd) ? conv_a(x, g, ap, gk) : 0.f;
        sw128_store1(at, arow, ahalf * 16 + j, v);
      }
    }
    // B: 64 output channels x 32 k values; consecutive threads take consecutive channels
    uint8_t* bt = st + CT_A_BYTES;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int it = tid + CT_THREADS * j;
      const int o = it & 63, word = it >> 6;
      const int gk = kb * CT_BK + word, go = o0 + o;
      sw128_store1(bt, o, word, (gk < g.Kd && go < g.K) ? conv_b(w, g, gk, go) : 0.f);
    }
  };

  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  const int wg = tid >> 7;

  gather(0, smem);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb & 1;
    ct_mma(acc, sbase + s * CT_STAGE, wg);
    // the other stage was last read by the products of kb-1, which completed before the barrier below
    if (kb + 1 < num_kb) gather(kb + 1, smem + (s ^ 1) * CT_STAGE);
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  }

  const int lane = tid & 31, wq = (tid >> 5) & 3;
  const int64_t r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t m = r0 + 8 * h;
      if (m >= g.M) continue;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int o = o0 + 8 * i + 2 * (lane & 3) + e;
        if (o < g.K) y[m * g.K + o] = act_apply(acc[4 * i + 2 * h + e] + (bias ? __ldg(bias + o) : 0.f), act);
      }
    }
  }
}

// Weight gradient partials: ws[split][r][o] = sum over this split's pixels of A'(r, m) dY(m, o), where
// A'(r, m) = A(m, r) for r < Kd and A'(Kd, m) = 1 (the bias row).
__global__ void __launch_bounds__(CT_THREADS)
conv_wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ ws, ConvGeom g,
                     int kb_per_split) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ Pix pix[2][CT_BK];
  __shared__ int pix_ok[2][CT_BK];
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;
  const int rows = g.Kd + 1;
  const int r0 = blockIdx.y * CT_BM;
  const int o0 = blockIdx.x * CT_BN;
  const int split = blockIdx.z;
  const int total_kb = (int)((g.M + CT_BK - 1) / CT_BK);
  const int kb0 = split * kb_per_split;
  const int num_kb = min(total_kb, kb0 + kb_per_split) - kb0;

  // A': thread owns row tid & 127 and the words (tid >> 7) + 2j
  const int arow = tid & 127, aw = tid >> 7;
  const int gr = r0 + arow;
  const bool is_bias = gr == g.Kd, row_ok = gr < g.Kd;
  int ky = 0, kx = 0, c = 0;
  if (row_ok) {
    const int tap = gr / g.C;
    c = gr - tap * g.C;
    ky = tap / g.k;
    kx = tap - ky * g.k;
  }
  const int dyo = ky - g.pt, dxo = kx - g.pl;

  auto decode = [&](int kb, int buf) {
    if (tid < CT_BK) {
      const int64_t m = (int64_t)(kb0 + kb) * CT_BK + tid;
      pix_ok[buf][tid] = m < g.M;
      pix[buf][tid] = conv_pix(g, m < g.M ? m : 0);
    }
  };
  auto gather = [&](int kb, int buf, uint8_t* st) {
#pragma unroll 4
    for (int j = 0; j < 16; ++j) {
      const int word = aw + 2 * j;
      float v = 0.f;
      if (pix_ok[buf][word]) {
        if (is_bias) {
          v = 1.f;
        } else if (row_ok) {
          const Pix p = pix[buf][word];
          const int iy = p.oy + dyo, ix = p.ox + dxo;
          if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
            v = __ldg(x + (p.base + (int64_t)iy * g.W + ix) * g.C + c);
        }
      }
      sw128_store1(st, arow, word, v);
    }
    uint8_t* bt = st + CT_A_BYTES;
    const int64_t mb = (int64_t)(kb0 + kb) * CT_BK;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int it = tid + CT_THREADS * j;
      const int o = it & 63, word = it >> 6;
      const int64_t m = mb + word;
      const int go = o0 + o;
      sw128_store1(bt, o, word, (m < g.M && go < g.K) ? __ldg(dy + m * g.K + go) : 0.f);
    }
  };

  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
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
    ct_mma(acc, sbase + s * CT_STAGE, wg);
    if (kb + 1 < num_kb) gather(kb + 1, s ^ 1, smem + (s ^ 1) * CT_STAGE);
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // the pixel table of kb+1 has been read; refill that slot for kb+2
    if (kb + 2 < num_kb) decode(kb + 2, s);
    __syncthreads();
  }

  float* out = ws + (int64_t)split * rows * g.K;
  const int lane = tid & 31, wq = (tid >> 5) & 3;
  const int rr = r0 + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rr + 8 * h;
      if (r >= rows) continue;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int o = o0 + 8 * i + 2 * (lane & 3) + e;
        if (o < g.K) out[(int64_t)r * g.K + o] = acc[4 * i + 2 * h + e];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Exact fp32 engine (NM_GEMM_SIMT): 64 x 64 tiles of gemm_simt.cuh, operands gathered the same way.
// ------------------------------------------------------------------------------------------------------------
constexpr int CS_BM = 64, CS_BN = 64, CS_TM = 4, CS_TN = 4;

__global__ void __launch_bounds__(SIMT_THREADS)
conv_fwd_simt_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ y, ConvGeom g, int act) {
  __shared__ SimtSmem<CS_BM, CS_BN, CS_TM, CS_TN> sm;
  const int64_t m0 = (int64_t)blockIdx.x * CS_BM;
  const int o0 = blockIdx.y * CS_BN;
  const int t = threadIdx.x;
  const int tx = t % (CS_BN / CS_TN), ty = t / (CS_BN / CS_TN);
  float acc[CS_TM][CS_TN] = {};
  for (int k0 = 0; k0 < g.Kd; k0 += SIMT_BK) {
#pragma unroll
    for (int i = 0; i < (CS_BM * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int m = idx / SIMT_BK, k = idx % SIMT_BK;
      const int64_t gm = m0 + m;
      const int gk = k0 + k;
      sm.a[k][m] = (gm < g.M && gk < g.Kd) ? conv_a(x, g, conv_pix(g, gm), gk) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < (CS_BN * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int k = idx / CS_BN, n = idx % CS_BN;
      const int gk = k0 + k, go = o0 + n;
      sm.b[k][n] = (gk < g.Kd && go < g.K) ? conv_b(w, g, gk, go) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SIMT_BK; ++k) {
      float av[CS_TM], bv[CS_TN];
#pragma unroll
      for (int i = 0; i < CS_TM; ++i) av[i] = sm.a[k][ty * CS_TM + i];
#pragma unroll
      for (int j = 0; j < CS_TN; ++j) bv[j] = sm.b[k][tx * CS_TN + j];
#pragma unroll
      for (int i = 0; i < CS_TM; ++i)
#pragma unroll
        for (int j = 0; j < CS_TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < CS_TM; ++i) {
    const int64_t m = m0 + ty * CS_TM + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < CS_TN; ++j) {
      const int o = o0 + tx * CS_TN + j;
      if (o < g.K) y[m * g.K + o] = act_apply(acc[i][j] + (bias ? bias[o] : 0.f), act);
    }
  }
}

__global__ void __launch_bounds__(SIMT_THREADS)
conv_wgrad_simt_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ ws,
                       ConvGeom g, int kb_per_split) {
  __shared__ SimtSmem<CS_BM, CS_BN, CS_TM, CS_TN> sm;
  const int rows = g.Kd + 1;
  const int r0 = blockIdx.y * CS_BM, o0 = blockIdx.x * CS_BN;
  const int64_t p_begin = (int64_t)blockIdx.z * kb_per_split * SIMT_BK;
  const int64_t p_end = min(g.M, p_begin + (int64_t)kb_per_split * SIMT_BK);
  const int t = threadIdx.x;
  const int tx = t % (CS_BN / CS_TN), ty = t / (CS_BN / CS_TN);
  float acc[CS_TM][CS_TN] = {};
  for (int64_t p0 = p_begin; p0 < p_end; p0 += SIMT_BK) {
#pragma unroll
    for (int i = 0; i < (CS_BM * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int k = idx / CS_BM, r = idx % CS_BM;      // consecutive threads: consecutive rows (channels)
      const int64_t m = p0 + k;
      const int gr = r0 + r;
      float v = 0.f;
      if (m < p_end) {
        if (gr == g.Kd) v = 1.f;
        else if (gr < g.Kd) v = conv_a(x, g, conv_pix(g, m), gr);
      }
      sm.a[k][r] = v;
    }
#pragma unroll
    for (int i = 0; i < (CS_BN * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int k = idx / CS_BN, n = idx % CS_BN;
      const int64_t m = p0 + k;
      const int go = o0 + n;
      sm.b[k][n] = (m < p_end && go < g.K) ? dy[m * g.K + go] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SIMT_BK; ++k) {
      float av[CS_TM], bv[CS_TN];
#pragma unroll
      for (int i = 0; i < CS_TM; ++i) av[i] = sm.a[k][ty * CS_TM + i];
#pragma unroll
      for (int j = 0; j < CS_TN; ++j) bv[j] = sm.b[k][tx * CS_TN + j];
#pragma unroll
      for (int i = 0; i < CS_TM; ++i)
#pragma unroll
        for (int j = 0; j < CS_TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* out = ws + (int64_t)blockIdx.z * rows * g.K;
#pragma unroll
  for (int i = 0; i < CS_TM; ++i) {
    const int r = r0 + ty * CS_TM + i;
    if (r >= rows) continue;
#pragma unroll
    for (int j = 0; j < CS_TN; ++j) {
      const int o = o0 + tx * CS_TN + j;
      if (o < g.K) out[(int64_t)r * g.K + o] = acc[i][j];
    }
  }
}

// dw[r, o] += sum_s ws[s][r][o] (r < Kd), db[o] += sum_s ws[s][Kd][o]; splits summed in index order.
__global__ void conv_wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, float* __restrict__ db,
                                         int64_t rows, int64_t K, int splits) {
  const int64_t total = rows * K;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < splits; ++j) s += ws[j * total + i];
    const int64_t r = i / K;
    if (r < rows - 1) dw[i] += s;
    else if (db) db[i - r * K] += s;
  }
}

// ------------------------------------------------------------------------------------------------------------
// Batch normalization over P = N*H*W rows of C channels.  Per-channel sums are accumulated in fp64: grid
// (ceil(C/32), S) partial blocks of 32 channels x 8 row lanes, then one thread per channel adds the S partials in
// index order, so the statistics do not depend on scheduling.
// ------------------------------------------------------------------------------------------------------------
constexpr int BN_SPLITS = 64;      // NM_BN_WS_DOUBLES_PER_CHANNEL = 2 * BN_SPLITS + 2

// mode 0: (sum x, sum x^2); mode 1: (sum dy', sum dy' * xhat), dy' = dy masked by the fused ReLU
__global__ void __launch_bounds__(256)
bn_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ gamma,
                  const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ invstd,
                  double* __restrict__ part, int64_t P, int C, int relu, int mode) {
  __shared__ double red[2][8][32];
  const int lc = threadIdx.x & 31, lr = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lc;
  double s0 = 0.0, s1 = 0.0;
  if (c < C) {
    float mu = 0.f, is = 0.f, ga = 0.f, be = 0.f;
    if (mode == 1) { mu = mean[c]; is = invstd[c]; ga = gamma[c]; be = beta[c]; }
    for (int64_t r = (int64_t)blockIdx.y * 8 + lr; r < P; r += (int64_t)gridDim.y * 8) {
      const float v = x[r * C + c];
      if (mode == 0) {
        s0 += v;
        s1 += (double)v * v;
      } else {
        const float xh = (v - mu) * is;
        float d = dy[r * C + c];
        if (relu && fmaf(ga, xh, be) <= 0.f) d = 0.f;
        s0 += d;
        s1 += (double)d * xh;
      }
    }
  }
  red[0][lr][lc] = s0;
  red[1][lr][lc] = s1;
  __syncthreads();
  if (lr == 0 && c < C) {
    for (int i = 1; i < 8; ++i) { s0 += red[0][i][lc]; s1 += red[1][i][lc]; }
    part[((int64_t)blockIdx.y * C + c) * 2] = s0;
    part[((int64_t)blockIdx.y * C + c) * 2 + 1] = s1;
  }
}

__global__ void bn_fwd_finalize_kernel(const double* __restrict__ part, int splits, float* __restrict__ moving_mean,
                                       float* __restrict__ moving_var, float* __restrict__ save_mean,
                                       float* __restrict__ save_invstd, int64_t P, int C, float momentum, float eps,
                                       int training) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (!training) {
    save_mean[c] = moving_mean[c];
    save_invstd[c] = (float)(1.0 / sqrt((double)moving_var[c] + (double)eps));
    return;
  }
  double s0 = 0.0, s1 = 0.0;
  for (int j = 0; j < splits; ++j) {
    s0 += part[((int64_t)j * C + c) * 2];
    s1 += part[((int64_t)j * C + c) * 2 + 1];
  }
  const double mu = s0 / (double)P;
  const double var = fmax(s1 / (double)P - mu * mu, 0.0);
  save_mean[c] = (float)mu;
  save_invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (moving_mean) {
    // moving statistics: the Bessel-corrected batch variance, as TF's fused batch norm returns it
    const double unbiased = P > 1 ? var * (double)P / (double)(P - 1) : var;
    moving_mean[c] = (float)((double)momentum * moving_mean[c] + (1.0 - momentum) * mu);
    moving_var[c] = (float)((double)momentum * moving_var[c] + (1.0 - momentum) * unbiased);
  }
}

__global__ void bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ mean,
                                const float* __restrict__ invstd, float* __restrict__ y, int64_t total, int C,
                                int relu) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float v = fmaf(gamma[c], (x[i] - mean[c]) * invstd[c], beta[c]);
    y[i] = relu ? fmaxf(v, 0.f) : v;
  }
}

// one thread per channel: the two sums of the backward pass; dgamma / dbeta accumulate
__global__ void bn_bwd_finalize_kernel(const double* __restrict__ part, int splits, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, double* __restrict__ sums, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s0 = 0.0, s1 = 0.0;
  for (int j = 0; j < splits; ++j) {
    s0 += part[((int64_t)j * C + c) * 2];
    s1 += part[((int64_t)j * C + c) * 2 + 1];
  }
  sums[2 * c] = s0;
  sums[2 * c + 1] = s1;
  if (dbeta) dbeta[c] += (float)s0;
  if (dgamma) dgamma[c] += (float)s1;
}

__global__ void bn_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ mean, const float* __restrict__ invstd,
                                 const double* __restrict__ sums, float* __restrict__ dx, int64_t total, int64_t P,
                                 int C, int relu, int training) {
  const float inv_p = 1.f / (float)P;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const float is = invstd[c], ga = gamma[c];
    const float xh = (x[i] - mean[c]) * is;
    float d = dy[i];
    if (relu && fmaf(ga, xh, beta[c]) <= 0.f) d = 0.f;
    if (training) d = d - (float)sums[2 * c] * inv_p - xh * ((float)sums[2 * c + 1] * inv_p);
    dx[i] = ga * is * d;
  }
}

// ------------------------------------------------------------------------------------------------------------
// Pooling (tf.layers.max_pooling2d / average_pooling2d): k x k window, stride s; `same` pads TF's way (odd pixel
// at the bottom / right) and averages over the pixels inside the image.
// ------------------------------------------------------------------------------------------------------------
struct PoolGeom {
  int N, H, W, C, k, s, pt, pl, Ho, Wo;
};

__global__ void pool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, PoolGeom g, int is_max) {
  const int64_t total = (int64_t)g.N * g.Ho * g.Wo * g.C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    int64_t r = i / g.C;
    const int ox = (int)(r % g.Wo);
    r /= g.Wo;
    const int oy = (int)(r % g.Ho);
    const int64_t n = r / g.Ho;
    const int y0 = oy * g.s - g.pt, x0 = ox * g.s - g.pl;
    float best = -INFINITY, sum = 0.f;
    int cnt = 0;
    for (int dy = 0; dy < g.k; ++dy) {
      const int iy = y0 + dy;
      if (iy < 0 || iy >= g.H) continue;
      for (int dx = 0; dx < g.k; ++dx) {
        const int ix = x0 + dx;
        if (ix < 0 || ix >= g.W) continue;
        const float v = x[((n * g.H + iy) * g.W + ix) * g.C + c];
        if (v > best) best = v;
        sum += v;
        ++cnt;
      }
    }
    y[i] = is_max ? best : sum / (float)cnt;
  }
}

// Gradient gathered per input pixel from every window that contains it (no atomics: same bits every call).  Max
// pooling routes a window's gradient to its first maximal pixel in row-major order.
__global__ void pool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx,
                                PoolGeom g, int is_max) {
  const int64_t total = (int64_t)g.N * g.H * g.W * g.C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    int64_t r = i / g.C;
    const int ix = (int)(r % g.W);
    r /= g.W;
    const int iy = (int)(r % g.H);
    const int64_t n = r / g.H;
    // windows oy with oy*s - pt <= iy < oy*s - pt + k
    const int oy_lo = max(0, (iy + g.pt - g.k + g.s) / g.s), oy_hi = min(g.Ho - 1, (iy + g.pt) / g.s);
    const int ox_lo = max(0, (ix + g.pl - g.k + g.s) / g.s), ox_hi = min(g.Wo - 1, (ix + g.pl) / g.s);
    float acc = 0.f;
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        const int y0 = oy * g.s - g.pt, x0 = ox * g.s - g.pl;
        if (iy < y0 || ix < x0) continue;    // (iy + pt - k + s) / s rounds toward zero for negative values
        const float d = dy[((n * g.Ho + oy) * g.Wo + ox) * g.C + c];
        if (is_max) {
          float best = -INFINITY;
          int by = -1, bx = -1;
          for (int yy = max(y0, 0); yy < min(y0 + g.k, g.H); ++yy)
            for (int xx = max(x0, 0); xx < min(x0 + g.k, g.W); ++xx) {
              const float v = x[((n * g.H + yy) * g.W + xx) * g.C + c];
              if (v > best || by < 0) { best = v; by = yy; bx = xx; }
            }
          if (by == iy && bx == ix) acc += d;
        } else {
          const int cy = min(y0 + g.k, g.H) - max(y0, 0), cx = min(x0 + g.k, g.W) - max(x0, 0);
          acc += d / (float)(cy * cx);
        }
      }
    }
    dx[i] = acc;
  }
}

static unsigned grid_for(int64_t total) {
  int64_t blocks = ceil_div(total, 256);
  const int64_t cap = (int64_t)sm_count() * 16;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

static int conv_geom(ConvGeom& g, int64_t N, int64_t H, int64_t W, int64_t C, int64_t K, int64_t k, int64_t pad_top,
                     int64_t pad_bottom, int64_t pad_left, int64_t pad_right, int flip, const char* name) {
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && K > 0 && k > 0 && pad_top >= 0 && pad_bottom >= 0 &&
                 pad_left >= 0 && pad_right >= 0 && pad_top < k && pad_bottom < k && pad_left < k && pad_right < k,
             NM_E_INVALID, "%s: bad sizes", name);
  const int64_t Ho = H + pad_top + pad_bottom - k + 1, Wo = W + pad_left + pad_right - k + 1;
  NM_REQUIRE(Ho > 0 && Wo > 0, NM_E_INVALID, "%s: window larger than the padded image", name);
  NM_REQUIRE(k * k * C < (1LL << 30) && K < (1LL << 24) && N * H * W * C < (1LL << 40) && H < (1 << 20) &&
                 W < (1 << 20),
             NM_E_UNSUPPORTED, "%s: sizes out of range", name);
  g.N = (int)N; g.H = (int)H; g.W = (int)W; g.C = (int)C; g.K = (int)K; g.k = (int)k;
  g.pt = (int)pad_top; g.pl = (int)pad_left; g.Ho = (int)Ho; g.Wo = (int)Wo; g.flip = flip;
  g.M = N * Ho * Wo;
  g.Kd = (int)(k * k * C);
  return NM_OK;
}

static int pool_geom(PoolGeom& g, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k, int64_t s, int same,
                     const char* name) {
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && k > 0 && s > 0 && H < (1 << 20) && W < (1 << 20),
             NM_E_INVALID, "%s: bad sizes", name);
  int64_t Ho, Wo, pt = 0, pl = 0;
  if (same) {
    Ho = ceil_div(H, s);
    Wo = ceil_div(W, s);
    const int64_t ph = (Ho - 1) * s + k - H, pw = (Wo - 1) * s + k - W;
    pt = ph > 0 ? ph / 2 : 0;
    pl = pw > 0 ? pw / 2 : 0;
  } else {
    NM_REQUIRE(H >= k && W >= k, NM_E_INVALID, "%s: window larger than the image", name);
    Ho = (H - k) / s + 1;
    Wo = (W - k) / s + 1;
  }
  g.N = (int)N; g.H = (int)H; g.W = (int)W; g.C = (int)C; g.k = (int)k; g.s = (int)s;
  g.pt = (int)pt; g.pl = (int)pl; g.Ho = (int)Ho; g.Wo = (int)Wo;
  return NM_OK;
}

// The weight-gradient launch: tile counts and how far the pixel reduction is split - until ~4 CTAs per SM are
// busy, within the workspace (ws_cap floats; < 0 = unbounded).  One place decides it, for the launch and for
// nm_conv2d_wgrad_workspace.
struct WgradPlan {
  int64_t rows, part, tiles_r, tiles_o, splits, kb_per;
};

static WgradPlan wgrad_plan(const ConvGeom& g, bool simt, int64_t ws_cap) {
  WgradPlan p;
  p.rows = (int64_t)g.Kd + 1;
  p.part = p.rows * g.K;
  const int bm = simt ? CS_BM : CT_BM, bn = simt ? CS_BN : CT_BN, bk = simt ? SIMT_BK : CT_BK;
  p.tiles_r = ceil_div(p.rows, bm);
  p.tiles_o = ceil_div(g.K, bn);
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

}  // namespace nm

using namespace nm;

extern "C" {

int nm_conv2d_fwd(const float* x, const float* w, const float* bias, float* y, int64_t N, int64_t H, int64_t W,
                  int64_t Cin, int64_t Cout, int64_t k, int64_t pad_top, int64_t pad_bottom, int64_t pad_left,
                  int64_t pad_right, int flip, int act, int backend, void* stream) {
  NM_REQUIRE(x && w && y, NM_E_INVALID, "nm_conv2d_fwd: null pointer");
  NM_REQUIRE(act == NM_ACT_NONE || act == NM_ACT_RELU, NM_E_INVALID, "nm_conv2d_fwd: act must be none or relu");
  ConvGeom g;
  const int rc = conv_geom(g, N, H, W, Cin, Cout, k, pad_top, pad_bottom, pad_left, pad_right, flip ? 1 : 0,
                           "nm_conv2d_fwd");
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  // pixel tiles along x (up to 2^31 - 1 of them), output-channel tiles along y
  if (backend == NM_GEMM_SIMT) {
    NM_REQUIRE(ceil_div(g.M, CS_BM) <= 0x7fffffffLL && ceil_div(Cout, CS_BN) <= 65535, NM_E_UNSUPPORTED,
               "nm_conv2d_fwd: grid too large");
    dim3 grid((unsigned)ceil_div(g.M, CS_BM), (unsigned)ceil_div(Cout, CS_BN));
    conv_fwd_simt_kernel<<<grid, SIMT_THREADS, 0, s>>>(x, w, bias, y, g, act);
    NM_LAUNCH_CHECK("nm_conv2d_fwd(simt)");
    return NM_OK;
  }
  NM_REQUIRE(backend == NM_GEMM_AUTO || backend == NM_GEMM_TC, NM_E_INVALID, "nm_conv2d_fwd: bad backend");
  NM_REQUIRE(ceil_div(g.M, CT_BM) <= 0x7fffffffLL && ceil_div(Cout, CT_BN) <= 65535, NM_E_UNSUPPORTED,
             "nm_conv2d_fwd: grid too large");
  static bool attr = false;
  if (!attr) {
    NM_CUDA_TRY(cudaFuncSetAttribute(conv_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM));
    attr = true;
  }
  dim3 grid((unsigned)ceil_div(g.M, CT_BM), (unsigned)ceil_div(Cout, CT_BN));
  conv_fwd_tc_kernel<<<grid, CT_THREADS, CT_SMEM, s>>>(x, w, bias, y, g, act);
  NM_LAUNCH_CHECK("nm_conv2d_fwd(tc)");
  return NM_OK;
}

int64_t nm_conv2d_wgrad_workspace(int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t k,
                                  int64_t pad_top, int64_t pad_bottom, int64_t pad_left, int64_t pad_right,
                                  int backend) {
  ConvGeom g;
  if (conv_geom(g, N, H, W, Cin, Cout, k, pad_top, pad_bottom, pad_left, pad_right, 0, "nm_conv2d_wgrad_workspace"))
    return -1;
  const WgradPlan p = wgrad_plan(g, backend == NM_GEMM_SIMT, -1);
  return p.splits * p.part;
}

int nm_conv2d_wgrad(const float* x, const float* dy, float* dw, float* db, float* workspace, int64_t workspace_floats,
                    int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t k, int64_t pad_top,
                    int64_t pad_bottom, int64_t pad_left, int64_t pad_right, int backend, void* stream) {
  NM_REQUIRE(x && dy && dw && workspace, NM_E_INVALID, "nm_conv2d_wgrad: null pointer");
  ConvGeom g;
  const int rc = conv_geom(g, N, H, W, Cin, Cout, k, pad_top, pad_bottom, pad_left, pad_right, 0, "nm_conv2d_wgrad");
  if (rc) return rc;
  const bool simt = backend == NM_GEMM_SIMT;
  NM_REQUIRE(simt || backend == NM_GEMM_AUTO || backend == NM_GEMM_TC, NM_E_INVALID, "nm_conv2d_wgrad: bad backend");
  const WgradPlan p = wgrad_plan(g, simt, workspace_floats);
  const int64_t rows = p.rows, part = p.part, tiles_r = p.tiles_r, tiles_o = p.tiles_o, splits = p.splits,
                kb_per = p.kb_per;
  NM_REQUIRE(workspace_floats >= part, NM_E_INVALID, "nm_conv2d_wgrad: workspace below (k*k*Cin+1)*Cout floats");
  NM_REQUIRE(tiles_r <= 65535 && tiles_o <= 65535, NM_E_UNSUPPORTED, "nm_conv2d_wgrad: filter too large");
  NM_REQUIRE(kb_per < (1LL << 31), NM_E_UNSUPPORTED, "nm_conv2d_wgrad: too many pixels");
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((unsigned)tiles_o, (unsigned)tiles_r, (unsigned)splits);
  if (simt) {
    conv_wgrad_simt_kernel<<<grid, SIMT_THREADS, 0, s>>>(x, dy, workspace, g, (int)kb_per);
  } else {
    static bool attr = false;
    if (!attr) {
      NM_CUDA_TRY(cudaFuncSetAttribute(conv_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM));
      attr = true;
    }
    conv_wgrad_tc_kernel<<<grid, CT_THREADS, CT_SMEM, s>>>(x, dy, workspace, g, (int)kb_per);
  }
  NM_LAUNCH_CHECK("nm_conv2d_wgrad");
  conv_wgrad_reduce_kernel<<<grid_for(part), 256, 0, s>>>(workspace, dw, db, rows, Cout, (int)splits);
  NM_LAUNCH_CHECK("nm_conv2d_wgrad(reduce)");
  return NM_OK;
}

int nm_batchnorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* moving_mean,
                     float* moving_var, float* save_mean, float* save_invstd, double* workspace, int64_t P, int64_t C,
                     float momentum, float eps, int training, int relu, void* stream) {
  NM_REQUIRE(x && gamma && beta && y && moving_mean && moving_var && save_mean && save_invstd, NM_E_INVALID,
             "nm_batchnorm_fwd: null pointer");
  NM_REQUIRE(P > 0 && C > 0 && C < (1 << 24), NM_E_INVALID, "nm_batchnorm_fwd: bad sizes");
  NM_REQUIRE(!training || workspace, NM_E_INVALID, "nm_batchnorm_fwd: training needs the workspace");
  cudaStream_t s = (cudaStream_t)stream;
  const int splits = (int)(ceil_div(P, 8) < BN_SPLITS ? ceil_div(P, 8) : BN_SPLITS);
  if (training) {
    bn_partial_kernel<<<dim3((unsigned)ceil_div(C, 32), splits), 256, 0, s>>>(x, nullptr, nullptr, nullptr, nullptr,
                                                                              nullptr, workspace, P, (int)C, 0, 0);
    NM_LAUNCH_CHECK("nm_batchnorm_fwd(stats)");
  }
  bn_fwd_finalize_kernel<<<(unsigned)ceil_div(C, 128), 128, 0, s>>>(workspace, splits, moving_mean, moving_var,
                                                                      save_mean, save_invstd, P, (int)C, momentum, eps,
                                                                      training);
  NM_LAUNCH_CHECK("nm_batchnorm_fwd(finalize)");
  bn_apply_kernel<<<grid_for(P * C), 256, 0, s>>>(x, gamma, beta, save_mean, save_invstd, y, P * C, (int)C, relu);
  NM_LAUNCH_CHECK("nm_batchnorm_fwd(apply)");
  return NM_OK;
}

int nm_batchnorm_bwd(const float* x, const float* dy, const float* gamma, const float* beta, const float* save_mean,
                     const float* save_invstd, float* dx, float* dgamma, float* dbeta, double* workspace, int64_t P,
                     int64_t C, int training, int relu, void* stream) {
  NM_REQUIRE(x && dy && gamma && beta && save_mean && save_invstd && workspace, NM_E_INVALID,
             "nm_batchnorm_bwd: null pointer");
  NM_REQUIRE(P > 0 && C > 0 && C < (1 << 24), NM_E_INVALID, "nm_batchnorm_bwd: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  const int splits = (int)(ceil_div(P, 8) < BN_SPLITS ? ceil_div(P, 8) : BN_SPLITS);
  double* sums = workspace + 2 * BN_SPLITS * C;
  bn_partial_kernel<<<dim3((unsigned)ceil_div(C, 32), splits), 256, 0, s>>>(x, dy, gamma, beta, save_mean,
                                                                            save_invstd, workspace, P, (int)C, relu, 1);
  NM_LAUNCH_CHECK("nm_batchnorm_bwd(sums)");
  bn_bwd_finalize_kernel<<<(unsigned)ceil_div(C, 128), 128, 0, s>>>(workspace, splits, dgamma, dbeta, sums, (int)C);
  NM_LAUNCH_CHECK("nm_batchnorm_bwd(finalize)");
  if (dx) {
    bn_bwd_dx_kernel<<<grid_for(P * C), 256, 0, s>>>(x, dy, gamma, beta, save_mean, save_invstd, sums, dx, P * C, P,
                                                     (int)C, relu, training);
    NM_LAUNCH_CHECK("nm_batchnorm_bwd(dx)");
  }
  return NM_OK;
}

int nm_pool2d_fwd(const float* x, float* y, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k, int64_t stride,
                  int same, int is_max, void* stream) {
  NM_REQUIRE(x && y, NM_E_INVALID, "nm_pool2d_fwd: null pointer");
  PoolGeom g;
  const int rc = pool_geom(g, N, H, W, C, k, stride, same, "nm_pool2d_fwd");
  if (rc) return rc;
  pool_fwd_kernel<<<grid_for((int64_t)N * g.Ho * g.Wo * C), 256, 0, (cudaStream_t)stream>>>(x, y, g, is_max);
  NM_LAUNCH_CHECK("nm_pool2d_fwd");
  return NM_OK;
}

int nm_pool2d_bwd(const float* x, const float* dy, float* dx, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k,
                  int64_t stride, int same, int is_max, void* stream) {
  NM_REQUIRE(dy && dx && (x || !is_max), NM_E_INVALID, "nm_pool2d_bwd: null pointer");
  PoolGeom g;
  const int rc = pool_geom(g, N, H, W, C, k, stride, same, "nm_pool2d_bwd");
  if (rc) return rc;
  pool_bwd_kernel<<<grid_for(N * H * W * C), 256, 0, (cudaStream_t)stream>>>(x, dy, dx, g, is_max);
  NM_LAUNCH_CHECK("nm_pool2d_bwd");
  return NM_OK;
}

}  // extern "C"
