// Implicit-GEMM convolution core of cnn.cu (conv2d), glu_conv.cu (the ConvS2S GLU conv1d) and conv.cu (the VGG 3x3):
// a stride-1 convolution of x [N,H,W,C] (NHWC fp32) by a kh x kw window, M = N*Ho*Wo output pixels, K = Cout,
// Kd = kh*kw*C:
//   A(m, (tap, c)) = x[n, oy + ky - pt, ox + kx - pl, c]   (zero outside the image), tap = ky*kw + kx
//   B((tap, c), o) = w[tap, c, o]                             (the filter viewed as [Kd, Cout], o-contiguous)
// No patch matrix is materialised: each CTA gathers its A tile from x straight into shared memory.  A data gradient
// is the same product over dY with the filter turned by 180 degrees and its channel axes swapped (FLIP: w is the
// forward filter [kh,kw,Cout,Cin], c-contiguous), with pads k-1-pad_fwd.  The weight gradient is the transposed
// product dW[(tap, c), o] = sum_m A(m, (tap, c)) dY(m, o), split over CTAs along m into a caller-owned workspace and
// summed in a fixed order; one extra row of ones in A gives the bias gradient in the same pass.
//
// The forward kernels also take an input policy: the ResNet-v2 convolutions (conv.cu) read x at a stride s,
// A(m, (tap, c)) = pre(x[n, oy*s + ky - pt, ox*s + kx - pl, c]) with an optional batch norm + ReLU `pre`; every other
// caller takes the stride-1 default.
//
// The GLU conv1d is the one-row case (ONE_ROW: H = kh = 1, pt = 0, W = T): row m of A is then one contiguous span
// of x cut at the row ends, so its gathers decode the window position only once.
//
// Two engines: wgmma with TF32 operands (cvt.rna, 128-byte swizzled K-major tiles, fp32 accumulators) and exact
// fp32 FMA tiles on the CUDA cores (NM_GEMM_SIMT).
#pragma once
#include "gemm_simt.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace nm {

struct ConvGeom {
  int H, W, C, K;          // input [N,H,W,C], output channels K
  int kh, kw, pt, pl;      // window and the pads before the image
  int Ho, Wo;
  int64_t M;               // N*Ho*Wo
  int Kd;                  // kh*kw*C
};

// The geometry of an output of Ho x Wo pixels; each caller checks its sizes first.
static inline ConvGeom conv_geom_of(int64_t N, int64_t H, int64_t W, int64_t C, int64_t K, int64_t kh, int64_t kw,
                                    int64_t pt, int64_t pl, int64_t Ho, int64_t Wo) {
  ConvGeom g;
  g.H = (int)H; g.W = (int)W; g.C = (int)C; g.K = (int)K;
  g.kh = (int)kh; g.kw = (int)kw; g.pt = (int)pt; g.pl = (int)pl; g.Ho = (int)Ho; g.Wo = (int)Wo;
  g.M = N * Ho * Wo;
  g.Kd = (int)(kh * kw * C);
  return g;
}

// B(gk, o); gk < Kd, o < K
template <bool FLIP, bool ONE_ROW>
__device__ __forceinline__ float conv_b(const float* __restrict__ w, const ConvGeom& g, int gk, int o) {
  if (!FLIP) return __ldg(w + (int64_t)gk * g.K + o);
  const int tap = gk / g.C, c = gk - tap * g.C;
  const int taps = ONE_ROW ? g.kw : g.kh * g.kw;
  return __ldg(w + ((int64_t)(taps - 1 - tap) * g.K + o) * g.C + c);
}

// pixel m -> (offset of image n, oy, ox); in a one-row image, base is the offset of pixel m - pl instead, where the
// span of x that row m of A reads begins
struct Pix {
  int64_t base;
  int oy, ox;
};
__device__ __forceinline__ Pix row_pix(const ConvGeom& g, int64_t m, int ox) {
  Pix p;
  p.base = (m - g.pl) * g.C;
  p.oy = 0;
  p.ox = ox;
  return p;
}
template <bool ONE_ROW>
__device__ __forceinline__ Pix conv_pix(const ConvGeom& g, int64_t m) {
  if (ONE_ROW) return row_pix(g, m, (int)(m % g.W));
  const int64_t hw = (int64_t)g.Ho * g.Wo;
  const int64_t n = m / hw;
  const int r = (int)(m - n * hw);
  Pix p;
  p.base = n * g.H * g.W;
  p.oy = r / g.Wo;
  p.ox = r - p.oy * g.Wo;
  return p;
}

// Where A(m, gk) of a decoded pixel lies in x; false in the zero padding.  gk < Kd
template <bool ONE_ROW>
__device__ __forceinline__ bool conv_a_at(const ConvGeom& g, const Pix& p, int gk, int64_t& off) {
  const int tap = gk / g.C;
  if (ONE_ROW) {
    const int ix = p.ox + tap - g.pl;
    off = p.base + gk;
    return ix >= 0 && ix < g.W;
  }
  const int c = gk - tap * g.C;
  // 3 x 3, the VGG window and the usual conv2d one, divides by a constant instead of once more at run time
  const int ky = g.kw == 3 ? tap / 3 : tap / g.kw, kx = tap - ky * g.kw;
  const int iy = p.oy + ky - g.pt, ix = p.ox + kx - g.pl;
  off = (p.base + (int64_t)iy * g.W + ix) * g.C + c;
  return iy >= 0 && iy < g.H && ix >= 0 && ix < g.W;
}
template <bool ONE_ROW>
__device__ __forceinline__ float conv_a(const float* __restrict__ x, const ConvGeom& g, const Pix& p, int gk) {
  int64_t off;
  return conv_a_at<ONE_ROW>(g, p, gk, off) ? __ldg(x + off) : 0.f;
}

__device__ __forceinline__ float act_apply(float v, int act) { return act == NM_ACT_RELU ? fmaxf(v, 0.f) : v; }

// ------------------------------------------------------------------------------------------------------------
// Input policies of the forward kernels: how a window reads x.  A stride s places output pixel (oy, ox)'s window at
// (oy*s - pt, ox*s - pl), so the decoded pixel carries oy*s, ox*s and conv_a_at stays the stride-1 code.
// ------------------------------------------------------------------------------------------------------------
// stride 1, A = x: every convolution but the ResNet-v2 ones (the template default)
struct PlainIn {
  static constexpr bool ON = false;
};

// stride s, and when scale is non-NULL A = relu(x * scale[c] + shift[c]) inside the image (0 in the padding): the
// batch-norm preactivation of a ResNet-v2 unit fused into the gathers of the convolutions that read it
struct BnReluIn {
  const float* __restrict__ scale;   // may be NULL
  const float* __restrict__ shift;
  int s;
  static constexpr bool ON = true;
  __device__ __forceinline__ void origin(Pix& p) const {
    p.oy *= s;
    p.ox *= s;
  }
  __device__ __forceinline__ float apply(float v, int c) const {
    return scale ? fmaxf(fmaf(v, __ldg(scale + c), __ldg(shift + c)), 0.f) : v;
  }
};

// ------------------------------------------------------------------------------------------------------------
// Output policies of the forward kernels.  cols() is the width of the output the grid's y axis tiles.  A GATED
// tile multiplies output column f and its gate column cols + f together and stores both through one call.
// ------------------------------------------------------------------------------------------------------------
// y[m, o] = act(acc + bias[o]): the conv2d forward and data gradient, the VGG 3x3
struct BiasAct {
  const float* __restrict__ bias;   // may be NULL
  float* __restrict__ y;
  int act;
  static constexpr bool GATED = false;
  __host__ __device__ int cols(const ConvGeom& g) const { return g.K; }
  __device__ __forceinline__ void operator()(const ConvGeom& g, int64_t m, int o, float v) const {
    y[m * g.K + o] = act_apply(v + (bias ? __ldg(bias + o) : 0.f), act);
  }
};

// y[m, o] = acc + res[m, o]: the GLU data gradient
struct AddRes {
  const float* __restrict__ res;
  float* __restrict__ y;
  static constexpr bool GATED = false;
  __host__ __device__ int cols(const ConvGeom& g) const { return g.K; }
  __device__ __forceinline__ void operator()(const ConvGeom& g, int64_t m, int o, float v) const {
    y[m * g.K + o] = v + __ldg(res + m * g.K + o);
  }
};

// z = acc + bias, y[m, f] = z_lin * sigmoid(z_gate) + res[m, f], z [M, 2F] stored when non-NULL: the GLU forward
struct Glu {
  const float* __restrict__ bias;
  const float* __restrict__ res;
  float* __restrict__ y;
  float* __restrict__ z;
  int64_t F;
  static constexpr bool GATED = true;
  __host__ __device__ int cols(const ConvGeom&) const { return (int)F; }
  __device__ __forceinline__ void operator()(const ConvGeom&, int64_t m, int f, float lin, float gate) const {
    const float zl = lin + __ldg(bias + f), zg = gate + __ldg(bias + F + f);
    if (z) {
      z[m * 2 * F + f] = zl;
      z[m * 2 * F + F + f] = zg;
    }
    y[m * F + f] = zl * sigmoidf_(zg) + __ldg(res + m * F + f);
  }
};

// y[m, o] = act(z + res[n, oy*rs, ox*rs, o]) with z = acc * scale[o] + shift[o] (an inference-mode batch norm) when
// scale is non-NULL, else acc + bias[o]; res [N, Hr, Wr, K] may be NULL.  The ResNet-v2 convolutions.
struct BnRes {
  const float* __restrict__ scale;   // may be NULL
  const float* __restrict__ shift;
  const float* __restrict__ bias;    // may be NULL
  const float* __restrict__ res;     // may be NULL
  float* __restrict__ y;
  int act, rs, Hr, Wr;
  static constexpr bool GATED = false;
  __host__ __device__ int cols(const ConvGeom& g) const { return g.K; }
  __device__ __forceinline__ void operator()(const ConvGeom& g, int64_t m, int o, float v) const {
    float z = scale ? fmaf(v, __ldg(scale + o), __ldg(shift + o)) : v + (bias ? __ldg(bias + o) : 0.f);
    if (res) {
      const int64_t hw = (int64_t)g.Ho * g.Wo;
      const int64_t n = m / hw;
      const int r = (int)(m - n * hw);
      const int oy = r / g.Wo, ox = r - oy * g.Wo;
      z += __ldg(res + ((n * Hr + (int64_t)oy * rs) * Wr + (int64_t)ox * rs) * g.K + o);
    }
    y[m * g.K + o] = act_apply(z, act);
  }
};

// ------------------------------------------------------------------------------------------------------------
// wgmma engine: 128 x BN output tile, 2 consumer warpgroups of 64 rows, 32-wide k-blocks in a 2-stage ring.
// All 256 threads gather the next k-block while the tensor cores work on the current one.  A gated tile holds the
// output columns c0 + n in [0, BN/2) and their gates in [BN/2, BN), so each thread holds a column and its gate in
// accumulators i and i + BN/16.
// ------------------------------------------------------------------------------------------------------------
constexpr int CT_BM = 128, CT_BK = 32, CT_THREADS = 256;
constexpr int CT_A_BYTES = CT_BM * 128;
// log2 of a tile width, for index arithmetic the compiler keeps in shifts
__host__ __device__ constexpr int tile_log2(int bn) { return bn > 1 ? 1 + tile_log2(bn / 2) : 0; }
template <int BN>
__host__ __device__ constexpr int ct_stage() { return CT_A_BYTES + BN * 128; }
template <int BN>
__host__ __device__ constexpr int ct_smem() { return 2 * ct_stage<BN>() + 1024; }   // + slack for 1 KB alignment

// Each warpgroup multiplies its 64 rows of the stage's A tile by the B tile (4 instructions of k = 8).
template <int BN>
__device__ __forceinline__ void ct_mma(float (&acc)[BN / 2], uint32_t stage_addr, int wg) {
  const uint32_t a = stage_addr + wg * 64 * 128, b = stage_addr + CT_A_BYTES;
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) Wgmma<BN, 4>::mma(acc, gmma_desc_sw128(a + k * 32), gmma_desc_sw128(b + k * 32));
  wgmma_commit();
}

// Forward / data gradient: epi(m, o, sum A(m, :) B(:, o)), A read through the input policy In.
template <int BN, bool FLIP, bool ONE_ROW, class Epi, class In = PlainIn>
__global__ void __launch_bounds__(CT_THREADS)
conv_fwd_tc_kernel(const float* __restrict__ x, const float* __restrict__ w, ConvGeom g, Epi epi, In in) {
  static_assert(!In::ON || (!FLIP && !ONE_ROW && !Epi::GATED), "the input policy reads a forward 2-D window");
  constexpr int TILE_COLS = Epi::GATED ? BN / 2 : BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * CT_BM;
  const int c0 = blockIdx.y * TILE_COLS;
  const int cols = epi.cols(g);
  const int num_kb = (g.Kd + CT_BK - 1) / CT_BK;
  const bool avec = (g.C & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const bool bvec = (g.C & 3) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0;

  // filter column of tile column n, or -1 past the output
  auto b_col = [&](int n) {
    const int o = c0 + (Epi::GATED ? (n & (BN / 2 - 1)) : n);
    if (o >= cols) return -1;
    return Epi::GATED && n >= BN / 2 ? cols + o : o;
  };

  // A: thread owns row tid/2 and the 16 k values of half tid&1
  const int arow = tid >> 1, ahalf = tid & 1;
  const int64_t am = m0 + arow;
  const bool arow_ok = am < g.M;
  Pix ap = ONE_ROW ? row_pix(g, am, arow_ok ? (int)(am % g.W) : 0) : conv_pix<false>(g, arow_ok ? am : 0);
  if constexpr (In::ON) in.origin(ap);

  auto gather = [&](int kb, uint8_t* st) {
    const int gk0 = kb * CT_BK + ahalf * 16;
    if (avec) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gk = gk0 + 4 * j;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        int64_t off;
        if (arow_ok && gk < g.Kd && conv_a_at<ONE_ROW>(g, ap, gk, off)) {
          v = __ldg(reinterpret_cast<const float4*>(x + off));
          if constexpr (In::ON) {
            const int c = gk % g.C;   // C % 4 == 0: the 4 channels share a tap
            v = make_float4(in.apply(v.x, c), in.apply(v.y, c + 1), in.apply(v.z, c + 2), in.apply(v.w, c + 3));
          }
        }
        sw128_store4(st, arow, ahalf * 4 + j, v);
      }
    } else {
#pragma unroll 4
      for (int j = 0; j < 16; ++j) {
        const int gk = gk0 + j;
        float v = 0.f;
        if constexpr (In::ON) {
          int64_t off;
          if (arow_ok && gk < g.Kd && conv_a_at<ONE_ROW>(g, ap, gk, off)) v = in.apply(__ldg(x + off), gk % g.C);
        } else {
          v = (arow_ok && gk < g.Kd) ? conv_a<ONE_ROW>(x, g, ap, gk) : 0.f;
        }
        sw128_store1(st, arow, ahalf * 16 + j, v);
      }
    }
    uint8_t* bt = st + CT_A_BYTES;
    if constexpr (!FLIP) {
      // B: BN tile columns x 32 k values; consecutive threads take consecutive columns (w is [Kd, K])
#pragma unroll
      for (int j = 0; j < BN * CT_BK / CT_THREADS; ++j) {
        const int it = tid + CT_THREADS * j;
        const int n = it & (BN - 1), word = it >> tile_log2(BN);
        const int gk = kb * CT_BK + word, o = b_col(n);
        sw128_store1(bt, n, word, (gk < g.Kd && o >= 0) ? conv_b<false, ONE_ROW>(w, g, gk, o) : 0.f);
      }
    } else {
      // B: each column's k values are contiguous within a tap of the flipped filter; a thread owns column bn and
      // BK_T of them
      static_assert(!Epi::GATED, "a gated tile reads the forward filter");
      constexpr int THR_PER_COL = CT_THREADS / BN, BK_T = CT_BK / THR_PER_COL;
      const int bn = tid / THR_PER_COL, bk0 = (tid % THR_PER_COL) * BK_T;
      const int o = c0 + bn;
      const int taps = ONE_ROW ? g.kw : g.kh * g.kw;
      if (bvec) {
#pragma unroll
        for (int j = 0; j < BK_T / 4; ++j) {
          const int gk = kb * CT_BK + bk0 + 4 * j;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (o < cols && gk < g.Kd) {
            const int tap = gk / g.C, c = gk - tap * g.C;
            v = __ldg(reinterpret_cast<const float4*>(w + ((int64_t)(taps - 1 - tap) * g.K + o) * g.C + c));
          }
          sw128_store4(bt, bn, bk0 / 4 + j, v);
        }
      } else {
#pragma unroll 4
        for (int j = 0; j < BK_T; ++j) {
          const int gk = kb * CT_BK + bk0 + j;
          sw128_store1(bt, bn, bk0 + j, (o < cols && gk < g.Kd) ? conv_b<true, ONE_ROW>(w, g, gk, o) : 0.f);
        }
      }
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  const int wg = tid >> 7;

  gather(0, smem);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb & 1;
    ct_mma<BN>(acc, sbase + s * ct_stage<BN>(), wg);
    // the other stage was last read by the products of kb-1, which completed before the barrier below
    if (kb + 1 < num_kb) gather(kb + 1, smem + (s ^ 1) * ct_stage<BN>());
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  }

  const int lane = tid & 31, wq = (tid >> 5) & 3;
  const int64_t r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < TILE_COLS / 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t m = r0 + 8 * h;
      if (m >= g.M) continue;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int o = c0 + 8 * i + 2 * (lane & 3) + e;
        if (o >= cols) continue;
        if constexpr (Epi::GATED)
          epi(g, m, o, acc[4 * i + 2 * h + e], acc[4 * (i + BN / 16) + 2 * h + e]);
        else
          epi(g, m, o, acc[4 * i + 2 * h + e]);
      }
    }
  }
}

// Weight gradient partials: ws[split][r][o] = sum over this split's pixels of A'(r, m) dY(m, o), where
// A'(r, m) = A(m, r) for r < Kd and A'(Kd, m) = 1 (the bias row).
template <int BN, bool ONE_ROW>
__global__ void __launch_bounds__(CT_THREADS)
conv_wgrad_tc_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ ws, ConvGeom g,
                     int kb_per_split) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ Pix pix[2][ONE_ROW ? 1 : CT_BK];   // the pixels of a k-block (a one-row image needs only ox)
  __shared__ int pix_x[2][CT_BK];               // -1 past M, else ox of a one-row image (0 otherwise)
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x;
  const int rows = g.Kd + 1;
  const int r0 = blockIdx.y * CT_BM;
  const int o0 = blockIdx.x * BN;
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
    if (ONE_ROW) {
      kx = tap;
    } else {
      ky = tap / g.kw;
      kx = tap - ky * g.kw;
    }
  }
  const int dyo = ky - g.pt, dxo = kx - g.pl;

  auto decode = [&](int kb, int buf) {
    if (tid < CT_BK) {
      const int64_t m = (int64_t)(kb0 + kb) * CT_BK + tid;
      if (ONE_ROW) {
        pix_x[buf][tid] = m < g.M ? (int)(m % g.W) : -1;
      } else {
        pix_x[buf][tid] = m < g.M ? 0 : -1;
        pix[buf][tid] = conv_pix<false>(g, m < g.M ? m : 0);
      }
    }
  };
  auto gather = [&](int kb, int buf, uint8_t* st) {
    const int64_t mb = (int64_t)(kb0 + kb) * CT_BK;
#pragma unroll 4
    for (int j = 0; j < 16; ++j) {
      const int word = aw + 2 * j;
      const int ox = pix_x[buf][word];
      float v = 0.f;
      if (ox >= 0) {
        if (is_bias) {
          v = 1.f;
        } else if (row_ok) {
          if (ONE_ROW) {
            const int ix = ox + dxo;
            if (ix >= 0 && ix < g.W) v = __ldg(x + (mb + word + dxo) * g.C + c);
          } else {
            const Pix p = pix[buf][word];
            const int iy = p.oy + dyo, ix = p.ox + dxo;
            if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
              v = __ldg(x + (p.base + (int64_t)iy * g.W + ix) * g.C + c);
          }
        }
      }
      sw128_store1(st, arow, word, v);
    }
    uint8_t* bt = st + CT_A_BYTES;
#pragma unroll
    for (int j = 0; j < BN * CT_BK / CT_THREADS; ++j) {
      const int it = tid + CT_THREADS * j;
      const int o = it & (BN - 1), word = it >> tile_log2(BN);
      const int64_t m = mb + word;
      const int go = o0 + o;
      sw128_store1(bt, o, word, (m < g.M && go < g.K) ? __ldg(dy + m * g.K + go) : 0.f);
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
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
    ct_mma<BN>(acc, sbase + s * ct_stage<BN>(), wg);
    if (kb + 1 < num_kb) gather(kb + 1, s ^ 1, smem + (s ^ 1) * ct_stage<BN>());
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
  for (int i = 0; i < BN / 8; ++i) {
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
// Exact fp32 engine (NM_GEMM_SIMT): 64 x 64 tiles of gemm_simt.cuh, operands gathered the same way.  A gated tile's
// column n is output column c0 + 2*(n/4) + (n & 1), its gate when (n/2) is odd, so the 4 columns of a thread are
// two outputs and their two gates.
// ------------------------------------------------------------------------------------------------------------
constexpr int CS_BM = 64, CS_BN = 64, CS_TM = 4, CS_TN = 4;

template <bool FLIP, bool ONE_ROW, class Epi, class In = PlainIn>
__global__ void __launch_bounds__(SIMT_THREADS)
conv_fwd_simt_kernel(const float* __restrict__ x, const float* __restrict__ w, ConvGeom g, Epi epi, In in) {
  static_assert(!In::ON || (!FLIP && !ONE_ROW && !Epi::GATED), "the input policy reads a forward 2-D window");
  constexpr int A_LOADS = (CS_BM * SIMT_BK) / SIMT_THREADS;
  __shared__ SimtSmem<CS_BM, CS_BN, CS_TM, CS_TN> sm;
  const int64_t m0 = (int64_t)blockIdx.x * CS_BM;
  const int c0 = blockIdx.y * (Epi::GATED ? CS_BN / 2 : CS_BN);
  const int cols = epi.cols(g);
  const int t = threadIdx.x;
  const int tx = t % (CS_BN / CS_TN), ty = t / (CS_BN / CS_TN);
  // the A rows this thread loads, (t + 256 i) / SIMT_BK = t / SIMT_BK + 16 i: -1 past M, else ox in a one-row image
  // (0 otherwise)
  int arow_x[A_LOADS];
#pragma unroll
  for (int i = 0; i < A_LOADS; ++i) {
    const int64_t gm = m0 + t / SIMT_BK + i * (SIMT_THREADS / SIMT_BK);
    arow_x[i] = gm < g.M ? (ONE_ROW ? (int)(gm % g.W) : 0) : -1;
  }
  float acc[CS_TM][CS_TN] = {};
  for (int k0 = 0; k0 < g.Kd; k0 += SIMT_BK) {
#pragma unroll
    for (int i = 0; i < A_LOADS; ++i) {
      const int mm = t / SIMT_BK + i * (SIMT_THREADS / SIMT_BK), kk = t % SIMT_BK;
      const int64_t gm = m0 + mm;
      const int gk = k0 + kk;
      float v = 0.f;
      if constexpr (In::ON) {
        Pix p = conv_pix<false>(g, gm);
        in.origin(p);
        int64_t off;
        if (arow_x[i] >= 0 && gk < g.Kd && conv_a_at<false>(g, p, gk, off)) v = in.apply(__ldg(x + off), gk % g.C);
      } else if (arow_x[i] >= 0 && gk < g.Kd) {
        v = conv_a<ONE_ROW>(x, g, ONE_ROW ? row_pix(g, gm, arow_x[i]) : conv_pix<false>(g, gm), gk);
      }
      sm.a[kk][mm] = v;
    }
#pragma unroll
    for (int i = 0; i < (CS_BN * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int kk = idx / CS_BN, n = idx % CS_BN;
      const int gk = k0 + kk;
      int o = c0 + n;
      if (Epi::GATED) {
        const int f = c0 + 2 * (n >> 2) + (n & 1);
        o = ((n >> 1) & 1) ? cols + f : f;
        if (f >= cols) o = -1;
      } else if (o >= cols) {
        o = -1;
      }
      sm.b[kk][n] = (gk < g.Kd && o >= 0) ? conv_b<FLIP, ONE_ROW>(w, g, gk, o) : 0.f;
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
    if constexpr (Epi::GATED) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int f = c0 + 2 * tx + j;
        if (f < cols) epi(g, m, f, acc[i][j], acc[i][j + 2]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < CS_TN; ++j) {
        const int o = c0 + tx * CS_TN + j;
        if (o < cols) epi(g, m, o, acc[i][j]);
      }
    }
  }
}

template <bool ONE_ROW>
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
        else if (gr < g.Kd) v = conv_a<ONE_ROW>(x, g, conv_pix<ONE_ROW>(g, m), gr);
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

// dw[r, o] += sum_s ws[s][r][o] (r < Kd), db[o] += sum_s ws[s][Kd][o] unless db is NULL; splits summed in index
// order.
static __global__ void conv_wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw,
                                                float* __restrict__ db, int64_t rows, int64_t K, int splits) {
  const int64_t total = rows * K;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < splits; ++j) s += ws[j * total + i];
    const int64_t r = i / K;
    if (r < rows - 1) dw[i] += s;
    else if (db) db[i - r * K] += s;
  }
}

// blocks of 256 threads for a grid-stride loop over `total` elements
static inline unsigned grid_for(int64_t total) {
  const int64_t blocks = ceil_div(total, 256), cap = (int64_t)sm_count() * 16;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// Forward / data-gradient launch on the engine `backend` selects, like nm_gemm's.
template <int BN, bool FLIP, bool ONE_ROW, class Epi, class In = PlainIn>
static int conv_fwd_launch(const float* x, const float* w, const ConvGeom& g, const Epi& epi, int backend,
                           cudaStream_t s, const char* name, const In& in = In{}) {
  // pixel tiles along x (up to 2^31 - 1 of them), output-column tiles along y
  const int64_t cols = epi.cols(g);
  if (backend == NM_GEMM_SIMT) {
    const int64_t tile_cols = Epi::GATED ? CS_BN / 2 : CS_BN;
    NM_REQUIRE(ceil_div(g.M, CS_BM) <= 0x7fffffffLL && ceil_div(cols, tile_cols) <= 65535, NM_E_UNSUPPORTED,
               "%s: grid too large", name);
    dim3 grid((unsigned)ceil_div(g.M, CS_BM), (unsigned)ceil_div(cols, tile_cols));
    conv_fwd_simt_kernel<FLIP, ONE_ROW, Epi, In><<<grid, SIMT_THREADS, 0, s>>>(x, w, g, epi, in);
    NM_LAUNCH_CHECK(name);
    return NM_OK;
  }
  NM_REQUIRE(backend == NM_GEMM_AUTO || backend == NM_GEMM_TC, NM_E_INVALID, "%s: bad backend", name);
  const int64_t tile_cols = Epi::GATED ? BN / 2 : BN;
  NM_REQUIRE(ceil_div(g.M, CT_BM) <= 0x7fffffffLL && ceil_div(cols, tile_cols) <= 65535, NM_E_UNSUPPORTED,
             "%s: grid too large", name);
  static bool attr = false;
  if (!attr) {
    NM_CUDA_TRY(cudaFuncSetAttribute(conv_fwd_tc_kernel<BN, FLIP, ONE_ROW, Epi, In>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, ct_smem<BN>()));
    attr = true;
  }
  dim3 grid((unsigned)ceil_div(g.M, CT_BM), (unsigned)ceil_div(cols, tile_cols));
  conv_fwd_tc_kernel<BN, FLIP, ONE_ROW, Epi, In><<<grid, CT_THREADS, ct_smem<BN>(), s>>>(x, w, g, epi, in);
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

// The weight-gradient launch: tile counts and how far the pixel reduction is split - until ~4 CTAs per SM are
// busy, within the workspace (ws_cap floats; < 0 = unbounded).  One place decides it, for the launch and for the
// workspace queries.
struct WgradPlan {
  int64_t rows, part, tiles_r, tiles_o, splits, kb_per;
};

static WgradPlan wgrad_plan(const ConvGeom& g, int bm, int bn, int bk, int64_t ws_cap) {
  WgradPlan p;
  p.rows = (int64_t)g.Kd + 1;
  p.part = p.rows * g.K;
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

// the plan of the engine `backend` selects; BN is the wgmma tile width
template <int BN>
static WgradPlan wgrad_plan(const ConvGeom& g, int backend, int64_t ws_cap) {
  return backend == NM_GEMM_SIMT ? wgrad_plan(g, CS_BM, CS_BN, SIMT_BK, ws_cap)
                                 : wgrad_plan(g, CT_BM, BN, CT_BK, ws_cap);
}

// dw [Kd, K] += the weight gradient, db [K] += the bias gradient (db may be NULL)
template <int BN, bool ONE_ROW>
static int conv_wgrad_launch(const float* x, const float* dy, float* dw, float* db, float* workspace,
                             int64_t workspace_floats, const ConvGeom& g, int backend, cudaStream_t s,
                             const char* name) {
  const bool simt = backend == NM_GEMM_SIMT;
  NM_REQUIRE(simt || backend == NM_GEMM_AUTO || backend == NM_GEMM_TC, NM_E_INVALID, "%s: bad backend", name);
  const WgradPlan p = wgrad_plan<BN>(g, backend, workspace_floats);
  NM_REQUIRE(workspace_floats >= p.part, NM_E_INVALID, "%s: workspace below (taps*Cin+1)*Cout floats", name);
  NM_REQUIRE(p.tiles_r <= 65535 && p.tiles_o <= 65535, NM_E_UNSUPPORTED, "%s: filter too large", name);
  NM_REQUIRE(p.kb_per < (1LL << 31), NM_E_UNSUPPORTED, "%s: too many pixels", name);
  dim3 grid((unsigned)p.tiles_o, (unsigned)p.tiles_r, (unsigned)p.splits);
  if (simt) {
    conv_wgrad_simt_kernel<ONE_ROW><<<grid, SIMT_THREADS, 0, s>>>(x, dy, workspace, g, (int)p.kb_per);
  } else {
    static bool attr = false;
    if (!attr) {
      NM_CUDA_TRY(cudaFuncSetAttribute(conv_wgrad_tc_kernel<BN, ONE_ROW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       ct_smem<BN>()));
      attr = true;
    }
    conv_wgrad_tc_kernel<BN, ONE_ROW><<<grid, CT_THREADS, ct_smem<BN>(), s>>>(x, dy, workspace, g, (int)p.kb_per);
  }
  NM_LAUNCH_CHECK(name);
  conv_wgrad_reduce_kernel<<<grid_for(p.part), 256, 0, s>>>(workspace, dw, db, p.rows, g.K, (int)p.splits);
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

}  // namespace nm
