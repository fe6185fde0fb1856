// K8: multi-head scaled dot-product attention core
// (attention/scaled_dot_product.py:160-214 of the reference) between the q/k/v
// projections and the output projection.  Reproduces the reference's masking
// semantics exactly: causal positions are REPLACED by -1e9 (tf.where), padded keys
// get E*m + (1-m)*(-1e9), both before the softmax; -1e9, not -inf.
//
// Two implementations: tiled kernels (below) for training shapes - one CTA per (32 query rows,
// head, sentence) with the head's K/V resident in shared memory - and the original row kernels
// (one CTA per query position) for everything else: single-query decoding steps, fewer than 8
// queries, odd or wide head sizes, more than 256 positions.  Both families take the attention-weight
// dropout mask (DROP below), so dropout works at every shape the row kernels' shared memory allows.
#include "common.cuh"

namespace nm {

constexpr int MHA_THREADS = 128;
constexpr float MHA_MASK = -1e9f;

// dynamic smem: qs[dh] | e[Tk].  DROP: as in mha_fwd_tile_kernel - the context is (p * drop) . V,
// `probs` keeps the undropped p.
template <bool DROP = false>
__global__ void __launch_bounds__(MHA_THREADS)
mha_fwd_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
               const float* __restrict__ key_mask, int causal, float* __restrict__ out,
               float* __restrict__ probs, int Tq, int Tk, int heads, int dh,
               const float* __restrict__ drop) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  float* qs = smem;
  float* e = smem + dh;
  const int tq = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * dh;
  const float scale = sqrtf((float)dh);
  for (int d = threadIdx.x; d < dh; d += MHA_THREADS)
    qs[d] = q[((int64_t)b * Tq + tq) * D + h * dh + d] / scale;
  __syncthreads();
  float lmax = -INFINITY;
  for (int tk = threadIdx.x; tk < Tk; tk += MHA_THREADS) {
    const float* kr = k + ((int64_t)b * Tk + tk) * D + h * dh;
    float acc = 0.f;
    for (int d = 0; d < dh; ++d) acc = fmaf(qs[d], kr[d], acc);
    if (causal && tk > tq) acc = MHA_MASK;
    if (key_mask) {
      const float m = key_mask[(int64_t)b * Tk + tk];
      acc = acc * m + (1.f - m) * MHA_MASK;
    }
    e[tk] = acc;
    lmax = fmaxf(lmax, acc);
  }
  const float mx = block_max(lmax, red);
  float lsum = 0.f;
  for (int tk = threadIdx.x; tk < Tk; tk += MHA_THREADS) {
    const float p = expf(e[tk] - mx);
    e[tk] = p;
    lsum += p;
  }
  const float s = block_sum(lsum, red);
  float* pr = probs + (((int64_t)b * heads + h) * Tq + tq) * Tk;
  const float* dr = DROP ? drop + (((int64_t)b * heads + h) * Tq + tq) * Tk : nullptr;
  for (int tk = threadIdx.x; tk < Tk; tk += MHA_THREADS) {
    const float p = e[tk] / s;
    e[tk] = DROP ? p * dr[tk] : p;
    pr[tk] = p;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < dh; d += MHA_THREADS) {
    const float* vc = v + (int64_t)b * Tk * D + h * dh + d;
    float acc = 0.f;
    for (int tk = 0; tk < Tk; ++tk) acc = fmaf(e[tk], vc[(int64_t)tk * D], acc);
    out[((int64_t)b * Tq + tq) * D + h * dh + d] = acc;
  }
}

// backward A: per query row: dE (pre-mask gradient) and dq.  smem: dos[dh] | de[Tk].
// DROP: d(softmax) = drop * (dO . V), and the row sum and dE are formed from it.
template <bool DROP = false>
__global__ void __launch_bounds__(MHA_THREADS)
mha_bwd_q_kernel(const float* __restrict__ k, const float* __restrict__ v,
                 const float* __restrict__ key_mask, int causal, const float* __restrict__ probs,
                 const float* __restrict__ dout, float* __restrict__ dq, float* __restrict__ de_out,
                 int Tq, int Tk, int heads, int dh, const float* __restrict__ drop) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  float* dos = smem;
  float* de = smem + dh;
  const int tq = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * dh;
  for (int d = threadIdx.x; d < dh; d += MHA_THREADS)
    dos[d] = dout[((int64_t)b * Tq + tq) * D + h * dh + d];
  __syncthreads();
  const float* pr = probs + (((int64_t)b * heads + h) * Tq + tq) * Tk;
  const float* dr = DROP ? drop + (((int64_t)b * heads + h) * Tq + tq) * Tk : nullptr;
  float lsum = 0.f;
  for (int tk = threadIdx.x; tk < Tk; tk += MHA_THREADS) {
    const float* vr = v + ((int64_t)b * Tk + tk) * D + h * dh;
    float dp = 0.f;
    for (int d = 0; d < dh; ++d) dp = fmaf(dos[d], vr[d], dp);
    if (DROP) dp *= dr[tk];
    de[tk] = dp;
    lsum += dp * pr[tk];
  }
  const float pdp = block_sum(lsum, red);
  float* der = de_out + (((int64_t)b * heads + h) * Tq + tq) * Tk;
  for (int tk = threadIdx.x; tk < Tk; tk += MHA_THREADS) {
    float g = pr[tk] * (de[tk] - pdp);
    if (key_mask) g *= key_mask[(int64_t)b * Tk + tk];  // d(E*m + c)/dE = m
    if (causal && tk > tq) g = 0.f;                     // tf.where: no gradient to replaced entries
    de[tk] = g;
    der[tk] = g;
  }
  __syncthreads();
  const float scale = sqrtf((float)dh);
  for (int d = threadIdx.x; d < dh; d += MHA_THREADS) {
    const float* kc = k + (int64_t)b * Tk * D + h * dh + d;
    float acc = 0.f;
    for (int tk = 0; tk < Tk; ++tk) acc = fmaf(de[tk], kc[(int64_t)tk * D], acc);
    dq[((int64_t)b * Tq + tq) * D + h * dh + d] = acc / scale;
  }
}

// backward B: per key row: dk and dv.  DROP: dV sees the dropped weights p * drop.
template <bool DROP = false>
__global__ void __launch_bounds__(MHA_THREADS)
mha_bwd_kv_kernel(const float* __restrict__ q, const float* __restrict__ probs,
                  const float* __restrict__ de, const float* __restrict__ dout,
                  float* __restrict__ dk, float* __restrict__ dv, int Tq, int Tk, int heads, int dh,
                  const float* __restrict__ drop) {
  const int tk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * dh;
  const float scale = sqrtf((float)dh);
  const float* pcol = probs + ((int64_t)b * heads + h) * Tq * Tk + tk;
  const float* dcol = de + ((int64_t)b * heads + h) * Tq * Tk + tk;
  const float* rcol = DROP ? drop + ((int64_t)b * heads + h) * Tq * Tk + tk : nullptr;
  for (int d = threadIdx.x; d < dh; d += MHA_THREADS) {
    float ak = 0.f, av = 0.f;
    for (int tq = 0; tq < Tq; ++tq) {
      const int64_t o = ((int64_t)b * Tq + tq) * D + h * dh + d;
      ak = fmaf(dcol[(int64_t)tq * Tk], q[o] / scale, ak);
      float p = pcol[(int64_t)tq * Tk];
      if (DROP) p *= rcol[(int64_t)tq * Tk];
      av = fmaf(p, dout[o], av);
    }
    const int64_t o = ((int64_t)b * Tk + tk) * D + h * dh + d;
    dk[o] = ak;
    dv[o] = av;
  }
}

// ---------------------------------------------------------------------------------------
// Tiled kernels (the path training takes): one CTA per (block of 32 query rows, head, sentence)
// keeps the head's K and V in shared memory, 8 threads share a query row.  Exact fp32.
//   smem (floats): Ks[TKP][dh+1] | Vs[TKP][dh+1] | Qs[32][dh+1] | Ps[32][TKP+1],  TKP = 8*NJ
// ---------------------------------------------------------------------------------------
constexpr int MT_QB = 32, MT_THREADS = 256;

__device__ __forceinline__ float group8_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
}
__device__ __forceinline__ float group8_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v + __shfl_xor_sync(0xffffffffu, v, 4);
}

// rows [0,nrows) x dh floats from a [*, D]-strided head slice into smem with pitch `pitch`;
// rows up to `fill_rows` are zero-filled.
__device__ __forceinline__ void mt_load_head(float* dst, int pitch, const float* src, int64_t row_stride,
                                             int nrows, int fill_rows, int dh, float mul) {
  const int q4 = dh >> 2;
  for (int idx = threadIdx.x; idx < fill_rows * q4; idx += MT_THREADS) {
    const int r = idx / q4, c = (idx - r * q4) << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < nrows) v = *reinterpret_cast<const float4*>(src + (int64_t)r * row_stride + c);
    float* d = dst + r * pitch + c;
    d[0] = v.x * mul; d[1] = v.y * mul; d[2] = v.z * mul; d[3] = v.w * mul;
  }
}

// DROP: attention-weight dropout (scaled_dot_product.py:208-214: weights = dropout(softmax(E)), context =
// weights . V).  `drop` is the mask already scaled by 1/keep_prob, [B, heads, Tq, Tk]; `probs` keeps the
// UNdropped softmax, which is what the backward of the softmax needs.  A trailing parameter and a
// template flag, so the instances without dropout are the code they were.
template <int NJ, bool DROP = false>
__global__ void __launch_bounds__(MT_THREADS)
mha_fwd_tile_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                    const float* __restrict__ key_mask, int causal, float* __restrict__ out,
                    float* __restrict__ probs, int Tq, int Tk, int heads, int dh,
                    const float* __restrict__ drop) {
  extern __shared__ float smem[];
  constexpr int TKP = 8 * NJ;
  const int kp = dh + 1;
  float* Ks = smem;
  float* Vs = Ks + TKP * kp;
  float* Qs = Vs + TKP * kp;
  float* Ps = Qs + MT_QB * kp;
  const int q0 = blockIdx.x * MT_QB, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * dh;
  const int nq = min(MT_QB, Tq - q0);
  const float inv_scale = 1.f / sqrtf((float)dh);
  mt_load_head(Ks, kp, k + (int64_t)b * Tk * D + h * dh, D, Tk, TKP, dh, 1.f);
  mt_load_head(Vs, kp, v + (int64_t)b * Tk * D + h * dh, D, Tk, TKP, dh, 1.f);
  mt_load_head(Qs, kp, q + ((int64_t)b * Tq + q0) * D + h * dh, D, nq, MT_QB, dh, inv_scale);
  __syncthreads();
  const int i = threadIdx.x >> 3, jg = threadIdx.x & 7;
  const int tq = q0 + i;
  float acc[NJ];
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) acc[jj] = 0.f;
  for (int d = 0; d < dh; ++d) {
    const float qv = Qs[i * kp + d];
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj) acc[jj] = fmaf(qv, Ks[(jg + 8 * jj) * kp + d], acc[jj]);
  }
  float mx = -INFINITY;
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) {
    const int j = jg + 8 * jj;
    float e = acc[jj];
    if (j < Tk) {
      if (causal && j > tq) e = MHA_MASK;
      if (key_mask) {
        const float m = key_mask[(int64_t)b * Tk + j];
        e = e * m + (1.f - m) * MHA_MASK;
      }
    } else {
      e = -INFINITY;
    }
    acc[jj] = e;
    mx = fmaxf(mx, e);
  }
  mx = group8_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) {
    acc[jj] = expf(acc[jj] - mx);
    sum += acc[jj];
  }
  sum = group8_sum(sum);
  float* pr = probs + (((int64_t)b * heads + h) * Tq + tq) * Tk;
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) {
    const int j = jg + 8 * jj;
    const float p = acc[jj] / sum;
    float pd = p;
    if (DROP) {
      if (i < nq && j < Tk) pd = p * drop[(((int64_t)b * heads + h) * Tq + tq) * Tk + j];
    }
    Ps[i * (TKP + 1) + j] = pd;
    if (i < nq && j < Tk) pr[j] = p;
  }
  __syncwarp();
  // O[i][d] = sum_j P[i][j] V[j][d];  this thread: d = jg + 8*dd
  float o[16];
#pragma unroll
  for (int dd = 0; dd < 16; ++dd) o[dd] = 0.f;
  const int nd = dh >> 3;
  for (int j = 0; j < Tk; ++j) {
    const float p = Ps[i * (TKP + 1) + j];
#pragma unroll
    for (int dd = 0; dd < 16; ++dd)
      if (dd < nd) o[dd] = fmaf(p, Vs[j * kp + jg + 8 * dd], o[dd]);
  }
  if (i < nq) {
    float* op = out + ((int64_t)b * Tq + tq) * D + h * dh;
#pragma unroll
    for (int dd = 0; dd < 16; ++dd)
      if (dd < nd) op[jg + 8 * dd] = o[dd];
  }
}

// backward A (per block of query rows): dE -> de_out, dq
template <int NJ, bool DROP = false>
__global__ void __launch_bounds__(MT_THREADS)
mha_bwd_q_tile_kernel(const float* __restrict__ k, const float* __restrict__ v,
                      const float* __restrict__ key_mask, int causal, const float* __restrict__ probs,
                      const float* __restrict__ dout, float* __restrict__ dq, float* __restrict__ de_out,
                      int Tq, int Tk, int heads, int dh, const float* __restrict__ drop) {
  extern __shared__ float smem[];
  constexpr int TKP = 8 * NJ;
  const int kp = dh + 1;
  float* Ks = smem;
  float* Vs = Ks + TKP * kp;
  float* Os = Vs + TKP * kp;             // dO block
  float* Ps = Os + MT_QB * kp;           // dE block
  const int q0 = blockIdx.x * MT_QB, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * dh;
  const int nq = min(MT_QB, Tq - q0);
  mt_load_head(Ks, kp, k + (int64_t)b * Tk * D + h * dh, D, Tk, TKP, dh, 1.f);
  mt_load_head(Vs, kp, v + (int64_t)b * Tk * D + h * dh, D, Tk, TKP, dh, 1.f);
  mt_load_head(Os, kp, dout + ((int64_t)b * Tq + q0) * D + h * dh, D, nq, MT_QB, dh, 1.f);
  __syncthreads();
  const int i = threadIdx.x >> 3, jg = threadIdx.x & 7;
  const int tq = q0 + i;
  const float* pr = probs + (((int64_t)b * heads + h) * Tq + tq) * Tk;
  float acc[NJ], p[NJ];
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) {
    const int j = jg + 8 * jj;
    acc[jj] = 0.f;
    p[jj] = (i < nq && j < Tk) ? pr[j] : 0.f;
  }
  for (int d = 0; d < dh; ++d) {
    const float ov = Os[i * kp + d];
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj) acc[jj] = fmaf(ov, Vs[(jg + 8 * jj) * kp + d], acc[jj]);
  }
  if (DROP) {   // d(dropped weights) -> d(softmax): times the same mask
#pragma unroll
    for (int jj = 0; jj < NJ; ++jj) {
      const int j = jg + 8 * jj;
      if (i < nq && j < Tk) acc[jj] *= drop[(((int64_t)b * heads + h) * Tq + tq) * Tk + j];
    }
  }
  float dot = 0.f;
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) dot = fmaf(acc[jj], p[jj], dot);
  dot = group8_sum(dot);
  float* der = de_out + (((int64_t)b * heads + h) * Tq + tq) * Tk;
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) {
    const int j = jg + 8 * jj;
    float g = p[jj] * (acc[jj] - dot);
    if (j < Tk) {
      if (key_mask) g *= key_mask[(int64_t)b * Tk + j];   // d(E*m + c)/dE = m
      if (causal && j > tq) g = 0.f;                       // tf.where: no gradient to replaced entries
    } else {
      g = 0.f;
    }
    Ps[i * (TKP + 1) + j] = g;
    if (i < nq && j < Tk) der[j] = g;
  }
  __syncwarp();
  float o[16];
#pragma unroll
  for (int dd = 0; dd < 16; ++dd) o[dd] = 0.f;
  const int nd = dh >> 3;
  for (int j = 0; j < Tk; ++j) {
    const float g = Ps[i * (TKP + 1) + j];
#pragma unroll
    for (int dd = 0; dd < 16; ++dd)
      if (dd < nd) o[dd] = fmaf(g, Ks[j * kp + jg + 8 * dd], o[dd]);
  }
  if (i < nq) {
    const float inv_scale = 1.f / sqrtf((float)dh);
    float* op = dq + ((int64_t)b * Tq + tq) * D + h * dh;
#pragma unroll
    for (int dd = 0; dd < 16; ++dd)
      if (dd < nd) op[jg + 8 * dd] = o[dd] * inv_scale;
  }
}

// backward B (per block of 32 key rows): dk, dv.  smem: Qs[Tq][dh] (scaled) | Os[Tq][dh] | Et[Tq][33] | Pt[Tq][33]
template <bool DROP = false>
__global__ void __launch_bounds__(MT_THREADS)
mha_bwd_kv_tile_kernel(const float* __restrict__ q, const float* __restrict__ probs,
                       const float* __restrict__ de, const float* __restrict__ dout,
                       float* __restrict__ dk, float* __restrict__ dv, int Tq, int Tk, int heads, int dh,
                       const float* __restrict__ drop) {
  extern __shared__ float smem[];
  float* Qs = smem;
  float* Os = Qs + Tq * dh;
  float* Et = Os + Tq * dh;
  float* Pt = Et + Tq * 33;
  const int j0 = blockIdx.x * MT_QB, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * dh;
  const int nj = min(MT_QB, Tk - j0);
  const float inv_scale = 1.f / sqrtf((float)dh);
  mt_load_head(Qs, dh, q + (int64_t)b * Tq * D + h * dh, D, Tq, Tq, dh, inv_scale);
  mt_load_head(Os, dh, dout + (int64_t)b * Tq * D + h * dh, D, Tq, Tq, dh, 1.f);
  const float* pb = probs + ((int64_t)b * heads + h) * Tq * Tk + j0;
  const float* eb = de + ((int64_t)b * heads + h) * Tq * Tk + j0;
  for (int idx = threadIdx.x; idx < Tq * 32; idx += MT_THREADS) {
    const int i = idx >> 5, jl = idx & 31;
    const bool ok = jl < nj;
    Et[i * 33 + jl] = ok ? eb[(int64_t)i * Tk + jl] : 0.f;
    float pv = ok ? pb[(int64_t)i * Tk + jl] : 0.f;
    if (DROP) {   // dV sees the dropped weights
      if (ok) pv *= drop[((int64_t)b * heads + h) * Tq * Tk + j0 + (int64_t)i * Tk + jl];
    }
    Pt[i * 33 + jl] = pv;
  }
  __syncthreads();
  const int jl = threadIdx.x >> 3, dg = threadIdx.x & 7;
  float ak[16], av[16];
#pragma unroll
  for (int dd = 0; dd < 16; ++dd) ak[dd] = av[dd] = 0.f;
  const int nd = dh >> 3;
  for (int i = 0; i < Tq; ++i) {
    const float ge = Et[i * 33 + jl], pp = Pt[i * 33 + jl];
#pragma unroll
    for (int dd = 0; dd < 16; ++dd)
      if (dd < nd) {
        ak[dd] = fmaf(ge, Qs[i * dh + dg + 8 * dd], ak[dd]);
        av[dd] = fmaf(pp, Os[i * dh + dg + 8 * dd], av[dd]);
      }
  }
  if (jl < nj) {
    const int64_t o = ((int64_t)b * Tk + j0 + jl) * D + h * dh;
#pragma unroll
    for (int dd = 0; dd < 16; ++dd)
      if (dd < nd) {
        dk[o + dg + 8 * dd] = ak[dd];
        dv[o + dg + 8 * dd] = av[dd];
      }
  }
}

// The tiled path needs dh % 8 == 0, dh <= 128, Tk <= 256 and a block of query rows worth tiling.
static bool mt_ok(int64_t Tq, int64_t Tk, int64_t dh, int64_t D) {
  return dh % 8 == 0 && dh <= 128 && Tk <= 256 && Tq >= 8 && Tq <= 256 && D % 4 == 0;
}
static size_t mt_smem_q(int64_t Tk, int64_t dh) {
  const int64_t TKP = Tk <= 64 ? 64 : (Tk <= 128 ? 128 : 256);
  return sizeof(float) * (size_t)(2 * TKP * (dh + 1) + MT_QB * (dh + 1) + MT_QB * (TKP + 1));
}
static size_t mt_smem_kv(int64_t Tq, int64_t dh) { return sizeof(float) * (size_t)(2 * Tq * dh + 2 * Tq * 33); }

template <class Kern>
static int mt_set_smem(Kern kern, size_t smem) {
  if (smem > 48 * 1024)
    NM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

static int mha_fwd_impl(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                        float* out, float* probs, int64_t B, int64_t Tq, int64_t Tk, int64_t heads,
                        int64_t dh, const float* drop, void* stream) {
  NM_REQUIRE(q && k && v && out && probs, NM_E_INVALID, "nm_mha_fwd: null pointer");
  NM_REQUIRE(B > 0 && Tq > 0 && Tk > 0 && heads > 0 && dh > 0, NM_E_INVALID, "nm_mha_fwd: bad sizes");
  NM_REQUIRE(B <= 65535 && heads <= 65535, NM_E_UNSUPPORTED, "nm_mha_fwd: grid too large");
  if (mt_ok(Tq, Tk, dh, heads * dh) && mt_smem_q(Tk, dh) <= 200 * 1024) {
    const size_t sm = mt_smem_q(Tk, dh);
    dim3 grid((unsigned)((Tq + MT_QB - 1) / MT_QB), (unsigned)heads, (unsigned)B);
    cudaStream_t s = (cudaStream_t)stream;
#define NM_MT_FWD(NJ)                                                                              \
  {                                                                                                \
    if (drop) {                                                                                    \
      int rc = mt_set_smem(mha_fwd_tile_kernel<NJ, true>, sm);                                     \
      if (rc != NM_OK) return rc;                                                                  \
      mha_fwd_tile_kernel<NJ, true><<<grid, MT_THREADS, sm, s>>>(q, k, v, key_mask, causal, out,   \
          probs, (int)Tq, (int)Tk, (int)heads, (int)dh, drop);                                     \
    } else {                                                                                       \
      int rc = mt_set_smem(mha_fwd_tile_kernel<NJ>, sm);                                           \
      if (rc != NM_OK) return rc;                                                                  \
      mha_fwd_tile_kernel<NJ><<<grid, MT_THREADS, sm, s>>>(q, k, v, key_mask, causal, out, probs,  \
          (int)Tq, (int)Tk, (int)heads, (int)dh, nullptr);                                         \
    }                                                                                              \
  }
    if (Tk <= 64) NM_MT_FWD(8) else if (Tk <= 128) NM_MT_FWD(16) else NM_MT_FWD(32)
#undef NM_MT_FWD
    NM_LAUNCH_CHECK("nm_mha_fwd(tile)");
    return NM_OK;
  }
  const size_t smem = sizeof(float) * (size_t)(dh + Tk);
  NM_REQUIRE(smem <= 48 * 1024, NM_E_UNSUPPORTED, "nm_mha_fwd: Tk+dh too large for this kernel");
  dim3 grid((unsigned)Tq, (unsigned)heads, (unsigned)B);
  cudaStream_t s = (cudaStream_t)stream;
  if (drop)
    mha_fwd_kernel<true><<<grid, MHA_THREADS, smem, s>>>(q, k, v, key_mask, causal, out, probs, (int)Tq,
                                                         (int)Tk, (int)heads, (int)dh, drop);
  else
    mha_fwd_kernel<<<grid, MHA_THREADS, smem, s>>>(q, k, v, key_mask, causal, out, probs, (int)Tq, (int)Tk,
                                                   (int)heads, (int)dh, nullptr);
  NM_LAUNCH_CHECK("nm_mha_fwd");
  return NM_OK;
}

int nm_mha_fwd(const float* q, const float* k, const float* v, const float* key_mask, int causal,
               float* out, float* probs, int64_t B, int64_t Tq, int64_t Tk, int64_t heads,
               int64_t dh, void* stream) {
  return mha_fwd_impl(q, k, v, key_mask, causal, out, probs, B, Tq, Tk, heads, dh, nullptr, stream);
}

int nm_mha_fwd_drop(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                    const float* drop_mask, float* out, float* probs, int64_t B, int64_t Tq, int64_t Tk,
                    int64_t heads, int64_t dh, void* stream) {
  NM_REQUIRE(drop_mask, NM_E_INVALID, "nm_mha_fwd_drop: null mask");
  return mha_fwd_impl(q, k, v, key_mask, causal, out, probs, B, Tq, Tk, heads, dh, drop_mask, stream);
}

static int mha_bwd_impl(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                        const float* probs, const float* dout, float* dq, float* dk, float* dv,
                        float* de_work, int64_t B, int64_t Tq, int64_t Tk, int64_t heads, int64_t dh,
                        const float* drop, void* stream) {
  NM_REQUIRE(q && k && v && probs && dout && dq && dk && dv && de_work, NM_E_INVALID,
             "nm_mha_bwd: null pointer");
  NM_REQUIRE(B > 0 && Tq > 0 && Tk > 0 && heads > 0 && dh > 0, NM_E_INVALID, "nm_mha_bwd: bad sizes");
  NM_REQUIRE(B <= 65535 && heads <= 65535, NM_E_UNSUPPORTED, "nm_mha_bwd: grid too large");
  cudaStream_t s = (cudaStream_t)stream;
  if (mt_ok(Tq, Tk, dh, heads * dh) && mt_smem_q(Tk, dh) <= 200 * 1024 && mt_smem_kv(Tq, dh) <= 200 * 1024) {
    const size_t sm = mt_smem_q(Tk, dh);
    dim3 gq((unsigned)((Tq + MT_QB - 1) / MT_QB), (unsigned)heads, (unsigned)B);
#define NM_MT_BWD(NJ)                                                                                 \
  {                                                                                                   \
    if (drop) {                                                                                       \
      int rc = mt_set_smem(mha_bwd_q_tile_kernel<NJ, true>, sm);                                      \
      if (rc != NM_OK) return rc;                                                                     \
      mha_bwd_q_tile_kernel<NJ, true><<<gq, MT_THREADS, sm, s>>>(k, v, key_mask, causal, probs, dout,  \
          dq, de_work, (int)Tq, (int)Tk, (int)heads, (int)dh, drop);                                  \
    } else {                                                                                          \
      int rc = mt_set_smem(mha_bwd_q_tile_kernel<NJ>, sm);                                            \
      if (rc != NM_OK) return rc;                                                                     \
      mha_bwd_q_tile_kernel<NJ><<<gq, MT_THREADS, sm, s>>>(k, v, key_mask, causal, probs, dout, dq,    \
          de_work, (int)Tq, (int)Tk, (int)heads, (int)dh, nullptr);                                   \
    }                                                                                                 \
  }
    if (Tk <= 64) NM_MT_BWD(8) else if (Tk <= 128) NM_MT_BWD(16) else NM_MT_BWD(32)
#undef NM_MT_BWD
    NM_LAUNCH_CHECK("nm_mha_bwd(q tile)");
    const size_t sk = mt_smem_kv(Tq, dh);
    dim3 gk((unsigned)((Tk + MT_QB - 1) / MT_QB), (unsigned)heads, (unsigned)B);
    if (drop) {
      int rc = mt_set_smem(mha_bwd_kv_tile_kernel<true>, sk);
      if (rc != NM_OK) return rc;
      mha_bwd_kv_tile_kernel<true><<<gk, MT_THREADS, sk, s>>>(q, probs, de_work, dout, dk, dv, (int)Tq,
                                                              (int)Tk, (int)heads, (int)dh, drop);
    } else {
      int rc = mt_set_smem(mha_bwd_kv_tile_kernel<false>, sk);
      if (rc != NM_OK) return rc;
      mha_bwd_kv_tile_kernel<false><<<gk, MT_THREADS, sk, s>>>(q, probs, de_work, dout, dk, dv, (int)Tq,
                                                               (int)Tk, (int)heads, (int)dh, nullptr);
    }
    NM_LAUNCH_CHECK("nm_mha_bwd(kv tile)");
    return NM_OK;
  }
  const size_t smem = sizeof(float) * (size_t)(dh + Tk);
  NM_REQUIRE(smem <= 48 * 1024, NM_E_UNSUPPORTED, "nm_mha_bwd: Tk+dh too large for this kernel");
  dim3 grid_q((unsigned)Tq, (unsigned)heads, (unsigned)B);
  if (drop)
    mha_bwd_q_kernel<true><<<grid_q, MHA_THREADS, smem, s>>>(k, v, key_mask, causal, probs, dout, dq, de_work,
                                                             (int)Tq, (int)Tk, (int)heads, (int)dh, drop);
  else
    mha_bwd_q_kernel<<<grid_q, MHA_THREADS, smem, s>>>(k, v, key_mask, causal, probs, dout, dq, de_work,
                                                       (int)Tq, (int)Tk, (int)heads, (int)dh, nullptr);
  NM_LAUNCH_CHECK("nm_mha_bwd(q)");
  dim3 grid_k((unsigned)Tk, (unsigned)heads, (unsigned)B);
  if (drop)
    mha_bwd_kv_kernel<true><<<grid_k, MHA_THREADS, 0, s>>>(q, probs, de_work, dout, dk, dv, (int)Tq, (int)Tk,
                                                           (int)heads, (int)dh, drop);
  else
    mha_bwd_kv_kernel<<<grid_k, MHA_THREADS, 0, s>>>(q, probs, de_work, dout, dk, dv, (int)Tq, (int)Tk,
                                                     (int)heads, (int)dh, nullptr);
  NM_LAUNCH_CHECK("nm_mha_bwd(kv)");
  return NM_OK;
}

int nm_mha_bwd(const float* q, const float* k, const float* v, const float* key_mask, int causal,
               const float* probs, const float* dout, float* dq, float* dk, float* dv,
               float* de_work, int64_t B, int64_t Tq, int64_t Tk, int64_t heads, int64_t dh,
               void* stream) {
  return mha_bwd_impl(q, k, v, key_mask, causal, probs, dout, dq, dk, dv, de_work, B, Tq, Tk, heads, dh,
                      nullptr, stream);
}

int nm_mha_bwd_drop(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                    const float* drop_mask, const float* probs, const float* dout, float* dq, float* dk,
                    float* dv, float* de_work, int64_t B, int64_t Tq, int64_t Tk, int64_t heads,
                    int64_t dh, void* stream) {
  NM_REQUIRE(drop_mask, NM_E_INVALID, "nm_mha_bwd_drop: null mask");
  return mha_bwd_impl(q, k, v, key_mask, causal, probs, dout, dq, dk, dv, de_work, B, Tq, Tk, heads, dh,
                      drop_mask, stream);
}

}  // extern "C"
