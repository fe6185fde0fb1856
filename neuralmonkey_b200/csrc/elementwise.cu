// HBM-bound kernels of the hot path: embedding gather/scatter (K1), activation
// backward, bias-gradient column sums, maxout and layer norm (K7).
// All are grid-stride / one-warp-per-row kernels with 16-byte vector accesses
// where the row length allows it.
#include "common.cuh"

namespace nm {

// ---------------------------------------------------------------------------
// K1 embedding
// ---------------------------------------------------------------------------
template <int VEC>
__global__ void embed_fwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ table,
                                 const float* __restrict__ mask, float* __restrict__ out,
                                 int64_t n, int64_t emb) {
  const int64_t per_row = emb / VEC;
  const int64_t total = n * per_row;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / per_row, c = (i - row * per_row) * VEC;
    const int64_t id = ids[row];
    const float m = mask ? mask[row] : 1.f;
    if (VEC == 4) {
      float4 v = *reinterpret_cast<const float4*>(table + id * emb + c);
      v.x *= m; v.y *= m; v.z *= m; v.w *= m;
      *reinterpret_cast<float4*>(out + row * emb + c) = v;
    } else {
      out[row * emb + c] = table[id * emb + c] * m;
    }
  }
}

__global__ void embed_bwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dout,
                                 const float* __restrict__ mask, float* __restrict__ dtable,
                                 int64_t n, int64_t emb) {
  const int64_t total = n * emb;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / emb, c = i - row * emb;
    const float m = mask ? mask[row] : 1.f;
    if (m != 0.f) atomicAdd(dtable + ids[row] * emb + c, dout[i] * m);
  }
}

// ---------------------------------------------------------------------------
// activation backward, column sums, maxout
// ---------------------------------------------------------------------------
__global__ void act_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy,
                               float* __restrict__ dx, int64_t n, int act) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float yy = y[i], g = dy[i];
    float d;
    switch (act) {
      case NM_ACT_TANH: d = g * (1.f - yy * yy); break;
      case NM_ACT_RELU: d = yy > 0.f ? g : 0.f; break;
      case NM_ACT_SIGMOID: d = g * yy * (1.f - yy); break;
      default: d = g;
    }
    dx[i] = d;
  }
}

// grid.x over 32-column strips, grid.y over row chunks; block (32, 8).
__global__ void colsum_kernel(const float* __restrict__ x, int64_t M, int64_t N, int64_t ldx,
                              float* __restrict__ out, int rows_per_block) {
  __shared__ float red[8][33];
  const int64_t col = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = min(M, r0 + rows_per_block);
  float s = 0.f;
  if (col < N)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) s += x[r * ldx + col];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    atomicAdd(out + col, t);
  }
}

__global__ void maxout_fwd_kernel(const float* __restrict__ z, float* __restrict__ y,
                                  uint8_t* __restrict__ which, int64_t M, int64_t O) {
  const int64_t total = M * O;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / O, j = i - m * O;
    const float a = z[m * 2 * O + j], b = z[m * 2 * O + O + j];
    // tf.nn.max_pool routes the gradient to the first maximal element.
    const bool second = b > a;
    y[i] = second ? b : a;
    which[i] = second ? 1 : 0;
  }
}
__global__ void maxout_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ which,
                                  float* __restrict__ dz, int64_t M, int64_t O) {
  const int64_t total = M * O;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / O, j = i - m * O;
    const float g = dy[i];
    const bool second = which[i] != 0;
    dz[m * 2 * O + j] = second ? 0.f : g;
    dz[m * 2 * O + O + j] = second ? g : 0.f;
  }
}

// ---------------------------------------------------------------------------
// K-major TF32 copies for the tensor-core GEMM: wgmma reads TF32 operands K-major only, and a K-major operand
// arrives by TMA.  dst[c, r] = tf32_rna(src[r, c]) through a 64 x 64 tile in shared memory: each source row
// segment is read with 16-byte loads (16 threads per row), each destination row segment written with 16-byte
// stores (16 threads per row); scalar accesses where a pitch, a base or the edge of the matrix does not allow a
// vector.  The rounding is the producer threads' cvt.rna.tf32 (low 13 bits cleared), so the GEMM sees the same
// operand bits either way.
// ---------------------------------------------------------------------------
constexpr int TT_EDGE = 64;

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u & 0xffffe000u);
}

__global__ void __launch_bounds__(256) transpose_tf32_kernel(const float* __restrict__ src, int64_t ld_src,
                                                             float* __restrict__ dst, int64_t ld_dst, int64_t rows,
                                                             int64_t cols, bool vec_in, bool vec_out) {
  __shared__ float tile[TT_EDGE][TT_EDGE + 1];     // [source column][source row]: 2-way bank conflicts at most
  const int64_t r0 = (int64_t)blockIdx.x * TT_EDGE, c0 = (int64_t)blockIdx.y * TT_EDGE;
  const int q = threadIdx.x & 15, sub = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < TT_EDGE; i += 16) {
    const int lr = sub + i;
    const int64_t r = r0 + lr, c = c0 + 4 * q;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < rows) {
      const float* p = src + r * ld_src + c;
      if (vec_in && c + 4 <= cols) {
        const float4 x = __ldg(reinterpret_cast<const float4*>(p));
        v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (c + j < cols) v[j] = __ldg(p + j);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) tile[4 * q + j][lr] = tf32_rna(v[j]);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < TT_EDGE; i += 16) {
    const int lc = sub + i;
    const int64_t c = c0 + lc, r = r0 + 4 * q;
    if (c >= cols || r >= rows) continue;
    float* p = dst + c * ld_dst + r;
    const float* t = tile[lc] + 4 * q;
    if (vec_out && r + 4 <= rows) {
      *reinterpret_cast<float4*>(p) = make_float4(t[0], t[1], t[2], t[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (r + j < rows) p[j] = t[j];
    }
  }
}

// ---------------------------------------------------------------------------
// K7 layer norm: one warp per row, the row cached in registers (PER_LANE values per
// lane, D <= 32*PER_LANE).  Parameter gradients are a separate column reduction.
// ---------------------------------------------------------------------------
constexpr int LN_MAX_D = 2048;

template <int PER_LANE>
__global__ void layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float* __restrict__ y,
                                     float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                     int64_t M, int D, float eps) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int64_t warp_global = blockIdx.x * (int64_t)warps_per_block + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * warps_per_block;
  for (int64_t row = warp_global; row < M; row += nwarps) {
    const float* xr = x + row * D;
    float vals[PER_LANE];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      vals[i] = (c < D) ? xr[c] : 0.f;
      s += vals[i];
    }
    const float mean = warp_sum(s) / (float)D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      const float d = (c < D) ? vals[i] - mean : 0.f;
      q += d * d;
    }
    const float var = warp_sum(q) / (float)D;
    const float rstd = rsqrtf(var + eps);
    float* yr = y + row * D;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      if (c < D) yr[c] = (vals[i] - mean) * rstd * gamma[c] + beta[c];
    }
    if (lane == 0) {
      mean_out[row] = mean;
      rstd_out[row] = rstd;
    }
  }
}

template <int PER_LANE>
__global__ void layernorm_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                        const float* __restrict__ mean,
                                        const float* __restrict__ rstd, const float* __restrict__ dy,
                                        float* __restrict__ dx, int64_t M, int D) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int64_t warp_global = blockIdx.x * (int64_t)warps_per_block + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * warps_per_block;
  for (int64_t row = warp_global; row < M; row += nwarps) {
    const float mu = mean[row], rs = rstd[row];
    const float* xr = x + row * D;
    const float* dyr = dy + row * D;
    float xh[PER_LANE], gy[PER_LANE];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      if (c < D) {
        xh[i] = (xr[c] - mu) * rs;
        gy[i] = dyr[c] * gamma[c];
        s1 += gy[i];
        s2 += gy[i] * xh[i];
      } else {
        xh[i] = gy[i] = 0.f;
      }
    }
    s1 = warp_sum(s1) / (float)D;
    s2 = warp_sum(s2) / (float)D;
    float* dxr = dx + row * D;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      if (c < D) dxr[c] = rs * (gy[i] - s1 - xh[i] * s2);
    }
  }
}

// dgamma[c] += sum_m dy*xhat ; dbeta[c] += sum_m dy.  grid (strips of 32 cols, row chunks), block (32,8).
__global__ void layernorm_bwd_param_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                           const float* __restrict__ rstd,
                                           const float* __restrict__ dy, float* __restrict__ dgamma,
                                           float* __restrict__ dbeta, int64_t M, int D,
                                           int rows_per_block) {
  __shared__ float rg[8][33], rb[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = min(M, r0 + rows_per_block);
  float sg = 0.f, sb = 0.f;
  if (col < D)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      const float g = dy[r * D + col];
      sg += g * (x[r * D + col] - mean[r]) * rstd[r];
      sb += g;
    }
  rg[threadIdx.y][threadIdx.x] = sg;
  rb[threadIdx.y][threadIdx.x] = sb;
  __syncthreads();
  if (threadIdx.y == 0 && col < D) {
    float tg = 0.f, tb = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { tg += rg[i][threadIdx.x]; tb += rb[i][threadIdx.x]; }
    atomicAdd(dgamma + col, tg);
    atomicAdd(dbeta + col, tb);
  }
}

static inline int grid_for(int64_t work_items, int threads, int blocks_per_sm = 8) {
  const int64_t need = ceil_div(work_items, threads);
  const int64_t cap = (int64_t)sm_count() * blocks_per_sm;
  return (int)(need < 1 ? 1 : (need < cap ? need : cap));
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_embed_fwd(const int64_t* ids, const float* table, const float* mask, float* out, int64_t n,
                 int64_t emb, int64_t vocab, void* stream) {
  NM_REQUIRE(ids && table && out, NM_E_INVALID, "nm_embed_fwd: null pointer");
  NM_REQUIRE(n >= 0 && emb > 0 && vocab > 0, NM_E_INVALID, "nm_embed_fwd: bad sizes");
  if (n == 0) return NM_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const bool vec = (emb % 4 == 0) && (((uintptr_t)table | (uintptr_t)out) % 16 == 0);
  if (vec)
    embed_fwd_kernel<4><<<grid_for(n * emb / 4, 256), 256, 0, s>>>(ids, table, mask, out, n, emb);
  else
    embed_fwd_kernel<1><<<grid_for(n * emb, 256), 256, 0, s>>>(ids, table, mask, out, n, emb);
  NM_LAUNCH_CHECK("nm_embed_fwd");
  return NM_OK;
}

int nm_embed_bwd(const int64_t* ids, const float* dout, const float* mask, float* dtable, int64_t n,
                 int64_t emb, int64_t vocab, void* stream) {
  NM_REQUIRE(ids && dout && dtable, NM_E_INVALID, "nm_embed_bwd: null pointer");
  NM_REQUIRE(n >= 0 && emb > 0 && vocab > 0, NM_E_INVALID, "nm_embed_bwd: bad sizes");
  if (n == 0) return NM_OK;
  embed_bwd_kernel<<<grid_for(n * emb, 256), 256, 0, (cudaStream_t)stream>>>(ids, dout, mask, dtable,
                                                                             n, emb);
  NM_LAUNCH_CHECK("nm_embed_bwd");
  return NM_OK;
}

int nm_act_bwd(const float* y, const float* dy, float* dx, int64_t n, int act, void* stream) {
  NM_REQUIRE(y && dy && dx, NM_E_INVALID, "nm_act_bwd: null pointer");
  NM_REQUIRE(n >= 0, NM_E_INVALID, "nm_act_bwd: negative size");
  if (n == 0) return NM_OK;
  act_bwd_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(y, dy, dx, n, act);
  NM_LAUNCH_CHECK("nm_act_bwd");
  return NM_OK;
}

int nm_colsum(const float* x, int64_t M, int64_t N, int64_t ldx, float* out, int accumulate,
              void* stream) {
  NM_REQUIRE(x && out, NM_E_INVALID, "nm_colsum: null pointer");
  NM_REQUIRE(M >= 0 && N > 0 && ldx >= N, NM_E_INVALID, "nm_colsum: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  if (!accumulate) NM_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * N, s));
  if (M == 0) return NM_OK;
  const int64_t strips = ceil_div(N, 32);
  // enough row chunks to fill the chip ~4x over, at least 64 rows each
  int64_t chunks = ceil_div((int64_t)sm_count() * 4, strips);
  if (chunks < 1) chunks = 1;
  int64_t rows_per_block = ceil_div(M, chunks);
  if (rows_per_block < 64) rows_per_block = 64;
  chunks = ceil_div(M, rows_per_block);
  dim3 grid((unsigned)strips, (unsigned)chunks), block(32, 8);
  colsum_kernel<<<grid, block, 0, s>>>(x, M, N, ldx, out, (int)rows_per_block);
  NM_LAUNCH_CHECK("nm_colsum");
  return NM_OK;
}

int nm_maxout_fwd(const float* z, float* y, uint8_t* which, int64_t M, int64_t O, void* stream) {
  NM_REQUIRE(z && y && which, NM_E_INVALID, "nm_maxout_fwd: null pointer");
  NM_REQUIRE(M >= 0 && O > 0, NM_E_INVALID, "nm_maxout_fwd: bad sizes");
  if (M == 0) return NM_OK;
  maxout_fwd_kernel<<<grid_for(M * O, 256), 256, 0, (cudaStream_t)stream>>>(z, y, which, M, O);
  NM_LAUNCH_CHECK("nm_maxout_fwd");
  return NM_OK;
}

int nm_maxout_bwd(const float* dy, const uint8_t* which, float* dz, int64_t M, int64_t O,
                  void* stream) {
  NM_REQUIRE(dy && which && dz, NM_E_INVALID, "nm_maxout_bwd: null pointer");
  NM_REQUIRE(M >= 0 && O > 0, NM_E_INVALID, "nm_maxout_bwd: bad sizes");
  if (M == 0) return NM_OK;
  maxout_bwd_kernel<<<grid_for(M * O, 256), 256, 0, (cudaStream_t)stream>>>(dy, which, dz, M, O);
  NM_LAUNCH_CHECK("nm_maxout_bwd");
  return NM_OK;
}

int nm_transpose_tf32(const float* src, int64_t ld_src, float* dst, int64_t ld_dst, int64_t rows, int64_t cols,
                      void* stream) {
  NM_REQUIRE(src && dst, NM_E_INVALID, "nm_transpose_tf32: null pointer");
  NM_REQUIRE(rows >= 0 && cols >= 0 && ld_src >= cols && ld_dst >= rows && ld_dst % 4 == 0, NM_E_INVALID,
             "nm_transpose_tf32: bad sizes (rows=%lld cols=%lld ld_src=%lld ld_dst=%lld)", (long long)rows,
             (long long)cols, (long long)ld_src, (long long)ld_dst);
  if (rows == 0 || cols == 0) return NM_OK;
  const int64_t gx = ceil_div(rows, TT_EDGE), gy = ceil_div(cols, TT_EDGE);
  NM_REQUIRE(gx <= 0x7fffffffLL && gy <= 65535, NM_E_UNSUPPORTED, "nm_transpose_tf32: %lld x %lld is too large",
             (long long)rows, (long long)cols);
  const bool vec_in = ld_src % 4 == 0 && (uintptr_t)src % 16 == 0;
  const bool vec_out = (uintptr_t)dst % 16 == 0;
  transpose_tf32_kernel<<<dim3((unsigned)gx, (unsigned)gy), 256, 0, (cudaStream_t)stream>>>(
      src, ld_src, dst, ld_dst, rows, cols, vec_in, vec_out);
  NM_LAUNCH_CHECK("nm_transpose_tf32");
  return NM_OK;
}

#define NM_LN_DISPATCH(D, CALL)                      \
  do {                                              \
    if ((D) <= 256) { constexpr int PL = 8; CALL; }       \
    else if ((D) <= 640) { constexpr int PL = 20; CALL; } \
    else if ((D) <= 1024) { constexpr int PL = 32; CALL; }\
    else { constexpr int PL = 64; CALL; }                 \
  } while (0)

int nm_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean,
                     float* rstd, int64_t M, int64_t D, float eps, void* stream) {
  NM_REQUIRE(x && gamma && beta && y && mean && rstd, NM_E_INVALID, "nm_layernorm_fwd: null pointer");
  NM_REQUIRE(M >= 0 && D > 0, NM_E_INVALID, "nm_layernorm_fwd: bad sizes");
  NM_REQUIRE(D <= LN_MAX_D, NM_E_UNSUPPORTED, "nm_layernorm_fwd: D=%lld > %d", (long long)D, LN_MAX_D);
  if (M == 0) return NM_OK;
  cudaStream_t s = (cudaStream_t)stream;
  NM_LN_DISPATCH(D, (layernorm_fwd_kernel<PL><<<grid_for(M, 4, 16), 128, 0, s>>>(
                        x, gamma, beta, y, mean, rstd, M, (int)D, eps)));
  NM_LAUNCH_CHECK("nm_layernorm_fwd");
  return NM_OK;
}

int nm_layernorm_bwd(const float* x, const float* gamma, const float* mean, const float* rstd,
                     const float* dy, float* dx, float* dgamma, float* dbeta, int64_t M, int64_t D,
                     void* stream) {
  NM_REQUIRE(x && gamma && mean && rstd && dy, NM_E_INVALID, "nm_layernorm_bwd: null pointer");
  NM_REQUIRE((dgamma == nullptr) == (dbeta == nullptr) && (dx || dgamma), NM_E_INVALID,
             "nm_layernorm_bwd: dgamma and dbeta come together, and dx or the pair must be asked for");
  NM_REQUIRE(M >= 0 && D > 0, NM_E_INVALID, "nm_layernorm_bwd: bad sizes");
  NM_REQUIRE(D <= LN_MAX_D, NM_E_UNSUPPORTED, "nm_layernorm_bwd: D too large");
  if (M == 0) return NM_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (dx) {
    NM_LN_DISPATCH(D, (layernorm_bwd_dx_kernel<PL><<<grid_for(M, 4, 16), 128, 0, s>>>(
                          x, gamma, mean, rstd, dy, dx, M, (int)D)));
    NM_LAUNCH_CHECK("nm_layernorm_bwd(dx)");
  }
  if (!dgamma) return NM_OK;
  const int64_t strips = ceil_div(D, 32);
  int64_t chunks = ceil_div((int64_t)sm_count() * 4, strips);
  int64_t rows_per_block = ceil_div(M, chunks < 1 ? 1 : chunks);
  if (rows_per_block < 64) rows_per_block = 64;
  chunks = ceil_div(M, rows_per_block);
  dim3 grid((unsigned)strips, (unsigned)chunks), block(32, 8);
  layernorm_bwd_param_kernel<<<grid, block, 0, s>>>(x, mean, rstd, dy, dgamma, dbeta, M, (int)D,
                                                    (int)rows_per_block);
  NM_LAUNCH_CHECK("nm_layernorm_bwd(param)");
  return NM_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// Gate arithmetic of the step-wise cell variants (SURVEY.md 8(f) N4): one launch per step
// instead of a chain of element-wise torch kernels.
// ---------------------------------------------------------------------------
namespace nm {

// NematusGRUCell (nn/ortho_gru_cell.py:57-105): sg [B,2H] = state_proj_g(state), gi [B,2H] = input_proj_g(x),
// sc [B,H] = state_proj_c(state), ci [B,H] = input_proj_c(x).
//   [r,u] = sigmoid(sg + gi);  cand = tanh(sc * r + ci);  new = u * state + (1 - u) * cand
// saved [B,3H] = (r, u, cand) for the backward pass.
__global__ void nematus_gate_fwd_kernel(const float* __restrict__ sg, const float* __restrict__ gi,
                                        const float* __restrict__ sc, const float* __restrict__ ci,
                                        const float* __restrict__ state, float* __restrict__ out,
                                        float* __restrict__ saved, int64_t B, int64_t H) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B * H; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / H, j = i - b * H;
    const float r = sigmoidf_(sg[b * 2 * H + j] + gi[b * 2 * H + j]);
    const float u = sigmoidf_(sg[b * 2 * H + H + j] + gi[b * 2 * H + H + j]);
    const float cand = tanhf(sc[i] * r + ci[i]);
    out[i] = u * state[i] + (1.f - u) * cand;
    saved[b * 3 * H + j] = r;
    saved[b * 3 * H + H + j] = u;
    saved[b * 3 * H + 2 * H + j] = cand;
  }
}

// dgates [B,2H] is the gradient of BOTH sg and gi, dcpre [B,H] of ci, dsc [B,H] of sc, dstate [B,H].
__global__ void nematus_gate_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ saved,
                                        const float* __restrict__ sc, const float* __restrict__ state,
                                        float* __restrict__ dgates, float* __restrict__ dcpre,
                                        float* __restrict__ dsc, float* __restrict__ dstate, int64_t B, int64_t H) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < B * H; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / H, j = i - b * H;
    const float r = saved[b * 3 * H + j], u = saved[b * 3 * H + H + j], cand = saved[b * 3 * H + 2 * H + j];
    const float g = dout[i];
    const float dpre = g * (1.f - u) * (1.f - cand * cand);
    const float du = g * (state[i] - cand);
    const float dr = dpre * sc[i];
    dstate[i] = g * u;
    dcpre[i] = dpre;
    dsc[i] = dpre * r;
    dgates[b * 2 * H + j] = dr * r * (1.f - r);
    dgates[b * 2 * H + H + j] = du * u * (1.f - u);
  }
}

// tf.nn.rnn_cell.LSTMCell defaults: z [B,4H] = (i, j, f, o);  c' = sigmoid(f + 1) * c + sigmoid(i) * tanh(j);
// h' = sigmoid(o) * tanh(c').  saved [B,5H] = (sig_i, tanh_j, sig_f, sig_o, tanh_c').
__global__ void lstm_gate_fwd_kernel(const float* __restrict__ z, const float* __restrict__ c,
                                     float* __restrict__ new_c, float* __restrict__ new_h,
                                     float* __restrict__ saved, int64_t B, int64_t H) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < B * H; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = idx / H, j = idx - b * H;
    const float* zr = z + b * 4 * H;
    const float si = sigmoidf_(zr[j]), tj = tanhf(zr[H + j]), sf = sigmoidf_(zr[2 * H + j] + 1.f),
                so = sigmoidf_(zr[3 * H + j]);
    const float nc = sf * c[idx] + si * tj;
    const float tc = tanhf(nc);
    new_c[idx] = nc;
    new_h[idx] = so * tc;
    float* sv = saved + b * 5 * H;
    sv[j] = si; sv[H + j] = tj; sv[2 * H + j] = sf; sv[3 * H + j] = so; sv[4 * H + j] = tc;
  }
}

__global__ void lstm_gate_bwd_kernel(const float* __restrict__ dnew_c, const float* __restrict__ dnew_h,
                                     const float* __restrict__ saved, const float* __restrict__ c,
                                     float* __restrict__ dz, float* __restrict__ dc, int64_t B, int64_t H) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < B * H; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = idx / H, j = idx - b * H;
    const float* sv = saved + b * 5 * H;
    const float si = sv[j], tj = sv[H + j], sf = sv[2 * H + j], so = sv[3 * H + j], tc = sv[4 * H + j];
    const float gh = dnew_h ? dnew_h[idx] : 0.f;
    const float gc = (dnew_c ? dnew_c[idx] : 0.f) + gh * so * (1.f - tc * tc);
    float* dzr = dz + b * 4 * H;
    dzr[j] = gc * tj * si * (1.f - si);
    dzr[H + j] = gc * si * (1.f - tj * tj);
    dzr[2 * H + j] = gc * c[idx] * sf * (1.f - sf);
    dzr[3 * H + j] = gh * tc * so * (1.f - so);
    dc[idx] = gc * sf;
  }
}

}  // namespace nm

extern "C" {

int nm_nematus_gate_fwd(const float* sg, const float* gi, const float* sc, const float* ci, const float* state,
                        float* out, float* saved, int64_t B, int64_t H, void* stream) {
  NM_REQUIRE(sg && gi && sc && ci && state && out && saved && B > 0 && H > 0, NM_E_INVALID,
             "nm_nematus_gate_fwd: bad arguments");
  nm::nematus_gate_fwd_kernel<<<nm::grid_for(B * H, 256), 256, 0, (cudaStream_t)stream>>>(sg, gi, sc, ci, state, out,
                                                                                         saved, B, H);
  NM_LAUNCH_CHECK("nm_nematus_gate_fwd");
  return NM_OK;
}

int nm_nematus_gate_bwd(const float* dout, const float* saved, const float* sc, const float* state, float* dgates,
                        float* dcpre, float* dsc, float* dstate, int64_t B, int64_t H, void* stream) {
  NM_REQUIRE(dout && saved && sc && state && dgates && dcpre && dsc && dstate && B > 0 && H > 0, NM_E_INVALID,
             "nm_nematus_gate_bwd: bad arguments");
  nm::nematus_gate_bwd_kernel<<<nm::grid_for(B * H, 256), 256, 0, (cudaStream_t)stream>>>(dout, saved, sc, state, dgates,
                                                                                         dcpre, dsc, dstate, B, H);
  NM_LAUNCH_CHECK("nm_nematus_gate_bwd");
  return NM_OK;
}

int nm_lstm_gate_fwd(const float* z, const float* c, float* new_c, float* new_h, float* saved, int64_t B, int64_t H,
                     void* stream) {
  NM_REQUIRE(z && c && new_c && new_h && saved && B > 0 && H > 0, NM_E_INVALID, "nm_lstm_gate_fwd: bad arguments");
  nm::lstm_gate_fwd_kernel<<<nm::grid_for(B * H, 256), 256, 0, (cudaStream_t)stream>>>(z, c, new_c, new_h, saved, B, H);
  NM_LAUNCH_CHECK("nm_lstm_gate_fwd");
  return NM_OK;
}

int nm_lstm_gate_bwd(const float* dnew_c, const float* dnew_h, const float* saved, const float* c, float* dz,
                     float* dc, int64_t B, int64_t H, void* stream) {
  NM_REQUIRE(saved && c && dz && dc && B > 0 && H > 0, NM_E_INVALID, "nm_lstm_gate_bwd: bad arguments");
  nm::lstm_gate_bwd_kernel<<<nm::grid_for(B * H, 256), 256, 0, (cudaStream_t)stream>>>(dnew_c, dnew_h, saved, c, dz, dc,
                                                                                      B, H);
  NM_LAUNCH_CHECK("nm_lstm_gate_bwd");
  return NM_OK;
}

}  // extern "C"
