// fp16-operand variant of the vocabulary projection (K5/K6), NOT the default path yet
// (ops.py selects it with NMB200_XENT16=1; see DESIGN.md section 8 item 1).
//
// The three kernels that touch dlogits [M,V] are a third of a training step; in fp32 the matrix is
// written once (1.6 GB at the bench shape) and read about three times.  Here it is stored as fp16,
// UNNORMALISED ((softmax - onehot) * mask, values in [-1, 1]: fp16 then has TF32's 10 mantissa bits;
// tools/fp16_dlogits_study.py), once row-major (for dX) and once transposed (for dW), so that every
// product is a K-major x K-major fp16 wgmma GEMM:
//     logits  = X16 [M,K]   . WT16 [V,K]^T          (forward and the recompute of the backward)
//     dX      = dl16 [M,V]  . W16  [K,V]^T           * row_scale[m]
//     dW^T    = dlT16 [V,M] . XT16 [K+1,M]^T         * alpha, stored transposed into dW (+ db row)
// The upstream per-row gradient is applied in fp32 in the consumers' epilogues.
#include <cuda_fp16.h>

#include "common.cuh"
#include "gemm_tc.h"

namespace nm {

// dst[r * ld_dst + c] = half(src[r * ld_src + c] * (row_scale ? row_scale[r] : 1)), c < cols; the
// `extra_ones` columns behind them hold the row's scale (the column of ones of the bias-gradient trick,
// scaled alike); the padding columns up to ld_dst are zeroed so that a padded K never feeds garbage
// to the MMA.
__global__ void cast_f16_kernel(const float* __restrict__ src, int64_t ld_src, __half* __restrict__ dst,
                                int64_t ld_dst, int64_t rows, int64_t cols,
                                const float* __restrict__ row_scale, int extra_ones) {
  const int64_t total = rows * ld_dst;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / ld_dst, c = i - r * ld_dst;
    float v = 0.f;
    const float sc = row_scale ? row_scale[r] : 1.f;
    if (c < cols) v = src[r * ld_src + c] * sc;
    else if (c < cols + extra_ones) v = sc;
    dst[i] = __float2half_rn(v);
  }
}

// dst [cols + extra_ones, ld_dst] = transpose of src [rows, cols] (scaled per source row), followed by
// `extra_ones` rows holding row_scale (the column of ones of the bias-gradient trick, scaled alike).
// 32x32 tiles through shared memory: coalesced on both sides.
__global__ void cast_transpose_f16_kernel(const float* __restrict__ src, int64_t ld_src,
                                          __half* __restrict__ dst, int64_t ld_dst, int64_t rows,
                                          int64_t cols, const float* __restrict__ row_scale,
                                          int extra_ones) {
  __shared__ float tile[32][33];
  const int64_t r0 = blockIdx.x * 32LL, c0 = blockIdx.y * 32LL;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t r = r0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (r < rows) {
      const float sc = row_scale ? row_scale[r] : 1.f;
      if (c < cols) v = src[r * ld_src + c] * sc;
      else if (c < cols + extra_ones) v = sc;
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t c = c0 + i, r = r0 + threadIdx.x;
    if (c < cols + extra_ones && r < ld_dst) dst[c * ld_dst + r] = __float2half_rn(tile[threadIdx.x][i]);
  }
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_cast_f16(const float* src, int64_t ld_src, void* dst, int64_t ld_dst, int64_t rows, int64_t cols,
                const float* row_scale, int transpose, int extra_ones, void* stream) {
  NM_REQUIRE(src && dst && rows > 0 && cols > 0 && ld_src >= cols, NM_E_INVALID, "nm_cast_f16: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  if (!transpose) {
    NM_REQUIRE(extra_ones >= 0 && ld_dst >= cols + extra_ones, NM_E_INVALID, "nm_cast_f16: bad destination pitch");
    const int64_t total = rows * ld_dst;
    const int64_t blocks = ceil_div(total, 256 * 4);
    const int64_t cap = (int64_t)sm_count() * 16;   // grid-stride: 16 blocks of 256 threads per SM
    cast_f16_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, s>>>(
        src, ld_src, reinterpret_cast<__half*>(dst), ld_dst, rows, cols, row_scale, extra_ones);
  } else {
    NM_REQUIRE(ld_dst >= rows && extra_ones >= 0, NM_E_INVALID, "nm_cast_f16: bad destination pitch");
    const dim3 grid((unsigned)ceil_div(ld_dst, 32), (unsigned)ceil_div(cols + extra_ones, 32));
    cast_transpose_f16_kernel<<<grid, dim3(32, 8), 0, s>>>(src, ld_src, reinterpret_cast<__half*>(dst), ld_dst,
                                                          rows, cols, row_scale, extra_ones);
  }
  NM_LAUNCH_CHECK("nm_cast_f16");
  return NM_OK;
}

int nm_gemm_f16(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16, int64_t ldb,
                float* C, int64_t ldc, const float* alpha_dev, const float* row_scale, float beta,
                int transposed, void* stream) {
  NM_REQUIRE(A16 && B16 && C, NM_E_INVALID, "nm_gemm_f16: null pointer");
  NM_REQUIRE(beta == 0.f || beta == 1.f, NM_E_INVALID, "nm_gemm_f16: beta must be 0 or 1");
  NM_REQUIRE(lda >= K && ldb >= K && ldc >= (transposed ? M : N), NM_E_INVALID, "nm_gemm_f16: bad pitches");
  TcEpilogue epi{};
  epi.mode = TC_EPI_DENSE;
  epi.C = C;
  epi.ldc = ldc;
  epi.act = NM_ACT_NONE;
  epi.beta = beta;
  epi.unk_index = -1;
  TcExt ext{};
  ext.alpha = alpha_dev;
  ext.row_scale = row_scale;
  ext.transposed = transposed;
  return tc_gemm16_launch(M, N, K, A16, lda, B16, ldb, epi, ext, (cudaStream_t)stream);
}

int nm_gemm_f16_tn(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16, int64_t ldb,
                   float* C, int64_t ldc, const float* alpha_dev, float beta, void* stream) {
  NM_REQUIRE(A16 && B16 && C, NM_E_INVALID, "nm_gemm_f16_tn: null pointer");
  NM_REQUIRE(beta == 0.f || beta == 1.f, NM_E_INVALID, "nm_gemm_f16_tn: beta must be 0 or 1");
  NM_REQUIRE(lda >= M && ldb >= N && ldc >= N, NM_E_INVALID, "nm_gemm_f16_tn: bad pitches");
  TcEpilogue epi{};
  epi.mode = TC_EPI_DENSE;
  epi.C = C;
  epi.ldc = ldc;
  epi.act = NM_ACT_NONE;
  epi.beta = beta;
  epi.unk_index = -1;
  TcExt ext{};
  ext.alpha = alpha_dev;
  return tc_gemm16_mn_launch(M, N, K, A16, lda, B16, ldb, epi, ext, (cudaStream_t)stream);
}

int nm_logits_xent_bwd16(const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                         int64_t unk_index, const int64_t* targets, const float* mask, const float* lse,
                         void* dl16, int64_t ldd, void* dlT16, int64_t lddt, int64_t M, int64_t V, int64_t K,
                         void* stream) {
  NM_REQUIRE(X16 && WT16 && targets && lse && dl16, NM_E_INVALID, "nm_logits_xent_bwd16: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= K && ldd >= V && (!dlT16 || lddt >= M),
             NM_E_INVALID, "nm_logits_xent_bwd16: bad sizes");
  TcEpilogue epi{};
  epi.mode = TC_EPI_XENT_BWD16;
  epi.bias = b;
  epi.unk_index = unk_index;
  epi.targets = targets;
  epi.weights = mask;
  epi.lse = lse;
  TcExt ext{};
  ext.C16 = dl16;
  ext.ldc16 = ldd;
  ext.C16T = dlT16;
  ext.ldc16t = lddt;
  return tc_gemm16_launch(M, V, K, X16, ldx, WT16, ldw, epi, ext, (cudaStream_t)stream);
}

}  // extern "C"
