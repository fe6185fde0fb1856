// Host interface of the wgmma GEMM (gemm_tc.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace nm {

enum TcEpiMode {
  TC_EPI_DENSE = 0,     // C = act(acc + bias) + beta*C
  TC_EPI_XENT_FWD = 1,  // per-(row, n-tile) softmax partials; optional logits store
  TC_EPI_XENT_BWD = 2,  // C = (exp(x - lse) - onehot) * weights * scale
  TC_EPI_XENT_BWD16 = 3,  // fp16 operands: C16 = half((exp(x - lse) - onehot) * weights)
  TC_EPI_SOFTMAX = 4,   // batched attention energies: C = softmax(mask(acc * scale)) (and C2 = C * drop)
  TC_EPI_DSOFTMAX = 5,  // batched: C = scale * mask' * P * (acc * drop - sum_j(acc * drop * P))
};

constexpr int TC_XENT_BN = 256;  // N tile used by the xent epilogues (sizes `part`)

struct TcEpilogue {
  int mode;
  float* C;  // dense: output; xent_fwd: logits (may be null); xent_bwd: dlogits
  int64_t ldc;
  const float* bias;  // [N] or null
  int act;
  float beta;
  // xent modes: x = acc + bias[n] + (n == unk_index ? -1e9 : 0)
  int64_t unk_index;       // < 0: none
  const int64_t* targets;  // [M] or null
  const float* weights;    // [M] or null (xent_bwd)
  const float* lse;        // [M] (xent_bwd)
  const float* scale;      // device scalar (xent_bwd)
  float4* part;            // [M][2*ceil(N/TC_XENT_BN)] (xent_fwd): (max, sumexp, argmax bits,
                           //   target logit or -inf) per (row, n-tile, epilogue half)
};

// Extra arguments of the fp16-operand instances; a separate
// trailing kernel parameter so the TF32 instances keep their parameter layout.
struct TcExt {
  void* C16;               // xent_bwd16: [M,N] fp16, row pitch ldc16 (elements)
  int64_t ldc16;
};

// Many small products in one launch: problem p = (o, i), o < count / inner, i < inner (sentence, head), all of the
// same M x N x K.  Operands are windows of two big 2-D tensors; a problem's window starts at
//   row o * row_outer + i * row_inner, column i * col_inner        (rows / columns of the STORED tensor)
// and its output at C + o * c_outer + i * c_inner.  Windows of neighbouring problems may be closer than a tile:
// rows / columns beyond M / N are computed and dropped; the reduction length K must be a multiple of 32 or be
// padded with zeros in one of the operands.  count = 0: an ordinary product.
struct TcBatch {
  int count, inner;
  int a_row_outer, a_row_inner, a_col_inner;
  int b_row_outer, b_row_inner, b_col_inner;
  int64_t c_outer, c_inner;
  // TC_EPI_SOFTMAX / TC_EPI_DSOFTMAX (scaled dot-product attention, attention/scaled_dot_product.py:160-214)
  float scale;               // 1 / sqrt(head size)
  int causal;                // future positions REPLACED by -1e9 (tf.where), no gradient through them
  const float* key_mask;     // [outer, N] or null: x * m + (1 - m) * (-1e9)
  const float* drop;         // [count, M, N] dropout mask (entries 0 or 1 / keep_prob) or null
  float* C2;                 // softmax: C * drop, same layout as C, or null
  const float* P;            // dsoftmax: the softmax output, same layout as C
  int m_pad, n_pad;          // rows [M, m_pad) and columns [N, n_pad) of C (and C2) are written as zeros
};

// op(A) . op(B) for every problem of `bt`; the operand tensors are [a_rows, a_cols] / [b_rows, b_cols] as stored
// (transA = 0: rows are M, columns K; transA = 1: rows K, columns M; transB = 1: rows N, columns K; 0: rows K,
// columns N).  epi.mode: TC_EPI_DENSE (bias / act / beta as usual), TC_EPI_SOFTMAX or TC_EPI_DSOFTMAX (N <= 128).
int tc_gemm_batched_launch(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A, int64_t a_rows,
                           int64_t a_cols, int64_t lda, const float* B, int64_t b_rows, int64_t b_cols,
                           int64_t ldb, const TcEpilogue& epi, const TcBatch& bt, cudaStream_t s);

// 2-D fp16 tensor [rows, cols] with row pitch ld (elements), K-major operand tile: box = {64 elements of K,
// box_rows}, 128-byte swizzle; elements outside [rows, cols] load as zeros.
int make_map16(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, uint32_t box_rows);

// The persistent fp16 vocabulary cross-entropy kernel (xent16.cu) for K <= XENT16_MAX_K:
// X16 [M,K] . WT16 [V,K]^T + b with
//   bwd = false: softmax partials into part ([M][2*ceil(V/TC_XENT_BN)] float4, see TcEpilogue::part) and the
//                logits into logits_out (fp32, row pitch ldl) unless it is null;
//   bwd = true:  dl16 [M,V] (fp16, row pitch ldd) = (softmax - onehot(targets)) * mask, with softmax from lse.
// Longer K runs the TC_EPI_XENT_FWD / TC_EPI_XENT_BWD16 instances of tc_gemm16_launch.
constexpr int64_t XENT16_MAX_K = 320;
int xent16_launch(bool bwd, const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                  int64_t unk_index, const int64_t* targets, const float* mask, const float* lse, float4* part,
                  float* logits_out, int64_t ldl, void* dl16, int64_t ldd, int64_t M, int64_t V, int64_t K,
                  cudaStream_t s);

// True when the operands can be addressed by TMA (16-byte aligned rows and bases).
bool tc_gemm_supported(int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, const void* A, const void* B);

// How tc_gemm_launch runs a dense product on `sms` SMs: bn-column tiles, and the reduction cut into `splits`
// slices of kb_per k-blocks (32 fp32 elements) whose partial tiles are added into C (splits = 1: no cut).
struct TcPlan {
  int bn, splits, kb_per;
};
TcPlan tc_dense_plan(int64_t M, int64_t N, int64_t K, int act, int sms);

// op(A)[M,K] . op(B)[K,N] with the given epilogue.  Same operand conventions as nm_gemm.
int tc_gemm_launch(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A,
                   int64_t lda, const float* B, int64_t ldb, const TcEpilogue& epi, cudaStream_t s);

// The same product with fp16 operands, both K-major: A is [M,K] (row pitch lda), B is [N,K] (row pitch
// ldb), pitches multiples of 8 elements, bases 16-byte aligned.  epi.mode: TC_EPI_XENT_FWD or
// TC_EPI_XENT_BWD16 (the dense fp16 products are nm_gemm_f16 / nm_gemm_f16_tn, gemm16.cu).
int tc_gemm16_launch(int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                     int64_t ldb, const TcEpilogue& epi, const TcExt& ext, cudaStream_t s);

}  // namespace nm
