// K8 on the tensor cores: multi-head scaled dot-product attention (attention/scaled_dot_product.py:160-214 of the
// reference) as BATCHED wgmma products - one 128 x N tile per (sentence, head), all heads of all sentences in
// one launch of the persistent GEMM kernel (gemm_tc.cu, TcBatch):
//
//   forward    P  = softmax(mask(Q K^T / sqrt(dh)))        K-major x K-major, softmax in the epilogue (TC_EPI_SOFTMAX)
//              O  = (P * drop) V                            K-major x MN-major
//   backward   dS = P * (dO V^T * drop - rowsum) / sqrt(dh) K-major x K-major, TC_EPI_DSOFTMAX
//              dQ = dS K                                    K-major x MN-major
//              dK = dS^T Q,  dV = (P * drop)^T dO           MN-major x MN-major
//
// q, k, v, out and their gradients stay in the model's [batch, time, heads * dh] layout: a head is a column
// window of the TMA tensor map, a sentence a row window, so nothing is split, transposed or copied.  The
// [B, heads, Tq, Tk] matrices (P, P * drop, dS) are stored with both time extents rounded up to 32 and the
// padding written as ZEROS by the epilogues: a reduction over time then runs over whole 32-element k-blocks,
// the rows it takes from the neighbouring sentence on the other operand meet zeros.  TF32 operands, fp32
// accumulation; the CUDA-core kernels of mha.cu remain the exact-fp32 engine (and serve the shapes this one does
// not: dh not a multiple of 32, more than 128 keys).
#include "common.cuh"
#include "gemm_tc.h"

using namespace nm;

namespace {

inline int64_t pad32(int64_t x) { return (x + 31) / 32 * 32; }

TcBatch attn_batch(int64_t B, int64_t heads) {
  TcBatch bt{};
  bt.count = (int)(B * heads);
  bt.inner = (int)heads;
  return bt;
}

}  // namespace

extern "C" {

int nm_mha_tc_supported(int64_t B, int64_t Tq, int64_t Tk, int64_t heads, int64_t dh) {
  if (B < 1 || Tq < 1 || Tk < 1 || heads < 1 || dh < 32) return 0;
  if (dh % 32 != 0 || dh > 128 || Tk > 128) return 0;
  if (B * heads > 0x7fffffffLL / 4 || B * heads * pad32(Tq) > 0x7fffffffLL || B * (Tq > Tk ? Tq : Tk) > 0x7fffffffLL)
    return 0;
  return 1;
}

int nm_mha_tc_fwd(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                  const float* drop_mask, float* out, float* probs, float* probs_drop, int64_t B, int64_t Tq,
                  int64_t Tk, int64_t heads, int64_t dh, void* stream) {
  NM_REQUIRE(q && k && v && out && probs, NM_E_INVALID, "nm_mha_tc_fwd: null pointer");
  NM_REQUIRE(nm_mha_tc_supported(B, Tq, Tk, heads, dh), NM_E_UNSUPPORTED,
             "nm_mha_tc_fwd: needs dh a multiple of 32 (<= 128) and at most 128 keys (Tq=%lld Tk=%lld dh=%lld)",
             (long long)Tq, (long long)Tk, (long long)dh);
  NM_REQUIRE((drop_mask == nullptr) == (probs_drop == nullptr), NM_E_INVALID,
             "nm_mha_tc_fwd: the dropped weights are stored exactly when a dropout mask is given");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t D = heads * dh, tqp = pad32(Tq), tkp = pad32(Tk);
  // P = softmax(mask(Q K^T * scale)) -> probs (and probs * drop)
  {
    TcBatch bt = attn_batch(B, heads);
    bt.a_row_outer = (int)Tq; bt.a_col_inner = (int)dh;
    bt.b_row_outer = (int)Tk; bt.b_col_inner = (int)dh;
    bt.c_outer = heads * tqp * tkp; bt.c_inner = tqp * tkp;
    bt.scale = 1.0f / sqrtf((float)dh);
    bt.causal = causal;
    bt.key_mask = key_mask;
    bt.drop = drop_mask;
    bt.C2 = probs_drop;
    bt.m_pad = (int)tqp; bt.n_pad = (int)tkp;
    TcEpilogue epi{};
    epi.mode = TC_EPI_SOFTMAX;
    epi.C = probs;
    epi.ldc = tkp;
    const int rc = tc_gemm_batched_launch(0, 1, Tq, Tk, dh, q, B * Tq, D, D, k, B * Tk, D, D, epi, bt, s);
    if (rc) return rc;
  }
  // O = (P * drop) V
  {
    TcBatch bt = attn_batch(B, heads);
    bt.a_row_outer = (int)(heads * tqp); bt.a_row_inner = (int)tqp;
    bt.b_row_outer = (int)Tk; bt.b_col_inner = (int)dh;
    bt.c_outer = Tq * D; bt.c_inner = dh;
    TcEpilogue epi{};
    epi.mode = TC_EPI_DENSE;
    epi.C = out;
    epi.ldc = D;
    const float* weights = probs_drop ? probs_drop : probs;
    return tc_gemm_batched_launch(0, 0, Tq, dh, tkp, weights, B * heads * tqp, tkp, tkp, v, B * Tk, D, D, epi, bt, s);
  }
}

int nm_mha_tc_bwd(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                  const float* drop_mask, const float* probs, const float* probs_drop, const float* dout,
                  float* dq, float* dk, float* dv, float* ds_work, int64_t B, int64_t Tq, int64_t Tk,
                  int64_t heads, int64_t dh, void* stream) {
  NM_REQUIRE(q && k && v && probs && dout && dq && dk && dv && ds_work, NM_E_INVALID, "nm_mha_tc_bwd: null pointer");
  NM_REQUIRE(nm_mha_tc_supported(B, Tq, Tk, heads, dh) && Tq <= 0x7fffffffLL, NM_E_UNSUPPORTED,
             "nm_mha_tc_bwd: needs dh a multiple of 32 (<= 128) and at most 128 keys (Tq=%lld Tk=%lld dh=%lld)",
             (long long)Tq, (long long)Tk, (long long)dh);
  NM_REQUIRE((drop_mask == nullptr) == (probs_drop == nullptr), NM_E_INVALID,
             "nm_mha_tc_bwd: the dropped weights come with the dropout mask");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t D = heads * dh, tqp = pad32(Tq), tkp = pad32(Tk);
  const float* weights = probs_drop ? probs_drop : probs;
  int rc;
  // dS = scale * mask' * P * (dO V^T * drop - rowsum(...))
  {
    TcBatch bt = attn_batch(B, heads);
    bt.a_row_outer = (int)Tq; bt.a_col_inner = (int)dh;
    bt.b_row_outer = (int)Tk; bt.b_col_inner = (int)dh;
    bt.c_outer = heads * tqp * tkp; bt.c_inner = tqp * tkp;
    bt.scale = 1.0f / sqrtf((float)dh);
    bt.causal = causal;
    bt.key_mask = key_mask;
    bt.drop = drop_mask;
    bt.P = probs;
    bt.m_pad = (int)tqp; bt.n_pad = (int)tkp;
    TcEpilogue epi{};
    epi.mode = TC_EPI_DSOFTMAX;
    epi.C = ds_work;
    epi.ldc = tkp;
    rc = tc_gemm_batched_launch(0, 1, Tq, Tk, dh, dout, B * Tq, D, D, v, B * Tk, D, D, epi, bt, s);
    if (rc) return rc;
  }
  // dQ = dS K
  {
    TcBatch bt = attn_batch(B, heads);
    bt.a_row_outer = (int)(heads * tqp); bt.a_row_inner = (int)tqp;
    bt.b_row_outer = (int)Tk; bt.b_col_inner = (int)dh;
    bt.c_outer = Tq * D; bt.c_inner = dh;
    TcEpilogue epi{};
    epi.mode = TC_EPI_DENSE;
    epi.C = dq;
    epi.ldc = D;
    rc = tc_gemm_batched_launch(0, 0, Tq, dh, tkp, ds_work, B * heads * tqp, tkp, tkp, k, B * Tk, D, D, epi, bt, s);
    if (rc) return rc;
  }
  // dK = dS^T Q and dV = (P * drop)^T dO: the [Tq, Tk] matrices are the MN-major A operand, reduction over Tq
  for (int which = 0; which < 2; ++which) {
    TcBatch bt = attn_batch(B, heads);
    bt.a_row_outer = (int)(heads * tqp); bt.a_row_inner = (int)tqp;
    bt.b_row_outer = (int)Tq; bt.b_col_inner = (int)dh;
    bt.c_outer = Tk * D; bt.c_inner = dh;
    TcEpilogue epi{};
    epi.mode = TC_EPI_DENSE;
    epi.C = which == 0 ? dk : dv;
    epi.ldc = D;
    rc = tc_gemm_batched_launch(1, 0, Tk, dh, tqp, which == 0 ? ds_work : weights, B * heads * tqp, tkp, tkp,
                                which == 0 ? q : dout, B * Tq, D, D, epi, bt, s);
    if (rc) return rc;
  }
  return NM_OK;
}

}  // extern "C"
