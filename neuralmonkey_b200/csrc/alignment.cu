// K21: supervised attention, decoders/word_alignment_decoder.py:100-108 of the reference:
//
//   loss = sum_{b,q} pad[b,q] * sum_t a[b,q,t] * (lse_t e[b,q,t] - e[b,q,t])
//   de[b,q,t] = g * pad[b,q] * (softmax_t(e)[b,q,t] * sum_t a[b,q,t] - a[b,q,t])
//
// softmax_cross_entropy_with_logits over the attention energies e (K4's pre-softmax scores) against a reference
// alignment a, over all Tx positions.  One warp per row; the log-sum-exp is a warp-shuffle reduction.  The row
// losses go to a workspace and one CTA sums them in a fixed order (no float atomics), so repeat calls give the
// same bits.
#include "common.cuh"

namespace nm {

constexpr int AX_THREADS = 256;   // 8 rows per CTA
constexpr int AX_SUM_THREADS = 1024;

// sum_t a (lse - e) = sa * log(s) - sum_t a (e - mx), with s = sum_t exp(e - mx), sa = sum_t a
__global__ void __launch_bounds__(AX_THREADS)
alignment_xent_rows_kernel(const float* __restrict__ e, const float* __restrict__ a,
                           const float* __restrict__ pad, float* __restrict__ row_loss, int64_t rows, int Tx) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (AX_THREADS / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* er = e + row * Tx;
  const float* ar = a + row * Tx;
  float mx = -INFINITY;
  for (int t = lane; t < Tx; t += 32) mx = fmaxf(mx, er[t]);
  mx = warp_max(mx);
  float s = 0.f, sa = 0.f, sae = 0.f;
  for (int t = lane; t < Tx; t += 32) {
    const float d = er[t] - mx, av = ar[t];
    s += expf(d);
    sa += av;
    sae = fmaf(av, d, sae);
  }
  s = warp_sum(s);
  sa = warp_sum(sa);
  sae = warp_sum(sae);
  if (lane == 0) row_loss[row] = pad[row] * (sa * logf(s) - sae);
}

// loss[0] = sum of the row losses: thread i sums rows i, i + 1024, ... in order, then a fixed-order block sum
__global__ void __launch_bounds__(AX_SUM_THREADS)
alignment_xent_sum_kernel(const float* __restrict__ row_loss, float* __restrict__ loss, int64_t rows) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < rows; i += AX_SUM_THREADS) acc += row_loss[i];
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) loss[0] = acc;
}

__global__ void __launch_bounds__(AX_THREADS)
alignment_xent_bwd_kernel(const float* __restrict__ e, const float* __restrict__ a,
                          const float* __restrict__ pad, const float* __restrict__ grad_loss,
                          float* __restrict__ de, int64_t rows, int Tx) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (AX_THREADS / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* er = e + row * Tx;
  const float* ar = a + row * Tx;
  float* dr = de + row * Tx;
  const float g = grad_loss[0] * pad[row];
  float mx = -INFINITY;
  for (int t = lane; t < Tx; t += 32) mx = fmaxf(mx, er[t]);
  mx = warp_max(mx);
  float s = 0.f, sa = 0.f;
  for (int t = lane; t < Tx; t += 32) {
    s += expf(er[t] - mx);
    sa += ar[t];
  }
  s = warp_sum(s);
  sa = warp_sum(sa);
  const float gsa = g * sa / s;
  for (int t = lane; t < Tx; t += 32) dr[t] = fmaf(gsa, expf(er[t] - mx), -g * ar[t]);
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_alignment_xent_fwd(const float* energies, const float* target, const float* pad, float* loss,
                          float* workspace, int64_t B, int64_t NQ, int64_t Tx, void* stream) {
  NM_REQUIRE(energies && target && pad && loss && workspace, NM_E_INVALID, "nm_alignment_xent_fwd: null pointer");
  NM_REQUIRE(B > 0 && NQ > 0 && Tx > 0, NM_E_INVALID, "nm_alignment_xent_fwd: bad sizes");
  NM_REQUIRE(Tx <= INT32_MAX, NM_E_UNSUPPORTED, "nm_alignment_xent_fwd: Tx > 2^31-1");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t rows = B * NQ;
  alignment_xent_rows_kernel<<<(unsigned)ceil_div(rows, AX_THREADS / 32), AX_THREADS, 0, s>>>(
      energies, target, pad, workspace, rows, (int)Tx);
  NM_LAUNCH_CHECK("nm_alignment_xent_fwd(rows)");
  alignment_xent_sum_kernel<<<1, AX_SUM_THREADS, 0, s>>>(workspace, loss, rows);
  NM_LAUNCH_CHECK("nm_alignment_xent_fwd(sum)");
  return NM_OK;
}

int nm_alignment_xent_bwd(const float* energies, const float* target, const float* pad, const float* grad_loss,
                          float* de_out, int64_t B, int64_t NQ, int64_t Tx, void* stream) {
  NM_REQUIRE(energies && target && pad && grad_loss && de_out, NM_E_INVALID,
             "nm_alignment_xent_bwd: null pointer");
  NM_REQUIRE(B > 0 && NQ > 0 && Tx > 0, NM_E_INVALID, "nm_alignment_xent_bwd: bad sizes");
  NM_REQUIRE(Tx <= INT32_MAX, NM_E_UNSUPPORTED, "nm_alignment_xent_bwd: Tx > 2^31-1");
  const int64_t rows = B * NQ;
  alignment_xent_bwd_kernel<<<(unsigned)ceil_div(rows, AX_THREADS / 32), AX_THREADS, 0, (cudaStream_t)stream>>>(
      energies, target, pad, grad_loss, de_out, rows, (int)Tx);
  NM_LAUNCH_CHECK("nm_alignment_xent_bwd");
  return NM_OK;
}

}  // extern "C"
