// Run-time (greedy / beam) side of the vocabulary projection: what get_body does with the logits of
// one step (decoders/autoregressive.py:446-480 of the reference)
//
//   logits = out.W + b (+ -1e9 on <unk>);  symbol = argmax(logits) * !finished;
//   finished |= (symbol == </s>);  mask = !finished
//
// as TWO launches: the wgmma GEMM whose epilogue keeps (max, sum exp, argmax) partials per 256-column
// tile (gemm_tc.cu, TC_EPI_XENT_FWD) and a combine kernel that also does the integer bookkeeping, so a
// decoding step is {nm_attn_decoder_step_fwd, GEMM, combine} with no host-side tensor arithmetic.
// With the exact-fp32 engine (NM_GEMM_SIMT) the logits are materialised by the CUDA-core GEMM and a
// row kernel does the rest.  Also here: the beam search's token back-tracking.
#include "common.cuh"
#include "gemm_simt.cuh"
#include "gemm_tc.h"

namespace nm {

struct DecodeSelect {
  const uint8_t* fin_in;   // [M] or null (nothing finished)
  int64_t* sym_out;        // [M] or null: no bookkeeping
  uint8_t* fin_out;        // [M] or null (may alias fin_in)
  uint8_t* mask_out;       // [M] or null: 1 while the hypothesis is unfinished AFTER this step
  int32_t* unfinished;     // device counter, += rows still unfinished (or null)
  const int64_t* targets;  // [M] gold symbols of this step or null: xent[m] = (lse - logit[target]) * weight
  const float* weights;    // [M] or null
  float* xent;             // [M] or null
};

__device__ __forceinline__ void decode_select(const DecodeSelect& s, int64_t row, int64_t arg) {
  if (!s.sym_out) return;
  const bool fin = s.fin_in && s.fin_in[row] != 0;
  const int64_t sym = fin ? 0 : arg;                 // PAD once finished (autoregressive.py:472-473)
  const bool fin2 = fin || sym == 2;                 // END_TOKEN_INDEX
  s.sym_out[row] = sym;
  if (s.fin_out) s.fin_out[row] = fin2 ? 1 : 0;
  if (s.mask_out) s.mask_out[row] = fin2 ? 0 : 1;
  if (s.unfinished && !fin2) atomicAdd(s.unfinished, 1);
}

// One warp per row: merge the per-tile partials the GEMM epilogue wrote (same arithmetic as
// xent_combine_kernel in xent_tc.cu), then the symbol bookkeeping.
__global__ void decode_combine_kernel(const float4* __restrict__ part, int64_t M, int64_t tiles_n,
                                      float* __restrict__ lse, int64_t* __restrict__ argmax, DecodeSelect sel) {
  const int lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  float mx = -INFINITY, tgt = -INFINITY;
  int32_t arg = 0x7fffffff;
  for (int64_t t = lane; t < tiles_n; t += 32) {
    const float4 p = part[row * tiles_n + t];
    const int32_t a = __float_as_int(p.z);
    if (p.x > mx || (p.x == mx && a < arg)) { mx = p.x; arg = a; }
    tgt = fmaxf(tgt, p.w);                           // -inf everywhere but in the target's tile
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float omx = __shfl_xor_sync(0xffffffffu, mx, o);
    const int32_t oarg = __shfl_xor_sync(0xffffffffu, arg, o);
    if (omx > mx || (omx == mx && oarg < arg)) { mx = omx; arg = oarg; }
    tgt = fmaxf(tgt, __shfl_xor_sync(0xffffffffu, tgt, o));
  }
  float s = 0.f;
  for (int64_t t = lane; t < tiles_n; t += 32) {
    const float4 p = part[row * tiles_n + t];
    s += p.y * expf(p.x - mx);
  }
  s = warp_sum(s);
  if (lane == 0) {
    const float l = mx + logf(s);
    if (lse) lse[row] = l;
    if (argmax) argmax[row] = (int64_t)arg;
    if (sel.targets && sel.xent) sel.xent[row] = (l - tgt) * (sel.weights ? sel.weights[row] : 1.f);
    decode_select(sel, row, (int64_t)arg);
  }
}

// One CTA per row of materialised logits: -1e9 on the <unk> column (written back), logsumexp,
// first-index argmax, bookkeeping.
__global__ void __launch_bounds__(256)
decode_rows_kernel(float* __restrict__ logits, int64_t V, int64_t ldl, int64_t unk_index,
                   float* __restrict__ lse, int64_t* __restrict__ argmax, DecodeSelect sel) {
  __shared__ float sv[8];
  __shared__ int32_t si[8];
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  float* lr = logits + row * ldl;
  if (unk_index >= 0 && unk_index < V) {
    if (threadIdx.x == 0) lr[unk_index] += -1e9f;
    __syncthreads();
  }
  float bv = -INFINITY;
  int32_t bi = 0x7fffffff;
  for (int64_t c = threadIdx.x; c < V; c += blockDim.x) {
    const float x = lr[c];
    if (x > bv) { bv = x; bi = (int32_t)c; }       // ascending c: the first maximum of this thread
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { sv[w] = bv; si[w] = bi; }
  __syncthreads();
  if (w == 0) {
    const int nw = blockDim.x >> 5;
    bv = lane < nw ? sv[lane] : -INFINITY;
    bi = lane < nw ? si[lane] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { sv[0] = bv; si[0] = bi; }
  }
  __syncthreads();
  const float mx = sv[0];
  float s = 0.f;
  for (int64_t c = threadIdx.x; c < V; c += blockDim.x) s += expf(lr[c] - mx);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float l = mx + logf(s);
    if (lse) lse[row] = l;
    if (argmax) argmax[row] = (int64_t)si[0];
    if (sel.targets && sel.xent)
      sel.xent[row] = (l - lr[sel.targets[row]]) * (sel.weights ? sel.weights[row] : 1.f);
    decode_select(sel, row, (int64_t)si[0]);
  }
}

struct BiasEpi {
  float* C;
  int64_t ldc;
  const float* bias;
  __device__ void operator()(int64_t m, int64_t n, float acc) const {
    C[m * ldc + n] = acc + (bias ? bias[n] : 0.f);
  }
};

// token_ids[t, b, j] of the hypotheses that survive: walk the (word, parent) records backwards
// (what re-gathering the whole token history at every step computes, beam_search_decoder.py:546-551).
__global__ void beam_backtrack_kernel(const int64_t* __restrict__ first, const int64_t* __restrict__ words,
                                      const int32_t* __restrict__ parents, int64_t* __restrict__ out,
                                      int64_t rows, int64_t k, int64_t steps) {
  const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // b*k + j
  if (o >= rows) return;
  const int64_t b = o / k;
  int64_t cur = o - b * k;
  for (int64_t t = steps; t >= 1; --t) {
    const int64_t src = (t - 1) * rows + b * k + cur;
    out[t * rows + o] = words[src];
    cur = parents[src];
  }
  out[o] = first[b * k + cur];
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_decode_logits_step(const float* X, int64_t ldx, const float* W, int64_t ldw, int transW, const float* b,
                          int64_t unk_index, const uint8_t* finished_in, const int64_t* targets,
                          const float* weights, float* lse, int64_t* argmax, float* xent,
                          int64_t* symbols_out, uint8_t* finished_out, uint8_t* mask_out,
                          int32_t* unfinished_count, float* part, float* logits_out, int64_t ldl, int64_t M,
                          int64_t V, int64_t K, int backend, void* stream) {
  NM_REQUIRE(X && W, NM_E_INVALID, "nm_decode_logits_step: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= (transW ? K : V), NM_E_INVALID,
             "nm_decode_logits_step: bad sizes");
  NM_REQUIRE(!logits_out || ldl >= V, NM_E_INVALID, "nm_decode_logits_step: ldl < V");
  NM_REQUIRE(V < 0x7fffffffLL, NM_E_UNSUPPORTED, "nm_decode_logits_step: vocabulary too large");
  NM_REQUIRE(backend >= NM_GEMM_AUTO && backend <= NM_GEMM_TC, NM_E_INVALID, "nm_decode_logits_step: bad backend");
  cudaStream_t s = (cudaStream_t)stream;
  const DecodeSelect sel{finished_in, symbols_out, finished_out, mask_out, unfinished_count,
                         targets, weights, xent};
  const bool tc_ok = part && (reinterpret_cast<uintptr_t>(part) & 15) == 0 &&
                     tc_gemm_supported(0, transW, M, V, K, ldx, ldw, V, X, W, nullptr);
  if (backend == NM_GEMM_TC)
    NM_REQUIRE(tc_ok, NM_E_UNSUPPORTED, "nm_decode_logits_step: operands not TMA-addressable or no scratch");
  if (tc_ok && backend != NM_GEMM_SIMT) {
    TcEpilogue epi{};
    epi.mode = TC_EPI_XENT_FWD;
    epi.C = logits_out;
    epi.ldc = ldl;
    epi.bias = b;
    epi.unk_index = unk_index;
    epi.targets = targets;
    epi.part = reinterpret_cast<float4*>(part);
    const int rc = tc_gemm_launch(0, transW, M, V, K, X, ldx, W, ldw, epi, s);
    if (rc) return rc;
    const int64_t tiles_n = 2 * ceil_div(V, TC_XENT_BN);
    decode_combine_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, s>>>(reinterpret_cast<const float4*>(part), M,
                                                                  tiles_n, lse, argmax, sel);
    NM_LAUNCH_CHECK("nm_decode_logits_step(combine)");
    return NM_OK;
  }
  NM_REQUIRE(logits_out, NM_E_INVALID,
             "nm_decode_logits_step: the CUDA-core engine needs a logits buffer (logits_out)");
  BiasEpi epi{logits_out, ldl, b};
  const int64_t sBk = transW ? 1 : ldw, sBn = transW ? ldw : 1;
  simt_gemm_launch(X, ldx, (int64_t)1, W, sBk, sBn, M, V, K, epi, s);
  NM_LAUNCH_CHECK("nm_decode_logits_step(simt gemm)");
  decode_rows_kernel<<<(unsigned)M, 256, 0, s>>>(logits_out, V, ldl, unk_index, lse, argmax, sel);
  NM_LAUNCH_CHECK("nm_decode_logits_step(rows)");
  return NM_OK;
}

int nm_beam_backtrack(const int64_t* first_symbols, const int64_t* words, const int32_t* parents,
                      int64_t* token_ids, int64_t B, int64_t k, int64_t steps, void* stream) {
  NM_REQUIRE(first_symbols && token_ids && B > 0 && k > 0 && steps >= 0, NM_E_INVALID,
             "nm_beam_backtrack: bad arguments");
  NM_REQUIRE(steps == 0 || (words && parents), NM_E_INVALID, "nm_beam_backtrack: null step records");
  const int64_t rows = B * k;
  beam_backtrack_kernel<<<(unsigned)ceil_div(rows, 128), 128, 0, (cudaStream_t)stream>>>(
      first_symbols, words, parents, token_ids, rows, k, steps);
  NM_LAUNCH_CHECK("nm_beam_backtrack");
  return NM_OK;
}

}  // extern "C"
