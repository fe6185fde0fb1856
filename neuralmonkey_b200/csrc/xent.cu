// K5/K6: the row-wise softmax statistics of the vocabulary projection - logsumexp, first-index argmax and
// the weighted cross-entropy (decoders/autoregressive.py:288-316,446-459 of the reference) - on either engine:
//
//   tensor cores      the wgmma GEMM's TC_EPI_XENT_FWD epilogue (gemm_tc.cu) or xent16_kernel (xent16.cu)
//                     keeps (max, sum exp, argmax, target logit) partials per 256-column tile, and
//                     xent_combine_kernel reduces them: the [M,V] logits need not be written;
//   materialised      xent_rows_kernel, one CTA per row of logits (nm_xent_fwd, and the exact-fp32 engine of
//                     nm_decode_logits_step)
//
// Both can also do what get_body does with one decoding step's argmax (autoregressive.py:446-480):
//
//   symbol = argmax * !finished;  finished |= (symbol == </s>);  mask = !finished
//
// so a decoding step is {nm_attn_decoder_step_fwd, GEMM, combine} with no host-side tensor arithmetic.
// Also here: the backward and the log-softmax over materialised logits.
#include "common.cuh"
#include "gemm_simt.cuh"
#include "gemm_tc.h"

namespace nm {

// The per-row outputs besides lse and argmax.  All null: none.
struct DecodeSelect {
  const uint8_t* fin_in;   // [M] or null (nothing finished)
  int64_t* sym_out;        // [M] or null: no bookkeeping
  uint8_t* fin_out;        // [M] or null (may alias fin_in)
  uint8_t* mask_out;       // [M] or null: 1 while the hypothesis is unfinished AFTER this step
  int32_t* unfinished;     // device counter, += rows still unfinished (or null)
  const int64_t* targets;  // [M] gold symbols or null: xent[m] = (lse - logit[target]) * weight
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

// One warp per row: merge the per-N-tile (max, sumexp, argmax, target) partials.
__global__ void xent_combine_kernel(const float4* __restrict__ part, int64_t M, int64_t tiles_n,
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

struct MaxIdx {
  float v;
  int64_t i;
};
__device__ __forceinline__ MaxIdx better(MaxIdx a, MaxIdx b) {
  // larger value wins; ties go to the lower index (tf.argmax / np.argmax order)
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
__device__ __forceinline__ MaxIdx warp_best(MaxIdx a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxIdx b;
    b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, a.i, o);
    a = better(a, b);
  }
  return a;
}

// One CTA per row of materialised logits: -1e9 on the <unk> column (unk_index >= 0; written back),
// logsumexp, first-index argmax, then xent and the bookkeeping.
__global__ void xent_rows_kernel(float* __restrict__ logits, int64_t V, int64_t ldl, int64_t unk_index,
                                 float* __restrict__ lse, int64_t* __restrict__ argmax, DecodeSelect sel) {
  __shared__ float red[32];
  __shared__ float sv[32];
  __shared__ int64_t si[32];
  const int64_t row = blockIdx.x;
  float* lr = logits + row * ldl;
  if (unk_index >= 0 && unk_index < V) {
    if (threadIdx.x == 0) lr[unk_index] += -1e9f;
    __syncthreads();
  }
  MaxIdx best{-INFINITY, (int64_t)0x7fffffffffffffffLL};
  for (int64_t c = threadIdx.x; c < V; c += blockDim.x) {
    const float x = lr[c];
    if (x > best.v) { best.v = x; best.i = c; }
  }
  best = warp_best(best);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { sv[w] = best.v; si[w] = best.i; }
  __syncthreads();
  if (w == 0) {
    const int nw = blockDim.x >> 5;
    MaxIdx b{lane < nw ? sv[lane] : -INFINITY, lane < nw ? si[lane] : (int64_t)0x7fffffffffffffffLL};
    b = warp_best(b);
    if (lane == 0) { sv[0] = b.v; si[0] = b.i; }
  }
  __syncthreads();
  const float mx = sv[0];
  float s = 0.f;
  for (int64_t c = threadIdx.x; c < V; c += blockDim.x) s += expf(lr[c] - mx);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float l = mx + logf(s);
    if (lse) lse[row] = l;
    if (argmax) argmax[row] = si[0];
    if (sel.targets && sel.xent)
      sel.xent[row] = (l - lr[sel.targets[row]]) * (sel.weights ? sel.weights[row] : 1.f);
    decode_select(sel, row, si[0]);
  }
}

__global__ void xent_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets,
                                const float* __restrict__ weights, const float* __restrict__ lse,
                                const float* __restrict__ scale, float* __restrict__ dlogits,
                                int64_t V, int64_t ldl) {
  const int64_t row = blockIdx.x;  // rows on grid.x (up to 2^31-1), column blocks on grid.y
  const float wgt = (weights ? weights[row] : 1.f) * scale[0];
  const float l = lse[row];
  const int64_t tgt = targets[row];
  const float* lr = logits + row * ldl;
  float* dr = dlogits + row * ldl;
  for (int64_t c = blockIdx.y * (int64_t)blockDim.x + threadIdx.x; c < V;
       c += (int64_t)gridDim.y * blockDim.x) {
    const float p = expf(lr[c] - l);
    dr[c] = (p - (c == tgt ? 1.f : 0.f)) * wgt;
  }
}

__global__ void log_softmax_kernel(const float* __restrict__ logits, const float* __restrict__ lse,
                                   float* __restrict__ out, int64_t V, int64_t ldl) {
  const int64_t row = blockIdx.x;  // as xent_bwd_kernel
  const float l = lse[row];
  for (int64_t c = blockIdx.y * (int64_t)blockDim.x + threadIdx.x; c < V;
       c += (int64_t)gridDim.y * blockDim.x)
    out[row * V + c] = logits[row * ldl + c] - l;
}

struct BiasEpi {
  float* C;
  int64_t ldc;
  const float* bias;
  __device__ void operator()(int64_t m, int64_t n, float acc) const {
    C[m * ldc + n] = acc + (bias ? bias[n] : 0.f);
  }
};

static int xent_rows_launch(float* logits, int64_t ldl, int64_t unk_index, float* lse, int64_t* argmax,
                            const DecodeSelect& sel, int64_t M, int64_t V, cudaStream_t s, const char* what) {
  const int threads = V >= 4096 ? 512 : (V >= 256 ? 128 : 32);
  xent_rows_kernel<<<(unsigned)M, threads, 0, s>>>(logits, V, ldl, unk_index, lse, argmax, sel);
  NM_LAUNCH_CHECK(what);
  return NM_OK;
}

static int xent_combine_launch(const float* part, float* lse, int64_t* argmax, const DecodeSelect& sel,
                               int64_t M, int64_t V, cudaStream_t s, const char* what) {
  const int64_t tiles_n = 2 * ceil_div(V, TC_XENT_BN);  // partials per row: two epilogue halves per n-tile
  xent_combine_kernel<<<(unsigned)ceil_div(M, 8), 256, 0, s>>>(reinterpret_cast<const float4*>(part), M, tiles_n,
                                                              lse, argmax, sel);
  NM_LAUNCH_CHECK(what);
  return NM_OK;
}

static TcEpilogue xent_fwd_epilogue(const float* b, int64_t unk_index, const int64_t* targets, float* part,
                                    float* logits_out, int64_t ldl) {
  TcEpilogue epi{};
  epi.mode = TC_EPI_XENT_FWD;
  epi.C = logits_out;
  epi.ldc = ldl;
  epi.bias = b;
  epi.unk_index = unk_index;
  epi.targets = targets;
  epi.part = reinterpret_cast<float4*>(part);
  return epi;
}

// TF32 wgmma GEMM with the softmax-partials epilogue, then the combine.
static int xent_tc_fwd(const float* X, int64_t ldx, const float* W, int64_t ldw, int transW, const float* b,
                       int64_t unk_index, float* part, float* logits_out, int64_t ldl, float* lse, int64_t* argmax,
                       const DecodeSelect& sel, int64_t M, int64_t V, int64_t K, cudaStream_t s, const char* what) {
  const int rc = tc_gemm_launch(0, transW, M, V, K, X, ldx, W, ldw,
                                xent_fwd_epilogue(b, unk_index, sel.targets, part, logits_out, ldl), s);
  if (rc) return rc;
  return xent_combine_launch(part, lse, argmax, sel, M, V, s, what);
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_xent_fwd(float* logits, int64_t unk_index, const int64_t* targets, const float* weights, float* lse,
                float* xent, int64_t* argmax, int64_t M, int64_t V, int64_t ldl, void* stream) {
  NM_REQUIRE(logits && lse, NM_E_INVALID, "nm_xent_fwd: null pointer");
  NM_REQUIRE(M >= 0 && V > 0 && ldl >= V, NM_E_INVALID, "nm_xent_fwd: bad sizes");
  if (M == 0) return NM_OK;
  const DecodeSelect sel{nullptr, nullptr, nullptr, nullptr, nullptr, targets, weights, xent};
  return xent_rows_launch(logits, ldl, unk_index, lse, argmax, sel, M, V, (cudaStream_t)stream, "nm_xent_fwd");
}

int nm_xent_bwd(const float* logits, const int64_t* targets, const float* weights, const float* lse,
                const float* scale, float* dlogits, int64_t M, int64_t V, int64_t ldl, void* stream) {
  NM_REQUIRE(logits && targets && lse && scale && dlogits, NM_E_INVALID, "nm_xent_bwd: null pointer");
  NM_REQUIRE(M >= 0 && V > 0 && ldl >= V, NM_E_INVALID, "nm_xent_bwd: bad sizes");
  NM_REQUIRE(M <= 0x7fffffffLL, NM_E_UNSUPPORTED, "nm_xent_bwd: M > 2^31-1 rows per call");
  if (M == 0) return NM_OK;
  dim3 grid((unsigned)M, (unsigned)(ceil_div(V, 256) < 64 ? ceil_div(V, 256) : 64));
  xent_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(logits, targets, weights, lse, scale,
                                                          dlogits, V, ldl);
  NM_LAUNCH_CHECK("nm_xent_bwd");
  return NM_OK;
}

int nm_log_softmax(const float* logits, const float* lse, float* logprobs, int64_t M, int64_t V,
                   int64_t ldl, void* stream) {
  NM_REQUIRE(logits && lse && logprobs, NM_E_INVALID, "nm_log_softmax: null pointer");
  NM_REQUIRE(M >= 0 && V > 0 && ldl >= V, NM_E_INVALID, "nm_log_softmax: bad sizes");
  NM_REQUIRE(M <= 0x7fffffffLL, NM_E_UNSUPPORTED, "nm_log_softmax: M > 2^31-1 rows per call");
  if (M == 0) return NM_OK;
  dim3 grid((unsigned)M, (unsigned)(ceil_div(V, 256) < 64 ? ceil_div(V, 256) : 64));
  log_softmax_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(logits, lse, logprobs, V, ldl);
  NM_LAUNCH_CHECK("nm_log_softmax");
  return NM_OK;
}

int64_t nm_logits_xent_scratch(int64_t M, int64_t V) {
  if (M <= 0 || V <= 0) return 0;
  return M * ceil_div(V, TC_XENT_BN) * 2 * 4;  // two epilogue halves per (row, n-tile)
}

int nm_logits_xent_fwd(const float* X, int64_t ldx, const float* W, int64_t ldw, int transW,
                       const float* b, int64_t unk_index, const int64_t* targets, const float* weights, float* lse,
                       float* xent, int64_t* argmax, float* part, float* logits_out, int64_t ldl,
                       int64_t M, int64_t V, int64_t K, void* stream) {
  NM_REQUIRE(X && W && lse && part, NM_E_INVALID, "nm_logits_xent_fwd: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= (transW ? K : V), NM_E_INVALID,
             "nm_logits_xent_fwd: bad sizes");
  NM_REQUIRE(!logits_out || ldl >= V, NM_E_INVALID, "nm_logits_xent_fwd: ldl < V");
  NM_REQUIRE((reinterpret_cast<uintptr_t>(part) & 15) == 0, NM_E_INVALID,
             "nm_logits_xent_fwd: part must be 16-byte aligned");
  NM_REQUIRE(tc_gemm_supported(M, V, K, ldx, ldw, X, W), NM_E_UNSUPPORTED,
             "nm_logits_xent_fwd: operands not TMA-addressable (use nm_gemm + nm_xent_fwd)");
  const DecodeSelect sel{nullptr, nullptr, nullptr, nullptr, nullptr, targets, weights, xent};
  return xent_tc_fwd(X, ldx, W, ldw, transW, b, unk_index, part, logits_out, ldl, lse, argmax, sel, M, V, K,
                     (cudaStream_t)stream, "nm_logits_xent_fwd(combine)");
}

int nm_logits_xent_bwd(const float* X, int64_t ldx, const float* W, int64_t ldw, int transW,
                       const float* b, int64_t unk_index, const int64_t* targets, const float* weights,
                       const float* lse, const float* scale, float* dlogits, int64_t ldd, int64_t M,
                       int64_t V, int64_t K, void* stream) {
  NM_REQUIRE(X && W && targets && lse && scale && dlogits, NM_E_INVALID,
             "nm_logits_xent_bwd: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= (transW ? K : V) && ldd >= V, NM_E_INVALID,
             "nm_logits_xent_bwd: bad sizes");
  NM_REQUIRE(tc_gemm_supported(M, V, K, ldx, ldw, X, W), NM_E_UNSUPPORTED,
             "nm_logits_xent_bwd: operands not TMA-addressable (use nm_gemm + nm_xent_bwd)");
  TcEpilogue epi{};
  epi.mode = TC_EPI_XENT_BWD;
  epi.C = dlogits;
  epi.ldc = ldd;
  epi.bias = b;
  epi.unk_index = unk_index;
  epi.targets = targets;
  epi.weights = weights;
  epi.lse = lse;
  epi.scale = scale;
  return tc_gemm_launch(0, transW, M, V, K, X, ldx, W, ldw, epi, (cudaStream_t)stream);
}

// fp16 operands (X16 [M,K], WT16 [V,K], both K-major): see xent16.cu
int nm_logits_xent_fwd16(const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                         int64_t unk_index, const int64_t* targets, const float* weights, float* lse,
                         float* xent, int64_t* argmax, float* part, float* logits_out, int64_t ldl,
                         int64_t M, int64_t V, int64_t K, void* stream) {
  NM_REQUIRE(X16 && WT16 && lse && part, NM_E_INVALID, "nm_logits_xent_fwd16: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= K, NM_E_INVALID, "nm_logits_xent_fwd16: bad sizes");
  NM_REQUIRE(!logits_out || ldl >= V, NM_E_INVALID, "nm_logits_xent_fwd16: ldl < V");
  NM_REQUIRE((reinterpret_cast<uintptr_t>(part) & 15) == 0, NM_E_INVALID,
             "nm_logits_xent_fwd16: part must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const int rc = K <= XENT16_MAX_K
      ? xent16_launch(false, X16, ldx, WT16, ldw, b, unk_index, targets, nullptr, nullptr,
                      reinterpret_cast<float4*>(part), logits_out, ldl, nullptr, 0, M, V, K, s)
      : tc_gemm16_launch(M, V, K, X16, ldx, WT16, ldw,
                         xent_fwd_epilogue(b, unk_index, targets, part, logits_out, ldl), TcExt{}, s);
  if (rc) return rc;
  const DecodeSelect sel{nullptr, nullptr, nullptr, nullptr, nullptr, targets, weights, xent};
  return xent_combine_launch(part, lse, argmax, sel, M, V, s, "nm_logits_xent_fwd16(combine)");
}

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
                     tc_gemm_supported(M, V, K, ldx, ldw, X, W);
  if (backend == NM_GEMM_TC)
    NM_REQUIRE(tc_ok, NM_E_UNSUPPORTED, "nm_decode_logits_step: operands not TMA-addressable or no scratch");
  if (tc_ok && backend != NM_GEMM_SIMT)
    return xent_tc_fwd(X, ldx, W, ldw, transW, b, unk_index, part, logits_out, ldl, lse, argmax, sel, M, V, K, s,
                       "nm_decode_logits_step(combine)");
  NM_REQUIRE(logits_out, NM_E_INVALID,
             "nm_decode_logits_step: the CUDA-core engine needs a logits buffer (logits_out)");
  BiasEpi epi{logits_out, ldl, b};
  const int64_t sBk = transW ? 1 : ldw, sBn = transW ? ldw : 1;
  simt_gemm_launch(X, ldx, (int64_t)1, W, sBk, sBn, M, V, K, epi, s);
  NM_LAUNCH_CHECK("nm_decode_logits_step(simt gemm)");
  return xent_rows_launch(logits_out, ldl, unk_index, lse, argmax, sel, M, V, s, "nm_decode_logits_step(rows)");
}

}  // extern "C"
