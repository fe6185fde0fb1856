// K11: one beam-search step (decoders/beam_search_decoder.py:440-496 of the reference):
// finished-row masking, hypothesis log-prob sums, length-normalised scores, top-k over
// the k*V candidates of every sentence, and the (batch, beam) index bookkeeping.
//
// HBM-bound: the step reads B*k*V fp32 log-probs once.  Phase 1 spreads the k*V
// candidates of each sentence over many CTAs (coalesced, 16 candidates per thread in
// registers) and keeps a per-CTA top-k; phase 2 merges the per-CTA lists in one CTA per
// sentence and writes the integer outputs.  Ordering is exactly tf.nn.top_k's: larger
// score first, equal scores by lower flat index.
#include "common.cuh"

namespace nm {

constexpr int BEAM_THREADS = 256;
constexpr int BEAM_ITEMS = 16;
constexpr int BEAM_CHUNK = BEAM_THREADS * BEAM_ITEMS;  // candidates per phase-1 CTA
constexpr int BEAM_MAX_K = 64;
constexpr float BEAM_INF = 1e9f;  // INF of beam_search_decoder.py:43

struct Cand {
  float s;
  int32_t i;
};
__device__ __forceinline__ bool cand_better(float s, int32_t i, float bs, int32_t bi) {
  return s > bs || (s == bs && i < bi);
}
__device__ __forceinline__ Cand warp_best_cand(Cand c) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float os = __shfl_xor_sync(0xffffffffu, c.s, o);
    const int32_t oi = __shfl_xor_sync(0xffffffffu, c.i, o);
    if (cand_better(os, oi, c.s, c.i)) { c.s = os; c.i = oi; }
  }
  return c;
}
// Block-wide best candidate; all threads receive it.  sm: 2*32 words.
__device__ __forceinline__ Cand block_best_cand(Cand c, float* sm_s, int32_t* sm_i) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  c = warp_best_cand(c);
  __syncthreads();
  if (lane == 0) { sm_s[w] = c.s; sm_i[w] = c.i; }
  __syncthreads();
  const int nw = blockDim.x >> 5;
  Cand r{lane < nw ? sm_s[lane] : -INFINITY, lane < nw ? sm_i[lane] : 0x7fffffff};
  r = warp_best_cand(r);
  return r;  // identical in every warp
}

// Top-k of the candidates a CTA holds in registers (ITEMS per thread), in (score desc, index asc) order:
// every warp extracts the k best of its own 32*ITEMS candidates with shuffles only (no block barrier),
// then warp 0 merges the (warps * k) survivors.  The order is total (indices are unique), so the result
// does not depend on how the candidates are spread over threads.  out_s/out_i: [k] in shared memory,
// valid after the trailing __syncthreads(); wk_s/wk_i: [warps * k] scratch in shared memory.
template <int ITEMS>
__device__ __forceinline__ void cta_topk(const float (&sc)[ITEMS], const int32_t (&ix)[ITEMS], int k,
                                         float* wk_s, int32_t* wk_i, float* out_s, int32_t* out_i) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint32_t taken = 0;
  for (int r = 0; r < k; ++r) {
    Cand best{-INFINITY, 0x7fffffff};
#pragma unroll
    for (int it = 0; it < ITEMS; ++it)
      if (!((taken >> it) & 1u) && ix[it] != 0x7fffffff && cand_better(sc[it], ix[it], best.s, best.i)) {
        best.s = sc[it];
        best.i = ix[it];
      }
    const Cand win = warp_best_cand(best);
#pragma unroll
    for (int it = 0; it < ITEMS; ++it)
      if (ix[it] == win.i && win.i != 0x7fffffff) taken |= (1u << it);
    if (lane == 0) { wk_s[w * k + r] = win.s; wk_i[w * k + r] = win.i; }
  }
  __syncthreads();
  if (w == 0) {
    const int n = nw * k;
    int32_t last_i = -1;
    float last_s = INFINITY;
    for (int r = 0; r < k; ++r) {
      Cand best{-INFINITY, 0x7fffffff};
      for (int c = lane; c < n; c += 32) {
        const float s2 = wk_s[c];
        const int32_t i2 = wk_i[c];
        if (i2 == 0x7fffffff) continue;
        const bool after = (r == 0) || s2 < last_s || (s2 == last_s && i2 > last_i);
        if (after && cand_better(s2, i2, best.s, best.i)) { best.s = s2; best.i = i2; }
      }
      const Cand win = warp_best_cand(best);
      last_s = win.s;
      last_i = win.i;
      if (lane == 0) { out_s[r] = win.s; out_i[r] = win.i; }
    }
  }
  __syncthreads();
}

// length penalty ((5+len)/6)^alpha, the fp32 division first (as the reference graph does),
// then a correctly rounded powf through double precision.
__device__ __forceinline__ float length_penalty(int32_t len, float alpha) {
  const float x = (5.f + (float)len) / 6.f;
  return (float)pow((double)x, (double)alpha);
}

// `lse` (may be null): the rows of `logprobs` hold LOGITS and log-prob = logit - lse[row], the
// same subtraction nm_log_softmax performs - the [B,k,V] log-prob tensor then never exists.
__device__ __forceinline__ float cand_hyp(const float* __restrict__ logprobs, const float* __restrict__ lse,
                                          const float* __restrict__ logprob_sum,
                                          const uint8_t* __restrict__ finished, int64_t b, int64_t k,
                                          int64_t V, int32_t flat) {
  const int64_t j = flat / V, w = flat - j * V;
  const bool fin = finished[b * k + j] != 0;
  float lp;
  if (fin) {
    lp = (w == 0 ? 0.f : -BEAM_INF);
  } else {
    lp = logprobs[(b * k + j) * V + w];
    if (lse) lp = lp - lse[b * k + j];
  }
  return logprob_sum[b * k + j] + lp;
}

// phase 1: grid (chunks, B).  cand_s/cand_i: [B, chunks, k]
// The per-hypothesis quantities (finished flag, logsumexp, log-prob sum, length penalty) sit in shared
// memory; a candidate's address is b*k*V + flat, and its hypothesis index needs no 64-bit division: the
// 4096 candidates of a chunk span at most two hypotheses when V >= 4096 (32-bit division otherwise).
__global__ void __launch_bounds__(BEAM_THREADS)
beam_local_topk_kernel(const float* __restrict__ logprobs, const float* __restrict__ lse,
                       const float* __restrict__ logprob_sum,
                       const int32_t* __restrict__ lengths, const uint8_t* __restrict__ finished,
                       float alpha, float* __restrict__ cand_s, int32_t* __restrict__ cand_i,
                       int64_t k, int64_t V) {
  __shared__ float pen[BEAM_MAX_K], s_lse[BEAM_MAX_K], s_lsum[BEAM_MAX_K];
  __shared__ uint8_t s_fin[BEAM_MAX_K];
  const int64_t b = blockIdx.y;
  const int64_t total = k * V;
  if (threadIdx.x < k) {
    const int32_t fin = finished[b * k + threadIdx.x] ? 1 : 0;
    pen[threadIdx.x] = length_penalty(lengths[b * k + threadIdx.x] + 1 - fin, alpha);
    s_fin[threadIdx.x] = (uint8_t)fin;
    s_lse[threadIdx.x] = lse ? lse[b * k + threadIdx.x] : 0.f;
    s_lsum[threadIdx.x] = logprob_sum[b * k + threadIdx.x];
  }
  __syncthreads();
  float sc[BEAM_ITEMS];
  const int64_t base = (int64_t)blockIdx.x * BEAM_CHUNK;
  const float* __restrict__ row = logprobs + b * total;
  const uint32_t v32 = (uint32_t)V;
  const uint32_t j_first = (uint32_t)base / v32;                    // hypothesis of the chunk's first candidate
  const uint32_t next_boundary = (j_first + 1u) * v32;
  const bool two_hyps_at_most = V >= BEAM_CHUNK;
#pragma unroll
  for (int it = 0; it < BEAM_ITEMS; ++it) {
    const int64_t flat = base + it * BEAM_THREADS + threadIdx.x;  // coalesced
    if (flat < total) {
      const uint32_t f32 = (uint32_t)flat;
      const uint32_t j = two_hyps_at_most ? (f32 >= next_boundary ? j_first + 1u : j_first) : f32 / v32;
      const uint32_t w = f32 - j * v32;
      float lp;
      if (s_fin[j]) {
        lp = (w == 0 ? 0.f : -BEAM_INF);
      } else {
        lp = row[flat];
        if (lse) lp = lp - s_lse[j];
      }
      sc[it] = (s_lsum[j] + lp) / pen[j];        // the arithmetic of cand_hyp, operands from shared memory
    } else {
      sc[it] = -INFINITY;
    }
  }
  int32_t ix[BEAM_ITEMS];
#pragma unroll
  for (int it = 0; it < BEAM_ITEMS; ++it) {
    const int64_t flat = base + it * BEAM_THREADS + threadIdx.x;
    ix[it] = flat < total ? (int32_t)flat : 0x7fffffff;   // 0x7fffffff = "no candidate here"
  }
  __shared__ float wk_s[(BEAM_THREADS / 32) * BEAM_MAX_K], out_s[BEAM_MAX_K];
  __shared__ int32_t wk_i[(BEAM_THREADS / 32) * BEAM_MAX_K], out_i[BEAM_MAX_K];
  // Pre-filter (k <= number of warps): every warp's best score is a candidate of its own, so the k-th
  // largest of the warp maxima is a lower bound of the chunk's k-th best score; only candidates at or
  // above it can be among the chunk's top k.  They are few (tens), get listed in shared memory and ranked
  // exactly by ONE warp - unless ties make the list overflow (a chunk inside a finished hypothesis holds
  // 4096 equal scores), which falls back to the full selection.  Same (score desc, index asc) order either way.
  constexpr int NW = BEAM_THREADS / 32, LIST_CAP = 32 * BEAM_ITEMS;
  __shared__ float wmax[NW], list_s[LIST_CAP];
  __shared__ int32_t list_i[LIST_CAP];
  __shared__ int list_n;
  bool done = false;
  if (k <= NW) {
    float tmax = sc[0];
#pragma unroll
    for (int it = 1; it < BEAM_ITEMS; ++it) tmax = fmaxf(tmax, sc[it]);
    tmax = warp_max(tmax);
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = tmax;
    if (threadIdx.x == 0) list_n = 0;
    __syncthreads();
    float thr;
    {   // k-th largest of the NW warp maxima (every thread computes it: NW = 8 values)
      float v[NW];
#pragma unroll
      for (int i = 0; i < NW; ++i) v[i] = wmax[i];
      thr = -INFINITY;
#pragma unroll
      for (int i = 0; i < NW; ++i) {
        int larger = 0;
#pragma unroll
        for (int j = 0; j < NW; ++j) larger += (v[j] > v[i]) || (v[j] == v[i] && j < i);
        if (larger == (int)k - 1) thr = v[i];
      }
    }
#pragma unroll
    for (int it = 0; it < BEAM_ITEMS; ++it)
      if (ix[it] != 0x7fffffff && sc[it] >= thr) {
        const int slot = atomicAdd(&list_n, 1);
        if (slot < LIST_CAP) { list_s[slot] = sc[it]; list_i[slot] = ix[it]; }
      }
    __syncthreads();
    const int n = list_n;
    if (n <= LIST_CAP) {
      done = true;
      if (threadIdx.x < 32) {          // one warp ranks the listed candidates exactly
        float ls[BEAM_ITEMS];
        int32_t li[BEAM_ITEMS];
#pragma unroll
        for (int it = 0; it < BEAM_ITEMS; ++it) {
          const int c = it * 32 + (int)threadIdx.x;
          ls[it] = c < n ? list_s[c] : -INFINITY;
          li[it] = c < n ? list_i[c] : 0x7fffffff;
        }
        uint32_t taken = 0;
        for (int r = 0; r < k; ++r) {
          Cand best{-INFINITY, 0x7fffffff};
#pragma unroll
          for (int it = 0; it < BEAM_ITEMS; ++it)
            if (!((taken >> it) & 1u) && li[it] != 0x7fffffff && cand_better(ls[it], li[it], best.s, best.i)) {
              best.s = ls[it];
              best.i = li[it];
            }
          const Cand win = warp_best_cand(best);
#pragma unroll
          for (int it = 0; it < BEAM_ITEMS; ++it)
            if (li[it] == win.i && win.i != 0x7fffffff) taken |= (1u << it);
          if (threadIdx.x == 0) { out_s[r] = win.s; out_i[r] = win.i; }
        }
      }
      __syncthreads();
    }
  }
  if (!done) cta_topk<BEAM_ITEMS>(sc, ix, (int)k, wk_s, wk_i, out_s, out_i);
  for (int r = threadIdx.x; r < k; r += BEAM_THREADS) {
    const int64_t o = (b * gridDim.x + blockIdx.x) * k + r;
    cand_s[o] = out_s[r];
    cand_i[o] = out_i[r];
  }
}

// phase 2: grid (B).  Merges chunks*k candidates, writes all outputs.
__global__ void __launch_bounds__(BEAM_THREADS)
beam_merge_kernel(const float* __restrict__ cand_s, const int32_t* __restrict__ cand_i,
                  int64_t chunks, const float* __restrict__ logprobs, const float* __restrict__ lse,
                  const float* __restrict__ logprob_sum, const int32_t* __restrict__ lengths,
                  const uint8_t* __restrict__ finished, float* __restrict__ scores,
                  int64_t* __restrict__ word_ids, int32_t* __restrict__ beam_ids,
                  float* __restrict__ logprob_sum_out, int32_t* __restrict__ lengths_out,
                  uint8_t* __restrict__ finished_out, int32_t* __restrict__ unfinished, int64_t k,
                  int64_t V) {
  __shared__ float sm_s[32];
  __shared__ int32_t sm_i[32];
  __shared__ float wk_s[(BEAM_THREADS / 32) * BEAM_MAX_K], out_s[BEAM_MAX_K];
  __shared__ int32_t wk_i[(BEAM_THREADS / 32) * BEAM_MAX_K], out_i[BEAM_MAX_K];
  const int64_t b = blockIdx.x;
  const int64_t n = chunks * k;
  const float* cs = cand_s + b * n;
  const int32_t* ci = cand_i + b * n;
  constexpr int MERGE_ITEMS = 8;
  if (n <= (int64_t)BEAM_THREADS * MERGE_ITEMS) {
    // the usual case (k = 8, V = 32k: 504 candidates): registers + warp shuffles, two block barriers
    float sc[MERGE_ITEMS];
    int32_t ix[MERGE_ITEMS];
#pragma unroll
    for (int it = 0; it < MERGE_ITEMS; ++it) {
      const int64_t c = (int64_t)it * BEAM_THREADS + threadIdx.x;
      sc[it] = c < n ? cs[c] : -INFINITY;
      ix[it] = c < n ? ci[c] : 0x7fffffff;
    }
    cta_topk<MERGE_ITEMS>(sc, ix, (int)k, wk_s, wk_i, out_s, out_i);
  } else {
    int32_t last_i = -1;
    float last_s = INFINITY;
    for (int r = 0; r < k; ++r) {
      // best candidate strictly after (last_s, last_i) in the (score desc, index asc) order
      Cand best{-INFINITY, 0x7fffffff};
      for (int64_t c = threadIdx.x; c < n; c += BEAM_THREADS) {
        const float s = cs[c];
        const int32_t i = ci[c];
        if (i == 0x7fffffff) continue;
        const bool after = (r == 0) || s < last_s || (s == last_s && i > last_i);
        if (after && cand_better(s, i, best.s, best.i)) { best.s = s; best.i = i; }
      }
      const Cand win = block_best_cand(best, sm_s, sm_i);
      last_s = win.s;
      last_i = win.i;
      if (threadIdx.x == 0) { out_s[r] = win.s; out_i[r] = win.i; }
    }
    __syncthreads();
  }
  // bookkeeping of the k winners, one thread each
  for (int r = threadIdx.x; r < k; r += BEAM_THREADS) {
    const int64_t o = b * k + r;
    const int32_t flat = out_i[r];
    const int64_t j = flat / V, w = flat - j * V;
    scores[o] = out_s[r];
    word_ids[o] = w;
    beam_ids[o] = (int32_t)j;
    logprob_sum_out[o] = cand_hyp(logprobs, lse, logprob_sum, finished, b, k, V, flat);
    const int32_t fin = finished[b * k + j] ? 1 : 0;
    lengths_out[o] = lengths[b * k + j] + 1 - fin;
    finished_out[o] = (fin || w == 2) ? 1 : 0;  // END_TOKEN_INDEX = 2
    if (unfinished && !(fin || w == 2)) atomicAdd(unfinished, 1);
  }
}

// gather_flat: out[(b*k+j), :] = x[(b*k+beam_ids[b,j]), :], rows of row_bytes bytes.
__global__ void beam_gather_kernel(const uint8_t* __restrict__ x, const int32_t* __restrict__ beam_ids,
                                   uint8_t* __restrict__ out, int64_t k, int64_t row_bytes) {
  const int64_t o = blockIdx.x;  // b*k + j
  const int64_t b = o / k;
  const int64_t src = b * k + beam_ids[o];
  const uint8_t* s = x + src * row_bytes;
  uint8_t* d = out + o * row_bytes;
  if (((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d) | (uintptr_t)row_bytes) & 15) == 0) {
    const int64_t n16 = row_bytes / 16;
    for (int64_t i = blockIdx.y * (int64_t)blockDim.x + threadIdx.x; i < n16;
         i += (int64_t)gridDim.y * blockDim.x)
      reinterpret_cast<uint4*>(d)[i] = reinterpret_cast<const uint4*>(s)[i];
  } else {
    for (int64_t i = blockIdx.y * (int64_t)blockDim.x + threadIdx.x; i < row_bytes;
         i += (int64_t)gridDim.y * blockDim.x)
      d[i] = s[i];
  }
}

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

int64_t nm_beam_scratch(int64_t B, int64_t k, int64_t V) {
  if (B <= 0 || k <= 0 || V <= 0) return 0;
  return 2 * B * ceil_div(k * V, BEAM_CHUNK) * k;  // 4-byte words: scores then indices
}

static int beam_step_impl(const float* logprobs, const float* lse, const float* logprob_sum,
                          const int32_t* lengths, const uint8_t* finished, float alpha, float* scores,
                          int64_t* word_ids, int32_t* beam_ids, float* logprob_sum_out, int32_t* lengths_out,
                          uint8_t* finished_out, int32_t* unfinished, void* scratch, int64_t B, int64_t k,
                          int64_t V, void* stream) {
  NM_REQUIRE(logprobs && logprob_sum && lengths && finished && scores && word_ids && beam_ids &&
                 logprob_sum_out && lengths_out && finished_out && scratch,
             NM_E_INVALID, "nm_beam_step: null pointer");
  NM_REQUIRE(B > 0 && k > 0 && V > 0, NM_E_INVALID, "nm_beam_step: bad sizes");
  NM_REQUIRE(k <= BEAM_MAX_K, NM_E_UNSUPPORTED, "nm_beam_step: beam %lld > %d", (long long)k, BEAM_MAX_K);
  NM_REQUIRE(k * V < 0x7fffffffLL && B <= 65535, NM_E_UNSUPPORTED, "nm_beam_step: k*V or B too large");
  NM_REQUIRE(k <= V * k, NM_E_INVALID, "nm_beam_step: beam larger than candidate set");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t chunks = ceil_div(k * V, BEAM_CHUNK);
  float* cand_s = reinterpret_cast<float*>(scratch);
  int32_t* cand_i = reinterpret_cast<int32_t*>(scratch) + B * chunks * k;
  dim3 grid1((unsigned)chunks, (unsigned)B);
  beam_local_topk_kernel<<<grid1, BEAM_THREADS, 0, s>>>(logprobs, lse, logprob_sum, lengths, finished, alpha,
                                                        cand_s, cand_i, k, V);
  NM_LAUNCH_CHECK("nm_beam_step(local)");
  beam_merge_kernel<<<(unsigned)B, BEAM_THREADS, 0, s>>>(cand_s, cand_i, chunks, logprobs, lse, logprob_sum,
                                                         lengths, finished, scores, word_ids, beam_ids,
                                                         logprob_sum_out, lengths_out, finished_out, unfinished,
                                                         k, V);
  NM_LAUNCH_CHECK("nm_beam_step(merge)");
  return NM_OK;
}

int nm_beam_step(const float* logprobs, const float* logprob_sum, const int32_t* lengths,
                 const uint8_t* finished, float alpha, float* scores, int64_t* word_ids,
                 int32_t* beam_ids, float* logprob_sum_out, int32_t* lengths_out,
                 uint8_t* finished_out, void* scratch, int64_t B, int64_t k, int64_t V,
                 void* stream) {
  return beam_step_impl(logprobs, nullptr, logprob_sum, lengths, finished, alpha, scores, word_ids, beam_ids,
                        logprob_sum_out, lengths_out, finished_out, nullptr, scratch, B, k, V, stream);
}

int nm_beam_step_logits(const float* logits, const float* lse, const float* logprob_sum,
                        const int32_t* lengths, const uint8_t* finished, float alpha, float* scores,
                        int64_t* word_ids, int32_t* beam_ids, float* logprob_sum_out, int32_t* lengths_out,
                        uint8_t* finished_out, int32_t* unfinished_count, void* scratch, int64_t B,
                        int64_t k, int64_t V, void* stream) {
  NM_REQUIRE(lse, NM_E_INVALID, "nm_beam_step_logits: null lse");
  return beam_step_impl(logits, lse, logprob_sum, lengths, finished, alpha, scores, word_ids, beam_ids,
                        logprob_sum_out, lengths_out, finished_out, unfinished_count, scratch, B, k, V, stream);
}

int nm_beam_gather(const void* x, const int32_t* beam_ids, void* out, int64_t B, int64_t k,
                   int64_t row_bytes, void* stream) {
  NM_REQUIRE(x && beam_ids && out, NM_E_INVALID, "nm_beam_gather: null pointer");
  NM_REQUIRE(B > 0 && k > 0 && row_bytes >= 0, NM_E_INVALID, "nm_beam_gather: bad sizes");
  NM_REQUIRE(x != out, NM_E_INVALID, "nm_beam_gather: in-place gather is not supported");
  if (row_bytes == 0) return NM_OK;
  int64_t gy = ceil_div(row_bytes / 16 + 1, 256);
  if (gy > 64) gy = 64;
  dim3 grid((unsigned)(B * k), (unsigned)gy);
  beam_gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint8_t*>(x),
                                                             beam_ids, reinterpret_cast<uint8_t*>(out),
                                                             k, row_bytes);
  NM_LAUNCH_CHECK("nm_beam_gather");
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
