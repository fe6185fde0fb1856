// K17: the two kernels of the reinforcement-learning objectives (trainers/self_critical_objective.py and
// trainers/rl_trainer.py of the reference).
//
// nm_sentence_ngram_reward: sentence-level BLEU / GLEU over token ids, one CTA per sentence with both token rows
// in shared memory.  The reference counts n-grams in a Counter keyed by str(ndarray) and decrements the
// reference count on every match (self_critical_objective.py:203-225).  Here the hypothesis n-gram at position i
// is matched when the number of equal n-grams BEFORE it in the hypothesis is smaller than its count in the
// reference: the same number of matches, with no hashing.  The scores are formed in fp64 and rounded to fp32 once,
// as numpy does.
//
// nm_sample_logits_step: one draw per row from softmax(logits / temperature) by the Gumbel-max trick,
// argmax_j(logits_j / T - log(-log u_j)), with u_j from Philox4x32-10.  Key: the runtime's {seed, step} state
// (the training step), as dropout.  Counter: (column quad, row, 0x80000000 | sample << 16 | loop step, step).
// Dropout's third counter word is its call site, a count of the dropout calls of one step, so the top bit keeps
// the two streams apart.
#include "common.cuh"

namespace nm {

constexpr int64_t kEndToken = 2;     // </s> (vocabulary.py: END_TOKEN_INDEX)
constexpr int kRewardThreads = 128;

// Number of n-grams of row x[0, len) that the reference's takewhile admits: windows are taken until the first
// one whose LAST token is </s> (self_critical_objective.py:228-231).
__device__ __forceinline__ int ngram_count(const int64_t* x, int len, int n) {
  int e = n - 1;
  while (e < len && x[e] != kEndToken) ++e;
  return e - (n - 1) > 0 ? e - (n - 1) : 0;
}

__device__ __forceinline__ bool same_ngram(const int64_t* a, const int64_t* b, int n) {
  for (int k = 0; k < n; ++k)
    if (a[k] != b[k]) return false;
  return true;
}

__global__ void __launch_bounds__(kRewardThreads)
ngram_reward_kernel(const int64_t* __restrict__ refs, int64_t rs_t, int64_t rs_b, const int64_t* __restrict__ hyps,
                    int64_t hs_t, int64_t hs_b, float* __restrict__ reward, int t_r, int t_h, int mode) {
  extern __shared__ int64_t toks[];
  int64_t* ref = toks;
  int64_t* hyp = toks + t_r;
  __shared__ int matched[4], counts[2][4], ref_len;
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < t_r; i += blockDim.x) ref[i] = refs[(int64_t)i * rs_t + (int64_t)b * rs_b];
  for (int i = threadIdx.x; i < t_h; i += blockDim.x) hyp[i] = hyps[(int64_t)i * hs_t + (int64_t)b * hs_b];
  if (threadIdx.x < 4) matched[threadIdx.x] = 0;
  __syncthreads();
  if (threadIdx.x < 4) {
    const int n = threadIdx.x + 1;
    counts[0][threadIdx.x] = ngram_count(hyp, t_h, n);
    counts[1][threadIdx.x] = ngram_count(ref, t_r, n);
  } else if (threadIdx.x == 4) {
    int e = 0;
    while (e < t_r && ref[e] != kEndToken) ++e;
    ref_len = e;
  }
  __syncthreads();
  for (int n = 1; n <= 4; ++n) {
    const int nh = counts[0][n - 1], nr = counts[1][n - 1];
    int mine = 0;
    for (int i = threadIdx.x; i < nh; i += blockDim.x) {
      const int64_t* g = hyp + i;
      int before = 0, in_ref = 0;
      for (int j = 0; j < i; ++j) before += same_ngram(hyp + j, g, n);
      for (int j = 0; j < nr && in_ref <= before; ++j) in_ref += same_ngram(ref + j, g, n);
      mine += before < in_ref;
    }
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&matched[n - 1], mine);
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double score;
  if (mode == NM_REWARD_BLEU) {
    // sentence_bleu (self_critical_objective.py:124-162): +1 smoothing of orders 2..4, 0 without unigrams
    if (counts[0][0] == 0) {
      score = 0.0;
    } else {
      int64_t pm = matched[0], pt = counts[0][0];
      for (int k = 1; k < 4; ++k) {
        pm *= matched[k] + 1;
        pt *= counts[0][k] + 1;
      }
      const double precision = pow((double)pm / (double)pt, 0.25);
      const double bp = fmin(1.0, exp(1.0 - (double)ref_len / (double)counts[0][0]));
      score = bp * precision;
    }
  } else {
    // sentence_gleu (:165-200): min(precision, recall) over the summed 1..4-gram counts.  Where either is 0/0
    // the reference's assert fails; the score is 0 here.
    const int64_t m = (int64_t)matched[0] + matched[1] + matched[2] + matched[3];
    const int64_t h = (int64_t)counts[0][0] + counts[0][1] + counts[0][2] + counts[0][3];
    const int64_t r = (int64_t)counts[1][0] + counts[1][1] + counts[1][2] + counts[1][3];
    score = (h == 0 || r == 0) ? 0.0 : fmin((double)m / (double)h, (double)m / (double)r);
  }
  reward[b] = __double2float_rn(score);
}

constexpr int kSampleThreads = 512;

__global__ void __launch_bounds__(kSampleThreads)
sample_logits_kernel(const float* __restrict__ logits, int64_t ldl, int64_t V, float temperature, int64_t unk_index,
                     const uint8_t* finished_in, int64_t* __restrict__ symbols,
                     uint8_t* finished_out, const int64_t* __restrict__ state, uint32_t site, int vec) {
  const int64_t row = blockIdx.x;
  const float* x = logits + row * ldl;
  const uint2 key = philox_step_key(state);
  const uint32_t step = (uint32_t)state[1];
  float best = -INFINITY;
  int64_t best_j = -1;
  const int64_t nquad = (V + 3) >> 2;
  for (int64_t q = threadIdx.x; q < nquad; q += blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)q, (uint32_t)row, site, step), key);
    const int64_t j0 = q << 2;
    float v[4];
    if (vec && j0 + 3 < V) {
      const float4 f = __ldg(reinterpret_cast<const float4*>(x + j0));
      v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = j0 + k < V ? __ldg(x + j0 + k) : -INFINITY;
    }
    const uint32_t bits[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int64_t j = j0 + k;
      if (j >= V || j == unk_index) continue;
      // 23 bits: (2^23 - 1 + 0.5) is exact in fp32, so u < 1 (with 24 bits the largest value rounds to 1.0,
      // -log(-log(1)) = +inf and that column would win whatever its logit)
      const float u = ((float)(bits[k] >> 9) + 0.5f) * 0x1p-23f;        // in (0, 1)
      const float s = v[k] / temperature - logf(-logf(u));
      if (s > best) {          // columns grow within a thread: a tie keeps the lower index
        best = s;
        best_j = j;
      }
    }
  }
  // block argmax, the lowest index among equal scores
  __shared__ float sv[kSampleThreads / 32];
  __shared__ int64_t sj[kSampleThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int64_t oj = __shfl_xor_sync(0xffffffffu, best_j, o);
    if (ov > best || (ov == best && oj >= 0 && (best_j < 0 || oj < best_j))) {
      best = ov;
      best_j = oj;
    }
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    sv[w] = best;
    sj[w] = best_j;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) {
    if (sv[i] > best || (sv[i] == best && sj[i] >= 0 && (best_j < 0 || sj[i] < best_j))) {
      best = sv[i];
      best_j = sj[i];
    }
  }
  const bool done = finished_in && finished_in[row];
  const int64_t sym = done || best_j < 0 ? 0 : best_j;
  symbols[row] = sym;
  if (finished_out) finished_out[row] = (uint8_t)(done || sym == kEndToken);
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_sentence_ngram_reward(const int64_t* references, int64_t ref_stride_t, int64_t ref_stride_b,
                             const int64_t* hypotheses, int64_t hyp_stride_t, int64_t hyp_stride_b, float* reward,
                             int64_t T_r, int64_t T_h, int64_t B, int mode, void* stream) {
  NM_REQUIRE(references && hypotheses && reward, NM_E_INVALID, "nm_sentence_ngram_reward: null pointer");
  NM_REQUIRE(T_r >= 0 && T_h >= 0 && B >= 0, NM_E_INVALID, "nm_sentence_ngram_reward: negative size");
  NM_REQUIRE(mode == NM_REWARD_BLEU || mode == NM_REWARD_GLEU, NM_E_INVALID,
             "nm_sentence_ngram_reward: mode must be NM_REWARD_BLEU or NM_REWARD_GLEU (got %d)", mode);
  NM_REQUIRE(T_r <= NM_REWARD_MAX_LEN && T_h <= NM_REWARD_MAX_LEN, NM_E_UNSUPPORTED,
             "nm_sentence_ngram_reward: sentences of at most %d tokens (T_r=%lld T_h=%lld)", NM_REWARD_MAX_LEN,
             (long long)T_r, (long long)T_h);
  if (B == 0) return NM_OK;
  NM_REQUIRE(B <= 0x7FFFFFFFLL, NM_E_UNSUPPORTED, "nm_sentence_ngram_reward: batch too large");
  const size_t smem = (size_t)(T_r + T_h) * sizeof(int64_t);
  ngram_reward_kernel<<<(unsigned)B, kRewardThreads, smem, (cudaStream_t)stream>>>(
      references, ref_stride_t, ref_stride_b, hypotheses, hyp_stride_t, hyp_stride_b, reward, (int)T_r, (int)T_h,
      mode);
  NM_LAUNCH_CHECK("nm_sentence_ngram_reward");
  return NM_OK;
}

int nm_sample_logits_step(const float* logits, int64_t ldl, float temperature, int64_t unk_index,
                          const uint8_t* finished_in, int64_t* symbols, uint8_t* finished_out, const int64_t* state,
                          int64_t loop_step, int64_t sample_index, int64_t rows, int64_t V, void* stream) {
  NM_REQUIRE(logits && symbols && state, NM_E_INVALID, "nm_sample_logits_step: null pointer");
  NM_REQUIRE(rows >= 0 && V > 0 && (ldl >= V || ldl == 0), NM_E_INVALID,
             "nm_sample_logits_step: rows >= 0, V > 0 and ldl >= V or 0 expected (rows=%lld V=%lld ldl=%lld)",
             (long long)rows, (long long)V, (long long)ldl);
  NM_REQUIRE(temperature > 0.f, NM_E_INVALID, "nm_sample_logits_step: the temperature must be positive (got %g)",
             (double)temperature);
  NM_REQUIRE(loop_step >= 0 && loop_step < 65536 && sample_index >= 0 && sample_index < 32768, NM_E_UNSUPPORTED,
             "nm_sample_logits_step: loop step < 65536 and sample index < 32768 expected (got %lld, %lld)",
             (long long)loop_step, (long long)sample_index);
  NM_REQUIRE(rows <= 0x7FFFFFFFLL && V <= 0x7FFFFFFFLL, NM_E_UNSUPPORTED, "nm_sample_logits_step: too many rows or columns");
  if (rows == 0) return NM_OK;
  const uint32_t site = 0x80000000u | ((uint32_t)sample_index << 16) | (uint32_t)loop_step;
  const bool vec = (reinterpret_cast<uintptr_t>(logits) & 15) == 0 && (ldl & 3) == 0;
  const int threads = V >= 4 * kSampleThreads ? kSampleThreads : 128;
  sample_logits_kernel<<<(unsigned)rows, threads, 0, (cudaStream_t)stream>>>(
      logits, ldl, V, temperature, unk_index, finished_in, symbols, finished_out, state, site, vec ? 1 : 0);
  NM_LAUNCH_CHECK("nm_sample_logits_step");
  return NM_OK;
}

}  // extern "C"
