// Connectionist temporal classification: the loss and the greedy decoder of decoders/ctc_decoder.py, i.e.
// tf.nn.ctc_loss(ignore_longer_outputs_than_inputs=True, ctc_merge_repeated=...) and tf.nn.ctc_greedy_decoder
// of the reference (decoders/ctc_decoder.py:73-112), restated from TF 1.12's published ctc_loss_calculator and
// ctc_decoder.  Logits are batch-major [B, T, C], the blank is class C-1.
//
// Loss, four launches over three kernels:
//   ctc_lse_kernel        one warp per frame: log-sum-exp of the logits row (frames past a sentence's end skipped);
//   ctc_alpha_kernel      one CTA per sentence, the S = 2L+1 states of the extended label l' = (blank, l1, blank,
//                         ..., blank) across its threads: the forward recursion in log space, alpha double-buffered
//                         in shared memory and spilled to the workspace for the backward pass; one barrier a frame.
//                         alpha and beta are sums of hundreds of log-probabilities, so they are carried in fp64 (in
//                         fp32 their rounding reaches 3e-4 in the gradient at T=128); the log1p(exp(-d)) terms of
//                         the log-additions are fp32;
//   ctc_beta_kernel       (backward) the same CTA shape walking the frames backwards: beta, the state occupancies
//                         exp(alpha + beta - log p), and their sums per class over the class's label positions,
//                         grouped once per sentence (one thread per class, one warp per class longer than 32 and
//                         for the blank) - in a fixed order, so two calls give identical bits (no float atomics);
//   ctc_grad_kernel       one warp per frame: dlogits = g * (softmax - occupancy), dense, zeros on frames past the
//                         end and for skipped sentences.
// Greedy decoding: ctc_greedy_kernel, one CTA per sentence: warp-per-frame argmax into shared memory, then the
// kept symbols compacted by a block-wide ballot scan, 256 frames at a time.
#include <algorithm>

#include "common.cuh"

namespace nm {

constexpr int CTC_GREEDY_CHUNK = 256;                      // frames per round of the greedy kernel (= its threads)

// Sentence status in the workspace: what the backward pass and the gradient kernel do with it.
constexpr int CTC_SKIP = 0;      // no alignment fits in the frames (or no frames): loss 0, gradient 0
constexpr int CTC_OK = 1;
constexpr int CTC_INVALID = 2;   // a label outside [0, C-1) or a label length outside [0, Lmax]: loss NaN, gradient 0

// Workspace layout (4-byte words), Lmax = the label tensor's width:
//   alpha [B*T*(2*Lmax+1)] f64 | logp [B] f64 | lse [B*T] | occ [B*T*(Lmax+1)] | slot_class [B*(Lmax+1)] i32 |
//   status [B] i32
struct CtcWs {
  double* alpha;
  double* logp;
  float* lse;
  float* occ;
  int32_t* slot_class;
  int32_t* status;
};

static inline int64_t ctc_ws_words(int64_t B, int64_t T, int64_t Lmax) {
  return B * T * (5 * Lmax + 4) + B * (Lmax + 4);
}

static inline CtcWs ctc_ws(void* base, int64_t B, int64_t T, int64_t Lmax) {
  CtcWs w;
  w.alpha = static_cast<double*>(base);
  w.logp = w.alpha + B * T * (2 * Lmax + 1);
  float* p = reinterpret_cast<float*>(w.logp + B);
  w.lse = p;
  p += B * T;
  w.occ = p;
  p += B * T * (Lmax + 1);
  w.slot_class = reinterpret_cast<int32_t*>(p);
  p += B * (Lmax + 1);
  w.status = reinterpret_cast<int32_t*>(p);
  return w;
}

// log(exp(a) + exp(b)): the large magnitudes added in fp64, the correction log1p(exp(-|a-b|)) <= log 2 in fp32.
__device__ __forceinline__ double log_add(double a, double b) {
  const double m = fmax(a, b);
  if (m == -INFINITY) return -INFINITY;
  return m + (double)log1pf(expf(-(float)fabs(a - b)));
}

__device__ __forceinline__ int ctc_frames(const int32_t* frames, int64_t b, int64_t T) {
  const int64_t f = frames[b];
  return (int)(f < 0 ? 0 : (f > T ? T : f));
}

// Per-state constants of the recursion: class of l'[s], and whether the transitions s -> s (self) and s-2 -> s (skip)
// exist.  merge (TF's ctc_merge_repeated): a state may repeat itself, the skip needs l'[s] non-blank and different
// from l'[s-2].  Without it only blanks repeat themselves and every non-blank label may be reached by a skip.
struct CtcState {
  int cls;
  bool self_ok, skip_ok;
};

__device__ __forceinline__ CtcState ctc_state(const int64_t* lab, int s, int S, int blank, bool merge) {
  CtcState st{blank, true, false};
  if (s < S && (s & 1)) {
    st.cls = (int)lab[s >> 1];
    st.self_ok = merge;
    st.skip_ok = s >= 3 && !(merge && lab[(s >> 1) - 1] == lab[s >> 1]);
  }
  return st;
}

// One warp per row (b, t): lse = log sum_c exp(logits[b, t, c]).  Frames past the sentence's end are not read.
__global__ void __launch_bounds__(256)
ctc_lse_kernel(const float* __restrict__ logits, const int32_t* __restrict__ frames, float* __restrict__ lse,
               int64_t B, int64_t T, int64_t C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * T) return;
  const int64_t b = row / T, t = row - b * T;
  if (t >= ctc_frames(frames, b, T)) return;
  const float* x = logits + row * C;
  float mx = -INFINITY;
  for (int64_t c = lane; c < C; c += 32) mx = fmaxf(mx, x[c]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int64_t c = lane; c < C; c += 32) s += expf(x[c] - mx);
  s = warp_sum(s);
  if (lane == 0) lse[row] = mx + logf(s);
}

__global__ void __launch_bounds__(1024)
ctc_alpha_kernel(const float* __restrict__ logits, const int32_t* __restrict__ frames,
                 const int64_t* __restrict__ labels, const int32_t* __restrict__ label_lengths, int merge,
                 float* __restrict__ loss, CtcWs ws, int64_t T, int64_t C, int Lmax) {
  extern __shared__ double a_sm[];                 // [2][S]
  __shared__ float red[32];
  const int64_t b = blockIdx.x;
  const int tid = threadIdx.x, bd = blockDim.x;
  const int L = label_lengths[b];
  const int f = ctc_frames(frames, b, T);
  const int64_t* lab = labels + b * Lmax;
  const int blank = (int)(C - 1);
  const bool mrg = merge != 0;

  // validity, and whether an alignment fits in the frames: L labels need L frames, plus one between each pair of
  // equal neighbours when they are merged (L is the same for the whole CTA, so no thread skips a barrier)
  int status = CTC_OK;
  if (L < 0 || L > Lmax) {
    status = CTC_INVALID;
  } else {
    int bad = 0, rep = 0;
    for (int i = tid; i < L; i += bd) {
      const int64_t l = lab[i];
      bad |= (l < 0 || l >= C - 1);
      rep += (mrg && i > 0 && l == lab[i - 1]);
    }
    bad = __syncthreads_or(bad);
    rep = (int)block_sum((float)rep, red);         // exact: at most 1022
    if (bad) status = CTC_INVALID;
    else if (f == 0 || L + rep > f) status = CTC_SKIP;
  }
  if (status != CTC_OK) {
    if (tid == 0) {
      ws.status[b] = status;
      loss[b] = status == CTC_SKIP ? 0.f : __int_as_float(0x7fc00000);
    }
    return;
  }

  const int S = 2 * L + 1;
  CtcState st[2];
  bool live[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int s = tid + k * bd;
    live[k] = s < S;
    st[k] = ctc_state(lab, s, S, blank, mrg);
  }
  const int64_t sst = 2 * (int64_t)Lmax + 1;       // state stride of the alpha workspace
  const float* xb = logits + b * T * C;
  const float* lb = ws.lse + b * T;
  double* ab = ws.alpha + b * T * sst;

  // frame 0: a path starts in the first blank or on the first label
  float lp[2], lp_next[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int s = tid + k * bd;
    lp[k] = live[k] ? xb[st[k].cls] - lb[0] : 0.f;
    lp_next[k] = (live[k] && f > 1) ? xb[C + st[k].cls] - lb[1] : 0.f;
    if (live[k]) {
      const double a0 = s <= 1 ? (double)lp[k] : -INFINITY;
      a_sm[s] = a0;
      ab[s] = a0;
    }
  }
  for (int t = 1; t < f; ++t) {
    __syncthreads();                               // alpha of frame t-1 complete
    const double* prev = a_sm + ((t - 1) & 1) * S;
    double* cur = a_sm + (t & 1) * S;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      lp[k] = lp_next[k];
      if (live[k] && t + 1 < f) lp_next[k] = xb[(int64_t)(t + 1) * C + st[k].cls] - lb[t + 1];
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (!live[k]) continue;
      const int s = tid + k * bd;
      double v = st[k].self_ok ? prev[s] : -INFINITY;
      if (s > 0) v = log_add(v, prev[s - 1]);
      if (st[k].skip_ok) v = log_add(v, prev[s - 2]);
      v += lp[k];
      cur[s] = v;
      ab[(int64_t)t * sst + s] = v;
    }
  }
  __syncthreads();
  if (tid == 0) {
    const double* last = a_sm + ((f - 1) & 1) * S;
    const double lp_all = S > 1 ? log_add(last[S - 1], last[S - 2]) : last[0];
    ws.logp[b] = lp_all;
    ws.status[b] = CTC_OK;
    loss[b] = (float)-lp_all;
  }
}

__global__ void __launch_bounds__(1024)
ctc_beta_kernel(const float* __restrict__ logits, const int32_t* __restrict__ frames,
                const int64_t* __restrict__ labels, const int32_t* __restrict__ label_lengths, int merge, CtcWs ws,
                int64_t T, int64_t C, int Lmax) {
  // nb [2][S] f64 | gam [2][S] f32 | lab, first_of, pos, tstart, tcount, tasks, long_tasks [Lmax] i32 each
  extern __shared__ double sm[];
  const int64_t b = blockIdx.x;
  const int tid = threadIdx.x, bd = blockDim.x;
  const int64_t nslot = (int64_t)Lmax + 1;
  int32_t* slot_class = ws.slot_class + b * nslot;
  const int status = ws.status[b];
  if (status != CTC_OK) {
    for (int j = tid; j < nslot; j += bd) slot_class[j] = -1;
    return;
  }
  const int L = label_lengths[b];
  const int S = 2 * L + 1;
  const int f = ctc_frames(frames, b, T);
  const int64_t* labg = labels + b * Lmax;
  const int blank = (int)(C - 1);
  const bool mrg = merge != 0;
  float* gam_base = reinterpret_cast<float*>(sm + 2 * S);
  int32_t* lab = reinterpret_cast<int32_t*>(gam_base + 2 * S);
  int32_t* first_of = lab + Lmax;     // label position -> position of the first occurrence of its class
  int32_t* pos = first_of + Lmax;     // label positions grouped by class (classes in order of first occurrence)
  int32_t* tstart = pos + Lmax;       // first occurrence -> where its class's positions start in pos
  int32_t* tcount = tstart + Lmax;    // first occurrence -> how many positions its class has
  int32_t* tasks = tcount + Lmax;     // the first occurrences, in order: one occupancy sum each
  int32_t* long_tasks = tasks + Lmax; // those whose class occurs more than 32 times

  // Group the label positions by class once.  The launch has more threads than labels (ctc_threads), so thread i
  // owns label position i in these loops.
  for (int i = tid; i < L; i += bd) lab[i] = (int32_t)labg[i];
  __syncthreads();
  for (int i = tid; i < L; i += bd) {
    int f0 = i;
    for (int j = 0; j < i; ++j)
      if (lab[j] == lab[i]) { f0 = j; break; }
    first_of[i] = f0;
    slot_class[i] = f0 == i ? lab[i] : -1;
  }
  for (int j = L + tid; j < nslot; j += bd) slot_class[j] = j == L ? blank : -1;
  __syncthreads();
  for (int i = tid; i < L; i += bd) {
    if (first_of[i] != i) continue;
    int start = 0, count = 0, task = 0;
    for (int k = 0; k < L; ++k) {
      start += first_of[k] < i;
      count += first_of[k] == i;
      task += k < i && first_of[k] == k;
    }
    tstart[i] = start;
    tcount[i] = count;
    tasks[task] = i;
  }
  const int ntask = __syncthreads_count(tid < L && first_of[tid] == tid);   // also orders tstart before its reads
  for (int j = tid; j < L; j += bd) {
    const int f0 = first_of[j];
    int rank = tstart[f0];
    for (int k = 0; k < j; ++k) rank += first_of[k] == f0;
    pos[rank] = j;
    if (f0 == j && tcount[j] > 32) {
      int idx = 0;
      for (int k = 0; k < j; ++k) idx += first_of[k] == k && tcount[k] > 32;
      long_tasks[idx] = j;
    }
  }
  const int nlong = __syncthreads_count(tid < L && first_of[tid] == tid && tcount[tid] > 32);

  CtcState st[2];
  bool live[2], next_skip[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int s = tid + k * bd;
    live[k] = s < S;
    st[k] = ctc_state(labg, s, S, blank, mrg);
    next_skip[k] = s + 2 < S && ctc_state(labg, s + 2, S, blank, mrg).skip_ok;   // the transition s -> s+2
  }
  const int64_t sst = 2 * (int64_t)Lmax + 1;
  const float* xb = logits + b * T * C;
  const float* lb = ws.lse + b * T;
  const double* ab = ws.alpha + b * T * sst;
  float* ob = ws.occ + b * T * nslot;
  const double logp = ws.logp[b];

  float lp[2], lp_next[2];
  double al[2], al_next[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int s = tid + k * bd;
    const int64_t t = f - 1;
    lp_next[k] = live[k] ? xb[t * C + st[k].cls] - lb[t] : 0.f;
    al_next[k] = live[k] ? ab[t * sst + s] : 0.f;
  }
  for (int t = f - 1; t >= 0; --t) {
    const int p = t & 1;
    float* gam = gam_base + p * S;                 // occupancies of frame t
    double* nb = sm + p * S;                       // lp(t) + beta(t), read at frame t-1
    const double* n1 = sm + (1 - p) * S;           // lp(t+1) + beta(t+1)
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      lp[k] = lp_next[k];
      al[k] = al_next[k];
      if (live[k] && t > 0) {
        lp_next[k] = xb[(int64_t)(t - 1) * C + st[k].cls] - lb[t - 1];
        al_next[k] = ab[(int64_t)(t - 1) * sst + tid + k * bd];
      }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (!live[k]) continue;
      const int s = tid + k * bd;
      double beta;
      if (t == f - 1) {
        beta = s >= S - 2 ? 0.0 : -INFINITY;       // a path ends on the last label or the final blank
      } else {
        beta = st[k].self_ok ? n1[s] : -INFINITY;
        if (s + 1 < S) beta = log_add(beta, n1[s + 1]);
        if (next_skip[k]) beta = log_add(beta, n1[s + 2]);
      }
      gam[s] = expf((float)(al[k] + beta - logp));
      nb[s] = lp[k] + beta;
    }
    __syncthreads();
    // occupancy per class in a fixed order, so the sums are the same bits on every call: a class occurring at
    // most 32 times is summed by one thread in label order; a longer one, and the blank, by one warp (lane-strided,
    // then a shuffle tree; warps taken from the top so they rarely also hold short classes): n occurrences cost
    // at most 32 + n/32 dependent steps
    float* orow = ob + (int64_t)t * nslot;
    for (int task = tid; task < ntask; task += bd) {
      const int slot = tasks[task];
      const int count = tcount[slot];
      if (count > 32) continue;
      const int32_t* ps = pos + tstart[slot];
      float sum = 0.f;
      for (int k = 0; k < count; ++k) sum += gam[2 * ps[k] + 1];
      orow[slot] = sum;
    }
    const int nw = bd >> 5, lane = tid & 31;
    for (int task = nw - 1 - (tid >> 5); task <= nlong; task += nw) {
      float sum = 0.f;
      int slot = L;
      if (task < nlong) {
        slot = long_tasks[task];
        const int32_t* ps = pos + tstart[slot];
        for (int k = lane; k < tcount[slot]; k += 32) sum += gam[2 * ps[k] + 1];
      } else {
        for (int j = lane; j <= L; j += 32) sum += gam[2 * j];
      }
      sum = warp_sum(sum);
      if (lane == 0) orow[slot] = sum;
    }
  }
}

// One warp per row (b, t): dlogits = g[b] * (softmax - occupancy of the class), zeros where the loss ignores the frame.
__global__ void __launch_bounds__(256)
ctc_grad_kernel(const float* __restrict__ logits, const int32_t* __restrict__ frames,
                const float* __restrict__ grad_loss, CtcWs ws, float* __restrict__ dlogits, int64_t B, int64_t T,
                int64_t C, int64_t Lmax) {
  const int lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * T) return;
  const int64_t b = row / T, t = row - b * T;
  float* dl = dlogits + row * C;
  if (ws.status[b] != CTC_OK || t >= ctc_frames(frames, b, T)) {
    for (int64_t c = lane; c < C; c += 32) dl[c] = 0.f;
    return;
  }
  const float* x = logits + row * C;
  const float g = grad_loss[b], l = ws.lse[row];
  for (int64_t c = lane; c < C; c += 32) dl[c] = g * expf(x[c] - l);
  __syncwarp();
  const int64_t nslot = Lmax + 1;
  const int32_t* cls = ws.slot_class + b * nslot;
  const float* occ = ws.occ + row * nslot;
  for (int64_t j = lane; j < nslot; j += 32) {
    const int k = cls[j];
    if (k >= 0) dl[k] = g * (expf(x[k] - l) - occ[j]);
  }
}

// One CTA of CTC_GREEDY_CHUNK threads per sentence.
__global__ void __launch_bounds__(CTC_GREEDY_CHUNK)
ctc_greedy_kernel(const float* __restrict__ logits, const int32_t* __restrict__ frames, int merge,
                  int64_t* __restrict__ ids, int32_t* __restrict__ lengths, int64_t T, int64_t C) {
  __shared__ int32_t am[CTC_GREEDY_CHUNK];
  __shared__ int32_t wcount[CTC_GREEDY_CHUNK / 32];
  const int64_t b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  constexpr int NW = CTC_GREEDY_CHUNK / 32;
  const int f = ctc_frames(frames, b, T);
  const int32_t blank = (int32_t)(C - 1);
  const float* xb = logits + b * T * C;
  int64_t* out = ids + b * T;
  int32_t prev = -1;                               // argmax of the frame before the chunk
  int n = 0;
  for (int base = 0; base < f; base += CTC_GREEDY_CHUNK) {
    const int rows = min(CTC_GREEDY_CHUNK, f - base);
    for (int r = w; r < rows; r += NW) {
      const float* x = xb + (int64_t)(base + r) * C;
      float bv = -INFINITY;
      int32_t bi = 0x7fffffff;
      for (int64_t c = lane; c < C; c += 32) {
        const float v = x[c];
        if (v > bv || bi == 0x7fffffff) { bv = v; bi = (int32_t)c; }   // ascending c: first maximum of the lane
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) am[r] = bi;
    }
    __syncthreads();
    int32_t a = -1;
    bool keep = false;
    if (tid < rows) {
      a = am[tid];
      const int32_t before = tid > 0 ? am[tid - 1] : prev;
      keep = a != blank && !(merge && a == before);
    }
    const unsigned ball = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) wcount[w] = __popc(ball);
    __syncthreads();
    int off = n, total = 0;
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      if (i < w) off += wcount[i];
      total += wcount[i];
    }
    if (keep) out[off + __popc(ball & ((1u << lane) - 1u))] = a;
    prev = am[rows - 1];
    n += total;
    __syncthreads();                               // am and wcount are rewritten by the next chunk
  }
  for (int64_t t = n + tid; t < T; t += CTC_GREEDY_CHUNK) out[t] = 2;   // END_TOKEN_INDEX
  if (tid == 0) lengths[b] = n;
}

static int ctc_threads(int64_t Lmax) {
  const int64_t S = 2 * Lmax + 1;
  const int64_t per = (S + 1) / 2;                 // two states per thread at most
  return (int)std::min<int64_t>(1024, std::max<int64_t>(32, (per + 31) / 32 * 32));
}

static int ctc_check(const char* fn, const float* logits, const int32_t* frames, const int64_t* labels,
                     const int32_t* label_lengths, const void* workspace, int64_t workspace_words, int64_t B,
                     int64_t T, int64_t C, int64_t Lmax) {
  NM_REQUIRE(logits && frames && label_lengths && workspace && (labels || Lmax == 0), NM_E_INVALID,
             "%s: null pointer", fn);
  NM_REQUIRE(B > 0 && T > 0 && C > 0 && Lmax >= 0, NM_E_INVALID, "%s: bad sizes B=%lld T=%lld C=%lld Lmax=%lld",
             fn, (long long)B, (long long)T, (long long)C, (long long)Lmax);
  NM_REQUIRE(Lmax <= NM_CTC_MAX_LABEL, NM_E_UNSUPPORTED,
             "%s: labels of up to %d symbols are supported, the label tensor is %lld wide", fn, NM_CTC_MAX_LABEL,
             (long long)Lmax);
  NM_REQUIRE(C < 0x7fffffffLL && T < 0x7fffffffLL && B < 0x7fffffffLL, NM_E_UNSUPPORTED, "%s: sizes too large", fn);
  NM_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, NM_E_INVALID, "%s: workspace not 8-byte aligned",
             fn);
  NM_REQUIRE(workspace_words >= ctc_ws_words(B, T, Lmax), NM_E_INVALID,
             "%s: workspace of %lld words, %lld needed", fn, (long long)workspace_words,
             (long long)ctc_ws_words(B, T, Lmax));
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_ctc_loss_fwd(const float* logits, const int32_t* frames, const int64_t* labels,
                    const int32_t* label_lengths, int merge_repeated, float* loss, void* workspace,
                    int64_t workspace_words, int64_t B, int64_t T, int64_t C, int64_t Lmax, void* stream) {
  int rc = ctc_check("nm_ctc_loss_fwd", logits, frames, labels, label_lengths, workspace, workspace_words, B, T, C,
                     Lmax);
  if (rc) return rc;
  NM_REQUIRE(loss, NM_E_INVALID, "nm_ctc_loss_fwd: null loss");
  cudaStream_t s = (cudaStream_t)stream;
  const CtcWs ws = ctc_ws(workspace, B, T, Lmax);
  ctc_lse_kernel<<<(unsigned)ceil_div(B * T, 8), 256, 0, s>>>(logits, frames, ws.lse, B, T, C);
  NM_LAUNCH_CHECK("nm_ctc_loss_fwd(lse)");
  const size_t smem = 2 * (2 * Lmax + 1) * sizeof(double);
  ctc_alpha_kernel<<<(unsigned)B, ctc_threads(Lmax), smem, s>>>(logits, frames, labels, label_lengths,
                                                                merge_repeated, loss, ws, T, C, (int)Lmax);
  NM_LAUNCH_CHECK("nm_ctc_loss_fwd(alpha)");
  return NM_OK;
}

int nm_ctc_loss_bwd(const float* logits, const int32_t* frames, const int64_t* labels,
                    const int32_t* label_lengths, int merge_repeated, const float* grad_loss, float* dlogits,
                    void* workspace, int64_t workspace_words, int64_t B, int64_t T, int64_t C, int64_t Lmax,
                    void* stream) {
  int rc = ctc_check("nm_ctc_loss_bwd", logits, frames, labels, label_lengths, workspace, workspace_words, B, T, C,
                     Lmax);
  if (rc) return rc;
  NM_REQUIRE(grad_loss && dlogits, NM_E_INVALID, "nm_ctc_loss_bwd: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const CtcWs ws = ctc_ws(workspace, B, T, Lmax);
  const size_t smem = 2 * (2 * Lmax + 1) * (sizeof(double) + sizeof(float)) + 7 * Lmax * sizeof(int32_t);
  NM_CUDA_TRY(cudaFuncSetAttribute(ctc_beta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ctc_beta_kernel<<<(unsigned)B, ctc_threads(Lmax), smem, s>>>(logits, frames, labels, label_lengths,
                                                               merge_repeated, ws, T, C, (int)Lmax);
  NM_LAUNCH_CHECK("nm_ctc_loss_bwd(beta)");
  ctc_grad_kernel<<<(unsigned)ceil_div(B * T, 8), 256, 0, s>>>(logits, frames, grad_loss, ws, dlogits, B, T, C,
                                                               Lmax);
  NM_LAUNCH_CHECK("nm_ctc_loss_bwd(grad)");
  return NM_OK;
}

int nm_ctc_greedy_decode(const float* logits, const int32_t* frames, int merge_repeated, int64_t* ids,
                         int32_t* lengths, int64_t B, int64_t T, int64_t C, void* stream) {
  NM_REQUIRE(logits && frames && ids && lengths, NM_E_INVALID, "nm_ctc_greedy_decode: null pointer");
  NM_REQUIRE(B > 0 && T > 0 && C > 0, NM_E_INVALID, "nm_ctc_greedy_decode: bad sizes");
  NM_REQUIRE(C < 0x7fffffffLL && T < 0x7fffffffLL && B < 0x7fffffffLL, NM_E_UNSUPPORTED,
             "nm_ctc_greedy_decode: sizes too large");
  ctc_greedy_kernel<<<(unsigned)B, CTC_GREEDY_CHUNK, 0, (cudaStream_t)stream>>>(logits, frames, merge_repeated, ids,
                                                                                 lengths, T, C);
  NM_LAUNCH_CHECK("nm_ctc_greedy_decode");
  return NM_OK;
}

}  // extern "C"
