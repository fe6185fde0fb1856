/*
 * nmb200.h -- C ABI of libnmb200.so: the H100 (sm_90a) kernels behind the
 * Neural Monkey encoder-decoder hot path.
 *
 * The reference (ufal/neuralmonkey @ 8b14652) has no FFI boundary: its hot
 * path is a TensorFlow-1.12 graph evaluated by `sess.run`
 * (neuralmonkey/tf_manager.py:179-180).  Every entry point below replaces the
 * TF op group named in its comment (reference file:line), and is what a
 * ctypes binding inside the reference's ModelPart classes would call
 * (see INTEGRATION.md).  89 entry points.
 *
 * Conventions
 *   - plain pointers + int64_t sizes; no torch / C++ types cross the ABI;
 *   - all pointers are DEVICE pointers unless the name ends in `_host`;
 *   - all tensors are dense row-major fp32 unless stated; ids are int64
 *     (the dtype `tf.contrib.lookup` tables emit, neuralmonkey/vocabulary.py:187-195),
 *     lengths/steps are int32, flags are uint8;
 *   - every function is asynchronous on `stream` (a cudaStream_t passed as
 *     void*), allocates no persistent device memory and keeps no pointer after
 *     it returns;
 *   - return value: 0 = ok, <0 = invalid argument (NM_E_*), >0 = cudaError_t.
 *     `nm_last_error()` returns a thread-local message.  No exceptions, no exit().
 */
#ifndef NMB200_H
#define NMB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NM_ABI_VERSION 1

#define NM_OK 0
#define NM_E_INVALID (-1)      /* bad argument (null pointer, negative size, ...) */
#define NM_E_UNSUPPORTED (-2)  /* shape / mode outside what the kernel handles    */
#define NM_E_NO_DEVICE (-3)    /* no sm_90 device visible                        */

/* activation codes for nm_gemm epilogues and nm_act_bwd */
#define NM_ACT_NONE 0
#define NM_ACT_TANH 1
#define NM_ACT_RELU 2
#define NM_ACT_SIGMOID 3

/* GEMM backends */
#define NM_GEMM_AUTO 0  /* wgmma when the shape is TMA-addressable, else SIMT */
#define NM_GEMM_SIMT 1  /* fp32 CUDA-core tiles (exact fp32 accumulate)         */
#define NM_GEMM_TC 2    /* wgmma tf32, TMA-staged, register accumulators       */

int nm_version(void);
const char* nm_last_error(void);
/* Number of CUDA kernels this library has launched in this process so far. */
int64_t nm_launch_count(void);
/* Fills SM count and compute capability of the current device. */
int nm_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- K1: embedding lookup -------------------------------------------------
 * Replaces tf.nn.embedding_lookup * mask (neuralmonkey/model/sequence.py:181-191)
 * and AutoregressiveDecoder.embed_input_symbols (decoders/autoregressive.py:269-272).
 * out[i,:] = table[ids[i],:] * (mask ? mask[i] : 1).  n = number of ids.  An id outside [0, vocab) gives a
 * zero row (tf.gather on the GPU) and no gradient. */
int nm_embed_fwd(const int64_t* ids, const float* table, const float* mask,
                 float* out, int64_t n, int64_t emb, int64_t vocab, void* stream);
/* dtable[ids[i],:] += dout[i,:] * mask[i]  (dtable is accumulated into). */
int nm_embed_bwd(const int64_t* ids, const float* dout, const float* mask,
                 float* dtable, int64_t n, int64_t emb, int64_t vocab, void* stream);

/* ---- dense projections (K2 input projection, K3, K5, K9, a5, a6) ----------
 * Replaces tf.layers.dense / tf.matmul / the 1x1 tf.nn.conv2d of
 * attention/feed_forward.py:111-118 and the logits matmul of
 * decoders/autoregressive.py:450-452.
 * C[M,N] = act(op(A) . op(B) + bias[N]) + beta * C      (beta in {0,1})
 * op(A) is [M,K]: A is [M,K] (transA=0, lda>=K) or [K,M] (transA=1, lda>=M);
 * op(B) is [K,N]: B is [K,N] (transB=0, ldb>=N) or [N,K] (transB=1, ldb>=K).
 * bias may be NULL.  backend: NM_GEMM_*. */
int nm_gemm(int transA, int transB, int64_t M, int64_t N, int64_t K,
            const float* A, int64_t lda, const float* B, int64_t ldb,
            float* C, int64_t ldc, const float* bias, int act, float beta,
            int backend, void* stream);
/* 1 if nm_gemm(AUTO) would take the wgmma path for this problem. */
int nm_gemm_uses_tc(int transA, int transB, int64_t M, int64_t N, int64_t K,
                    int64_t lda, int64_t ldb, int64_t ldc);
/* The wgmma plan nm_gemm would use for a dense product: tile width, number of split-K slices and
 * k-blocks (32 fp32 elements) per slice.  sms <= 0: this device's SM count. */
int nm_gemm_tc_plan(int64_t M, int64_t N, int64_t K, int act, int sms, int* bn, int* splits, int* kb_per_split);

/* dst[c * ld_dst + r] = tf32(src[r * ld_src + c]) for a [rows, cols] source (a strided column slice is fine):
 * the transpose of src rounded to TF32 with cvt.rna (low 13 bits zero), i.e. the K-major copy of an operand
 * whose reduction dimension is strided, which the wgmma GEMM then loads by TMA with the same operand bits its
 * producer threads would have made.  ld_dst >= rows and a multiple of 4 (TMA-addressable rows); the padding
 * columns [rows, ld_dst) of dst are not written.  HBM-bound: 64 x 64 tiles through shared memory, 16-byte
 * loads / stores where pitches and bases allow. */
int nm_transpose_tf32(const float* src, int64_t ld_src, float* dst, int64_t ld_dst, int64_t rows,
                      int64_t cols, void* stream);
/* dx = dy * act'(y) expressed through the activation OUTPUT y (tanh: 1-y^2,
 * relu: y>0, sigmoid: y(1-y)); n elements; dx may alias dy. */
int nm_act_bwd(const float* y, const float* dy, float* dx, int64_t n, int act,
               void* stream);
/* out[n] (+)= sum_m x[m,n]  -- bias gradients. accumulate in {0,1}. */
int nm_colsum(const float* x, int64_t M, int64_t N, int64_t ldx, float* out,
              int accumulate, void* stream);
/* Dropout (tf.nn.dropout selected by train_mode: nn/utils.py:6-22) in one pass, the keep decisions drawn inside
 * the kernel (Philox4x32-10; key = seed, counter = (element / 4, site, step)) - no random tensor and no mask in
 * memory.  `state` = device int64[2] {seed, step}; the host bumps `step` once per training step, `site` numbers
 * the dropout calls of a step in program order.
 *   nm_dropout_apply: y[i] = keep_i ? x[i] / keep_prob : 0   (+ residual[i] when residual != NULL); y may alias x.
 *     The backward pass is the same call on the incoming gradient with the same (site, step).
 *   nm_dropout_mask:  mask[i] = keep_i ? 1 / keep_prob : 0  (for kernels that take a mask operand: nm_mha_fwd_drop,
 *     the drop_mask of nm_gru_seq_fwd). */
int nm_dropout_apply(const float* x, const float* residual, float* y, int64_t n, float keep_prob,
                     const int64_t* state, int64_t site, void* stream);
int nm_dropout_mask(float* mask, int64_t n, float keep_prob, const int64_t* state, int64_t site,
                    void* stream);
/* maxout of nn/projection.py:7-35: y[m,j] = max(z[m,j], z[m,O+j]); z is [M,2*O].
 * fwd writes y and the uint8 winner (0: first half, 1: second half). */
int nm_maxout_fwd(const float* z, float* y, uint8_t* which, int64_t M, int64_t O,
                  void* stream);
int nm_maxout_bwd(const float* dy, const uint8_t* which, float* dz, int64_t M,
                  int64_t O, void* stream);

/* ---- K7: layer normalisation ----------------------------------------------
 * Replaces tf_utils.layer_norm (neuralmonkey/tf_utils.py:189-219): biased
 * variance, eps inside the rsqrt, over the last dim.  rstd/mean are saved [M]. */
int nm_layernorm_fwd(const float* x, const float* gamma, const float* beta,
                     float* y, float* mean, float* rstd, int64_t M, int64_t D,
                     float eps, void* stream);
/* dgamma/dbeta are accumulated into (two call sites share LayerNorm/{gamma,beta}
 * in RecurrentEncoder: encoders/recurrent.py:215-216).  dx == NULL: parameter gradients only;
 * dgamma == dbeta == NULL: input gradient only (two launches that a caller may put on different streams). */
int nm_layernorm_bwd(const float* x, const float* gamma, const float* mean,
                     const float* rstd, const float* dy, float* dx, float* dgamma,
                     float* dbeta, int64_t M, int64_t D, void* stream);

/* ---- K2: GRU over a whole sequence ------------------------------------------
 * Replaces tf.nn.dynamic_rnn / bidirectional_dynamic_rnn over
 * tf.contrib.rnn.GRUCell (encoders/recurrent.py:71-110, nn/ortho_gru_cell.py:44-53)
 * and, in teacher-forced training, the GRU part of Decoder.next_state
 * (decoders/decoder.py:279-289).  TF-1.12 GRUCell semantics:
 *     [r,u] = sigmoid(xg_t + h.Wgh)          (xg already holds x.Wgx + b_g)
 *     c     = tanh(xc_t + (r*h).Wch)         (xc already holds x.Wcx + b_c)
 *     h'    = u*h + (1-u)*c
 * xproj is [B,T,3H] = [xg(2H) | xc(H)] per step.  lengths (int32 [B], may be
 * NULL) gives dynamic_rnn masking: for t >= len the output is 0 and the state
 * is carried.  reverse=1 walks t = len-1 .. 0 (tf.reverse_sequence semantics:
 * outputs land at their original time index).  drop_mask ([B,T,H], already scaled
 * by 1/keep_prob, may be NULL) multiplies each new state BEFORE it is emitted and fed
 * back: the reference decoder's recurrence runs on the dropped-out cell output
 * (decoders/decoder.py:288-289,333-334,351).
 * Outputs: states [B,T,H]; raw_states [B,T,H] (cell outputs before drop_mask, the
 * attention query of decoder.py:291-297; may be NULL); final [B,H]; and, saved for
 * the backward pass (sm_budget > 0 limits the launch to that many SMs so that two
 * directions can run side by side on two streams; 0 = whole chip):
 * gates [B,T,3H] = (r,u,c), hprev [B,T,H] = the state each step consumed,
 * rh [B,T,H] = r*hprev (the A operand of the candidate matmul). */
int nm_gru_seq_fwd(const float* xproj, const float* Wgh, const float* Wch,
                   const float* h0, const int32_t* lengths,
                   const float* drop_mask, int reverse, float* states,
                   float* raw_states, float* final_state, float* gates,
                   float* hprev, float* rh, int64_t B, int64_t T, int64_t H,
                   int sm_budget, void* stream);
/* Number of 8-CTA clusters of the persistent GRU kernel that are co-resident on the
 * current device (forward: backward=0).  Diagnostic. */
int nm_gru_resident_clusters(int backward);
/* Diagnostic: 8 int64 device counters receiving the cycles thread 0 of CTA 0 of the forward and
 * backward cluster kernels spends per section of a step (see tools/gru_probe.py). NULL = off. */
int nm_gru_debug_profile(void* counters);
/* Inputs: dstates [B,T,H] (may be NULL), dfinal [B,H] (may be NULL).
 * Outputs: dxproj [B,T,3H] (pre-activation grads = grads of xproj), dh0 [B,H]
 * (may be NULL).  Weight grads are NOT produced here: they are the hoisted
 * GEMMs hprev^T.dxproj[:, :2H] and rh^T.dxproj[:, 2H:], which the host issues
 * through nm_gemm.  work is a scratch buffer of 2*B*H floats. */
int nm_gru_seq_bwd(const float* Wgh, const float* Wch, const int32_t* lengths,
                   const float* drop_mask, int reverse, const float* gates,
                   const float* hprev, const float* dstates,
                   const float* draw /* grad of raw_states, may be NULL */,
                   const float* dfinal, float* dxproj, float* dh0, float* work,
                   int64_t B, int64_t T, int64_t H, int sm_budget, void* stream);

/* Both directions of a bidirectional layer (tf.nn.bidirectional_dynamic_rnn, encoders/recurrent.py:82-95):
 * sequence a, then sequence b, each as one nm_gru_seq_fwd / nm_gru_seq_bwd call on the whole GPU.  Same
 * arguments as nm_gru_seq_fwd / nm_gru_seq_bwd per sequence, without h0 / drop_mask / raw_states (encoder
 * layers have none); `lengths` is shared. */
int nm_gru_seq_fwd_pair(const float* xproj_a, const float* Wgh_a, const float* Wch_a, int reverse_a,
                        float* states_a, float* final_a, float* gates_a, float* hprev_a, float* rh_a,
                        const float* xproj_b, const float* Wgh_b, const float* Wch_b, int reverse_b,
                        float* states_b, float* final_b, float* gates_b, float* hprev_b, float* rh_b,
                        const int32_t* lengths, int64_t B, int64_t T, int64_t H, void* stream);
int nm_gru_seq_bwd_pair(const float* Wgh_a, const float* Wch_a, int reverse_a, const float* gates_a,
                        const float* hprev_a, const float* dstates_a, const float* dfinal_a,
                        float* dxproj_a, const float* Wgh_b, const float* Wch_b, int reverse_b,
                        const float* gates_b, const float* hprev_b, const float* dstates_b,
                        const float* dfinal_b, float* dxproj_b, const int32_t* lengths, float* work,
                        int64_t B, int64_t T, int64_t H, void* stream);

/* ---- K4: Bahdanau attention -------------------------------------------------
 * Replaces Attention.attention (attention/feed_forward.py:125-166) for NQ query
 * steps at once (NQ = Ty in teacher-forced training, 1 in step-wise decoding):
 *     e[b,q,t] = sum_a v[a]*tanh(keys[b,t,a] + qproj[b,q,a]) + bias
 *     w        = softmax_t(e) * mask ;  w /= (sum_t w + 1e-8)
 *     ctx[b,q] = sum_t w[b,q,t] * values[b,t,:]
 * keys [B,Tx,A] (hidden_features), values [B,Tx,C] (attention_states),
 * mask [B,Tx] fp32 (may be NULL = no masking: plain softmax),
 * qproj [B,NQ,A] (= query.W_q + b_p), v [A], bias [1] (device scalar).
 * Outputs: energies [B,NQ,Tx] (pre-softmax e, saved for backward; may be NULL),
 * weights [B,NQ,Tx], ctx [B,NQ,C]. */
int nm_bahdanau_fwd(const float* keys, const float* values, const float* mask,
                    const float* qproj, const float* v, const float* bias,
                    float* energies, float* weights, float* ctx, int64_t B,
                    int64_t Tx, int64_t NQ, int64_t A, int64_t C, void* stream);
/* Backward.  dkeys [B,Tx,A], dvalues [B,Tx,C], dqproj [B,NQ,A] are overwritten;
 * dv [A] and dbias [1] are accumulated into.  Gradient reaches the energies of
 * masked positions too (the softmax runs before the mask), as in the reference.
 * de_in [B,NQ,Tx] (may be NULL = none) is a gradient of a loss on the energies
 * themselves (K21); it is added to the energy gradient derived from dctx before
 * that reaches keys, qproj, v and bias.  de_work is scratch of B*NQ*Tx floats. */
int nm_bahdanau_bwd(const float* keys, const float* values, const float* mask,
                    const float* qproj, const float* v, const float* energies,
                    const float* weights, const float* dctx, const float* de_in, float* dkeys,
                    float* dvalues, float* dqproj, float* dv, float* dbias,
                    float* de_work, int64_t B, int64_t Tx, int64_t NQ, int64_t A,
                    int64_t C, void* stream);

/* ---- Coverage attention --------------------------------------------------------
 * Replaces CoverageAttention (attention/coverage.py:37-61 with
 * attention/feed_forward.py:125-166) for NQ decoder steps at once, as a scan:
 *     fert[b,t]  = 1e-8 + max_fertility*sigmoid(sum_c fertility_w[c]*S[b,t,c])
 *     sum_0      = cov_in (0 when NULL);  sum_{q+1} = sum_q + w[b,q,:]
 *     cov[b,q,t] = sum_q[t] / fert[b,t] * mask[b,t]
 *     e[b,q,t]   = sum_a v[a]*tanh(keys[b,t,a] + qproj[b,q,a] + coverage_w[a]*cov[b,q,t])
 *     w          = softmax_t(e) * mask ;  w /= (sum_t w + 1e-8)   (as K4, no bias)
 *     ctx[b,q]   = sum_t w[b,q,t] * values[b,t,:];   cov_out = sum_NQ
 * Fertility: states [B,Tx,C] -> fert [B,Tx], fp32 dot products.  Its backward
 * overwrites dstates and accumulates into dfertility_w [C]; work is B*C floats. */
int nm_coverage_fertility_fwd(const float* states, const float* fertility_w,
                              float max_fertility, float* fert, int64_t B,
                              int64_t Tx, int64_t C, void* stream);
int nm_coverage_fertility_bwd(const float* states, const float* fertility_w,
                              float max_fertility, const float* dfert,
                              float* dstates, float* dfertility_w, float* work,
                              int64_t B, int64_t Tx, int64_t C, void* stream);
/* Attention scan.  keys [B,Tx,A], values [B,Tx,C], mask [B,Tx] (may be NULL),
 * fert [B,Tx], qproj [B,NQ,A], v [A], coverage_w [A], cov_in [B,Tx] (may be
 * NULL = zero coverage).  Outputs: energies, weights and coverage [B,NQ,Tx]
 * (the first and last saved for backward), ctx [B,NQ,C], cov_out [B,Tx].  Each
 * step's arithmetic is independent of NQ: NQ chained one-step calls give the
 * bits of one NQ-step call.  Refuses (NM_E_UNSUPPORTED) shapes whose shared
 * memory, 4*(3A + 4Tx) bytes, exceeds 200 KB. */
int nm_coverage_attention_fwd(const float* keys, const float* values,
                              const float* mask, const float* fert,
                              const float* qproj, const float* v,
                              const float* coverage_w, const float* cov_in,
                              float* energies, float* weights, float* coverage,
                              float* ctx, float* cov_out, int64_t B, int64_t Tx,
                              int64_t NQ, int64_t A, int64_t C, void* stream);
/* Reverse scan.  dkeys, dvalues, dqproj, dfert and dcov_in (may be NULL) are
 * overwritten; dv and dcoverage_w [A] are accumulated into.  dcov_out may be
 * NULL (zero).  No atomics: repeated calls give identical bits.  work is 2*B*A
 * floats.  Refuses B > 65535, 4*(51A + C + 6Tx) bytes of shared memory above
 * 200 KB, or 4*NQ*(Tx rounded up to 8 + 128) bytes above 200 KB. */
int nm_coverage_attention_bwd(const float* keys, const float* values,
                              const float* mask, const float* fert,
                              const float* qproj, const float* v,
                              const float* coverage_w, const float* energies,
                              const float* weights, const float* coverage,
                              const float* dctx, const float* dcov_out,
                              float* dkeys, float* dvalues, float* dqproj,
                              float* dfert, float* dcov_in, float* dv,
                              float* dcoverage_w, float* work, int64_t B,
                              int64_t Tx, int64_t NQ, int64_t A, int64_t C,
                              void* stream);

/* ---- Joint multi-source attention --------------------------------------------
 * Replaces FlatMultiAttention.attention (attention/combination.py:240-321) and
 * HierarchicalMultiAttention.attention (:394-463) for NQ query steps at once:
 *     e[b,q,t]    = sum_a v[a]*tanh(keys[b,t,a] + qproj[b,q,a]) + seg_bias[seg(t)]
 *     e[b,q,Tx+j] = sum_a v[a]*tanh(ckeys[b,q,j,a] + qproj[b,q,a]) + cand_bias[j]
 *     p = softmax over all L = Tx + J positions
 *     mask given: w = p*m / (sum p*m + 1e-8), m = mask[b,t] (t < Tx), 1 (candidates)
 *     mask NULL:  w = p
 *     ctx[b,q] = sum_t w[b,q,t]*values[b,t,:] + sum_j w[b,q,Tx+j]*cvalues[b,q,j,:]
 * keys [B,Tx,A], values [B,Tx,C], mask [B,Tx] (may be NULL), seg_ends: HOST array
 * of S cumulative segment ends (the last is Tx; S = 0 iff Tx = 0; S <= 8),
 * seg_bias [S], ckeys [B,NQ,J,A], cvalues [B,NQ,J,C], cand_bias [J], qproj
 * [B,NQ,A], v [A].  Tx = 0 or J = 0 is allowed (not both); the pointers of an
 * empty part may be NULL.  Outputs: energies [B,NQ,L] (saved for backward; may
 * be NULL), weights [B,NQ,L], ctx [B,NQ,C].  fp32 throughout. */
int nm_joint_attention_fwd(const float* keys, const float* values,
                           const float* mask, const int64_t* seg_ends,
                           const float* seg_bias, const float* ckeys,
                           const float* cvalues, const float* cand_bias,
                           const float* qproj, const float* v, float* energies,
                           float* weights, float* ctx, int64_t B, int64_t Tx,
                           int64_t S, int64_t J, int64_t NQ, int64_t A,
                           int64_t C, void* stream);
/* Backward.  dkeys, dvalues, dqproj, dckeys, dcvalues are overwritten; dv [A],
 * dseg_bias [S] and dcand_bias [J] are accumulated into.  The gradient reaches
 * masked energies too.  No atomics: repeated calls give identical bits.  work is
 * scratch of B*NQ*(Tx+J) + B*A + B*(S+J) floats. */
int nm_joint_attention_bwd(const float* keys, const float* values,
                           const float* mask, const int64_t* seg_ends,
                           const float* ckeys, const float* cvalues,
                           const float* qproj, const float* v,
                           const float* energies, const float* weights,
                           const float* dctx, float* dkeys, float* dvalues,
                           float* dqproj, float* dckeys, float* dcvalues,
                           float* dv, float* dseg_bias, float* dcand_bias,
                           float* work, int64_t B, int64_t Tx, int64_t S,
                           int64_t J, int64_t NQ, int64_t A, int64_t C,
                           void* stream);

/* ---- K5/K6: vocabulary projection loss ---------------------------------------
 * Replaces log_softmax + tf.contrib.seq2seq.sequence_loss
 * (decoders/autoregressive.py:288-316) and the greedy argmax (:446-480).
 * logits [M,V] (already includes the bias).  unk_index >= 0: -1e9 is added to
 * column unk_index of every row and written back to logits (the <unk> mask).
 * Per row m: lse[m] = logsumexp_v logits; xent[m] = (lse - logits[m,target[m]])
 * * weight[m]; argmax[m] = first index of the row maximum (tf.argmax order).
 * targets may be NULL (then xent is not written). */
int nm_xent_fwd(float* logits, int64_t unk_index, const int64_t* targets, const float* weights,
                float* lse, float* xent, int64_t* argmax, int64_t M, int64_t V,
                int64_t ldl, void* stream);
/* dlogits[m,v] = (exp(logits[m,v]-lse[m]) - [v==target[m]]) * weights[m] * scale[0]
 * (scale is a DEVICE scalar: upstream dloss / sum(mask)). May be in place. */
int nm_xent_bwd(const float* logits, const int64_t* targets, const float* weights,
                const float* lse, const float* scale, float* dlogits, int64_t M,
                int64_t V, int64_t ldl, void* stream);
/* logprobs[m,v] = logits[m,v] - lse[m]  (runtime_logprobs of the runner API). */
int nm_log_softmax(const float* logits, const float* lse, float* logprobs,
                   int64_t M, int64_t V, int64_t ldl, void* stream);

/* Fused vocabulary projection + loss statistics (K5 without materialising the
 * [M,V] logits): logits = X[M,K].W + b (+ -1e9 at unk_index if >= 0), W stored
 * [K,V] (transW=0) or [V,K] (transW=1: tied embeddings, decoders/autoregressive.py:231-233), on
 * wgmma; writes lse, xent, argmax as nm_xent_fwd.  part is scratch of
 * nm_logits_xent_scratch(M,V) floats (16-byte aligned).  logits_out (may be NULL)
 * additionally receives the [M,V] logits (runtime_logits of the runner API).
 * Returns NM_E_UNSUPPORTED when X/W are not TMA-addressable (rows not multiples
 * of 16 bytes): callers then use nm_gemm + nm_xent_fwd. */
int64_t nm_logits_xent_scratch(int64_t M, int64_t V);
int nm_logits_xent_fwd(const float* X, int64_t ldx, const float* W, int64_t ldw,
                       int transW, const float* b, int64_t unk_index, const int64_t* targets,
                       const float* weights, float* lse, float* xent,
                       int64_t* argmax, float* part, float* logits_out,
                       int64_t ldl, int64_t M, int64_t V, int64_t K, void* stream);
/* Recomputes the logits tile-by-tile and writes
 * dlogits = (softmax - onehot) * weights[m] * scale[0]   [M,V]. */
int nm_logits_xent_bwd(const float* X, int64_t ldx, const float* W, int64_t ldw,
                       int transW, const float* b, int64_t unk_index, const int64_t* targets,
                       const float* weights, const float* lse, const float* scale,
                       float* dlogits, int64_t ldd, int64_t M, int64_t V,
                       int64_t K, void* stream);

/* ---- K5/K6 with fp16 operands: the default path of ops.logits_xent ----
 * Every product is K-major x K-major: X16 [M,K], WT16 [V,K] (the projection matrix transposed),
 * row pitches multiples of 8 elements, bases 16-byte aligned.
 * nm_cast_f16: dst = half(src * row_scale[row]) (row_scale may be NULL) followed by `extra_ones` columns
 *   holding row_scale (the ones column of the bias-gradient trick); transpose != 0 writes
 *   dst [cols + extra_ones, ld_dst] = the transpose of that; padding up to ld_dst is zeroed.
 * nm_gemm_f16: C[M,N] (or C^T when transposed != 0: element (m,n) -> C[n*ldc+m])
 *   = alpha_dev[0] * row_scale[m] * A16[M,K] . B16[N,K]^T  (+ C when beta == 1).
 * nm_logits_xent_fwd16: as nm_logits_xent_fwd.
 * nm_logits_xent_bwd16: dl16 [M,V] = half((softmax - onehot) * mask[m]), row pitch ldd (a multiple of 8,
 *   base 16-byte aligned); the upstream scale is applied by the consumers (replaces autoregressive.py:292-316
 *   backward). */
int nm_cast_f16(const float* src, int64_t ld_src, void* dst, int64_t ld_dst, int64_t rows,
                int64_t cols, const float* row_scale, int transpose, int extra_ones, void* stream);
int nm_gemm_f16(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16,
                int64_t ldb, float* C, int64_t ldc, const float* alpha_dev, const float* row_scale,
                float beta, int transposed, void* stream);
/* C[M,N] = alpha_dev[0] * A16^T . B16 (+ C when beta == 1) with both operands stored reduction-major:
 * A16 [K,M] (row pitch lda), B16 [K,N] (row pitch ldb) - the weight-gradient product X^T . dY of the
 * vocabulary projection straight from the row-major fp16 matrices (MN-major wgmma operands), no
 * transposed copies. */
int nm_gemm_f16_tn(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16,
                   int64_t ldb, float* C, int64_t ldc, const float* alpha_dev, float beta, void* stream);
/* nm_gemm_f16_tn on at most max_ctas SMs (<= 0: all of them), leaving the others to work issued concurrently
 * on other streams: the product runs one persistent CTA per SM it is given, which no other kernel can share. */
int nm_gemm_f16_tn_ctas(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16,
                        int64_t ldb, float* C, int64_t ldc, const float* alpha_dev, float beta, int max_ctas,
                        void* stream);
int nm_logits_xent_fwd16(const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                         int64_t unk_index, const int64_t* targets, const float* weights, float* lse,
                         float* xent, int64_t* argmax, float* part, float* logits_out, int64_t ldl,
                         int64_t M, int64_t V, int64_t K, void* stream);
int nm_logits_xent_bwd16(const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                         int64_t unk_index, const int64_t* targets, const float* mask, const float* lse,
                         void* dl16, int64_t ldd, int64_t M, int64_t V, int64_t K, void* stream);

/* ---- K11: beam-search step ----------------------------------------------------
 * Replaces steps (1)-(8) of BeamSearchDecoder body
 * (decoders/beam_search_decoder.py:440-496).  Per batch item b with beam k:
 *   rows of finished hypotheses become {PAD:0, others:-1e9}; hyp = logprob_sum +
 *   logprobs; len' = len + 1 - finished; score = hyp / ((5+len')/6)^alpha;
 *   top-k over the k*V candidates (ties: lower flat index first, tf.nn.top_k);
 *   word = idx % V (int64), beam = idx / V (int32); gathers lengths, the
 *   UN-normalised logprob_sum and finished by (b, beam); finished |= word==2.
 * In:  logprobs [B,k,V], logprob_sum [B,k], lengths [B,k] i32, finished [B,k] u8.
 * Out: scores [B,k], word_ids [B,k] i64, beam_ids [B,k] i32, logprob_sum_out,
 *      lengths_out, finished_out (may NOT alias the inputs).  The length penalty
 *      is evaluated as fp32 (5+len)/6 followed by a correctly rounded powf, so the
 *      scores and therefore the selected indices are bit-identical to an IEEE fp32
 *      CPU evaluation of the same graph.  k <= 64. */
int nm_beam_step(const float* logprobs, const float* logprob_sum,
                 const int32_t* lengths, const uint8_t* finished, float alpha,
                 float* scores, int64_t* word_ids, int32_t* beam_ids,
                 float* logprob_sum_out, int32_t* lengths_out,
                 uint8_t* finished_out, void* scratch, int64_t B, int64_t k,
                 int64_t V, void* stream);
/* Size of nm_beam_step's scratch in 4-byte words. */
int64_t nm_beam_scratch(int64_t B, int64_t k, int64_t V);
/* gather_flat (tf_utils.py:106-131): out[b*k+j, :] = x[b*k+beam_ids[b,j], :],
 * row = `row_bytes` bytes (any dtype). */
int nm_beam_gather(const void* x, const int32_t* beam_ids, void* out, int64_t B,
                   int64_t k, int64_t row_bytes, void* stream);

/* ---- K13: per-tensor clip + Adam over a flat parameter arena --------------------
 * Replaces GenericTrainer.{regularization_losses,gradients,train_op}
 * (trainers/generic_trainer.py:84-195) with tf.train.AdamOptimizer semantics:
 *   g += 2*l2*p + l1*sign(p)            (only where seg_reg[s] != 0)
 *   g *= min(1, clip/||g_s||)           per tensor s (tf.clip_by_norm), clip<=0: off
 *   m = b1*m+(1-b1)*g ; v = b2*v+(1-b2)*g^2 ; p -= lr_t * m/(sqrt(v)+eps)
 * with lr_t = lr*sqrt(1-b2^t)/(1-b1^t) computed by the caller.
 * The arena holds `n` floats split into `nseg` tensors: seg_off [nseg+1] int64
 * (device), seg_reg [nseg] uint8 (device).  norms [nseg] scratch (device).
 * grad_scale multiplies g first (1/k for delayed updates); grad_denominator (a
 * DEVICE scalar, may be NULL) then divides it: the all-reduced global token count of
 * a data-parallel step, so the host never has to read it back.  l1l2_out [2] (device, may be NULL) receives sum|p|, sum p^2 over
 * regularised tensors (the "L1"/"L2" losses the trainer reports).  * seg_reg flags per segment: bit 0 = receives the L1/L2 terms (generic_trainer.py:87-91),
 * bit 1 = lazy (tf.contrib.opt.LazyAdamOptimizer): entries whose gradient is exactly zero keep
 * their moments and value. */
int nm_clip_adam_step(float* params, float* grads, float* m, float* v,
                      const int64_t* seg_off, const uint8_t* seg_reg, float* norms,
                      int64_t n, int64_t nseg, float grad_scale,
                      const float* grad_denominator, float lr_t,
                      float beta1, float beta2, float eps, float clip_norm,
                      float l1, float l2, float* l1l2_out,
                      const float* lr_t_dev /* optional device scalar that replaces lr_t, so a
                                               captured CUDA graph of the step can be replayed
                                               with the schedule's next value */,
                      void* stream);

/* tf.train.AdadeltaOptimizer (trainers/generic_trainer.py:172-190 with an Adadelta optimizer, tests/str.ini) after
 * the same regularisation and per-tensor clip_by_norm as nm_clip_adam_step, over the same arena and segment tables:
 *   accum = rho*accum + (1-rho)*g^2;  update = sqrt(accum_update + eps) / sqrt(accum + eps) * g;
 *   accum_update = rho*accum_update + (1-rho)*update^2;  p -= lr*update
 * Segments flagged lazy (bit 1) skip entries whose gradient is exactly zero.  lr_dev: as lr_t_dev above. */
int nm_clip_adadelta_step(float* params, float* grads, float* accum, float* accum_update, const int64_t* seg_off,
                          const uint8_t* seg_reg, float* norms, int64_t n, int64_t nseg, float grad_scale,
                          const float* grad_denominator, float lr, float rho, float eps, float clip_norm, float l1,
                          float l2, float* l1l2_out, const float* lr_dev, void* stream);

/* ---- K8: multi-head scaled dot-product attention core ---------------------------
 * Replaces attention() of attention/scaled_dot_product.py:98-226 between the
 * q/k/v projections and the output projection:
 *   E = (q/sqrt(dh)).k^T ; causal: where(tril, E, -1e9) ; key mask:
 *   E*m + (1-m)*(-1e9) ; P = softmax(E) ; out = P.v
 * q [B,Tq,h*dh], k/v [B,Tk,h*dh] (heads interleaved on the feature axis as
 * split_for_heads does), key_mask [B,Tk] fp32 or NULL.  probs [B,h,Tq,Tk] saved. */
int nm_mha_fwd(const float* q, const float* k, const float* v,
               const float* key_mask, int causal, float* out, float* probs,
               int64_t B, int64_t Tq, int64_t Tk, int64_t heads, int64_t dh,
               void* stream);
int nm_mha_bwd(const float* q, const float* k, const float* v,
               const float* key_mask, int causal, const float* probs,
               const float* dout, float* dq, float* dk, float* dv,
               float* de_work /* scratch, B*heads*Tq*Tk floats */, int64_t B,
               int64_t Tq, int64_t Tk, int64_t heads, int64_t dh, void* stream);
/* The same with attention-weight dropout (attention/scaled_dot_product.py:208-214): drop_mask
 * [B, heads, Tq, Tk] holds 0 or 1/keep_prob; context = (softmax * drop_mask) . V, while `probs`
 * keeps the undropped softmax (what the softmax backward needs).  Supported wherever nm_mha_fwd /
 * nm_mha_bwd are: both the tiled and the row kernels apply the mask. */
int nm_mha_fwd_drop(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                    const float* drop_mask, float* out, float* probs, int64_t B, int64_t Tq,
                    int64_t Tk, int64_t heads, int64_t dh, void* stream);
int nm_mha_bwd_drop(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                    const float* drop_mask, const float* probs, const float* dout, float* dq,
                    float* dk, float* dv, float* de_work, int64_t B, int64_t Tq, int64_t Tk,
                    int64_t heads, int64_t dh, void* stream);

/* The same attention on the tensor cores: every product a batched wgmma GEMM over all (sentence, head)
 * pairs - P = softmax(mask(Q.K^T/sqrt(dh))) with the softmax in the GEMM epilogue, O = (P*drop).V; backward
 * dS = P*(dO.V^T*drop - rowsum)/sqrt(dh) in the epilogue, dQ = dS.K, dK = dS^T.Q, dV = (P*drop)^T.dO.  TF32
 * operands, fp32 accumulation; q/k/v/out and their gradients keep the [B, T, heads*dh] layout (a head is a
 * column window of the TMA tensor map).  probs, probs_drop and ds_work are [B, heads, Tq32, Tk32] with both
 * time extents rounded up to 32 and the padding written as zeros; probs_drop (= probs * drop_mask) exists
 * exactly when drop_mask [B, heads, Tq, Tk] is given.  Supported: dh % 32 == 0, dh <= 128, Tk <= 128
 * (nm_mha_tc_supported returns 1), otherwise NM_E_UNSUPPORTED - nm_mha_fwd / nm_mha_bwd serve the rest and
 * remain the exact-fp32 engine. */
int nm_mha_tc_supported(int64_t B, int64_t Tq, int64_t Tk, int64_t heads, int64_t dh);
int nm_mha_tc_fwd(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                  const float* drop_mask, float* out, float* probs, float* probs_drop, int64_t B,
                  int64_t Tq, int64_t Tk, int64_t heads, int64_t dh, void* stream);
int nm_mha_tc_bwd(const float* q, const float* k, const float* v, const float* key_mask, int causal,
                  const float* drop_mask, const float* probs, const float* probs_drop, const float* dout,
                  float* dq, float* dk, float* dv, float* ds_work, int64_t B, int64_t Tq, int64_t Tk,
                  int64_t heads, int64_t dh, void* stream);

/* ---- K12: VGG convolution stack primitives (forward only; the encoder is frozen,
 * encoders/imagenet_encoder.py:212,234) -----------------------------------------
 * NHWC fp32; 3x3, stride 1, SAME padding, + bias + ReLU (slim vgg_arg_scope);
 * w is [3,3,Cin,Cout] (HWIO, the slim checkpoint layout).  Exact fp32 on the CUDA cores: the NM_GEMM_SIMT
 * forward of nm_conv2d_fwd (csrc/conv_igemm.cuh).  Any batch whose ceil(N*H*W / 64) pixel tiles stay below 2^31
 * is accepted; earlier versions returned NM_E_UNSUPPORTED for some very large batches. */
int nm_conv3x3_bias_relu_fwd(const float* x, const float* w, const float* bias,
                             float* y, int64_t N, int64_t H, int64_t W,
                             int64_t Cin, int64_t Cout, void* stream);
/* Patch matrix of the same convolution for the tensor-core path (the conv is then nm_gemm with
 * the bias+ReLU epilogue; output rows are NHWC pixels): cols[(n,y,x)][tap*Cin + c], row pitch ldc
 * floats (>= 9*Cin; a multiple of 4 keeps the rows TMA-addressable), zeros outside the image.
 * Same layer as above: slim vgg_arg_scope conv2d (encoders/imagenet_encoder.py:52-68). */
int nm_im2col3x3(const float* x, float* cols, int64_t N, int64_t H, int64_t W,
                 int64_t Cin, int64_t ldc, void* stream);
/* 2x2 / stride 2 max pool, NHWC (H, W even). */
int nm_maxpool2x2_fwd(const float* x, float* y, int64_t N, int64_t H, int64_t W,
                      int64_t C, void* stream);

/* ---- K12: ResNet-v2 convolutions (forward only; the encoder is frozen, encoders/imagenet_encoder.py:70-99
 * builds slim nets/resnet_v2.py) ---------------------------------------------------------------------------------
 * y [N,Ho,Wo,Cout] = act(z + r), NHWC fp32, w [k,k,Cin,Cout] (HWIO), with
 *   A = relu(x * in_scale[c] + in_shift[c]) inside the image and 0 in the padding when in_scale is non-NULL, else x
 *       (the preactivation batch norm of a v2 unit, never written to memory);
 *   acc[n,oy,ox,o] = sum over the k x k window at (oy*stride - pad_top, ox*stride - pad_left) of A * w;
 *   z = acc * out_scale[o] + out_shift[o] when out_scale is non-NULL (an inference-mode batch norm), else acc + bias[o]
 *       (bias may be NULL; out_scale and bias exclude each other);
 *   r = res[n, oy*res_stride, ox*res_stride, o] when res is non-NULL (res [N,res_H,res_W,Cout], res_stride 1 or 2,
 *       ceil(res_H / res_stride) = Ho, ceil(res_W / res_stride) = Wo: the identity shortcut, subsampled in a strided
 *       unit), else 0.
 * Ho = (H + pad_top + pad_bottom - k) / stride + 1 (Wo likewise); pads lie in [0, k).  The scale / shift pairs come
 * together.  act is NM_ACT_NONE or NM_ACT_RELU.  backend: NM_GEMM_SIMT = exact fp32 on the CUDA cores, NM_GEMM_AUTO /
 * NM_GEMM_TC = wgmma with TF32 operands (the implicit-GEMM kernels of csrc/conv_igemm.cuh).  Bad arguments return
 * NM_E_INVALID or NM_E_UNSUPPORTED with a message and launch nothing. */
int nm_conv2d_bn_fwd(const float* x, const float* w, const float* in_scale, const float* in_shift,
                     const float* out_scale, const float* out_shift, const float* bias, const float* res,
                     int64_t res_H, int64_t res_W, int64_t res_stride, float* y, int64_t N, int64_t H, int64_t W,
                     int64_t Cin, int64_t Cout, int64_t k, int64_t stride, int64_t pad_top, int64_t pad_bottom,
                     int64_t pad_left, int64_t pad_right, int act, int backend, void* stream);

/* ---- K12b: trainable CNN layers (encoders/cnn_encoder.py:209-320: tf.layers.conv2d, batch_normalization,
 * max_pooling2d / average_pooling2d) --------------------------------------------------------------------------
 * NHWC fp32, filters HWIO.  Convolutions have stride 1 (the reference never strides them).
 *
 * nm_conv2d_fwd: y [N,Ho,Wo,Cout] = act(conv(x [N,H,W,Cin], w) + bias), Ho = H + pad_top + pad_bottom - k + 1
 * (Wo likewise); `same` in TF's convention is pad_top = (k-1)/2, pad_bottom = k-1-pad_top, `valid` all zero.
 * w is [k,k,Cin,Cout]; with flip = 1 it is [k,k,Cout,Cin] and is applied turned by 180 degrees with its channel
 * axes swapped: the data gradient of a forward convolution with pads (t, b, l, r) is this call on dY with
 * pads (k-1-t, k-1-b, k-1-l, k-1-r), flip = 1, no bias.  bias may be NULL; act is NM_ACT_NONE or NM_ACT_RELU.
 * An implicit GEMM (no patch matrix): backend NM_GEMM_SIMT = exact fp32 on the CUDA cores, NM_GEMM_AUTO /
 * NM_GEMM_TC = wgmma with TF32 operands.
 * nm_conv2d_wgrad: dw [k,k,Cin,Cout] += sum over the output pixels of patch(x)^T dy, db [Cout] += sum dy (db may
 * be NULL).  The pixel reduction is split over CTAs into `workspace` (>= (k*k*Cin+1)*Cout floats; more lets it
 * split further) and the partials are added in a fixed order: two calls give identical bits.
 * nm_conv2d_wgrad_workspace: the workspace (floats) at which nm_conv2d_wgrad splits as far as it wants to for that
 * shape and backend, or -1 for invalid sizes. */
int nm_conv2d_fwd(const float* x, const float* w, const float* bias, float* y, int64_t N, int64_t H, int64_t W,
                  int64_t Cin, int64_t Cout, int64_t k, int64_t pad_top, int64_t pad_bottom, int64_t pad_left,
                  int64_t pad_right, int flip, int act, int backend, void* stream);
int64_t nm_conv2d_wgrad_workspace(int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t k,
                                  int64_t pad_top, int64_t pad_bottom, int64_t pad_left, int64_t pad_right,
                                  int backend);
int nm_conv2d_wgrad(const float* x, const float* dy, float* dw, float* db, float* workspace, int64_t workspace_floats,
                    int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t k, int64_t pad_top,
                    int64_t pad_bottom, int64_t pad_left, int64_t pad_right, int backend, void* stream);
/* tf.layers.batch_normalization over the P = N*H*W rows of x [P,C] (+ the ReLU after it when relu = 1):
 * y = gamma * (x - mean) * invstd + beta, invstd = 1/sqrt(var + eps).  training = 1: mean and the biased var of the
 * batch (sums in fp64), and in the same call moving = momentum*moving + (1-momentum)*batch value, with the
 * Bessel-corrected batch variance for moving_var (TF 1.x fused batch norm); training = 0: the moving statistics.
 * save_mean / save_invstd [C] receive what was used.  workspace: NM_BN_WS_DOUBLES_PER_CHANNEL * C doubles (may
 * be NULL when training = 0).  Backward: dx (may be NULL) and dgamma, dbeta += (may be NULL), summed in a fixed
 * order. */
#define NM_BN_WS_DOUBLES_PER_CHANNEL 130
int nm_batchnorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* moving_mean,
                     float* moving_var, float* save_mean, float* save_invstd, double* workspace, int64_t P, int64_t C,
                     float momentum, float eps, int training, int relu, void* stream);
int nm_batchnorm_bwd(const float* x, const float* dy, const float* gamma, const float* beta, const float* save_mean,
                     const float* save_invstd, float* dx, float* dgamma, float* dbeta, double* workspace, int64_t P,
                     int64_t C, int training, int relu, void* stream);
/* k x k pooling with stride `stride`, max (is_max = 1) or average, NHWC.  same = 0: `valid`, Ho = (H-k)/stride+1;
 * same = 1: Ho = ceil(H/stride), padded TF's way (odd pixel at the bottom / right), averages over the pixels inside
 * the image.  The backward pass writes dx [N,H,W,C] (x is only read for max pooling); max pooling routes each
 * window's gradient to its first maximal pixel in row-major order, as TF does. */
int nm_pool2d_fwd(const float* x, float* y, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k, int64_t stride,
                  int same, int is_max, void* stream);
int nm_pool2d_bwd(const float* x, const float* dy, float* dx, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k,
                  int64_t stride, int same, int is_max, void* stream);

/* ---- gate arithmetic of the step-wise cell variants (SURVEY.md 8(f) N4) ------------------------------
 * NematusGRUCell (nn/ortho_gru_cell.py:57-105) after its four projections: sg = state_proj_g(state) [B,2H],
 * gi = input_proj_g(x) [B,2H], sc = state_proj_c(state) [B,H], ci = input_proj_c(x) [B,H]:
 *   [r,u] = sigmoid(sg + gi);  cand = tanh(sc * r + ci);  out = u * state + (1 - u) * cand
 * saved [B,3H] = (r, u, cand).  Backward: dgates [B,2H] (gradient of sg AND of gi), dcpre [B,H] (of ci),
 * dsc [B,H], dstate [B,H] (the direct path only; the projections' backward adds theirs). */
int nm_nematus_gate_fwd(const float* sg, const float* gi, const float* sc, const float* ci,
                        const float* state, float* out, float* saved, int64_t B, int64_t H, void* stream);
int nm_nematus_gate_bwd(const float* dout, const float* saved, const float* sc, const float* state,
                        float* dgates, float* dcpre, float* dsc, float* dstate, int64_t B, int64_t H,
                        void* stream);
/* tf.nn.rnn_cell.LSTMCell with its defaults (encoders/recurrent.py:21, decoders/decoder.py:29; forget_bias 1):
 * z [B,4H] = (i, j, f, o) = [x, h].kernel + bias;  c' = sigmoid(f + 1) * c + sigmoid(i) * tanh(j);
 * h' = sigmoid(o) * tanh(c').  saved [B,5H].  Backward: dnew_c / dnew_h may be NULL. */
int nm_lstm_gate_fwd(const float* z, const float* c, float* new_c, float* new_h, float* saved, int64_t B,
                     int64_t H, void* stream);
int nm_lstm_gate_bwd(const float* dnew_c, const float* dnew_h, const float* saved, const float* c,
                     float* dz, float* dc, int64_t B, int64_t H, void* stream);

/* ---- K4 (inference): the fused attention-decoder step ---------------------------------
 * Replaces ONE iteration of the decoding while_loop between the previous symbol and the vector the
 * vocabulary projection consumes: embed_input_symbols (decoders/autoregressive.py:269-272),
 * Decoder.next_state with a GRU cell (decoders/decoder.py:279-358: GRUCell on [emb; h], TF-1.12 gate
 * order, candidate on r*h), Attention.attention (attention/feed_forward.py:125-166: query projection,
 * energies, softmax over ALL Tx, mask, +1e-8 renormalisation, context) and the deep output
 * (decoders/output_projection.py:115-160: tanh/relu/sigmoid dense, or maxout).  Inference only:
 * no dropout.  One kernel launch; exact fp32.
 *   rows            hypotheses (batch, or batch*beam beam-minor); `group` consecutive rows share
 *                   encoder row (row / group): 1 for greedy decoding, the beam size for beam search
 *                   - the encoder tensors are NOT tiled;
 *   symbols [rows] i64 + emb_table [V,E], or x_in [rows,E] (already embedded; then symbols is ignored);
 *   h_prev [rows,H]; parent [rows] i32 or NULL: row r continues hypothesis
 *                   (r/group)*group + parent[r] of the previous step (the gather_flat of
 *                   beam_search_decoder.py:499-532 folded into the load); h_out must not alias h_prev;
 *   Wg [E+H,2H], bg [2H], Wc [E+H,H], bc [H]  (gates/candidate kernels of the GRUCell);
 *   Wq [H,A], bq [A], v [A], att_bias [1];  keys [NB,Tx,A] (hidden_features), values [NB,Tx,C]
 *                   (attention_states), mask [NB,Tx] fp32 or NULL, NB = rows/group;
 *   Wo [H+E+C, O] (or [H+E+C, 2*O] with maxout != 0), bo; act = NM_ACT_* (ignored with maxout).
 * Outputs: h_out [rows,H]; out [rows,O]; optional x_out [rows,E] (embedded input), ctx_out [rows,C],
 * weights_out [rows,Tx].  16-byte loads and TMA-staged key/value tiles need E,H,A,C,O % 4 == 0 and
 * 16-byte aligned bases; other shapes take a scalar variant of the same kernel.  Shapes the kernel cannot
 * take (nm_attn_decoder_step_supported returns 0) return NM_E_UNSUPPORTED before anything is launched. */
int nm_attn_decoder_step_fwd(const int64_t* symbols, const float* emb_table, const float* x_in,
                             const float* h_prev, const int32_t* parent, const float* Wg, const float* bg,
                             const float* Wc, const float* bc, const float* Wq, const float* bq,
                             const float* v, const float* att_bias, const float* keys,
                             const float* values, const float* mask, const float* Wo, const float* bo,
                             float* x_out, float* h_out, float* ctx_out, float* weights_out, float* out,
                             int64_t rows, int64_t group, int64_t E, int64_t H, int64_t A, int64_t C,
                             int64_t Tx, int64_t O, int act, int maxout, void* stream);

/* 1 when nm_attn_decoder_step_fwd takes this shape on the current device (its SM count picks the cluster
 * size, which sizes the shared memory), else 0: the context (C <= 512, or C <= 2048 on the vector variant),
 * one key / value tile and the step's shared memory must fit one CTA.  `aligned` != 0: Wg, Wc, Wq, Wo, keys
 * and values are 16-byte aligned. */
int nm_attn_decoder_step_supported(int64_t rows, int64_t group, int64_t E, int64_t H, int64_t A, int64_t C,
                                   int64_t Tx, int64_t O, int maxout, int aligned);

/* Diagnostic: 8 int64 device counters receiving the cycle counter of CTA 0 at the phase boundaries of the
 * following nm_attn_decoder_step_fwd launches; NULL switches it off. */
int nm_attn_decoder_step_debug(void* counters);

/* ---- K5/K6 at run time: logits, argmax and the symbol bookkeeping of one decoding step ------
 * Replaces get_body of decoders/autoregressive.py:446-480 after next_state: logits = X.W + b
 * (+ -1e9 at unk_index >= 0), lse[m], argmax[m] (first index), and - when symbols_out is given -
 *   symbol = finished_in[m] ? 0 : argmax;  finished_out = finished_in | (symbol == 2);
 *   mask_out = !finished_out;  *unfinished_count += number of rows still unfinished.
 * finished_in/finished_out (u8) may alias.  backend NM_GEMM_AUTO/TC: the wgmma GEMM with the
 * softmax-partials epilogue + one combine kernel (`part`: nm_logits_xent_scratch(M,V) floats;
 * logits_out optional).  NM_GEMM_SIMT: exact fp32 CUDA-core GEMM into logits_out (required) + one
 * row kernel.  With targets [M] (gold symbols of this step) xent[m] = (lse - logit[target]) * weights[m]
 * (runtime_xents, autoregressive.py:351-366).  lse / argmax / xent / the bookkeeping outputs may be NULL. */
int nm_decode_logits_step(const float* X, int64_t ldx, const float* W, int64_t ldw, int transW,
                          const float* b, int64_t unk_index, const uint8_t* finished_in,
                          const int64_t* targets, const float* weights, float* lse, int64_t* argmax,
                          float* xent, int64_t* symbols_out, uint8_t* finished_out, uint8_t* mask_out,
                          int32_t* unfinished_count, float* part, float* logits_out, int64_t ldl,
                          int64_t M, int64_t V, int64_t K, int backend, void* stream);

/* nm_beam_step reading LOGITS [B,k,V] and their logsumexp [B,k]: log-prob = logit - lse, the
 * subtraction nm_log_softmax performs, so the selected indices and scores are bit-identical while
 * the [B,k,V] log-prob tensor (beam_search_decoder.py:537-544) is never written.  unfinished_count
 * (device int32, may be NULL) += hypotheses still unfinished after this step (the loop criterion of
 * beam_search_decoder.py:330-355 without a host round trip per step). */
int nm_beam_step_logits(const float* logits, const float* lse, const float* logprob_sum,
                        const int32_t* lengths, const uint8_t* finished, float alpha, float* scores,
                        int64_t* word_ids, int32_t* beam_ids, float* logprob_sum_out,
                        int32_t* lengths_out, uint8_t* finished_out, int32_t* unfinished_count,
                        void* scratch, int64_t B, int64_t k, int64_t V, void* stream);
/* token_ids [steps+1, B, k] of the surviving hypotheses from the per-step records words
 * [steps,B,k] i64 / parents [steps,B,k] i32 and first_symbols [B,k] (slot 0): what re-gathering
 * the whole token history at every step computes (beam_search_decoder.py:546-551). */
int nm_beam_backtrack(const int64_t* first_symbols, const int64_t* words, const int32_t* parents,
                      int64_t* token_ids, int64_t B, int64_t k, int64_t steps, void* stream);

/* ---- K16: CTC loss and greedy CTC decoding ---------------------------------------------------------
 * Replace tf.nn.ctc_loss(ignore_longer_outputs_than_inputs=True, ctc_merge_repeated=merge_repeated) and
 * tf.nn.ctc_greedy_decoder of decoders/ctc_decoder.py:73-112 (TF 1.12 semantics; preprocess_collapse_repeated
 * is the caller's job).  logits [B,T,C] batch-major, the blank is class C-1; frames [B] i32: frames
 * t >= frames[b] are ignored; labels [B,Lmax] i64, row b holding label_lengths[b] (i32) labels in [0, C-1).
 * nm_ctc_loss_fwd: loss[b] = -log p(labels_b | logits_b), summed over the alignments of the extended label
 *   (blank, l1, blank, ..., blank) in log space.  merge_repeated != 0 (standard CTC): a state may repeat and
 *   the skip over a blank needs two different labels; 0: labels do not repeat, every label may be skipped to.
 *   A sentence whose labels need more frames than it has (L, plus one per pair of equal neighbours with
 *   merging), or that has no frames, gets loss 0; a label outside [0, C-1) or a length outside [0, Lmax]
 *   gives NaN.  Both get a zero gradient.
 * nm_ctc_loss_bwd: dlogits [B,T,C] = grad_loss[b] * (softmax - sum of the occupancies of the states of class k),
 *   dense, zeros on ignored frames; reads what the forward call left in the workspace and is deterministic.
 * workspace: at least B*T*(5*Lmax+4) + B*(Lmax+4) 4-byte words (8-byte aligned), passed to both calls;
 *   workspace_words is its size.  Lmax <= NM_CTC_MAX_LABEL, otherwise NM_E_UNSUPPORTED.
 * nm_ctc_greedy_decode: per frame the first index of the row maximum; blanks dropped, and with
 *   merge_repeated a symbol equal to the previous frame's maximum; ids [B,T] i64 padded with 2 (</s>),
 *   lengths [B] i32 = number of symbols kept. */
#define NM_CTC_MAX_LABEL 1023
int nm_ctc_loss_fwd(const float* logits, const int32_t* frames, const int64_t* labels,
                    const int32_t* label_lengths, int merge_repeated, float* loss, void* workspace,
                    int64_t workspace_words, int64_t B, int64_t T, int64_t C, int64_t Lmax, void* stream);
int nm_ctc_loss_bwd(const float* logits, const int32_t* frames, const int64_t* labels,
                    const int32_t* label_lengths, int merge_repeated, const float* grad_loss, float* dlogits,
                    void* workspace, int64_t workspace_words, int64_t B, int64_t T, int64_t C, int64_t Lmax,
                    void* stream);
int nm_ctc_greedy_decode(const float* logits, const int32_t* frames, int merge_repeated, int64_t* ids,
                         int32_t* lengths, int64_t B, int64_t T, int64_t C, void* stream);

/* ---- K17: rewards and sampling of the reinforcement-learning objectives ----------------------------------------
 * nm_sentence_ngram_reward replaces the tf.py_func over sentence_bleu / sentence_gleu of
 * trainers/self_critical_objective.py:124-231.  references [T_r,B] and hypotheses [T_h,B] are int64 token ids,
 * element (t,b) at t*stride_t + b*stride_b (any strides); reward [B] fp32.  Per sentence and n = 1..4, n-grams are
 * taken until the first window whose LAST token is </s> (2); <pad> before it is an ordinary token, and a row
 * without </s> contributes every window.  A hypothesis n-gram is matched while fewer equal n-grams precede it in
 * the hypothesis than the reference holds (clipped counts).
 *   NM_REWARD_BLEU: 0 without hypothesis unigrams, else min(1, exp(1 - ref_len / hyp_1grams)) *
 *     (m1 (m2+1)(m3+1)(m4+1) / (h1 (h2+1)(h3+1)(h4+1)))^(1/4), ref_len = tokens before the first </s>;
 *   NM_REWARD_GLEU: min(sum m / sum h, sum m / sum r); 0 where either denominator is 0 (the reference's assert
 *     fails there).
 * Computed in fp64, rounded to fp32 once.  T_r, T_h <= NM_REWARD_MAX_LEN, otherwise NM_E_UNSUPPORTED. */
#define NM_REWARD_BLEU 0
#define NM_REWARD_GLEU 1
#define NM_REWARD_MAX_LEN 2048
int nm_sentence_ngram_reward(const int64_t* references, int64_t ref_stride_t, int64_t ref_stride_b,
                             const int64_t* hypotheses, int64_t hyp_stride_t, int64_t hyp_stride_b, float* reward,
                             int64_t T_r, int64_t T_h, int64_t B, int mode, void* stream);
/* One draw per row of logits [rows,V] (row stride ldl >= V, or 0: every row reads the same logits) from
 * softmax(logits / temperature): tf.multinomial of get_body (decoders/autoregressive.py:463-465,492-493) as the
 * reference's RL sampling pass (trainers/rl_trainer.py:120-126) runs it.  Gumbel-max over Philox4x32-10 keyed by
 * the runtime state {seed, step} (the one nm_dropout_apply reads), with the row, loop_step (< 65536) and
 * sample_index (< 32768) in the counter: every row, loop step, sample and training step draws afresh, the same
 * arguments draw the same symbols.  Column unk_index (>= 0) is never drawn.  Then the bookkeeping of get_body:
 *   symbols[r] = finished_in[r] ? 0 : draw;  finished_out[r] = finished_in[r] | (symbols[r] == 2).
 * finished_in / finished_out (u8, may alias, may be NULL). */
int nm_sample_logits_step(const float* logits, int64_t ldl, float temperature, int64_t unk_index,
                          const uint8_t* finished_in, int64_t* symbols, uint8_t* finished_out, const int64_t* state,
                          int64_t loop_step, int64_t sample_index, int64_t rows, int64_t V, void* stream);

/* ---- K18: sentence classification and regression (csrc/classify.cu) -------------------------------------------
 * Time-major spans: sentence b, position t is row b*T + t of a [rows, D] matrix (D contiguous floats per row);
 * mask [B,T] (0/1 floats) may be NULL (every position valid).  Reductions run in a fixed order: repeat calls give
 * identical bits.
 * nm_seq_max_pool_fwd: y[b,d] = max_{t<L} (x*m + 1e-15*(1-m)), i.e. reduce_max of encoders/pooling.py:49-57 (a
 *   sentence whose valid values are all negative pools to 1e-15); relu != 0 gives max(y, 0), which is
 *   reduce_max(relu(x)) of encoders/sequence_cnn_encoder.py:125-129.  1 <= L <= T.
 * nm_seq_max_pool_bwd: TF's reduce_max gradient: dy split equally among ALL positions equal to the maximum, times
 *   the mask; with relu, zero unless the maximum is positive (ReluGrad).  Writes every row r < rows of dx
 *   (rows in [(B-1)*T + L, B*T]), zero at positions t >= L.
 * nm_seq_mean_pool_fwd/bwd: y[b,d] = sum_t x*m / (sum_t m + 1e-8) (encoders/pooling.py:60-70).
 * nm_attentive_pool_fwd: the self-attentive pooling of encoders/attentive.py:58-90 after its two dense layers:
 *   energies [B,T,R], states [B,T,D]; weights [B,T,R] = softmax over all T positions, times the mask,
 *   renormalised with +1e-8 (no renormalisation without a mask); out [B,R,D] = weights^T . states.
 *   R <= 32 and T*R <= 16384, otherwise NM_E_UNSUPPORTED.
 * nm_attentive_pool_bwd: from dout [B,R,D] (and dweights [B,T,R], may be NULL) and the forward's weights:
 *   denergies [B,T,R] and dstates [B,T,D].
 * nm_squared_error_fwd: loss[0] = mean over [B,dim] of (pred[b,i] - target[b])^2 (decoders/sequence_regressor.py:
 *   78-87); nm_squared_error_bwd: dpred = dloss[0] * 2 (pred - target) / (B*dim), dloss a device scalar. */
int nm_seq_max_pool_fwd(const float* x, const float* mask, float* y, int64_t B, int64_t L, int64_t T, int64_t D,
                        int relu, void* stream);
int nm_seq_max_pool_bwd(const float* x, const float* mask, const float* dy, float* dx, int64_t B, int64_t L,
                        int64_t T, int64_t D, int64_t rows, int relu, void* stream);
int nm_seq_mean_pool_fwd(const float* x, const float* mask, float* y, int64_t B, int64_t T, int64_t D, void* stream);
int nm_seq_mean_pool_bwd(const float* mask, const float* dy, float* dx, int64_t B, int64_t T, int64_t D,
                         void* stream);
int nm_attentive_pool_fwd(const float* energies, const float* mask, const float* states, float* weights, float* out,
                          int64_t B, int64_t T, int64_t R, int64_t D, void* stream);
int nm_attentive_pool_bwd(const float* energies, const float* mask, const float* states, const float* weights,
                          const float* dout, const float* dweights, float* denergies, float* dstates, int64_t B,
                          int64_t T, int64_t R, int64_t D, void* stream);
int nm_squared_error_fwd(const float* pred, const float* target, float* loss, int64_t B, int64_t dim, void* stream);
int nm_squared_error_bwd(const float* pred, const float* target, const float* dloss, float* dpred, int64_t B,
                         int64_t dim, void* stream);

/* ---- K19: one layer of the convolutional seq2seq encoder (encoders/facebook_conv.py, csrc/glu_conv.cu on the
 * implicit-GEMM kernels of csrc/conv_igemm.cuh: a 1 x k window over [B, 1, T, F]) ------------------------------
 * x [B,T,F], w [k,F,2F], bias [2F], fp32, row-major; M = B*T.
 *   z = conv1d(x, w) + bias       TF's SAME padding at stride 1: (k-1)/2 zeros before each sequence, the rest after;
 *                                 positions inside [0,T) always take part, padded batch positions included
 *   y = z[..., :F] * sigmoid(z[..., F:]) + x
 * Any B, T (T < k and T = 1 included), F and k.  backend: NM_GEMM_SIMT = exact fp32 on the CUDA cores,
 * NM_GEMM_AUTO / NM_GEMM_TC = wgmma with TF32 operands.  Implicit GEMMs: no patch matrix.
 * nm_glu_conv1d_fwd: y [B,T,F]; z [B,T,2F] is written only when non-NULL (training keeps it for the backward).
 * nm_glu_conv1d_dz: dz [M,2F] = the gradient of z from dy [M,F] and the saved z.
 * nm_glu_conv1d_dgrad: dx [B,T,F] = conv1d of dz with w's taps reversed and channel axes swapped, + dy (the
 * residual); dx must not alias dz or dy.
 * nm_glu_conv1d_wgrad: dw [k,F,2F] += sum over positions of patch(x)^T dz, db [2F] += sum dz.  The position sum is
 * split over CTAs into `workspace` (>= (k*F+1)*2F floats; more lets it split further) and the partials are added
 * in a fixed order: two calls give identical bits.  db is that product's row of ones, so on the wgmma engine it sums
 * dz rounded to TF32 like every other operand (2^-11 relative per term); NM_GEMM_SIMT sums it in fp32.
 * nm_glu_conv1d_wgrad_workspace: the workspace (floats) at which nm_glu_conv1d_wgrad splits as far as it wants to
 * for that shape and backend, or -1 for invalid sizes. */
int nm_glu_conv1d_fwd(const float* x, const float* w, const float* bias, float* y, float* z, int64_t B, int64_t T,
                      int64_t F, int64_t k, int backend, void* stream);
int nm_glu_conv1d_dz(const float* dy, const float* z, float* dz, int64_t M, int64_t F, void* stream);
int nm_glu_conv1d_dgrad(const float* dz, const float* w, const float* dy, float* dx, int64_t B, int64_t T, int64_t F,
                        int64_t k, int backend, void* stream);
int64_t nm_glu_conv1d_wgrad_workspace(int64_t B, int64_t T, int64_t F, int64_t k, int backend);
int nm_glu_conv1d_wgrad(const float* x, const float* dz, float* dw, float* db, float* workspace,
                        int64_t workspace_floats, int64_t B, int64_t T, int64_t F, int64_t k, int backend,
                        void* stream);

/* ---- K20: speech features ---------------------------------------------------------------------------
 * Replace python_speech_features 0.6.1's mfcc / fbank / logfbank / ssc and delta, which the reference's
 * processors/speech.py:43-62 calls once per utterance (SpeechFeaturesPreprocessor).  All arithmetic is fp64.
 * nm_speech_features: signal [samples] f64 is pre-emphasised (y[0] = x[0], y[n] = x[n] - preemph*x[n-1]), cut into
 *   `frames` frames of frame_len samples every frame_step samples (zeros past the end), each multiplied by window
 *   [frame_len] f64, truncated or zero-padded to nfft (a power of two, 2..8192); pspec = |rfft|^2 / nfft over the
 *   nfft/2+1 bins.  fbank [nfilt, nfft/2+1] f64 is the filterbank matrix; filter j reads only the bins
 *   [fb_first[j], fb_last[j]) (i32), which must hold all its nonzero entries; nfilt <= 1024.  Per frame, into the
 *   first `width` columns of row f of out (row stride out_stride):
 *     NM_SPEECH_FBANK     pspec . fbank^T, zeros replaced by DBL_EPSILON (width = nfilt);
 *     NM_SPEECH_LOGFBANK  its log;
 *     NM_SPEECH_MFCC      DCT-II (ortho) of the log, the first width = min(numcep, nfilt) coefficients, times
 *                         1 + (ceplifter/2) sin(pi n / ceplifter) when ceplifter > 0, column 0 replaced by
 *                         log(sum pspec) (zero energy -> DBL_EPSILON) when append_energy != 0;
 *     NM_SPEECH_SSC       (pspec' * R) . fbank^T / (pspec' . fbank^T) with pspec' = pspec, zeros -> DBL_EPSILON,
 *                         R = linspace(1, rate/2, nfft/2+1); an all-zero filter gives NaN (width = nfilt).
 * nm_speech_deltas: columns [(block+1)*width, (block+2)*width) of out [frames, out_stride] f64 become the deltas of
 *   columns [block*width, (block+1)*width): d[t] = sum_{n=-N..N} n x[clamp(t+n, 0, frames-1)] / (2 sum_{n=1..N} n^2),
 *   N = window (1..1024). */
#define NM_SPEECH_MFCC 0
#define NM_SPEECH_FBANK 1
#define NM_SPEECH_LOGFBANK 2
#define NM_SPEECH_SSC 3
int nm_speech_features(const double* signal, int64_t samples, const double* window, int64_t frame_len,
                       int64_t frame_step, int64_t nfft, double preemph, const double* fbank,
                       const int32_t* fb_first, const int32_t* fb_last, int64_t nfilt, int kind, int64_t numcep,
                       double ceplifter, int append_energy, double rate, double* out, int64_t frames,
                       int64_t out_stride, void* stream);
int nm_speech_deltas(double* out, int64_t frames, int64_t width, int64_t out_stride, int64_t block, int64_t window,
                     void* stream);

/* ---- K21: supervised attention: cross-entropy of attention energies against word alignments ------------------
 * Replaces the training loss of decoders/word_alignment_decoder.py:100-108, softmax_cross_entropy_with_logits over
 * the K4 energies (all Tx positions, padding included) times the decoder's training padding, summed:
 *     loss = sum_{b,q} pad[b,q] * sum_t target[b,q,t] * (lse_t energies[b,q,t] - energies[b,q,t])
 * energies, target [B,NQ,Tx], pad [B,NQ] fp32 (all device).
 * nm_alignment_xent_fwd: loss [1]; workspace holds B*NQ floats (the row losses), which one CTA sums in a fixed
 *   order: repeat calls give identical bits.
 * nm_alignment_xent_bwd: de_out [B,NQ,Tx] = grad_loss[0] * pad * (softmax_t(energies) * sum_t target - target),
 *   overwritten; grad_loss [1] is a device scalar.  de_out is what nm_bahdanau_bwd takes as de_in. */
int nm_alignment_xent_fwd(const float* energies, const float* target, const float* pad, float* loss,
                          float* workspace, int64_t B, int64_t NQ, int64_t Tx, void* stream);
int nm_alignment_xent_bwd(const float* energies, const float* target, const float* pad, const float* grad_loss,
                          float* de_out, int64_t B, int64_t NQ, int64_t Tx, void* stream);

/* ---- K22: the character-level sentence encoder (encoders/sentence_cnn_encoder.py, nn/highway.py; csrc/
 * sentence_cnn.cu on the implicit-GEMM kernels of csrc/conv_igemm.cuh: a 1 x k window over [B, 1, T, Cin]) -----
 * x [B,T,Cin], w [k,Cin,Cout], bias [Cout], fp32, row-major; M = B*T.
 *   y = act(conv1d(x, w) + bias)   tf.nn.conv1d at stride 1 with SAME padding: (k-1)/2 zeros before each sequence,
 *                                  the rest after; positions inside [0,T) always take part, padded batch positions
 *                                  included.  act is NM_ACT_NONE or NM_ACT_RELU.
 * Any B, T (T < k and T = 1 included), Cin, Cout and k.  backend: NM_GEMM_SIMT = exact fp32 on the CUDA cores,
 * NM_GEMM_AUTO / NM_GEMM_TC = wgmma with TF32 operands.  Implicit GEMMs: no patch matrix.
 * nm_conv1d_fwd: y [B,T,Cout]; bias may be NULL.
 * nm_conv1d_dgrad: dx [B,T,Cin] = conv1d of dy [B,T,Cout] (the gradient of the pre-activation) with w's taps
 *   reversed and channel axes swapped; dx must not alias dy.
 * nm_conv1d_wgrad: dw [k,Cin,Cout] += sum over positions of patch(x)^T dy, db [Cout] += sum dy (db may be NULL).
 *   The position sum is split over CTAs into `workspace` (>= (k*Cin+1)*Cout floats; more lets it split further)
 *   and the partials are added in a fixed order: two calls give identical bits.
 * nm_conv1d_wgrad_workspace: the workspace (floats) at which nm_conv1d_wgrad splits as far as it wants to for that
 *   shape and backend, or -1 for invalid sizes.
 * nm_highway_fwd: the highway gate over the n elements of the two dense products' outputs zh = x W_H + b_H and
 *   zt = x W_T + b_T and of x:  y = relu(zh) * sigmoid(zt) + x * (1 - sigmoid(zt)).
 * nm_highway_bwd: dzh = dy t [zh > 0], dzt = dy (relu(zh) - x) t (1 - t), dx = dy (1 - t) with t = sigmoid(zt):
 *   the gradients of both products' outputs and the carry term of dx.  Element by element: repeat calls give
 *   identical bits. */
int nm_conv1d_fwd(const float* x, const float* w, const float* bias, float* y, int64_t B, int64_t T, int64_t Cin,
                  int64_t Cout, int64_t k, int act, int backend, void* stream);
int nm_conv1d_dgrad(const float* dy, const float* w, float* dx, int64_t B, int64_t T, int64_t Cin, int64_t Cout,
                    int64_t k, int backend, void* stream);
int64_t nm_conv1d_wgrad_workspace(int64_t B, int64_t T, int64_t Cin, int64_t Cout, int64_t k, int backend);
int nm_conv1d_wgrad(const float* x, const float* dy, float* dw, float* db, float* workspace, int64_t workspace_floats,
                    int64_t B, int64_t T, int64_t Cin, int64_t Cout, int64_t k, int backend, void* stream);
int nm_highway_fwd(const float* zh, const float* zt, const float* x, float* y, int64_t n, void* stream);
int nm_highway_bwd(const float* dy, const float* zh, const float* zt, const float* x, float* dzh, float* dzt,
                   float* dx, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NMB200_H */
