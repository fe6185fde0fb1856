// wgmma GEMM for sm_90a: D[M,N] = op(A)[M,K] . op(B)[K,N], fp32 operands consumed as
// TF32 (or fp16 operands), fp32 accumulation in registers.
//
//   * one CTA per 128 x BN output tile (per split-K slice / batched problem);
//   * warpgroup 0 = producer, warpgroups 1 and 2 = consumers: each issues wgmma.mma_async
//     m64nBNk8 (tf32) / m64nBNk16 (fp16) for 64 of the tile's rows;
//   * STAGES-deep smem ring of {A 128 x 128 B, B BN x 128 B} K-major tiles in the 128-byte
//     swizzle.  K-major operands arrive by cp.async.bulk.tensor (OOB rows / cols as zeros);
//     wgmma takes TF32 operands K-major only, so MN-major TF32 operands (reduction dim strided)
//     are loaded by the producer warpgroup's threads and written K-major (transposed, rounded to
//     TF32) into the same layout; MN-major fp16 operands arrive by TMA as they are stored and
//     wgmma reads them transposed;
//   * after the main loop the accumulators go through shared memory (the ring is free by then)
//     and the epilogue warps read whole 32-column row chunks: one thread = one output row;
//   * epilogues: dense (bias/activation/accumulate), and the fused vocabulary
//     cross-entropy forward (online softmax partials + argmax + target logit) and
//     backward (softmax - onehot), which never materialise fp32 logits twice.
//
// Descriptor bit layouts follow the PTX ISA "Matrix Descriptor Format" of the wgmma section.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "gemm_tc.h"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace nm {

constexpr int TC_BM = 128;
constexpr int TC_BK = 32;                      // fp32 elements = 128 bytes = one swizzle row
constexpr int TC_THREADS = 384;                // producer warpgroup, two consumer warpgroups
constexpr int TC_EPI_WARPS = 8;                // the consumer warps run the epilogue
constexpr int TC_A_BYTES = TC_BM * 128;        // 16 KB
constexpr int TC_RING_BUDGET = 192 * 1024;

template <int BN>
struct TcCfg {
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES;
  static constexpr int STAGES = (TC_RING_BUDGET / STAGE_BYTES) > 4 ? 4 : (TC_RING_BUDGET / STAGE_BYTES);
  static constexpr int CT_PITCH = BN + 4;      // floats per row of the accumulator tile
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int CT_BYTES = TC_BM * CT_PITCH * 4;
  static constexpr int UNION_BYTES = RING_BYTES > CT_BYTES ? RING_BYTES : CT_BYTES;
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + UNION_BYTES + 256 /*barriers*/ +
                                    TC_EPI_WARPS * 4096 /*per-warp store staging*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "more shared memory than an sm_90 block may have");
};
// ---------------------------------------------------------------------------
// epilogue for one 32-column chunk owned by one thread (= one output row).
// The epilogue runs once per output element, so it is written for instruction count:
// 32-bit column arithmetic, bias fetched as 8 x 16-byte uniform loads, exp as one FFMA +
// one MUFU.EX2, and the rare cases (the <unk> column, the row's target column, ragged
// right edge) handled in branches only the affected chunk takes.
// ---------------------------------------------------------------------------
struct RowStats {
  float mx, sum, tgt;
  int32_t arg;
};

constexpr float TC_LOG2E = 1.4426950408889634f;

// 2^x as ONE MUFU instruction.  exp2f() wraps the same MUFU.EX2 in a range fix for results below 2^-126
// (compare, halve, square: three more issue slots per element in epilogues that run once per logit); here such
// results flush to zero, which is what they contribute to a sum of probabilities anyway.
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void load_bias32(const float* __restrict__ bias, int col0, int ncols,
                                            float (&b)[32]) {
  if (bias == nullptr) {
#pragma unroll
    for (int j = 0; j < 32; ++j) b[j] = 0.f;
    return;
  }
  if (ncols == 32 && ((reinterpret_cast<uintptr_t>(bias + col0) & 15) == 0)) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(bias + col0 + j));
      b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) b[j] = (j < ncols) ? __ldg(bias + col0 + j) : 0.f;
  }
}

__device__ __forceinline__ void store32(float* __restrict__ c, const float (&x)[32], int ncols,
                                        bool vec_ok) {
  if (vec_ok && ncols == 32) {
#pragma unroll
    for (int j = 0; j < 32; j += 4)
      *reinterpret_cast<float4*>(c + j) = make_float4(x[j], x[j + 1], x[j + 2], x[j + 3]);
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j < ncols) c[j] = x[j];
  }
}

// Coalesced store of a warp's 32x32 chunk.  The epilogue hands every thread one ROW (32 columns),
// so direct stores scatter 16-byte pieces over 32 different cache lines per instruction - the L2
// request rate, not DRAM, then bounds a kernel that writes a large C (the 1.6 GB dlogits).  Going
// through a 4 KB per-warp staging tile (XOR-swizzled float4 slots: conflict-free both ways) turns
// each store instruction into four full 128-byte row segments.
__device__ __forceinline__ void store32_coalesced(float* __restrict__ stage, float* __restrict__ C,
                                                  int64_t ldc, int64_t row_base, int col0, int64_t M,
                                                  const float (&x)[32], int lane) {
  float4* st4 = reinterpret_cast<float4*>(stage);
#pragma unroll
  for (int j = 0; j < 8; ++j)
    st4[lane * 8 + (j ^ (lane & 7))] = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
  __syncwarp();
  const int sub = lane >> 3, slot = lane & 7;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = 4 * i + sub;
    const float4 v = st4[r * 8 + (slot ^ (r & 7))];
    const int64_t grow = row_base + r;
    if (grow < M) *reinterpret_cast<float4*>(C + grow * ldc + col0 + 4 * slot) = v;
  }
  __syncwarp();
}

// mode is a compile-time constant so each kernel instance carries one epilogue only.
template <int MODE>
__device__ __forceinline__ void epilogue_chunk(const TcEpilogue& e, float (&x)[32], int64_t row,
                                               int col0, int64_t M, int N, RowStats& st,
                                               int target, float row_lse2, float row_w,
                                               bool vec_ok, float* __restrict__ stage, int lane) {
  if (col0 >= N) return;                                     // warp-uniform
  const int ncols = min(32, N - col0);
  // full, aligned chunks leave through the staging tile (all 32 lanes take part, rows >= M are
  // masked at the store); everything else keeps the per-row path
  const bool coalesced = vec_ok && ncols == 32 &&
                         (MODE == TC_EPI_XENT_BWD || (MODE == TC_EPI_DENSE && e.beta == 0.f));
  if (row >= M && !coalesced) return;
  float b[32];
  load_bias32(e.bias, col0, ncols, b);
  if (MODE == TC_EPI_DENSE) {
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] = apply_act(x[j] + b[j], e.act);
    if (coalesced) {
      store32_coalesced(stage, e.C, e.ldc, row - lane, col0, M, x, lane);
      return;
    }
    float* c = e.C + row * e.ldc + col0;
    if (e.beta != 0.f) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < ncols) x[j] += c[j];
    }
    store32(c, x, ncols, vec_ok);
    return;
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) x[j] += b[j];
  const int unk_rel = (int)e.unk_index - col0;  // rare: only the chunk holding <unk>
  if (unk_rel >= 0 && unk_rel < 32) {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j == unk_rel) x[j] += -1e9f;
  }
  if (MODE == TC_EPI_XENT_FWD) {
    if (ncols < 32) {  // ragged right edge: padding columns must not win the max
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j >= ncols) x[j] = -INFINITY;
    }
    float cmx = x[0];
#pragma unroll
    for (int j = 1; j < 32; ++j) cmx = fmaxf(cmx, x[j]);
    if (cmx > st.mx) {  // strict: earlier chunks (lower columns) keep ties
      int carg = 0;
#pragma unroll
      for (int j = 31; j >= 0; --j)
        if (x[j] == cmx) carg = j;  // lowest index among equals
      st.sum *= fast_ex2((st.mx - cmx) * TC_LOG2E);
      st.mx = cmx;
      st.arg = col0 + carg;
    }
    const float m2 = st.mx * TC_LOG2E;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;   // four chains of 8 dependent adds instead of one of 32
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      s0 += fast_ex2(fmaf(x[j], TC_LOG2E, -m2));
      s1 += fast_ex2(fmaf(x[j + 1], TC_LOG2E, -m2));
      s2 += fast_ex2(fmaf(x[j + 2], TC_LOG2E, -m2));
      s3 += fast_ex2(fmaf(x[j + 3], TC_LOG2E, -m2));
    }
    st.sum += (s0 + s1) + (s2 + s3);
    const int t_rel = target - col0;  // rare: the chunk holding this row's target
    if (t_rel >= 0 && t_rel < ncols) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j == t_rel) st.tgt = x[j];
    }
    if (e.C) store32(e.C + row * e.ldc + col0, x, ncols, vec_ok);
  } else {  // TC_EPI_XENT_BWD: (softmax - onehot) * row weight
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] = fast_ex2(fmaf(x[j], TC_LOG2E, -row_lse2)) * row_w;
    const int t_rel = target - col0;
    if (t_rel >= 0 && t_rel < ncols) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j == t_rel) x[j] -= row_w;
    }
    if (coalesced)
      store32_coalesced(stage, e.C, e.ldc, row - lane, col0, M, x, lane);
    else
      store32(e.C + row * e.ldc + col0, x, ncols, vec_ok);
  }
}

// split-K partial tile: C += x (+ bias once, from split 0); no activation.
__device__ __forceinline__ void red_add_v4(float* addr, const float4& v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

__device__ __forceinline__ void epilogue_chunk_atomic(const TcEpilogue& e, const float (&x)[32],
                                                      int64_t row, int col0, int64_t M, int N,
                                                      bool add_bias, bool vec_ok,
                                                      float* __restrict__ stage, int lane) {
  if (col0 >= N) return;                                   // warp-uniform
  const int ncols = min(32, N - col0);
  if (vec_ok && ncols == 32) {
    // same transposition as store32_coalesced: one vector reduction covers 16 bytes of a row
    // and a warp instruction four full 128-byte row segments, instead of 32 scalar atomics
    // scattered over 32 rows
    float4* st4 = reinterpret_cast<float4*>(stage);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float4 v = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
      if (add_bias && e.bias) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(e.bias + col0 + 4 * j));
        v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
      }
      st4[lane * 8 + (j ^ (lane & 7))] = v;
    }
    __syncwarp();
    const int sub = lane >> 3, slot = lane & 7;
    const int64_t row_base = row - lane;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = 4 * i + sub;
      const float4 v = st4[r * 8 + (slot ^ (r & 7))];
      const int64_t grow = row_base + r;
      if (grow < M) red_add_v4(e.C + grow * e.ldc + col0 + 4 * slot, v);
    }
    __syncwarp();
    return;
  }
  if (row >= M) return;
  float* c = e.C + row * e.ldc + col0;
#pragma unroll
  for (int j = 0; j < 32; ++j)
    if (j < ncols) {
      float v = x[j];
      if (add_bias && e.bias) v += __ldg(e.bias + col0 + j);
      atomicAdd(c + j, v);
    }
}

// ---------------------------------------------------------------------------
// epilogues of the fp16-operand instances (ESZ == 2)
// ---------------------------------------------------------------------------
// Transposed store of a warp's 32x32 chunk: lane = row, so for one column the 32 lanes write 32
// consecutive elements of the transposed matrix - a full segment without any staging.
template <typename T>
__device__ __forceinline__ void store32_transposed(T* __restrict__ ct, int64_t ldt, int64_t row, int col0,
                                                   int64_t M, int ncols, const float (&x)[32], float beta) {
  if (row >= M) return;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if (j < ncols) {
      T* dst = ct + (int64_t)(col0 + j) * ldt + row;
      if constexpr (sizeof(T) == 2) {
        *dst = __float2half_rn(x[j]);
      } else {
        *dst = (beta != 0.f) ? (x[j] + *dst) : x[j];
      }
    }
  }
}

// Row-major fp16 store of a warp's 32x32 chunk through the per-warp staging tile (32 rows x 64 B,
// 16-byte slots XOR-swizzled): every store instruction then writes eight full 64-byte row segments.
__device__ __forceinline__ void store32_half_coalesced(float* __restrict__ stage, __half* __restrict__ C,
                                                       int64_t ldc, int64_t row_base, int col0, int64_t M,
                                                       const float (&x)[32], int lane) {
  uint4* st4 = reinterpret_cast<uint4*>(stage);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    __half2 h0 = __floats2half2_rn(x[8 * j], x[8 * j + 1]), h1 = __floats2half2_rn(x[8 * j + 2], x[8 * j + 3]);
    __half2 h2 = __floats2half2_rn(x[8 * j + 4], x[8 * j + 5]), h3 = __floats2half2_rn(x[8 * j + 6], x[8 * j + 7]);
    uint4 v;
    v.x = *reinterpret_cast<uint32_t*>(&h0); v.y = *reinterpret_cast<uint32_t*>(&h1);
    v.z = *reinterpret_cast<uint32_t*>(&h2); v.w = *reinterpret_cast<uint32_t*>(&h3);
    st4[lane * 4 + (j ^ ((lane >> 1) & 3))] = v;     // rows 2q, 2q+1 share a swizzle: conflict-free both ways
  }
  __syncwarp();
  const int sub = lane >> 2, slot = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = 8 * i + sub;
    const uint4 v = st4[r * 4 + (slot ^ ((r >> 1) & 3))];
    const int64_t grow = row_base + r;
    if (grow < M) *reinterpret_cast<uint4*>(C + grow * ldc + col0 + 8 * slot) = v;
  }
  __syncwarp();
}

// TC_EPI_XENT_BWD16: (softmax - onehot) * row weight, stored as fp16 row-major and transposed.
// The row weight is the 0/1 mask here (the caller applies the upstream scale in the consumers), so
// the stored values lie in [-1, 1] and fp16 keeps TF32's 10 mantissa bits for them.
__device__ __forceinline__ void epilogue_chunk_xent_bwd16(const TcEpilogue& e, const TcExt& ext, float (&x)[32],
                                                          int64_t row, int col0, int64_t M, int N, int target,
                                                          float row_lse2, float row_w,
                                                          float* __restrict__ stage, int lane) {
  if (col0 >= N) return;                                     // warp-uniform
  const int ncols = min(32, N - col0);
  float b[32];
  load_bias32(e.bias, col0, ncols, b);
#pragma unroll
  for (int j = 0; j < 32; ++j) x[j] += b[j];
  const int unk_rel = (int)e.unk_index - col0;
  if (unk_rel >= 0 && unk_rel < 32) {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j == unk_rel) x[j] += -1e9f;
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) x[j] = fast_ex2(fmaf(x[j], TC_LOG2E, -row_lse2)) * row_w;
  const int t_rel = target - col0;
  if (t_rel >= 0 && t_rel < ncols) {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j == t_rel) x[j] -= row_w;
  }
  __half* c16 = reinterpret_cast<__half*>(ext.C16);
  const bool vec_ok = ncols == 32 && ((ext.ldc16 & 7) == 0) && ((reinterpret_cast<uintptr_t>(c16) & 15) == 0);
  if (vec_ok) {
    store32_half_coalesced(stage, c16, ext.ldc16, row - lane, col0, M, x, lane);
  } else if (row < M) {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j < ncols) c16[row * ext.ldc16 + col0 + j] = __float2half_rn(x[j]);
  }
  if (ext.C16T)
    store32_transposed(reinterpret_cast<__half*>(ext.C16T), ext.ldc16t, row, col0, M, ncols, x, 0.f);
}

// TC_EPI_DENSE of the fp16 instances: C (or C^T) = alpha * row_scale[m] * acc + bias (+ C).
__device__ __forceinline__ void epilogue_chunk_dense16(const TcEpilogue& e, const TcExt& ext, float (&x)[32],
                                                       int64_t row, int col0, int64_t M, int N, float factor,
                                                       bool vec_ok, float* __restrict__ stage, int lane,
                                                       RowStats& st) {
#pragma unroll
  for (int j = 0; j < 32; ++j) x[j] *= factor;
  if (!ext.transposed) {
    epilogue_chunk<TC_EPI_DENSE>(e, x, row, col0, M, N, st, -1, 0.f, 0.f, vec_ok, stage, lane);
    return;
  }
  if (col0 >= N) return;
  const int ncols = min(32, N - col0);
  if (e.bias) {
    float b[32];
    load_bias32(e.bias, col0, ncols, b);
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] += b[j];
  }
  store32_transposed(e.C, e.ldc, row, col0, M, ncols, x, e.beta);
}

// ---------------------------------------------------------------------------
// TC_EPI_SOFTMAX / TC_EPI_DSOFTMAX: one thread owns one query row of one (sentence, head) problem; the whole
// row of energies sits in this thread's row of the accumulator tile (N <= BN), so the row reductions need no
// exchange - the row is simply read again from shared memory for every pass.  Mask semantics of the reference
// (scaled_dot_product.py:160-206): causal positions are REPLACED by -1e9, padded keys get x*m + (1-m)*(-1e9),
// both before the softmax; dropout multiplies the softmax output (:208-214).
//
// Everything a row needs from memory - its slice of the dropout mask, of the saved softmax - and everything it
// writes goes through the warp's staging tile, 32 rows x 32 columns at a time (the inverse of
// store32_coalesced), so global memory sees full 128-byte row segments; the key mask of the sentence is copied
// once per tile into the idle partner warp's staging tile.  (The first version read and wrote per-thread rows
// element by element: 99 us per launch at the bench shape, six times the products themselves.)
__device__ __forceinline__ void load32_coalesced(float* __restrict__ stage, const float* __restrict__ src,
                                                 int64_t ld, int64_t row_base, int col0, int64_t M,
                                                 float (&x)[32], int lane) {
  float4* st4 = reinterpret_cast<float4*>(stage);
  const int sub = lane >> 3, slot = lane & 7;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = 4 * i + sub;
    const int64_t grow = row_base + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (grow < M) v = *reinterpret_cast<const float4*>(src + grow * ld + col0 + 4 * slot);
    st4[r * 8 + (slot ^ (r & 7))] = v;
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 v = st4[lane * 8 + (j ^ (lane & 7))];
    x[4 * j] = v.x; x[4 * j + 1] = v.y; x[4 * j + 2] = v.z; x[4 * j + 3] = v.w;
  }
  __syncwarp();
}

// 32 consecutive accumulators of this thread's row of the tile (16-byte aligned)
__device__ __forceinline__ void ld_row32(const float* __restrict__ p, float (&x)[32]) {
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const float4 v = *reinterpret_cast<const float4*>(p + j);
    x[j] = v.x; x[j + 1] = v.y; x[j + 2] = v.z; x[j + 3] = v.w;
  }
}

template <int MODE>
__device__ __forceinline__ void attn_epilogue(const TcEpilogue& e, const TcBatch& bt, const float* crow, int r,
                                              int M, int N, int o, int p, int64_t c_off,
                                              float* __restrict__ stage, int lane) {
  const int nchunks = bt.n_pad >> 5;                 // n_pad is a multiple of 32
  float* km_s = stage + 4 * 1024;                    // the partner warp's tile (idle in these modes)
  const bool has_km = bt.key_mask != nullptr;
  if (has_km) {
    const float* km = bt.key_mask + (int64_t)o * N;
    for (int c = lane; c < nchunks * 32; c += 32) km_s[c] = c < N ? km[c] : 1.f;
    __syncwarp();
  }
  const bool row_ok = r < M;
  const int64_t row_base = r - lane;
  float* cbase = e.C + c_off;
  const float* dbase = bt.drop ? bt.drop + (int64_t)p * M * N : nullptr;
  const bool drop_vec = dbase && (N & 3) == 0 && (reinterpret_cast<uintptr_t>(dbase) & 15) == 0;
  // this row's 32 entries of the dropout mask from column col0 (1 where there is no mask, 0 outside the matrix)
  auto load_drop = [&](int col0, float (&d)[32]) {
    if (!dbase) {
#pragma unroll
      for (int j = 0; j < 32; ++j) d[j] = 1.f;
    } else if (drop_vec && col0 + 32 <= N) {
      load32_coalesced(stage, dbase, N, row_base, col0, M, d, lane);
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) d[j] = (row_ok && col0 + j < N) ? dbase[(int64_t)r * N + col0 + j] : 0.f;
    }
  };
  // the rows this tile will read from memory (dropout mask, saved softmax): on their way into L2 while the
  // shared-memory passes run
  if (row_ok) {
    if (dbase) asm volatile("prefetch.global.L2 [%0];" ::"l"(dbase + (int64_t)r * N) : "memory");
    if (MODE == TC_EPI_DSOFTMAX) asm volatile("prefetch.global.L2 [%0];" ::"l"(bt.P + c_off + (int64_t)r * e.ldc) : "memory");
  }
  float v[32];
  if (MODE == TC_EPI_SOFTMAX) {
    // energies in units of log2: 2^(x*log2e - max) is ONE MUFU instruction (fast_ex2), the masks' -1e9 stays -1e9*log2e
    const float sc2 = bt.scale * TC_LOG2E;
    constexpr float MASKED2 = -1e9f * TC_LOG2E;
    auto energy = [&](float acc, int col) {
      float x = acc * sc2;
      if (bt.causal && col > r) x = MASKED2;
      if (has_km) {
        const float m = km_s[col];
        x = x * m + (1.f - m) * MASKED2;
      }
      return x;
    };
    float mx = -INFINITY;
    for (int c = 0; c < nchunks; ++c) {
      ld_row32(crow + c * 32, v);
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (c * 32 + j < N) mx = fmaxf(mx, energy(v[j], c * 32 + j));
    }
    float sum = 0.f;
    for (int c = 0; c < nchunks; ++c) {
      ld_row32(crow + c * 32, v);
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (c * 32 + j < N) sum += fast_ex2(energy(v[j], c * 32 + j) - mx);
    }
    const float inv = 1.f / sum;
    for (int c = 0; c < nchunks; ++c) {
      ld_row32(crow + c * 32, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = c * 32 + j;
        v[j] = (row_ok && col < N) ? fast_ex2(energy(v[j], col) - mx) * inv : 0.f;
      }
      store32_coalesced(stage, cbase, e.ldc, row_base, c * 32, bt.m_pad, v, lane);   // padding rows: zeros
      if (bt.C2) {
        float d[32];
        load_drop(c * 32, d);
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] *= d[j];
        store32_coalesced(stage, bt.C2 + c_off, e.ldc, row_base, c * 32, bt.m_pad, v, lane);
      }
    }
  } else {   // TC_EPI_DSOFTMAX: acc = d(dropped weights)
    const float* pbase = bt.P + c_off;
    float pr[32], d[32];
    float dot = 0.f;
    for (int c = 0; c < nchunks; ++c) {
      ld_row32(crow + c * 32, v);
      load32_coalesced(stage, pbase, e.ldc, row_base, c * 32, M, pr, lane);   // zero beyond the rows / columns
      load_drop(c * 32, d);
#pragma unroll
      for (int j = 0; j < 32; ++j) dot = fmaf(v[j] * d[j], pr[j], dot);
    }
    for (int c = 0; c < nchunks; ++c) {
      ld_row32(crow + c * 32, v);
      load32_coalesced(stage, pbase, e.ldc, row_base, c * 32, M, pr, lane);
      load_drop(c * 32, d);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int col = c * 32 + j;
        float g = pr[j] * (v[j] * d[j] - dot);             // pr = 0 in the padding: g = 0 there
        if (has_km) g *= km_s[col];                         // d(x*m + c)/dx = m
        if (bt.causal && col > r) g = 0.f;                  // tf.where: no gradient into replaced entries
        v[j] = row_ok ? g * bt.scale : 0.f;
      }
      store32_coalesced(stage, cbase, e.ldc, row_base, c * 32, bt.m_pad, v, lane);
    }
  }
}

// An MN-major operand (reduction dimension strided) as the kernel reads it: [rows, cols] stored with row pitch ld
// (elements), rows = K, cols = M or N.  Elements outside [rows, cols] read as zeros, as TMA would fill them.
struct TcOperand {
  const void* ptr;
  int64_t rows, cols, ld;
};

// One k-block of an MN-major operand: R MN rows x 128 bytes of K, written K-major into the 128-byte swizzle
// (16-byte chunk c of row m at chunk c ^ (m & 7)).  An item is one 32-bit word of a row (one tf32 or two fp16
// k values); a warp covers 8 rows x 4 words, so the shared-memory stores hit 32 different banks and the loads of
// one k row are 8 consecutive MN elements.  Called by the 128 threads of the producer warpgroup.
template <int ESZ, int R>
__device__ __forceinline__ void load_mn_tile(uint8_t* __restrict__ dst, const TcOperand& op, int64_t k_row0,
                                             int64_t mn0, int tid) {
  constexpr int PER = R * 32 / 128;
#pragma unroll 8
  for (int j = 0; j < PER; ++j) {
    const int it = tid + 128 * j;
    const int b = it & 3, a = (it >> 2) & 7, rest = it >> 5;
    const int m = (rest % (R / 8)) * 8 + a;
    const int word = (rest / (R / 8)) * 4 + b;
    const int64_t col = mn0 + m;
    const bool col_ok = col < op.cols;
    uint32_t packed;
    if constexpr (ESZ == 4) {
      const int64_t r = k_row0 + word;
      const float* f = reinterpret_cast<const float*>(op.ptr);
      packed = to_tf32((col_ok && r < op.rows) ? __ldg(f + r * op.ld + col) : 0.f);
    } else {
      const int64_t r = k_row0 + 2 * word;
      const __half* h = reinterpret_cast<const __half*>(op.ptr);
      const __half zero = __float2half_rn(0.f);
      const __half lo = (col_ok && r < op.rows) ? h[r * op.ld + col] : zero;
      const __half hi = (col_ok && r + 1 < op.rows) ? h[(r + 1) * op.ld + col] : zero;
      const __half2 v = __halves2half2(lo, hi);
      packed = *reinterpret_cast<const uint32_t*>(&v);
    }
    *reinterpret_cast<uint32_t*>(dst + m * 128 + (((word >> 2) ^ (m & 7)) << 4) + ((word & 3) << 2)) = packed;
  }
}

// ESZ = operand element size: 4 = fp32 consumed as TF32, 2 = fp16.  A k-block is 128 bytes of K either way
// (32 or 64 elements) and one instruction consumes 32 of them, so the smem ring and the descriptors are the same.
// PAIR: a cluster of two CTAs computes a 256 x BN tile (128 rows each) and shares its B tile: each CTA loads half
// of every B k-block with a multicast TMA that lands in both CTAs, so a pair pulls B through L2 once instead of
// twice.  A stage is refilled only when the consumers of BOTH CTAs have released it (their empty barriers count
// the peer's warps too).  B must be K-major (TMA-loaded).
template <int BN, bool A_MN, bool B_MN, int MODE, int ESZ = 4, bool PAIR = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               TcOperand opa, TcOperand opb, int64_t M, int64_t N, int64_t K, TcEpilogue epi, int splits,
               int kb_per_split, TcExt ext, TcBatch bt) {
  static_assert(ESZ == 2 || MODE != TC_EPI_XENT_BWD16, "the fp16 epilogue belongs to the fp16 instances");
  static_assert(!PAIR || (!B_MN && BN % 16 == 0), "a pair multicasts whole 8-row swizzle atoms of a TMA-loaded B");
  constexpr int BK = 128 / ESZ;                // elements per 128-byte k-block
  constexpr bool MN16 = ESZ == 2 && A_MN && B_MN;   // fp16, both MN-major: TMA boxes, transposed wgmma operands
  constexpr bool A_MANUAL = A_MN && !MN16, B_MANUAL = B_MN && !MN16;
  constexpr bool MANUAL = A_MANUAL || B_MANUAL;      // the producer threads write (some of) the tiles
  using Cfg = TcCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SW128 tiles: 1 KB aligned
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_base + Cfg::UNION_BYTES;
  // barrier layout (8 B each): full[STAGES] | empty[STAGES]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int TILE_M = PAIR ? 2 * TC_BM : TC_BM;
  const uint32_t cta_rank = PAIR ? cluster_ctarank() : 0u;
  const int64_t tiles_m = (M + TILE_M - 1) / TILE_M;
  const int64_t tiles_n = (N + BN - 1) / BN;
  // split-K: the reduction is cut into `splits` slices, each an independent work item whose
  // epilogue adds its partial tile into C with red.global.add (weight-gradient products
  // have tiny outputs and very long K: without this only a handful of SMs would work)
  // batched: bt.count independent problems of this M x N x K, each a window of the operand tensors (no split-K)
  const bool batched = bt.count > 0;
  const int64_t tiles_per = tiles_m * tiles_n;
  const int64_t tile = PAIR ? (int64_t)(blockIdx.x >> 1) : (int64_t)blockIdx.x;
  const int64_t tm = tile % tiles_m, tn = (tile / tiles_m) % tiles_n;
  const int num_kb_total = (int)((K + BK - 1) / BK);  // host guarantees no empty split
  const int split = batched ? 0 : (int)(tile / tiles_per);
  const int kb_begin = batched ? 0 : split * kb_per_split;
  const int num_kb = batched ? num_kb_total : min(num_kb_total, kb_begin + kb_per_split) - kb_begin;
  int prob = 0, prob_o = 0;
  int32_t a_row = 0, a_col = 0, b_row = 0, b_col = 0;   // this problem's operand windows
  if (batched) {
    prob = (int)(tile / tiles_per);
    prob_o = prob / bt.inner;
    const int i = prob - prob_o * bt.inner;
    a_row = prob_o * bt.a_row_outer + i * bt.a_row_inner;
    a_col = i * bt.a_col_inner;
    b_row = prob_o * bt.b_row_outer + i * bt.b_row_inner;
    b_col = i * bt.b_col_inner;
  }
  const int32_t m0 = (int32_t)(tm * TILE_M) + (int32_t)cta_rank * TC_BM, n0 = (int32_t)(tn * BN);

  if (threadIdx.x == 0) {
    if (!A_MANUAL) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
    if (!B_MANUAL) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b)) : "memory");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), MANUAL ? 128 : 1);
      mbar_init(empty_bar(s), TC_EPI_WARPS * (PAIR ? 2 : 1));   // one arrive per consumer warp (of both CTAs)
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if constexpr (PAIR) cluster_sync_all();   // the peer's barriers exist before anything arrives on them
  // Programmatic dependent launch (NMB200_TC_PDL): the barrier set-up above touches no global memory and may run
  // while the previous kernel of the stream drains; from here on its results are needed.  Without the launch
  // attribute both instructions do nothing.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");

  if (warp < 4) {
    // ===================== producer warpgroup =====================
    const int ptid = threadIdx.x;
    for (int kb = 0; kb < num_kb && (MANUAL || ptid == 0); ++kb) {
      const int s = kb % STAGES;
      const uint32_t phase = (uint32_t)((kb / STAGES) & 1);
      if constexpr (PAIR) mbar_wait_cluster(empty_bar(s), phase ^ 1u);   // the peer's releases are cluster-scope
      else mbar_wait(empty_bar(s), phase ^ 1u);
      const uint32_t a_dst = smem_base + s * Cfg::STAGE_BYTES;
      const uint32_t b_dst = a_dst + TC_A_BYTES;
      const int32_t k0 = (kb_begin + kb) * BK;
      if (ptid == 0) {
        constexpr uint32_t TX = (A_MANUAL ? 0u : (uint32_t)TC_A_BYTES) + (B_MANUAL ? 0u : (uint32_t)Cfg::B_BYTES);
        if (TX) mbar_expect_tx_only(full_bar(s), TX);
        if constexpr (MN16) {   // boxes {64 MN elements, one k-block of rows}, 8 KB each
#pragma unroll
          for (int j = 0; j < TC_BM / 64; ++j)
            tma_load_2d(a_dst + j * 8192, &map_a, full_bar(s), m0 + a_col + 64 * j, k0 + a_row);
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_2d(b_dst + j * 8192, &map_b, full_bar(s), n0 + b_col + 64 * j, k0 + b_row);
        } else if (!A_MN) {
          tma_load_2d(a_dst, &map_a, full_bar(s), k0 + a_col, m0 + a_row);  // box {one k-block, 128 rows}
        }
        if constexpr (PAIR) {   // this CTA's half of the B tile, into both CTAs
          tma_load_2d_multicast(b_dst + cta_rank * (Cfg::B_BYTES / 2), &map_b, full_bar(s), k0 + b_col,
                                n0 + b_row + (int32_t)cta_rank * (BN / 2), (uint16_t)3);
        } else if (!B_MN) {   // (MN16 loaded it above)
          tma_load_2d(b_dst, &map_b, full_bar(s), k0 + b_col, n0 + b_row);  // box {one k-block, BN rows}
        }
      }
      uint8_t* ring = smem + s * Cfg::STAGE_BYTES;
      if constexpr (A_MANUAL) load_mn_tile<ESZ, TC_BM>(ring, opa, k0 + a_row, m0 + a_col, ptid);
      if constexpr (B_MANUAL) load_mn_tile<ESZ, BN>(ring + TC_A_BYTES, opb, k0 + b_row, n0 + b_col, ptid);
      // the generic-proxy stores above become visible to wgmma (async proxy) before the arrive
      if constexpr (MANUAL) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_arrive(full_bar(s));
    }
  } else {
  // ===================== consumer warpgroups: main loop =====================
  const int wg = (warp >> 2) - 1;              // rows [64*wg, 64*wg + 64) of the tile
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int prev_s = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(full_bar(s), (uint32_t)((kb / STAGES) & 1));
    const uint32_t a_addr = smem_base + s * Cfg::STAGE_BYTES + wg * 64 * 128;   // K-major: 64 rows; MN16: one box
    const uint32_t b_addr = smem_base + s * Cfg::STAGE_BYTES + TC_A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if constexpr (MN16)
        Wgmma<BN, 2, true>::mma(acc, gmma_desc_sw128_mn(a_addr + k * 2048), gmma_desc_sw128_mn(b_addr + k * 2048));
      else
        Wgmma<BN, ESZ>::mma(acc, gmma_desc_sw128(a_addr + k * 32), gmma_desc_sw128(b_addr + k * 32));
    }
    wgmma_commit();
    wgmma_wait<1>();                           // the previous k-block's products are done with their stage
    wgmma_fence_operands(acc);
    if (prev_s >= 0 && lane == 0) {
      mbar_arrive(empty_bar(prev_s));
      if constexpr (PAIR) mbar_arrive_cluster(mapa_u32(empty_bar(prev_s), cta_rank ^ 1u));   // the peer refills it too
    }
    prev_s = s;
  }
  wgmma_wait<0>();
  wgmma_fence_operands(acc);

  // ===================== accumulators -> shared memory =====================
  // the ring is free once both consumer warpgroups are past their last product
  asm volatile("bar.sync 1, 256;" ::: "memory");
  float* ctile = reinterpret_cast<float*>(smem);
  {
    const int wt = threadIdx.x & 127;
    const int r0 = wg * 64 + (wt >> 5) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      *reinterpret_cast<float2*>(ctile + r0 * Cfg::CT_PITCH + 8 * i + c0) = make_float2(acc[4 * i], acc[4 * i + 1]);
      *reinterpret_cast<float2*>(ctile + (r0 + 8) * Cfg::CT_PITCH + 8 * i + c0) =
          make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");

  // ===================== epilogue warps =====================
  // Two warps per 32-row quadrant; the pair splits the tile's 32-column chunks (even / odd).
  const int ew = warp - 4;
  const int quad = ew & 3;                     // rows [32*quad, 32*quad+32)
  const int half = ew >> 2;                    // 0: even chunks, 1: odd chunks
  const bool vec_ok = ((epi.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(epi.C) & 15) == 0);
  float* stage = reinterpret_cast<float*>(smem + Cfg::UNION_BYTES + 256) + ew * 1024;   // per-warp staging tile
  const int n32 = (int)N;
  const int64_t row = m0 + quad * 32 + lane;
  const float* crow = ctile + (quad * 32 + lane) * Cfg::CT_PITCH;
  int64_t c_off = 0;   // batched: this problem's output window
  if (batched)
    c_off = (int64_t)prob_o * bt.c_outer + (int64_t)(prob - prob_o * bt.inner) * bt.c_inner;
  RowStats st{-INFINITY, 0.f, -INFINITY, 0x7fffffff};
  int target = -1;
  float row_lse2 = 0.f, row_w = 0.f;
  if (MODE != TC_EPI_DENSE && row < M) {
    if (epi.targets) target = (int)epi.targets[row];
    if (MODE == TC_EPI_XENT_BWD) {
      row_lse2 = epi.lse[row] * TC_LOG2E;
      row_w = (epi.weights ? epi.weights[row] : 1.f) * epi.scale[0];
    }
    if (MODE == TC_EPI_XENT_BWD16) {
      row_lse2 = epi.lse[row] * TC_LOG2E;
      row_w = epi.weights ? epi.weights[row] : 1.f;
    }
  }
  float factor16 = 1.f;
  if (ESZ == 2 && MODE == TC_EPI_DENSE) {
    if (ext.alpha) factor16 = ext.alpha[0];
    if (ext.row_scale && row < M) factor16 *= ext.row_scale[row];
  }
  if constexpr (MODE == TC_EPI_SOFTMAX || MODE == TC_EPI_DSOFTMAX) {
    // whole rows per thread: the first warp of each quadrant does the tile (a handful of columns)
    if (half == 0) attn_epilogue<MODE>(epi, bt, crow, (int)row, (int)M, n32, prob_o, prob, c_off, stage, lane);
  } else {
    TcEpilogue epi_p = epi;               // this problem's window of C
    if (batched) epi_p.C += c_off;
    const TcEpilogue& epi = epi_p;
#pragma unroll 1
    for (int c = half; c < BN / 32; c += 2) {
      float v[32];
      ld_row32(crow + c * 32, v);
      if constexpr (MODE == TC_EPI_XENT_BWD16) {
        epilogue_chunk_xent_bwd16(epi, ext, v, row, (int)(tn * BN) + c * 32, M, n32, target, row_lse2,
                                  row_w, stage, lane);
      } else if constexpr (ESZ == 2 && MODE == TC_EPI_DENSE) {
        epilogue_chunk_dense16(epi, ext, v, row, (int)(tn * BN) + c * 32, M, n32, factor16, vec_ok,
                               stage, lane, st);
      } else {
        if (MODE == TC_EPI_DENSE && splits > 1)
          epilogue_chunk_atomic(epi, v, row, (int)(tn * BN) + c * 32, M, n32, split == 0,
                                vec_ok && ((reinterpret_cast<uintptr_t>(epi.bias) & 15) == 0), stage, lane);
        else
          epilogue_chunk<MODE>(epi, v, row, (int)(tn * BN) + c * 32, M, n32, st, target, row_lse2,
                               row_w, vec_ok, stage, lane);
      }
    }
  }
  if (MODE == TC_EPI_XENT_FWD && row < M)
    epi.part[(row * tiles_n + tn) * 2 + half] = make_float4(st.mx, st.sum, __int_as_float(st.arg), st.tgt);
  }
  // a pair: neither CTA leaves while the other may still arrive on its barriers
  if constexpr (PAIR) cluster_sync_all();
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D fp32 tensor [rows, cols] with row pitch ld (elements), K-major operand tile: box = {one k-block, box_rows},
// 128-byte swizzle; the TMA unit rounds the fp32 values to TF32 on the way.
static int make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t cols, int64_t ld, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  NM_REQUIRE(fn != nullptr, NM_E_NO_DEVICE, "tc_gemm: cuTensorMapEncodeTiled not available");
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)TC_BK, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  NM_REQUIRE(r == CUDA_SUCCESS, NM_E_INVALID,
             "tc_gemm: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", (int)r,
             (long long)rows, (long long)cols, (long long)ld);
  return NM_OK;
}

static int make_map16(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld,
                      uint32_t box_rows);

// One operand: a tensor map when it is K-major, the plain description the producer threads read otherwise.
static int make_operand(CUtensorMap* map, TcOperand* op, bool mn_major, const void* base, int64_t rows, int64_t cols,
                        int64_t ld, uint32_t box_rows, int esz) {
  memset(map, 0, sizeof(*map));
  *op = TcOperand{base, rows, cols, ld};
  if (mn_major) return NM_OK;
  if (esz == 4) return make_map(map, reinterpret_cast<const float*>(base), rows, cols, ld, box_rows);
  return make_map16(map, base, rows, cols, ld, box_rows);
}

bool tc_gemm_supported(int transA, int transB, int64_t M, int64_t N, int64_t K, int64_t lda,
                       int64_t ldb, int64_t ldc, const void* A, const void* B, const void* C) {
  (void)transA; (void)transB; (void)ldc; (void)C;
  if (M < 1 || N < 1 || K < 1) return false;
  if ((lda & 3) || (ldb & 3)) return false;  // TMA global strides are multiples of 16 bytes
  if (A && (reinterpret_cast<uintptr_t>(A) & 15)) return false;
  if (B && (reinterpret_cast<uintptr_t>(B) & 15)) return false;
  if (M > 0x7fffffffLL || N > 0x7fffffffLL || K > 0x7fffffffLL) return false;
  return true;
}

// NMB200_TC_PDL=1: launch with programmatic stream serialization, so that a kernel's prologue overlaps the tail of
// its predecessor (the kernel waits with griddepcontrol.wait before it touches global memory)
static bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("NMB200_TC_PDL");
    return e && atoi(e) != 0;
  }();
  return on;
}

// one CTA per work item (tile x split-K slice, or tile x batched problem); PAIR: a cluster of two CTAs per
// 256-row work item
template <int BN, bool A_MN, bool B_MN, int MODE, int ESZ, bool PAIR = false>
static int launch_tiles(const CUtensorMap& ma, const CUtensorMap& mb, const TcOperand& oa, const TcOperand& ob,
                        int64_t M, int64_t N, int64_t K, const TcEpilogue& epi, int splits, int kb_per_split,
                        const TcExt& ext, const TcBatch& bt, cudaStream_t s, const char* name) {
  using Cfg = TcCfg<BN>;
  auto kern = tc_gemm_kernel<BN, A_MN, B_MN, MODE, ESZ, PAIR>;
  static bool attr_done = false;
  if (!attr_done) {
    NM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_done = true;
  }
  const int64_t items = ceil_div(M, PAIR ? 2 * TC_BM : TC_BM) * ceil_div(N, BN) * (bt.count > 0 ? bt.count : splits);
  NM_REQUIRE(items <= (PAIR ? 0x3fffffffLL : 0x7fffffffLL), NM_E_INVALID, "%s: %lld tiles", name, (long long)items);
  if (kb_per_split <= 0) kb_per_split = (int)ceil_div(K, 128 / ESZ);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(PAIR ? 2 * items : items));
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = (size_t)Cfg::SMEM_BYTES;
  cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int nattr = 0;
  if (PAIR) {
    attr[nattr].id = cudaLaunchAttributeClusterDimension;
    attr[nattr].val.clusterDim.x = 2;
    attr[nattr].val.clusterDim.y = 1;
    attr[nattr].val.clusterDim.z = 1;
    ++nattr;
  }
  if (pdl_enabled()) {
    attr[nattr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[nattr].val.programmaticStreamSerializationAllowed = 1;
    ++nattr;
  }
  cfg.attrs = attr;
  cfg.numAttrs = nattr;
  NM_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, ma, mb, oa, ob, M, N, K, epi, splits, kb_per_split, ext, bt));
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

template <int BN, bool A_MN, bool B_MN, int MODE, bool PAIR = false>
static int launch_cfg(const CUtensorMap& ma, const CUtensorMap& mb, const TcOperand& oa, const TcOperand& ob,
                      int64_t M, int64_t N, int64_t K, const TcEpilogue& epi, cudaStream_t s, int splits = 1,
                      int kb_per_split = 0) {
  return launch_tiles<BN, A_MN, B_MN, MODE, 4, PAIR>(ma, mb, oa, ob, M, N, K, epi, splits, kb_per_split, TcExt{},
                                               TcBatch{}, s, "tc_gemm_kernel");
}

// fp16 operands: no split-K.  MN = both operands MN-major (the reduction dimension strided: X^T . dY products),
// otherwise both K-major.
template <int BN, int MODE, bool MN = false, bool PAIR = false>
static int launch_cfg16(const CUtensorMap& ma, const CUtensorMap& mb, const TcOperand& oa, const TcOperand& ob,
                        int64_t M, int64_t N, int64_t K, const TcEpilogue& epi, const TcExt& ext, cudaStream_t s) {
  return launch_tiles<BN, MN, MN, MODE, 2, PAIR>(ma, mb, oa, ob, M, N, K, epi, 1, 0, ext, TcBatch{}, s,
                                           "tc_gemm_kernel(fp16)");
}

// 2-D fp16 tensor [rows, cols] with row pitch ld (elements), K-major operand tile: box = {64 elements of K,
// box_rows}, 128-byte swizzle.
static int make_map16(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld,
                      uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  NM_REQUIRE(fn != nullptr, NM_E_NO_DEVICE, "tc_gemm16: cuTensorMapEncodeTiled not available");
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {64, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstride, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  NM_REQUIRE(r == CUDA_SUCCESS, NM_E_INVALID,
             "tc_gemm16: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld", (int)r,
             (long long)rows, (long long)cols, (long long)ld);
  return NM_OK;
}

template <int BN, bool A_MN, bool B_MN, int MODE>
static int launch_batched(const CUtensorMap& ma, const CUtensorMap& mb, const TcOperand& oa, const TcOperand& ob,
                          int64_t M, int64_t N, int64_t K, const TcEpilogue& epi, const TcBatch& bt, cudaStream_t s) {
  return launch_tiles<BN, A_MN, B_MN, MODE, 4>(ma, mb, oa, ob, M, N, K, epi, 1, 0, TcExt{}, bt, s,
                                               "tc_gemm_kernel(batched)");
}

int tc_gemm_batched_launch(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A, int64_t a_rows,
                           int64_t a_cols, int64_t lda, const float* B, int64_t b_rows, int64_t b_cols,
                           int64_t ldb, const TcEpilogue& epi, const TcBatch& bt, cudaStream_t s) {
  const bool a_mn = transA != 0, b_mn = transB == 0;
  NM_REQUIRE(bt.count >= 1 && bt.inner >= 1 && bt.count % bt.inner == 0, NM_E_INVALID,
             "tc_gemm_batched: %d problems do not split into groups of %d", bt.count, bt.inner);
  NM_REQUIRE(M >= 1 && N >= 1 && K >= 1 && (lda & 3) == 0 && (ldb & 3) == 0 &&
                 (reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
             NM_E_INVALID, "tc_gemm_batched: operands must be 16-byte aligned with 16-byte row pitches");
  const bool attn = epi.mode == TC_EPI_SOFTMAX || epi.mode == TC_EPI_DSOFTMAX;
  NM_REQUIRE(attn || epi.mode == TC_EPI_DENSE, NM_E_INVALID, "tc_gemm_batched: unsupported epilogue %d", epi.mode);
  NM_REQUIRE(((bt.c_outer | bt.c_inner | epi.ldc) & 3) == 0 && (reinterpret_cast<uintptr_t>(epi.C) & 15) == 0,
             NM_E_INVALID, "tc_gemm_batched: output windows must be 16-byte aligned");
  const int bn = attn ? 128 : (N <= 64 ? 64 : 128);
  NM_REQUIRE(!attn || (N <= 128 && bt.n_pad >= N && bt.n_pad <= 128 && bt.m_pad >= M && !a_mn && !b_mn),
             NM_E_UNSUPPORTED, "tc_gemm_batched: attention epilogues take K-major operands and N <= 128 (N=%lld)",
             (long long)N);
  CUtensorMap ma, mb;
  TcOperand oa, ob;
  int rc = make_operand(&ma, &oa, a_mn, A, a_rows, a_cols, lda, TC_BM, 4);
  if (rc) return rc;
  rc = make_operand(&mb, &ob, b_mn, B, b_rows, b_cols, ldb, (uint32_t)bn, 4);
  if (rc) return rc;
  if (epi.mode == TC_EPI_SOFTMAX)
    return launch_batched<128, false, false, TC_EPI_SOFTMAX>(ma, mb, oa, ob, M, N, K, epi, bt, s);
  if (epi.mode == TC_EPI_DSOFTMAX)
    return launch_batched<128, false, false, TC_EPI_DSOFTMAX>(ma, mb, oa, ob, M, N, K, epi, bt, s);
  NM_REQUIRE(b_mn, NM_E_UNSUPPORTED, "tc_gemm_batched: dense products take an MN-major B operand");
  if (bn == 64) {
    if (a_mn) return launch_batched<64, true, true, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, bt, s);
    return launch_batched<64, false, true, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, bt, s);
  }
  if (a_mn) return launch_batched<128, true, true, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, bt, s);
  return launch_batched<128, false, true, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, bt, s);
}

// CTA pairs (tc_gemm_set_pair_mode): 0 = never, 1 = wherever the shape allows, -1 = the library's policy, which
// is one CTA per tile (pairs are not measured to be faster on any product of the workloads).  NMB200_TC_PAIR
// presets the mode.
static int g_pair_override = -2;   // -2 = not set
static int pair_mode() {
  static const int mode = [] {
    const char* e = getenv("NMB200_TC_PAIR");
    return (e && *e) ? atoi(e) : -1;
  }();
  return g_pair_override != -2 ? g_pair_override : mode;
}
int tc_gemm_set_pair_mode(int mode) {
  const int before = pair_mode();
  g_pair_override = mode;
  return before;
}
// a pair shares a TMA-loaded (K-major) B tile of 128 or 256 columns between two 128-row halves
static bool pair_wanted(int64_t M, int bn, bool b_tma) {
  return pair_mode() == 1 && b_tma && (bn == 128 || bn == 256) && M > TC_BM;
}

static int pick_bn(int64_t M, int64_t N, int64_t K) {
  static const int forced = [] {   // NMB200_TC_BN={64,128,160,256}: tile-width experiments (tools/gemm_sweep.py)
    const char* e = getenv("NMB200_TC_BN");
    const int v = e ? atoi(e) : 0;
    return (v == 64 || v == 128 || v == 160 || v == 256) ? v : 0;
  }();
  if (forced) return forced;
  if (N <= 64) return 64;
  if (N <= 128) return 128;
  // skinny output, very long reduction (dX of the vocabulary projection: 12800 x 300 x 32000):
  // the A stream dominates and is re-read once per N tile, so cover N with the fewest equal tiles
  if (K >= 8192 && N > 256 && N <= 320) return 160;
  const int64_t pad128 = ceil_div(N, 128) * 128, pad256 = ceil_div(N, 256) * 256;
  const int64_t tiles256 = ceil_div(M, TC_BM) * ceil_div(N, 256);
  if (pad256 == pad128 && tiles256 >= sm_count()) return 256;
  if (pad256 * 10 <= pad128 * 11 && tiles256 >= 2 * (int64_t)sm_count()) return 256;
  return 128;
}

int tc_gemm_launch(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A,
                   int64_t lda, const float* B, int64_t ldb, const TcEpilogue& epi, cudaStream_t s) {
  // op(A) is [M,K]: transA=0 -> A stored [M,K], K contiguous (K-major);
  //                 transA=1 -> A stored [K,M], M contiguous (MN-major).
  // op(B) is [K,N]: transB=0 -> B stored [K,N], N contiguous (MN-major);
  //                 transB=1 -> B stored [N,K], K contiguous (K-major).
  const bool a_mn = transA != 0, b_mn = transB == 0;
  const int bn = (epi.mode == TC_EPI_DENSE) ? pick_bn(M, N, K) : TC_XENT_BN;
  // split-K when the output alone cannot occupy the chip (and nothing forbids partial sums)
  int splits = 1;
  int kb_per = (int)ceil_div(K, TC_BK);
  if (epi.mode == TC_EPI_DENSE) {
    const int64_t tiles = ceil_div(M, TC_BM) * ceil_div(N, bn);
    const int64_t num_kb = ceil_div(K, TC_BK);
    if (epi.act == NM_ACT_NONE && tiles * 2 <= sm_count() && num_kb >= 16) {
      int64_t want = ceil_div(sm_count(), tiles);
      if (want > num_kb / 8) want = num_kb / 8;
      if (want > 1) {
        kb_per = (int)ceil_div(num_kb, want);
        splits = (int)ceil_div(num_kb, kb_per);  // every split owns >= 1 k-block
      }
    } else if (epi.act == NM_ACT_NONE && num_kb >= 256 && tiles < 4 * (int64_t)sm_count()) {
      // a few waves of very long tiles: the last, partly filled wave costs a whole tile time.
      // Cut K so that the work items fill the waves (static round-robin: ceil(items/SMs) rounds).
      int best = 1;
      double best_cost = (double)ceil_div(tiles, sm_count());
      for (int sp = 2; sp <= 8; ++sp) {
        if (num_kb / sp < 64) break;
        const double cost = (double)ceil_div(tiles * sp, sm_count()) / sp;
        if (cost < best_cost * 0.93) { best_cost = cost; best = sp; }
      }
      if (best > 1) {
        kb_per = (int)ceil_div(num_kb, best);
        splits = (int)ceil_div(num_kb, kb_per);
      }
    }
  }
  CUtensorMap ma, mb;
  TcOperand oa, ob;
  int rc = a_mn ? make_operand(&ma, &oa, true, A, K, M, lda, TC_BM, 4) : make_operand(&ma, &oa, false, A, M, K, lda, TC_BM, 4);
  if (rc) return rc;
  const bool pair = pair_wanted(M, bn, !b_mn);
  rc = b_mn ? make_operand(&mb, &ob, true, B, K, N, ldb, (uint32_t)bn, 4)
            : make_operand(&mb, &ob, false, B, N, K, ldb, (uint32_t)(pair ? bn / 2 : bn), 4);
  if (rc) return rc;
  if (splits > 1 && epi.beta == 0.f)  // partial sums are added: start from zero
    NM_CUDA_TRY(cudaMemset2DAsync(epi.C, sizeof(float) * epi.ldc, 0, sizeof(float) * N, M, s));
#define NM_TC_DISPATCH(BN_, MODE_)                                                                               \
  do {                                                                                                           \
    if (!a_mn && !b_mn) return launch_cfg<BN_, false, false, MODE_>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per); \
    if (!a_mn && b_mn) return launch_cfg<BN_, false, true, MODE_>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per);   \
    if (a_mn && !b_mn) return launch_cfg<BN_, true, false, MODE_>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per);   \
    return launch_cfg<BN_, true, true, MODE_>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per);                       \
  } while (0)
  if (pair) {   // B K-major
    if (epi.mode == TC_EPI_XENT_FWD) return launch_cfg<256, false, false, TC_EPI_XENT_FWD, true>(ma, mb, oa, ob, M, N, K, epi, s);
    if (epi.mode == TC_EPI_XENT_BWD) return launch_cfg<256, false, false, TC_EPI_XENT_BWD, true>(ma, mb, oa, ob, M, N, K, epi, s);
    if (bn == 128) {
      if (a_mn) return launch_cfg<128, true, false, TC_EPI_DENSE, true>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per);
      return launch_cfg<128, false, false, TC_EPI_DENSE, true>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per);
    }
    if (a_mn) return launch_cfg<256, true, false, TC_EPI_DENSE, true>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per);
    return launch_cfg<256, false, false, TC_EPI_DENSE, true>(ma, mb, oa, ob, M, N, K, epi, s, splits, kb_per);
  }
  if (epi.mode == TC_EPI_XENT_FWD) {  // A is always K-major for the vocabulary projection
    if (b_mn) return launch_cfg<256, false, true, TC_EPI_XENT_FWD>(ma, mb, oa, ob, M, N, K, epi, s);
    return launch_cfg<256, false, false, TC_EPI_XENT_FWD>(ma, mb, oa, ob, M, N, K, epi, s);
  }
  if (epi.mode == TC_EPI_XENT_BWD) {
    if (b_mn) return launch_cfg<256, false, true, TC_EPI_XENT_BWD>(ma, mb, oa, ob, M, N, K, epi, s);
    return launch_cfg<256, false, false, TC_EPI_XENT_BWD>(ma, mb, oa, ob, M, N, K, epi, s);
  }
  if (bn == 64) NM_TC_DISPATCH(64, TC_EPI_DENSE);
  if (bn == 128) NM_TC_DISPATCH(128, TC_EPI_DENSE);
  if (bn == 160) NM_TC_DISPATCH(160, TC_EPI_DENSE);
  NM_TC_DISPATCH(256, TC_EPI_DENSE);
#undef NM_TC_DISPATCH
}

int tc_gemm16_mn_launch(int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                        int64_t ldb, const TcEpilogue& epi, const TcExt& ext, cudaStream_t s) {
  // A stored [K, M] (row pitch lda), B stored [K, N] (row pitch ldb): both MN-major
  NM_REQUIRE(M >= 1 && N >= 1 && K >= 1 && M <= 0x7fffffffLL && N <= 0x7fffffffLL && K <= 0x7fffffffLL,
             NM_E_INVALID, "tc_gemm16_mn: bad shape %lld x %lld x %lld", (long long)M, (long long)N, (long long)K);
  NM_REQUIRE((lda & 7) == 0 && (ldb & 7) == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(B) & 15) == 0,
             NM_E_INVALID, "tc_gemm16_mn: fp16 operands need 16-byte aligned bases and row pitches");
  NM_REQUIRE(epi.mode == TC_EPI_DENSE, NM_E_INVALID, "tc_gemm16_mn: dense epilogue only");
  CUtensorMap ma, mb;   // [K, M] and [K, N] as stored, boxes of 64 columns x one 64-row k-block
  int rc = make_map16(&ma, A, K, M, lda, 64);
  if (rc) return rc;
  rc = make_map16(&mb, B, K, N, ldb, 64);
  if (rc) return rc;
  const TcOperand oa{A, K, M, lda}, ob{B, K, N, ldb};
  int bn = 256;
  if (N <= 64) bn = 64;
  else if (N <= 128) bn = 128;
  else if (ceil_div(M, TC_BM) * ceil_div(N, 256) < sm_count()) bn = 128;
  if (bn == 64) return launch_cfg16<64, TC_EPI_DENSE, true>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  if (bn == 128) return launch_cfg16<128, TC_EPI_DENSE, true>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  return launch_cfg16<256, TC_EPI_DENSE, true>(ma, mb, oa, ob, M, N, K, epi, ext, s);
}

int tc_gemm16_launch(int64_t M, int64_t N, int64_t K, const void* A, int64_t lda, const void* B,
                     int64_t ldb, const TcEpilogue& epi, const TcExt& ext, cudaStream_t s) {
  NM_REQUIRE(M >= 1 && N >= 1 && K >= 1 && M <= 0x7fffffffLL && N <= 0x7fffffffLL && K <= 0x7fffffffLL,
             NM_E_INVALID, "tc_gemm16: bad shape %lld x %lld x %lld", (long long)M, (long long)N, (long long)K);
  NM_REQUIRE((lda & 7) == 0 && (ldb & 7) == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(B) & 15) == 0,
             NM_E_INVALID, "tc_gemm16: fp16 operands need 16-byte aligned bases and row pitches");
  const int bn = (epi.mode == TC_EPI_DENSE) ? pick_bn(M, N, K) : TC_XENT_BN;
  CUtensorMap ma, mb;
  TcOperand oa, ob;
  int rc = make_operand(&ma, &oa, false, A, M, K, lda, TC_BM, 2);
  if (rc) return rc;
  const bool pair = pair_wanted(M, bn, true);
  rc = make_operand(&mb, &ob, false, B, N, K, ldb, (uint32_t)(pair ? bn / 2 : bn), 2);
  if (rc) return rc;
  if (pair) {
    if (epi.mode == TC_EPI_XENT_FWD) return launch_cfg16<256, TC_EPI_XENT_FWD, false, true>(ma, mb, oa, ob, M, N, K, epi, ext, s);
    if (epi.mode == TC_EPI_XENT_BWD16)
      return launch_cfg16<256, TC_EPI_XENT_BWD16, false, true>(ma, mb, oa, ob, M, N, K, epi, ext, s);
    NM_REQUIRE(epi.mode == TC_EPI_DENSE, NM_E_INVALID, "tc_gemm16: unsupported epilogue %d", epi.mode);
    if (bn == 128) return launch_cfg16<128, TC_EPI_DENSE, false, true>(ma, mb, oa, ob, M, N, K, epi, ext, s);
    return launch_cfg16<256, TC_EPI_DENSE, false, true>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  }
  if (epi.mode == TC_EPI_XENT_FWD) return launch_cfg16<256, TC_EPI_XENT_FWD>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  if (epi.mode == TC_EPI_XENT_BWD16) return launch_cfg16<256, TC_EPI_XENT_BWD16>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  NM_REQUIRE(epi.mode == TC_EPI_DENSE, NM_E_INVALID, "tc_gemm16: unsupported epilogue %d", epi.mode);
  if (bn == 64) return launch_cfg16<64, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  if (bn == 128) return launch_cfg16<128, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  if (bn == 160) return launch_cfg16<160, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, ext, s);
  return launch_cfg16<256, TC_EPI_DENSE>(ma, mb, oa, ob, M, N, K, epi, ext, s);
}

}  // namespace nm
