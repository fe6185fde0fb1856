// The vocabulary projection with fp16 operands (K5/K6), the default of ops.logits_xent on the tensor-core engine
// (ops._LogitsXent16; tied embeddings, the exact engine and weights without gradient-buffer sinks keep every
// product in TF32, xent.cu).
//
// The three kernels that touch dlogits [M,V] are a large part of a training step; in fp32 the matrix is
// written once (1.6 GB at the bench shape) and read about three times.  Here it is stored once as fp16,
// UNNORMALISED ((softmax - onehot) * mask, values in [-1, 1]: fp16 then has TF32's 10 mantissa bits;
// tools/fp16_dlogits_study.py), row-major, and every product is an fp16 wgmma GEMM:
//     logits  = X16 [M,K]   . WT16 [V,K]^T          forward, and the recompute of the backward (xent16_kernel)
//     dX      = dl16 [M,V]  . W16  [K,V]^T           * row_scale[m]                (nm_gemm_f16, gemm16.cu)
//     dW      = XS16 [M,K+1]^T . dl16 [M,V]         * alpha, MN-major operands    (nm_gemm_f16_tn, gemm16.cu)
// The upstream per-row gradient is applied in fp32 in the consumers' epilogues.
//
// xent16_kernel: a persistent CTA per SM works through a contiguous range of 64 x 256 output tiles, row tiles
// fastest.  At K <= 320 the 256-column slice of WT16 (five 32 KB k-blocks) stays in shared memory while the CTA
// walks down the rows: only the 8 KB k-blocks of X16 stream from L2 (a third of the traffic of re-loading W for
// every 128-row tile), and a CTA loads one or two W slices in all.  Longer K (the slice no longer fits) runs the
// fused epilogues of the generic wgmma GEMM (tc_gemm16_launch), which re-load W for every 128-row tile.
//   * warpgroup 0: one thread issues the TMA loads (operand boxes bounded at K: the padding columns of X16 / WT16
//     are never read, they arrive as zeros); it gives its registers to the consumers (setmaxnreg);
//   * warpgroups 1 and 2 take alternate tiles (wgmma m64n256k16, accumulators in registers) and ping-pong on two
//     named barriers: one issues its products while the other runs its epilogue, so the exp / store work of one
//     tile hides under the products of the next;
//   * the epilogues work on the accumulator fragment in registers (thread = 2 rows x 64 columns, a quad of lanes
//     covers the tile's 256 columns of both rows).  Forward: max / sum of 2^(x log2e - max) / argmax / target
//     logit per thread, merged over lane pairs, written as the two partials per (row, 256-column tile) of the
//     `part` layout.  Backward: P16 through a per-warp stmatrix staging tile into whole 256-byte row segments,
//     marked evict-first so that the 0.8 GB stream does not push X16 and WT16 out of L2.
#include <cuda_fp16.h>

#include "common.cuh"
#include "gemm_tc.h"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace nm {

__global__ void cast_f16_kernel(const float* __restrict__ src, int64_t ld_src, __half* __restrict__ dst,
                                int64_t ld_dst, int64_t rows, int64_t cols,
                                const float* __restrict__ row_scale, int extra_ones) {
  const int64_t total = rows * ld_dst;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / ld_dst, c = i - r * ld_dst;
    float v = 0.f;
    const float sc = row_scale ? row_scale[r] : 1.f;
    if (c < cols) v = src[r * ld_src + c] * sc;
    else if (c < cols + extra_ones) v = sc;
    dst[i] = __float2half_rn(v);
  }
}

// dst [cols + extra_ones, ld_dst] = transpose of src [rows, cols] (scaled per source row), followed by
// `extra_ones` rows holding row_scale (the column of ones of the bias-gradient trick, scaled alike).
// 32x32 tiles through shared memory: coalesced on both sides.
__global__ void cast_transpose_f16_kernel(const float* __restrict__ src, int64_t ld_src,
                                          __half* __restrict__ dst, int64_t ld_dst, int64_t rows,
                                          int64_t cols, const float* __restrict__ row_scale,
                                          int extra_ones) {
  __shared__ float tile[32][33];
  const int64_t r0 = blockIdx.x * 32LL, c0 = blockIdx.y * 32LL;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t r = r0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (r < rows) {
      const float sc = row_scale ? row_scale[r] : 1.f;
      if (c < cols) v = src[r * ld_src + c] * sc;
      else if (c < cols + extra_ones) v = sc;
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t c = c0 + i, r = r0 + threadIdx.x;
    if (c < cols + extra_ones && r < ld_dst) dst[c * ld_dst + r] = __float2half_rn(tile[threadIdx.x][i]);
  }
}

constexpr int X16_BM = 64;                     // rows of one consumer tile
constexpr int X16_BN = TC_XENT_BN;             // columns of one tile
constexpr int X16_A_BYTES = X16_BM * 128;      // one 64-element k-block of a tile's X16 rows: 8 KB
constexpr int X16_B_BYTES = X16_BN * 128;      // one k-block of the tile's WT16 rows: 32 KB
constexpr int X16_B_SLOTS = XENT16_MAX_K / 64;   // the W slice's k-blocks, resident
constexpr int X16_STAGE_WARP = 16 * 128 * 2;   // bwd staging: a warp's 16 rows x 128 columns of fp16
constexpr int X16_THREADS = 384;

template <bool BWD>
struct X16Cfg {
  static constexpr int A_STAGES = BWD ? 4 : 8;
  static constexpr int A_OFF = X16_B_SLOTS * X16_B_BYTES;
  static constexpr int ST_OFF = A_OFF + A_STAGES * X16_A_BYTES;
  static constexpr int BAR_OFF = ST_OFF + (BWD ? 8 * X16_STAGE_WARP : 0);
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + BAR_OFF + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "more shared memory than an sm_90 block may have");
  static_assert((2 * A_STAGES + 2 * X16_B_SLOTS) * 8 <= 256, "barrier area");
};

struct X16Args {
  const float* bias;         // [V] or null
  int64_t unk;               // column that gets -1e9, < 0: none
  const int64_t* targets;    // [M] or null (fwd)
  const float* mask;         // [M] or null (bwd: row weight)
  const float* lse;          // [M] (bwd)
  float4* part;              // fwd
  float* logits;             // fwd, may be null
  int64_t ldl;
  __half* dl16;              // bwd
  int64_t ldd;
  int M, V, K;
};

__device__ __forceinline__ void named_sync(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void named_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// merge the (max, sum, argmax, target) of two disjoint column sets; the lower column wins among equal maxima
__device__ __forceinline__ void merge_stats(float& mx, float& sum, int& arg, float& tgt, float omx, float osum,
                                            int oarg, float otgt) {
  const float nm = fmaxf(mx, omx);
  if (nm != -INFINITY) sum = sum * fast_ex2((mx - nm) * TC_LOG2E) + osum * fast_ex2((omx - nm) * TC_LOG2E);
  if (omx > mx || (omx == mx && oarg < arg)) arg = oarg;
  mx = nm;
  tgt = fmaxf(tgt, otgt);
}

template <bool BWD>
__global__ void __launch_bounds__(X16_THREADS, 1)
xent16_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, X16Args p) {
  using Cfg = X16Cfg<BWD>;
  constexpr int AST = Cfg::A_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SW128 tiles: 1 KB aligned
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bars = sbase + Cfg::BAR_OFF;
  auto full_a = [&](int s) { return bars + 8u * s; };
  auto empty_a = [&](int s) { return bars + 8u * (AST + s); };
  auto full_b = [&](int s) { return bars + 8u * (2 * AST + s); };
  auto empty_b = [&](int s) { return bars + 8u * (2 * AST + X16_B_SLOTS + s); };

  const int tiles_m = (p.M + X16_BM - 1) / X16_BM;
  const int units = tiles_m * ((p.V + X16_BN - 1) / X16_BN);
  // a contiguous range of tiles per CTA (static: the launch may be replayed from a CUDA graph), row tiles
  // fastest, so that consecutive tiles share their W slice
  const int first = (int)((int64_t)blockIdx.x * units / gridDim.x);
  const int count = (int)((int64_t)(blockIdx.x + 1) * units / gridDim.x) - first;
  const int KB = (p.K + 63) / 64;              // <= X16_B_SLOTS

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_x)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
    for (int s = 0; s < AST; ++s) {
      mbar_init(full_a(s), 1);
      mbar_init(empty_a(s), 4);   // one arrive per warp of the consuming warpgroup
    }
    for (int s = 0; s < X16_B_SLOTS; ++s) {
      mbar_init(full_b(s), 1);
      mbar_init(empty_b(s), 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp < 4) {
    // ===================== producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (threadIdx.x != 0) return;
    int loads = 0, prev_tn = -1;
    for (int j = 0; j < count; ++j) {
      const int u = first + j, tm = u % tiles_m, tn = u / tiles_m;
      const bool reload = tn != prev_tn;   // a new W slice: once the last tile reading the old one is done
      loads += reload;
      prev_tn = tn;
      for (int kb = 0; kb < KB; ++kb) {
        const int ia = j * KB + kb, sa = ia % AST;
        mbar_wait(empty_a(sa), ((ia / AST) & 1) ^ 1u);
        mbar_expect_tx(full_a(sa), X16_A_BYTES);
        tma_load_2d(sbase + Cfg::A_OFF + sa * X16_A_BYTES, &map_x, full_a(sa), kb * 64, tm * X16_BM);
        if (reload) {
          mbar_wait(empty_b(kb), ((loads - 1) & 1) ^ 1u);
          mbar_expect_tx(full_b(kb), X16_B_BYTES);
          tma_load_2d(sbase + kb * X16_B_BYTES, &map_w, full_b(kb), kb * 64, tn * X16_BN);
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int c = (warp >> 2) - 1;      // consumer warpgroup: tiles j with j % 2 == c
  const int w = warp & 3, q = lane & 3;
  uint64_t evict_first = 0;
  if (BWD) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(evict_first));
  if (c == 1) named_arrive(1);        // the first tile's products go first
  float acc[128];
  int loads = 0, prev_tn = -1;
  for (int j = 0; j < count; ++j) {
    const int u = first + j, tm = u % tiles_m, tn = u / tiles_m;
    loads += tn != prev_tn;
    prev_tn = tn;
    if ((j & 1) != c) continue;
    // the last tile of this CTA that reads the resident W slice hands its slots back to the producer
    const bool last_use = j + 1 == count || (u + 1) / tiles_m != tn;

    // ---- products: this warpgroup's turn on the tensor cores ----
    named_sync(1 + c);
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < KB; ++kb) {
      const int ia = j * KB + kb, sa = ia % AST;
      mbar_wait(full_a(sa), (ia / AST) & 1);
      mbar_wait(full_b(kb), (loads - 1) & 1);
      const uint32_t a_addr = sbase + Cfg::A_OFF + sa * X16_A_BYTES, b_addr = sbase + kb * X16_B_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Wgmma<256, 2>::mma(acc, gmma_desc_sw128(a_addr + k * 32), gmma_desc_sw128(b_addr + k * 32));
      wgmma_commit();
      wgmma_wait<1>();                 // the previous k-block's products are done with their stages
      wgmma_fence_operands(acc);
      if (kb > 0 && lane == 0) mbar_arrive(empty_a((ia - 1) % AST));
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (lane == 0) {
      mbar_arrive(empty_a((j * KB + KB - 1) % AST));
      if (last_use)
        for (int kb = 0; kb < KB; ++kb) mbar_arrive(empty_b(kb));
    }
    // products complete before the other warpgroup starts: a W slice is handed back only when no tile still
    // reads it
    if (j + 1 < count) named_arrive(2 - c);

    // ---- epilogue, on the fragment: acc[4i + 2h + e] = (row r0 + 8h, column cb + 8i + e) ----
    const int r0 = tm * X16_BM + 16 * w + (lane >> 2);
    const int n0 = tn * X16_BN, cb = n0 + 2 * q;
    const int V = p.V;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = cb + 8 * i + e;
        const float b = (p.bias != nullptr && col < V) ? __ldg(p.bias + col) : 0.f;
        acc[4 * i + e] += b;
        acc[4 * i + 2 + e] += b;
      }
    }
    const int unk_rel = (int)(p.unk - cb);   // rare: only the tile (and the lane) holding <unk>
    if (p.unk >= 0 && unk_rel >= 0 && unk_rel < X16_BN && (unk_rel & 6) == 0) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * i + e == unk_rel) {
            acc[4 * i + e] += -1e9f;
            acc[4 * i + 2 + e] += -1e9f;
          }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      const bool row_ok = row < p.M;
      const int target = (row_ok && p.targets) ? (int)p.targets[row] : -1;
      const int t_rel = target - cb;      // this lane holds the target column when (t_rel & 7) < 2
      const bool has_t = target >= 0 && t_rel >= 0 && t_rel < X16_BN && (t_rel & 6) == 0;
      if constexpr (!BWD) {
        if (p.logits && row_ok) {
          float* lrow = p.logits + (int64_t)row * p.ldl + cb;
          const int ncols = V - cb;       // >= 256 except in the last column tile
#pragma unroll
          for (int i = 0; i < 32; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * i + e < ncols) lrow[8 * i + e] = acc[4 * i + 2 * h + e];
        }
        if (n0 + X16_BN > V) {             // ragged right edge: padding columns must not win the max
#pragma unroll
          for (int i = 0; i < 32; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (cb + 8 * i + e >= V) acc[4 * i + 2 * h + e] = -INFINITY;
        }
        float mx = -INFINITY;
        int arg = 0x7fffffff;
#pragma unroll
        for (int i = 0; i < 32; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (acc[4 * i + 2 * h + e] > mx) {   // strict, columns ascending: the lowest of equal maxima
              mx = acc[4 * i + 2 * h + e];
              arg = cb + 8 * i + e;
            }
        const float m2 = mx == -INFINITY ? 0.f : mx * TC_LOG2E;
        float s[4] = {0.f, 0.f, 0.f, 0.f};   // four chains of 16 dependent adds instead of one of 64
#pragma unroll
        for (int i = 0; i < 32; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            s[(2 * i + e) & 3] += fast_ex2(fmaf(acc[4 * i + 2 * h + e], TC_LOG2E, -m2));
        float sum = (s[0] + s[1]) + (s[2] + s[3]);
        float tgt = -INFINITY;
        if (has_t) {
#pragma unroll
          for (int i = 0; i < 32; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * i + e == t_rel) tgt = acc[4 * i + 2 * h + e];
        }
        merge_stats(mx, sum, arg, tgt, __shfl_xor_sync(0xffffffffu, mx, 1), __shfl_xor_sync(0xffffffffu, sum, 1),
                    __shfl_xor_sync(0xffffffffu, arg, 1), __shfl_xor_sync(0xffffffffu, tgt, 1));
        // lanes 2k, 2k+1 now hold the same partial of columns {8i + 4k .. 8i + 4k + 3}: lane q writes row
        // r0 + 8 (q & 1) of slot q >> 1
        if (row_ok && (q & 1) == h) {
          const int tiles_n2 = 2 * ((V + X16_BN - 1) / X16_BN);
          p.part[(int64_t)row * tiles_n2 + 2 * tn + (q >> 1)] = make_float4(mx, sum, __int_as_float(arg), tgt);
        }
      } else {
        const float lse2 = row_ok ? p.lse[row] * TC_LOG2E : 0.f;
        const float wt = row_ok ? (p.mask ? p.mask[row] : 1.f) : 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            acc[4 * i + 2 * h + e] = fast_ex2(fmaf(acc[4 * i + 2 * h + e], TC_LOG2E, -lse2)) * wt;
        if (has_t) {
#pragma unroll
          for (int i = 0; i < 32; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * i + e == t_rel) acc[4 * i + 2 * h + e] -= wt;
        }
      }
    }
    if constexpr (BWD) {
      // P16: the warp's 16 rows x 256 columns in two halves through its staging tile (16-byte chunk c of row r
      // at chunk c ^ (r & 7): conflict-free for stmatrix and for the row reads), then 16-byte row pieces
      uint8_t* stage = smem + Cfg::ST_OFF + (warp - 4) * X16_STAGE_WARP;
      const uint32_t stage_u = smem_u32(stage);
      const int srow_w = (lane & 7) + ((lane >> 3) & 1) * 8;   // the matrix row this lane addresses
#pragma unroll
      for (int half = 0; half < 2; ++half) {
#pragma unroll
        for (int jj = 0; jj < 16; jj += 2) {
          const int i = 16 * half + jj;
          const int chunk = jj + (lane >> 4);
          const uint32_t addr = stage_u + srow_w * 256 + ((chunk ^ (srow_w & 7)) << 4);
          asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr),
                       "r"(pack_half2(acc[4 * i], acc[4 * i + 1])), "r"(pack_half2(acc[4 * i + 2], acc[4 * i + 3])),
                       "r"(pack_half2(acc[4 * i + 4], acc[4 * i + 5])), "r"(pack_half2(acc[4 * i + 6], acc[4 * i + 7]))
                       : "memory");
        }
        __syncwarp();
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int idx = it * 32 + lane, srow = idx >> 4, ch = idx & 15;
          const uint4 v = *reinterpret_cast<const uint4*>(stage + srow * 256 + ((ch ^ (srow & 7)) << 4));
          const int grow = tm * X16_BM + 16 * w + srow;
          const int gcol = n0 + 128 * half + 8 * ch;
          if (grow < p.M && gcol < V) {
            __half* dst = p.dl16 + (int64_t)grow * p.ldd + gcol;
            if (gcol + 8 <= V) {
              asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(dst), "r"(v.x),
                           "r"(v.y), "r"(v.z), "r"(v.w), "l"(evict_first)
                           : "memory");
            } else {
              const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
              for (int e = 0; e < 8; ++e)
                if (gcol + e < V) dst[e] = __ushort_as_half((unsigned short)(wv[e >> 1] >> (16 * (e & 1))));
            }
          }
        }
        __syncwarp();
      }
    }
  }
}

template <bool BWD>
static int launch_xent16(const CUtensorMap& mx, const CUtensorMap& mw, const X16Args& a, int grid, cudaStream_t s,
                         const char* name) {
  auto kern = xent16_kernel<BWD>;
  static bool attr_done = false;
  if (!attr_done) {
    NM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, X16Cfg<BWD>::SMEM_BYTES));
    attr_done = true;
  }
  kern<<<grid, X16_THREADS, X16Cfg<BWD>::SMEM_BYTES, s>>>(mx, mw, a);
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

int xent16_launch(bool bwd, const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                  int64_t unk_index, const int64_t* targets, const float* mask, const float* lse, float4* part,
                  float* logits_out, int64_t ldl, void* dl16, int64_t ldd, int64_t M, int64_t V, int64_t K,
                  cudaStream_t s) {
  const char* name = bwd ? "nm_logits_xent_bwd16" : "nm_logits_xent_fwd16";
  NM_REQUIRE(ceil_div(M, X16_BM) * ceil_div(V, X16_BN) <= 0x7fffffffLL && M * 2 * ceil_div(V, X16_BN) <= 0x7fffffffLL &&
                 K <= XENT16_MAX_K,
             NM_E_INVALID, "%s: shape %lld x %lld x %lld too large", name, (long long)M, (long long)V, (long long)K);
  NM_REQUIRE((ldx & 7) == 0 && (ldw & 7) == 0 && (reinterpret_cast<uintptr_t>(X16) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(WT16) & 15) == 0,
             NM_E_INVALID, "%s: fp16 operands need 16-byte aligned bases and row pitches", name);
  NM_REQUIRE(!bwd || ((ldd & 7) == 0 && (reinterpret_cast<uintptr_t>(dl16) & 15) == 0), NM_E_INVALID,
             "%s: dl16 needs a 16-byte aligned base and row pitch", name);
  CUtensorMap mx, mw;
  int rc = make_map16(&mx, X16, M, K, ldx, X16_BM);
  if (rc) return rc;
  rc = make_map16(&mw, WT16, V, K, ldw, X16_BN);
  if (rc) return rc;
  X16Args a{b, unk_index, targets, mask, lse, part, logits_out, ldl, reinterpret_cast<__half*>(dl16), ldd,
            (int)M, (int)V, (int)K};
  const int64_t units = ceil_div(M, X16_BM) * ceil_div(V, X16_BN);
  const int grid = (int)(units < sm_count() ? units : sm_count());
  return bwd ? launch_xent16<true>(mx, mw, a, grid, s, name) : launch_xent16<false>(mx, mw, a, grid, s, name);
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_cast_f16(const float* src, int64_t ld_src, void* dst, int64_t ld_dst, int64_t rows, int64_t cols,
                const float* row_scale, int transpose, int extra_ones, void* stream) {
  NM_REQUIRE(src && dst && rows > 0 && cols > 0 && ld_src >= cols, NM_E_INVALID, "nm_cast_f16: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  if (!transpose) {
    NM_REQUIRE(extra_ones >= 0 && ld_dst >= cols + extra_ones, NM_E_INVALID, "nm_cast_f16: bad destination pitch");
    const int64_t total = rows * ld_dst;
    const int64_t blocks = ceil_div(total, 256 * 4);
    const int64_t cap = (int64_t)sm_count() * 16;   // grid-stride: 16 blocks of 256 threads per SM
    cast_f16_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, s>>>(
        src, ld_src, reinterpret_cast<__half*>(dst), ld_dst, rows, cols, row_scale, extra_ones);
  } else {
    NM_REQUIRE(ld_dst >= rows && extra_ones >= 0, NM_E_INVALID, "nm_cast_f16: bad destination pitch");
    const dim3 grid((unsigned)ceil_div(ld_dst, 32), (unsigned)ceil_div(cols + extra_ones, 32));
    cast_transpose_f16_kernel<<<grid, dim3(32, 8), 0, s>>>(src, ld_src, reinterpret_cast<__half*>(dst), ld_dst,
                                                          rows, cols, row_scale, extra_ones);
  }
  NM_LAUNCH_CHECK("nm_cast_f16");
  return NM_OK;
}

int nm_logits_xent_bwd16(const void* X16, int64_t ldx, const void* WT16, int64_t ldw, const float* b,
                         int64_t unk_index, const int64_t* targets, const float* mask, const float* lse,
                         void* dl16, int64_t ldd, int64_t M, int64_t V, int64_t K, void* stream) {
  NM_REQUIRE(X16 && WT16 && targets && lse && dl16, NM_E_INVALID, "nm_logits_xent_bwd16: null pointer");
  NM_REQUIRE(M > 0 && V > 0 && K > 0 && ldx >= K && ldw >= K && ldd >= V, NM_E_INVALID,
             "nm_logits_xent_bwd16: bad sizes");
  if (K <= XENT16_MAX_K)
    return xent16_launch(true, X16, ldx, WT16, ldw, b, unk_index, targets, mask, lse, nullptr, nullptr, 0, dl16,
                         ldd, M, V, K, (cudaStream_t)stream);
  TcEpilogue epi{};
  epi.mode = TC_EPI_XENT_BWD16;
  epi.bias = b;
  epi.unk_index = unk_index;
  epi.targets = targets;
  epi.weights = mask;
  epi.lse = lse;
  TcExt ext{};
  ext.C16 = dl16;
  ext.ldc16 = ldd;
  return tc_gemm16_launch(M, V, K, X16, ldx, WT16, ldw, epi, ext, (cudaStream_t)stream);
}

}  // extern "C"
