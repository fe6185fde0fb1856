// The dense fp16 products (nm_gemm_f16, nm_gemm_f16_tn): the vocabulary gradients dX and [dW; db] of
// ops._LogitsXent16 (csrc/xent16.cu has the forward and the P16 recompute).
//
// gemm16_kernel: D[R, Cn] = A'[R, K] . B'[Cn, K]^T in 128 x 320 output tiles, both operands K-major (!MN) or both
// MN-major (MN: A' stored [K, R], B' stored [K, Cn], read transposed by wgmma), fp32 accumulators in registers.
//   * one persistent CTA per SM (or per SM of a budget, nm_gemm_f16_tn_ctas).  The (tile, 64-wide k-block) space is linearised, k-blocks fastest, and every CTA
//     takes an equal contiguous range of it (stream-K): at the bench shape both products are 50,000 k-blocks of
//     128 x 320 x 64 (dX 100 tiles x 500, [dW; db] 250 x 200), about 379 per SM, so no SM idles in a last,
//     partly filled wave.  A tile cut by a range boundary is summed in C by red.global.add from each CTA holding
//     a piece (into C zeroed by the host when beta = 0); no CTA ever waits for another, so the kernel stays
//     correct when only part of the grid is resident (a concurrent launch on the weight-gradient stream);
//   * warpgroup 0: one thread issues the TMA loads into a 4-stage ring of {A' 128 rows, B' 320 rows} k-blocks
//     (boxes bounded at the matrix edges: padding columns are never read, they arrive as zeros); the A' stream
//     (P16, 0.8 GB at the bench shape, larger than L2) is marked evict-first, the small B' (W16 19 MB, XS16 8 MB)
//     evict-last; it gives its registers to the consumers (setmaxnreg);
//   * warpgroups 1 and 2 own rows [0, 64) and [64, 128) of the tile: one m64n256k16 + one m64n64k16 per 16-deep
//     step (on MN-major 128-byte-swizzle operands N must be a multiple of 64), 160 accumulators per thread;
//   * the epilogue works on the fragment in registers: alpha * row_scale[r] * acc, stored (or added) as 2-column
//     pieces; a warp instruction then covers eight 32-byte row segments of C, or four 32-byte column segments of
//     C^T, whole sectors either way.
#include <cuda_fp16.h>

#include "common.cuh"
#include "gemm_tc.h"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace nm {

constexpr int G16_BM = 128;
constexpr int G16_BN = 320;
constexpr int G16_A_BYTES = G16_BM * 128;       // one 64-element k-block of the tile's A' rows: 16 KB
constexpr int G16_B_BYTES = G16_BN * 128;       // ... of its B' rows: 40 KB
constexpr int G16_STAGE_BYTES = G16_A_BYTES + G16_B_BYTES;
constexpr int G16_STAGES = 4;
constexpr int G16_BAR_OFF = G16_STAGES * G16_STAGE_BYTES;
constexpr int G16_SMEM_BYTES = 1024 /*align slack*/ + G16_BAR_OFF + 256 /*barriers*/;
constexpr int G16_THREADS = 384;
static_assert(G16_SMEM_BYTES <= 227 * 1024, "more shared memory than an sm_90 block may have");

struct G16Args {
  float* C;
  int64_t ldc;
  const float* alpha;       // device scalar or null (1)
  const float* row_scale;   // [R] or null (1)
  int R, Cn, K;
  int trans_out;            // element (r, c) goes to C[c * ldc + r]
  int beta;                 // 1: add into C
  int vec2;                 // row-major C with 8-byte aligned column pairs
};

__device__ __forceinline__ void tma_load_2d_hint(uint32_t dst, const CUtensorMap* map, uint32_t bar, int32_t c0,
                                                 int32_t c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

// out(r, c) and out(r, c + 1), c < Cn; `add`: red.global.add into C
__device__ __forceinline__ void put2(const G16Args& p, int r, int c, float v0, float v1, bool add) {
  const bool ok1 = c + 1 < p.Cn;
  if (p.trans_out) {
    float* d = p.C + (int64_t)c * p.ldc + r;
    if (add) {
      atomicAdd(d, v0);
      if (ok1) atomicAdd(d + p.ldc, v1);
    } else {
      *d = v0;
      if (ok1) d[p.ldc] = v1;
    }
    return;
  }
  float* d = p.C + (int64_t)r * p.ldc + c;
  if (p.vec2 && ok1) {
    if (add)
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d), "f"(v0), "f"(v1) : "memory");
    else
      *reinterpret_cast<float2*>(d) = make_float2(v0, v1);
    return;
  }
  if (add) {
    atomicAdd(d, v0);
    if (ok1) atomicAdd(d + 1, v1);
  } else {
    d[0] = v0;
    if (ok1) d[1] = v1;
  }
}

template <bool MN>
__global__ void __launch_bounds__(G16_THREADS, 1)
gemm16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, G16Args p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SW128 tiles: 1 KB aligned
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bars = sbase + G16_BAR_OFF;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (G16_STAGES + s); };

  const int tiles_r = (p.R + G16_BM - 1) / G16_BM;
  const int KB = (p.K + 63) / 64;
  const int64_t total = (int64_t)tiles_r * ((p.Cn + G16_BN - 1) / G16_BN) * KB;
  // this CTA's range of (tile, k-block) units; static, so the launch may be replayed from a CUDA graph
  const int64_t begin = blockIdx.x * total / gridDim.x, end = (blockIdx.x + 1) * total / gridDim.x;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b)) : "memory");
    for (int s = 0; s < G16_STAGES; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 8);   // one arrive per consumer warp
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
    uint64_t stream_pol, keep_pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(stream_pol));
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep_pol));
    int it = 0;
    for (int64_t u = begin; u < end;) {
      const int t = (int)(u / KB), kb0 = (int)(u - (int64_t)t * KB);
      const int kb1 = (int)min((int64_t)KB, end - (int64_t)t * KB);
      const int r0 = (t % tiles_r) * G16_BM, c0 = (t / tiles_r) * G16_BN;
      // 64-wide boxes wholly beyond the matrix are not loaded: their stale rows only reach discarded outputs
      const int nb = min(G16_BN / 64, (p.Cn - c0 + 63) / 64);
      const int na = MN ? min(G16_BM / 64, (p.R - r0 + 63) / 64) : 1;
      const uint32_t bytes = (MN ? na * 8192 : G16_A_BYTES) + nb * 8192;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % G16_STAGES;
        mbar_wait(empty(s), ((it / G16_STAGES) & 1) ^ 1u);
        mbar_expect_tx(full(s), bytes);
        const uint32_t a_dst = sbase + s * G16_STAGE_BYTES, b_dst = a_dst + G16_A_BYTES;
        if (MN) {   // boxes {64 MN elements, one k-block of rows}, 8 KB each
          for (int j = 0; j < na; ++j) tma_load_2d_hint(a_dst + j * 8192, &map_a, full(s), r0 + 64 * j, kb * 64, stream_pol);
          for (int j = 0; j < nb; ++j) tma_load_2d_hint(b_dst + j * 8192, &map_b, full(s), c0 + 64 * j, kb * 64, keep_pol);
        } else {    // boxes {one k-block, 128 / 64 rows}
          tma_load_2d_hint(a_dst, &map_a, full(s), kb * 64, r0, stream_pol);
          for (int j = 0; j < nb; ++j) tma_load_2d_hint(b_dst + j * 8192, &map_b, full(s), kb * 64, c0 + 64 * j, keep_pol);
        }
      }
      u = (int64_t)t * KB + kb1;
    }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = (warp >> 2) - 1, w = warp & 3, q = lane & 3;
  const float alpha = p.alpha ? __ldg(p.alpha) : 1.f;
  constexpr int KSTEP = MN ? 2048 : 32;     // bytes per 16-deep step within a k-block
  float acc[128], acc2[32];                 // columns [0, 256) and [256, 320) of the warpgroup's 64 rows
  int it = 0;
  for (int64_t u = begin; u < end;) {
    const int t = (int)(u / KB), kb0 = (int)(u - (int64_t)t * KB);
    const int kb1 = (int)min((int64_t)KB, end - (int64_t)t * KB);
    const int r0 = (t % tiles_r) * G16_BM, c0 = (t / tiles_r) * G16_BN;
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) acc2[i] = 0.f;
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const int s = it % G16_STAGES;
      mbar_wait(full(s), (it / G16_STAGES) & 1);
      const uint32_t a_addr = sbase + s * G16_STAGE_BYTES + wg * 8192;   // K-major: 64 rows; MN: one box
      const uint32_t b_addr = sbase + s * G16_STAGE_BYTES + G16_A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t da = MN ? gmma_desc_sw128_mn(a_addr + k * KSTEP) : gmma_desc_sw128(a_addr + k * KSTEP);
        const uint64_t db = MN ? gmma_desc_sw128_mn(b_addr + k * KSTEP) : gmma_desc_sw128(b_addr + k * KSTEP);
        const uint64_t db2 = MN ? gmma_desc_sw128_mn(b_addr + 32768 + k * KSTEP)
                                : gmma_desc_sw128(b_addr + 32768 + k * KSTEP);
        Wgmma<256, 2, MN>::mma(acc, da, db);
        Wgmma<64, 2, MN>::mma(acc2, da, db2);
      }
      wgmma_commit();
      wgmma_wait<1>();                       // the previous k-block's products are done with their stage
      wgmma_fence_operands(acc);
      wgmma_fence_operands(acc2);
      if (kb > kb0 && lane == 0) mbar_arrive(empty((it - 1) % G16_STAGES));
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    wgmma_fence_operands(acc2);
    if (lane == 0) mbar_arrive(empty((it - 1) % G16_STAGES));

    // ---- epilogue, on the fragment: acc[4i + 2h + e] = (row rw + 8h, column c0 + 8i + 2q + e) ----
    const bool add = p.beta != 0 || kb0 != 0 || kb1 != KB;   // beta = 1, or a piece of a cut tile
    const int rw = r0 + 64 * wg + 16 * w + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rw + 8 * h;
      if (r >= p.R) continue;
      const float f = p.row_scale ? alpha * __ldg(p.row_scale + r) : alpha;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c = c0 + 8 * i + 2 * q;
        if (c < p.Cn) put2(p, r, c, acc[4 * i + 2 * h] * f, acc[4 * i + 2 * h + 1] * f, add);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = c0 + 256 + 8 * i + 2 * q;
        if (c < p.Cn) put2(p, r, c, acc2[4 * i + 2 * h] * f, acc2[4 * i + 2 * h + 1] * f, add);
      }
    }
    u = (int64_t)t * KB + kb1;
  }
}

// D[R, Cn] = A' . B'^T (see the kernel), then C = alpha * row_scale[r] * D (+ C), stored as D or D^T, on at most
// max_ctas SMs (<= 0: all).  !mn: A' is A [R, K] (row pitch lda), B' is B [Cn, K]; mn: A' is stored [K, R], B'
// [K, Cn].
static int gemm16_run(const char* name, bool mn, int64_t R, int64_t Cn, int64_t K, const void* A, int64_t lda,
                      const void* B, int64_t ldb, float* C, int64_t ldc, const float* alpha, const float* row_scale,
                      float beta, bool trans_out, int max_ctas, cudaStream_t s) {
  NM_REQUIRE(R >= 1 && Cn >= 1 && K >= 1 && R <= 0x7fffffffLL && Cn <= 0x7fffffffLL && K <= 0x7fffffffLL,
             NM_E_INVALID, "%s: bad shape", name);
  NM_REQUIRE((lda & 7) == 0 && (ldb & 7) == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(B) & 15) == 0,
             NM_E_INVALID, "%s: fp16 operands need 16-byte aligned bases and row pitches", name);
  const int64_t tiles = ceil_div(R, G16_BM) * ceil_div(Cn, G16_BN);
  const int64_t KB = ceil_div(K, 64);
  NM_REQUIRE(tiles <= 0x7fffffffLL, NM_E_INVALID, "%s: %lld tiles", name, (long long)tiles);
  CUtensorMap ma, mb;
  int rc = mn ? make_map16(&ma, A, K, R, lda, 64) : make_map16(&ma, A, R, K, lda, G16_BM);
  if (rc) return rc;
  rc = mn ? make_map16(&mb, B, K, Cn, ldb, 64) : make_map16(&mb, B, Cn, K, ldb, 64);
  if (rc) return rc;
  const int64_t total = tiles * KB;
  const int sms = max_ctas > 0 && max_ctas < sm_count() ? max_ctas : sm_count();
  const int grid = (int)(total < sms ? total : sms);
  if (beta == 0.f) {
    // tiles cut by a range boundary are summed in C: start those from zero (the whole C, one memset)
    bool cut = false;
    for (int b = 1; b < grid && !cut; ++b) cut = (b * total / grid) % KB != 0;
    if (cut) {
      const int64_t rows = trans_out ? Cn : R, cols = trans_out ? R : Cn;
      NM_CUDA_TRY(cudaMemset2DAsync(C, sizeof(float) * ldc, 0, sizeof(float) * cols, rows, s));
    }
  }
  G16Args a{C, ldc, alpha, row_scale, (int)R, (int)Cn, (int)K, trans_out ? 1 : 0, beta != 0.f ? 1 : 0,
            (!trans_out && (ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(C) & 7) == 0) ? 1 : 0};
  auto kern = mn ? gemm16_kernel<true> : gemm16_kernel<false>;
  static bool attr_done[2] = {false, false};
  if (!attr_done[mn]) {
    NM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, G16_SMEM_BYTES));
    attr_done[mn] = true;
  }
  kern<<<grid, G16_THREADS, G16_SMEM_BYTES, s>>>(ma, mb, a);
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_gemm_f16(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16, int64_t ldb,
                float* C, int64_t ldc, const float* alpha_dev, const float* row_scale, float beta,
                int transposed, void* stream) {
  NM_REQUIRE(A16 && B16 && C, NM_E_INVALID, "nm_gemm_f16: null pointer");
  NM_REQUIRE(beta == 0.f || beta == 1.f, NM_E_INVALID, "nm_gemm_f16: beta must be 0 or 1");
  NM_REQUIRE(lda >= K && ldb >= K && ldc >= (transposed ? M : N), NM_E_INVALID, "nm_gemm_f16: bad pitches");
  return gemm16_run("nm_gemm_f16", false, M, N, K, A16, lda, B16, ldb, C, ldc, alpha_dev, row_scale, beta,
                    transposed != 0, 0, (cudaStream_t)stream);
}

int nm_gemm_f16_tn_ctas(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16,
                        int64_t ldb, float* C, int64_t ldc, const float* alpha_dev, float beta, int max_ctas,
                        void* stream) {
  NM_REQUIRE(A16 && B16 && C, NM_E_INVALID, "nm_gemm_f16_tn: null pointer");
  NM_REQUIRE(beta == 0.f || beta == 1.f, NM_E_INVALID, "nm_gemm_f16_tn: beta must be 0 or 1");
  NM_REQUIRE(lda >= M && ldb >= N && ldc >= N, NM_E_INVALID, "nm_gemm_f16_tn: bad pitches");
  // both operands MN-major, so the roles are symmetric: the larger of M and N runs down the 128-row tiles, the
  // smaller across the 320-column ones ([dW; db]: 32000 rows, 301 columns, C^T = B^T A stored transposed)
  if (M < N)
    return gemm16_run("nm_gemm_f16_tn", true, N, M, K, B16, ldb, A16, lda, C, ldc, alpha_dev, nullptr, beta, true,
                      max_ctas, (cudaStream_t)stream);
  return gemm16_run("nm_gemm_f16_tn", true, M, N, K, A16, lda, B16, ldb, C, ldc, alpha_dev, nullptr, beta, false,
                    max_ctas, (cudaStream_t)stream);
}

int nm_gemm_f16_tn(int64_t M, int64_t N, int64_t K, const void* A16, int64_t lda, const void* B16, int64_t ldb,
                   float* C, int64_t ldc, const float* alpha_dev, float beta, void* stream) {
  return nm_gemm_f16_tn_ctas(M, N, K, A16, lda, B16, ldb, C, ldc, alpha_dev, beta, 0, stream);
}

}  // extern "C"
