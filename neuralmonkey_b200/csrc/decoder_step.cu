// K4 (inference): ONE launch per decoding step of the RNN attention decoder - everything
// Decoder.next_state (decoders/decoder.py:279-358 of the reference) does between the previous
// symbol and the vector the vocabulary projection consumes:
//
//   x      = word_embeddings[symbol]                         (autoregressive.py:269-272)
//   [r,u]  = sigmoid([x,h].W_g + b_g)                        (TF-1.12 GRUCell, ortho_gru_cell.py:44-53)
//   c      = tanh([x, r*h].W_c + b_c);  h' = u*h + (1-u)*c
//   y      = h'.W_q + b_p                                    (feed_forward.py:131-137)
//   e_t    = sum_a v_a tanh(keys[t,a] + y_a) + b;  w = softmax(e) over ALL Tx, then *mask,
//            / (sum + 1e-8);  ctx = sum_t w_t values[t]       (feed_forward.py:139-156)
//   out    = tanh([h', x, ctx].W_o + b_o)   or maxout        (output_projection.py:115-160)
//
// Inference only (no dropout).  Exact fp32 on the CUDA cores: the step is a chain of five
// dependent matrix-vector products per hypothesis, i.e. latency- and weight-streaming bound, not
// tensor-pipe bound, and greedy / beam token parity wants fp32.
//
// Work split.  A thread-block CLUSTER of CL CTAs (1, 2, 4 or 8) owns DS_R = 8 rows (hypotheses).
// Every product is split over the cluster by OUTPUT columns: a CTA streams only 1/CL of each
// weight matrix (coalesced 16-byte loads, 8 in flight per thread) and multiplies it with all 8 rows
// held transposed in shared memory ([k][row]: two LDS.128 feed 32 FMAs); the K range of a column
// group is split over the threads of the CTA and reduced through shared memory in a fixed order
// (deterministic).  The slices a CTA produces (r*h, h', the query projection, the context) are
// written straight into the peers' shared memory (DSMEM) and a cluster barrier separates the phases.
// The attention itself is split by rows: each CTA attends for 8/CL rows.  Its key / value tiles
// are staged by 1-D TMA (cp.async.bulk + mbarrier ring) - the first ring of tiles is requested
// before the GRU phases start, so the HBM-bound part of the step hides behind the latency-bound
// part - and hypotheses of one sentence (beam search: `group` rows share an encoder row) reuse a
// staged tile.  The softmax over Tx is a warp-shuffle reduction.
#include <cooperative_groups.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace cg = cooperative_groups;

namespace nm {

constexpr int DS_R = 8;          // rows (hypotheses) per cluster
constexpr int DS_THREADS = 512;
constexpr int DS_WARPS = DS_THREADS / 32;
constexpr int DS_UNROLL = 8;     // weight rows in flight per thread
constexpr int DS_SLOTS = 4;      // TMA ring depth
constexpr int DS_RED_FLOATS = 128 * 32;   // K-split scratch of ds_panel: up to 128 partial sums of 32 floats

struct DecStep {
  int rows, E, H, A, C, Tx, O, group, act, maxout;
  int cl;            // cluster size
  int tck, tcv;      // time steps per staged keys / values tile (TMA path)
  int slot_floats;   // floats per ring slot (TMA path)
  const int64_t* symbols;
  const float* table;
  const float* x_in;
  const float* h_prev;
  const int32_t* parent;
  const float *Wg, *bg, *Wc, *bc, *Wq, *bq, *v, *abias;
  const float *keys, *values, *mask;
  const float *Wo, *bo;
  float *x_out, *h_out, *ctx_out, *w_out, *out;
  long long* prof;   // diagnostic: 8 clock64 stamps of CTA 0 (phase boundaries), or null
};

// Shared-memory carve-up (float offsets), the same arithmetic on host and device.
struct DsLayout {
  int xT, hT, rhT, hnT, ctxT, ug, res, red, qs, es, vs, ring, bars, total;
  int res_ld;
};

__host__ __device__ inline int ds_align4(int x) { return (x + 3) & ~3; }

__host__ __device__ inline DsLayout ds_layout(const DecStep& p, bool tma) {
  DsLayout L;
  const int rpc = DS_R / p.cl;
  int maxn = 2 * p.H;
  if (p.A > maxn) maxn = p.A;
  const int no = (p.maxout ? 2 : 1) * p.O;
  if (no > maxn) maxn = no;
  L.res_ld = ds_align4((maxn + p.cl - 1) / p.cl + 16);
  int o = 0;
  L.xT = o;   o += ds_align4(p.E * DS_R);
  L.hT = o;   o += ds_align4(p.H * DS_R);
  L.rhT = o;  o += ds_align4(p.H * DS_R);
  L.hnT = o;  o += ds_align4(p.H * DS_R);
  L.ctxT = o; o += ds_align4(p.C * DS_R);
  L.ug = o;   o += ds_align4(DS_R * ((p.H + p.cl - 1) / p.cl + 8));
  L.res = o;  o += DS_R * L.res_ld;
  L.red = o;  o += DS_RED_FLOATS;
  L.qs = o;   o += ds_align4(rpc * p.A);
  L.es = o;   o += ds_align4(rpc * p.Tx);
  L.vs = o;   o += ds_align4(p.A);
  L.ring = o; o += tma ? DS_SLOTS * p.slot_floats : 0;
  L.bars = o; o += 4 * DS_SLOTS;            // DS_SLOTS mbarriers (8 bytes each) + padding
  L.total = o;
  return L;
}

__device__ __forceinline__ float ds_fast_tanh(float x) {   // the form attention.cu uses
  return 1.f - __fdividef(2.f, 1.f + __expf(2.f * x));
}

// Key / value tiles are read once per step and are 15x the size of everything the step re-reads (its
// weights, the vocabulary matrix of the GEMM that follows): they pass through L2 with evict-first priority so
// that the re-read data stays resident from one step to the next.
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  uint64_t policy;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}

// Weights: streamed once per CTA and step (no reuse inside the SM: no L1 allocation), re-read by every cluster
// and every step (kept in L2: evict-last).
__device__ __forceinline__ uint64_t l2_evict_last_policy() {
  uint64_t policy;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(policy));
  return policy;
}
__device__ __forceinline__ float4 ldg_weight4(const float* p, uint64_t policy) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(policy));
  return v;
}

struct DsSeg {
  const float* inT;   // [len][DS_R] in shared memory
  int len;
};

// res[r][local column] = sum_k in[r][k] * W[k][column] for this CTA's columns: two ranges of
// G-wide column groups (nA groups from column colA, nB groups from column colB); local columns are
// range A first, then range B.  K = sum of the segment lengths, weight row of segment element i =
// (start of the segment in the virtual K range) + i.
//
// Thread mapping (the first version split K over threads of DIFFERENT warps and reduced through shared
// memory behind three block barriers: ncu put 27 % of the kernel's samples on those barriers).  A warp owns
// DS_GW adjacent column groups (64 contiguous bytes of every weight row: full sectors) times DS_KSL
// k-slices; the k-slices of a group are lanes of ONE warp, so their partial sums meet in three shuffle rounds.
// When the CTA has fewer group quads than warps, several warps share a quad (K split once more) and a
// single barrier joins them.  NOT inlined: four call sites, ~10 KB of unrolled FMAs each.
constexpr int DS_GW_MAX = 16;   // a warp owns gw = 2..16 adjacent column groups x (32 / gw) k-slices; gw is
                                // chosen per call so that as many of the 16 warps as possible have work

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}

template <int G>
__device__ __noinline__ void ds_panel(const DsSeg* segs, int nseg, int K, const float* __restrict__ W,
                                      int ldw, int colA, int nA, int colB, int nB,
                                      float* __restrict__ res, int res_ld, float* __restrict__ red) {
  const int ng = nA + nB;
  if (ng == 0) return;   // a CTA of a large cluster may own no columns of a small product (uniform per CTA)
  constexpr int RG = DS_R * G;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // groups per warp: the choice that keeps most warps busy (38 groups: gw = 8 -> 5 quads x 3 warps; gw = 4
  // would leave 6 of 16 warps idle and every busy lane with twice the k range)
  int DS_GW = 4, best_busy = 0;
#pragma unroll
  for (int cand = 2; cand <= DS_GW_MAX; cand <<= 1) {
    const int nqc = (ng + cand - 1) / cand;
    const int busy = nqc >= DS_WARPS ? DS_WARPS : nqc * (DS_WARPS / nqc);
    const bool fits = nqc >= DS_WARPS || (DS_WARPS / nqc) * nqc * cand * RG <= DS_RED_FLOATS;   // K-split scratch
    if (fits && (busy > best_busy || (busy == best_busy && cand == 4))) { best_busy = busy; DS_GW = cand; }
  }
  const int DS_KSL = 32 / DS_GW;
  const int gl = lane % DS_GW, ksl = lane / DS_GW;
  const uint64_t wpolicy = l2_evict_last_policy();
  const int nquads = (ng + DS_GW - 1) / DS_GW;
#pragma unroll 1
  for (int qb = 0; qb < nquads; qb += DS_WARPS) {
    const int nq = min(DS_WARPS, nquads - qb);
    const int wsplit = DS_WARPS / nq;                 // warps sharing one quad (K split across them)
    const int quad = warp % nq, ws = warp / nq;
    const int gg = (qb + quad) * DS_GW + gl;          // this lane's column group
    const bool active = ws < wsplit && gg < ng;
    const int col = gg < nA ? colA + gg * G : colB + (gg - nA) * G;
    const int kslices = DS_KSL * wsplit;
    const int kper = (K + kslices - 1) / kslices;
    const int k0 = min(K, (ws * DS_KSL + ksl) * kper);
    const int k1 = min(K, k0 + kper);
    float acc[DS_R][G];
#pragma unroll
    for (int r = 0; r < DS_R; ++r)
#pragma unroll
      for (int c = 0; c < G; ++c) acc[r][c] = 0.f;
    if (active) {
      int start = 0;
#pragma unroll 1
      for (int s = 0; s < nseg; ++s) {
        const int len = segs[s].len;
        const int lo = max(k0, start), hi = min(k1, start + len);
        if (lo < hi) {
          const float* wp = W + (int64_t)lo * ldw + col;
          uint32_t ip = smem_u32(segs[s].inT) + (uint32_t)(lo - start) * DS_R * 4u;
          // batches of DS_UNROLL weight rows: all loads of a batch are in flight together; the last,
          // partial batch is predicated instead of falling back to one dependent load per row
#pragma unroll 1
          for (int k = lo; k < hi; k += DS_UNROLL) {
            float w[DS_UNROLL][G];
#pragma unroll
            for (int u = 0; u < DS_UNROLL; ++u) {
              if (k + u < hi) {
                if constexpr (G == 4) {
                  const float4 t = ldg_weight4(wp + (int64_t)u * ldw, wpolicy);
                  w[u][0] = t.x; w[u][1] = t.y; w[u][2] = t.z; w[u][3] = t.w;
                } else {
                  w[u][0] = __ldg(wp + (int64_t)u * ldw);
                }
              } else {
#pragma unroll
                for (int c = 0; c < G; ++c) w[u][c] = 0.f;
              }
            }
#pragma unroll
            for (int u = 0; u < DS_UNROLL; ++u) {
              if (k + u < hi) {
                float in[DS_R];
#pragma unroll
                for (int q = 0; q < DS_R / 4; ++q) {
                  const float4 t4 = lds128(ip + u * DS_R * 4 + 16 * q);
                  in[4 * q] = t4.x; in[4 * q + 1] = t4.y; in[4 * q + 2] = t4.z; in[4 * q + 3] = t4.w;
                }
#pragma unroll
                for (int r = 0; r < DS_R; ++r)
#pragma unroll
                  for (int c = 0; c < G; ++c) acc[r][c] = fmaf(in[r], w[u][c], acc[r][c]);
              }
            }
            wp += (int64_t)DS_UNROLL * ldw;
            ip += DS_UNROLL * DS_R * 4;
          }
        }
        start += len;
      }
    }
    // the k-slices of a column group are the lanes gl, gl + gw, gl + 2 gw, ... of this warp
#pragma unroll
    for (int off = 2; off < 32; off <<= 1) {
      if (off >= DS_GW) {        // warp-uniform
#pragma unroll
        for (int r = 0; r < DS_R; ++r)
#pragma unroll
          for (int c = 0; c < G; ++c) acc[r][c] += __shfl_xor_sync(0xffffffffu, acc[r][c], off);
      }
    }
    if (wsplit == 1) {
      if (active && ksl == 0) {
#pragma unroll
        for (int r = 0; r < DS_R; ++r)
#pragma unroll
          for (int c = 0; c < G; ++c) res[r * res_ld + gg * G + c] = acc[r][c];
      }
    } else {
      // several warps per quad: one barrier joins their partial sums (fixed order: deterministic)
      const int S = wsplit * nq * DS_GW;              // S * RG <= DS_RED_FLOATS by the choice of gw above
      if (ws < wsplit && ksl == 0) {
        const int slot = ws * nq * DS_GW + quad * DS_GW + gl;
#pragma unroll
        for (int r = 0; r < DS_R; ++r)
#pragma unroll
          for (int c = 0; c < G; ++c) red[(r * G + c) * S + slot] = acc[r][c];
      }
      __syncthreads();
#pragma unroll 1
      for (int idx = threadIdx.x; idx < nq * DS_GW * RG; idx += DS_THREADS) {
        const int e = idx / (nq * DS_GW), g2 = idx - e * (nq * DS_GW);
        const int gout = qb * DS_GW + g2;
        if (gout < ng) {
          float sum = 0.f;
#pragma unroll 1
          for (int h = 0; h < wsplit; ++h) sum += red[e * S + h * nq * DS_GW + g2];
          res[(e / G) * res_ld + gout * G + (e % G)] = sum;
        }
      }
    }
    __syncthreads();
  }
}

// The slice of `total` G-wide groups CTA `rank` of `cl` owns: [first, first + count).
__device__ __forceinline__ void ds_slice(int total, int cl, int rank, int& first, int& count) {
  const int per = (total + cl - 1) / cl;
  first = min(total, rank * per);
  count = min(total, first + per) - first;
}

// Attention schedule of one CTA: runs of owned rows that share an encoder row, each at most `jt` rows
// (a thread of the context pass owns one (row, column group) pair).  Computed by thread 0 into shared memory.
struct DsRuns {
  int n;
  int e[DS_R], first[DS_R], cnt[DS_R];
};

template <int G>
__global__ void __launch_bounds__(DS_THREADS, 1) attn_decoder_step_kernel(const __grid_constant__ DecStep p) {
  constexpr bool TMA = (G == 4);
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = p.cl;
  const int rank = (int)cluster.block_rank();
  const int row0 = (int)(blockIdx.x / CL) * DS_R;
  const int rpc = DS_R / CL;                // rows this CTA attends for
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const DsLayout L = ds_layout(p, TMA);

  extern __shared__ __align__(128) float smem[];
  float* xT = smem + L.xT;
  float* hT = smem + L.hT;
  float* rhT = smem + L.rhT;
  float* hnT = smem + L.hnT;
  float* ctxT = smem + L.ctxT;
  float* ugs = smem + L.ug;
  float* res = smem + L.res;
  float* red = smem + L.red;
  float* qs = smem + L.qs;
  float* es = smem + L.es;
  float* vs = smem + L.vs;
  float* ring = smem + L.ring;
  const uint32_t bar0 = smem_u32(smem + L.bars);
  const int res_ld = L.res_ld;
  __shared__ DsRuns runs;

  const int my0 = row0 + rank * rpc;                      // first global row this CTA attends for
  const int nmy = max(0, min(rpc, p.rows - my0));         // valid ones
  const int nk = TMA ? (p.Tx + p.tck - 1) / p.tck : 1;    // tiles per run: keys, then values
  const int nv = TMA ? (p.Tx + p.tcv - 1) / p.tcv : 1;
  const int ncg = (p.C + G - 1) / G;                      // context column groups (host: <= DS_THREADS)
  const int jt = min(DS_R, DS_THREADS / ncg);          // rows per run

  // tile i of this CTA's schedule (run-major: the key tiles of a run, then its value tiles)
  auto issue_tile = [&](int i) {   // one thread
    const int run = i / (nk + nv), j = i - run * (nk + nv);
    const int e = runs.e[run];
    const float* src;
    uint32_t bytes;
    if (j < nk) {
      const int t0 = j * p.tck, nt = min(p.tck, p.Tx - t0);
      src = p.keys + ((int64_t)e * p.Tx + t0) * p.A;
      bytes = (uint32_t)(nt * p.A * 4);
    } else {
      const int t0 = (j - nk) * p.tcv, nt = min(p.tcv, p.Tx - t0);
      src = p.values + ((int64_t)e * p.Tx + t0) * p.C;
      bytes = (uint32_t)(nt * p.C * 4);
    }
    const int slot = i % DS_SLOTS;
    mbar_expect_tx(bar0 + 8u * slot, bytes);
    bulk_load_1d(smem_u32(ring + slot * p.slot_floats), src, bytes, bar0 + 8u * slot);
  };

  if (tid == 0) {
    int n = 0, prev = -1;
#pragma unroll 1
    for (int j = 0; j < nmy; ++j) {
      const int e = (my0 + j) / p.group;
      if (e != prev || runs.cnt[n - 1] >= jt) {
        runs.e[n] = e; runs.first[n] = j; runs.cnt[n] = 1;
        ++n;
        prev = e;
      } else {
        ++runs.cnt[n - 1];
      }
    }
    runs.n = n;
    if (TMA) {
#pragma unroll 1
      for (int s2 = 0; s2 < DS_SLOTS; ++s2) mbar_init(bar0 + 8u * s2, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      const int first = min(n * (nk + nv), DS_SLOTS);
#pragma unroll 1
      for (int i = 0; i < first; ++i) issue_tile(i);   // in flight while the GRU phases run
    }
  }

  // ---- phase 0: inputs of the 8 rows, transposed into shared memory -----------------------------
  // lane -> (row = lane & 7, k offset = lane >> 3): the stores walk shared memory linearly (no bank
  // conflicts); the global side reads 16 contiguous bytes of each of the 8 rows per warp instruction
  {
    const int r = lane & (DS_R - 1);
    const int grow = row0 + r;
    const bool ok = grow < p.rows;
    const float* xsrc = nullptr;
    const float* hsrc = nullptr;
    if (ok) {
      xsrc = p.x_in ? p.x_in + (int64_t)grow * p.E : p.table + (int64_t)p.symbols[grow] * p.E;
      const int src = p.parent ? (grow / p.group) * p.group + p.parent[grow] : grow;
      hsrc = p.h_prev + (int64_t)src * p.H;
    }
#pragma unroll 1
    for (int k = tid / DS_R; k < p.E; k += DS_THREADS / DS_R) {
      const float val = ok ? xsrc[k] : 0.f;
      if (ok && p.x_out && rank == 0) p.x_out[(int64_t)grow * p.E + k] = val;
      xT[k * DS_R + r] = val;
    }
#pragma unroll 1
    for (int k = tid / DS_R; k < p.H; k += DS_THREADS / DS_R) hT[k * DS_R + r] = ok ? hsrc[k] : 0.f;
  }
#pragma unroll 1
  for (int a = tid; a < p.A; a += DS_THREADS) vs[a] = p.v[a];
  __syncthreads();
  const bool prof = p.prof != nullptr && blockIdx.x == 0 && tid == 0;
  if (prof) p.prof[0] = clock64();
  cluster.sync();   // every CTA of the cluster has started: its shared memory may be written remotely
  if (prof) p.prof[1] = clock64();

  const int r_w = warp & (DS_R - 1), half_w = warp / DS_R;   // element-wise passes: warp -> (row, half)
  constexpr int NHALF = DS_WARPS / DS_R;

  // ---- phase 1: gates of this CTA's hidden units -------------------------------------------------
  int uf, un;   // first unit group / number of unit groups
  ds_slice((p.H + G - 1) / G, CL, rank, uf, un);
  const int u0 = uf * G;
  const int nu = min(p.H, u0 + un * G) - u0;   // units this CTA owns (0 when H is small and CL large)
  {
    const DsSeg segs[2] = {{xT, p.E}, {hT, p.H}};
    ds_panel<G>(segs, 2, p.E + p.H, p.Wg, 2 * p.H, u0, un, p.H + u0, un, res, res_ld, red);
#pragma unroll 1
    for (int ul = lane + 32 * half_w; ul < nu; ul += 32 * NHALF) {
      const int r = r_w, u = u0 + ul;
      const float rr = sigmoidf_(res[r * res_ld + ul] + p.bg[u]);
      const float uu = sigmoidf_(res[r * res_ld + un * G + ul] + p.bg[p.H + u]);
      ugs[r * nu + ul] = uu;
      const float rh = rr * hT[u * DS_R + r];
#pragma unroll 1
      for (int c = 0; c < CL; ++c) cluster.map_shared_rank(rhT, c)[u * DS_R + r] = rh;
    }
  }
  cluster.sync();
  if (prof) p.prof[2] = clock64();

  // ---- phase 2: candidate and new state ------------------------------------------------------------
  {
    const DsSeg segs[2] = {{xT, p.E}, {rhT, p.H}};
    ds_panel<G>(segs, 2, p.E + p.H, p.Wc, p.H, u0, un, 0, 0, res, res_ld, red);
#pragma unroll 1
    for (int ul = lane + 32 * half_w; ul < nu; ul += 32 * NHALF) {
      const int r = r_w, u = u0 + ul;
      const float c = tanhf(res[r * res_ld + ul] + p.bc[u]);
      const float uu = ugs[r * nu + ul];
      const float hn = uu * hT[u * DS_R + r] + (1.f - uu) * c;
#pragma unroll 1
      for (int cc = 0; cc < CL; ++cc) cluster.map_shared_rank(hnT, cc)[u * DS_R + r] = hn;
      if (row0 + r < p.rows) p.h_out[(int64_t)(row0 + r) * p.H + u] = hn;
    }
  }
  cluster.sync();
  if (prof) p.prof[3] = clock64();

  // ---- phase 3: query projection, delivered to the CTA that attends for the row --------------------
  {
    int af, an;
    ds_slice((p.A + G - 1) / G, CL, rank, af, an);
    const int a0 = af * G;
    const int na = min(p.A, a0 + an * G) - a0;
    const DsSeg segs[1] = {{hnT, p.H}};
    ds_panel<G>(segs, 1, p.H, p.Wq, p.A, a0, an, 0, 0, res, res_ld, red);
    float* qdst = cluster.map_shared_rank(qs, r_w / rpc) + (r_w % rpc) * p.A;
#pragma unroll 1
    for (int al = lane + 32 * half_w; al < na; al += 32 * NHALF)
      qdst[a0 + al] = res[r_w * res_ld + al] + p.bq[a0 + al];
  }
  cluster.sync();
  if (prof) p.prof[4] = clock64();

  // ---- phase 4: attention for the rows this CTA owns ---------------------------------------------------
  {
    const float abias = p.abias[0];
    const int ntiles = runs.n * (nk + nv);
    int tile = 0;          // position in the TMA schedule
#pragma unroll 1
    for (int run = 0; run < runs.n; ++run) {
      const int e = runs.e[run], j0 = runs.first[run], cnt = runs.cnt[run];
      // energies: one warp per (time step, row) pair, lanes over A
#pragma unroll 1
      for (int kt = 0; kt < nk; ++kt) {
        const float* kc;
        int t0, nt;
        if (TMA) {
          mbar_wait(bar0 + 8u * (tile % DS_SLOTS), (uint32_t)((tile / DS_SLOTS) & 1));
          kc = ring + (tile % DS_SLOTS) * p.slot_floats;
          t0 = kt * p.tck;
          nt = min(p.tck, p.Tx - t0);
        } else {
          kc = p.keys + (int64_t)e * p.Tx * p.A;
          t0 = 0;
          nt = p.Tx;
        }
#pragma unroll 1
        for (int it = warp; it < nt * cnt; it += DS_WARPS) {
          const int tl = it / cnt, j = it - tl * cnt;
          const float* kr = kc + tl * p.A;
          const float* qr = qs + (j0 + j) * p.A;
          float acc = 0.f;
          if constexpr (G == 4) {
#pragma unroll 1
            for (int a4 = lane; a4 < p.A / 4; a4 += 32) {
              const float4 k4 = *reinterpret_cast<const float4*>(kr + 4 * a4);
              const float4 v4 = *reinterpret_cast<const float4*>(vs + 4 * a4);
              const float4 q4 = *reinterpret_cast<const float4*>(qr + 4 * a4);
              acc = fmaf(v4.x, ds_fast_tanh(k4.x + q4.x), acc);
              acc = fmaf(v4.y, ds_fast_tanh(k4.y + q4.y), acc);
              acc = fmaf(v4.z, ds_fast_tanh(k4.z + q4.z), acc);
              acc = fmaf(v4.w, ds_fast_tanh(k4.w + q4.w), acc);
            }
          } else {
#pragma unroll 1
            for (int a = lane; a < p.A; a += 32) acc = fmaf(vs[a], ds_fast_tanh(kr[a] + qr[a]), acc);
          }
          const float en = warp_sum(acc) + abias;
          if (lane == 0) es[(j0 + j) * p.Tx + t0 + tl] = en;
        }
        __syncthreads();   // the tile is consumed (and, after the last one, the energies are complete)
        if (TMA) {
          if (tid == 0 && tile + DS_SLOTS < ntiles) issue_tile(tile + DS_SLOTS);
          ++tile;
        }
      }
      // softmax over ALL Tx, then mask and renormalise: one warp per row of the run
#pragma unroll 1
      for (int j = warp; j < cnt; j += DS_WARPS) {
        float* er = es + (j0 + j) * p.Tx;
        const int64_t grow = my0 + j0 + j;
        float mx = -INFINITY;
        for (int t = lane; t < p.Tx; t += 32) mx = fmaxf(mx, er[t]);
        mx = warp_max(mx);
        float s = 0.f;
        for (int t = lane; t < p.Tx; t += 32) s += expf(er[t] - mx);
        s = warp_sum(s);
        float ws = 0.f;
        for (int t = lane; t < p.Tx; t += 32) {
          float pr = expf(er[t] - mx) / s;
          if (p.mask) pr *= p.mask[(int64_t)e * p.Tx + t];
          er[t] = pr;
          ws += pr;
        }
        if (p.mask) {
          const float norm = warp_sum(ws) + 1e-8f;
          for (int t = lane; t < p.Tx; t += 32) er[t] = er[t] / norm;
        }
        __syncwarp();
        if (p.w_out)
          for (int t = lane; t < p.Tx; t += 32) p.w_out[grow * p.Tx + t] = er[t];
      }
      __syncthreads();
      // context: thread = (row of the run, column group), all time steps; the sum stays in registers
      const int cj = tid / ncg, cgi = tid - cj * ncg;
      const bool cact = cj < cnt;
      float cacc[G];
#pragma unroll
      for (int c = 0; c < G; ++c) cacc[c] = 0.f;
#pragma unroll 1
      for (int vt = 0; vt < nv; ++vt) {
        const float* vc;
        int t0, nt;
        if (TMA) {
          mbar_wait(bar0 + 8u * (tile % DS_SLOTS), (uint32_t)((tile / DS_SLOTS) & 1));
          vc = ring + (tile % DS_SLOTS) * p.slot_floats;
          t0 = vt * p.tcv;
          nt = min(p.tcv, p.Tx - t0);
        } else {
          vc = p.values + (int64_t)e * p.Tx * p.C;
          t0 = 0;
          nt = p.Tx;
        }
        if (cact) {
          const float* wr = es + (j0 + cj) * p.Tx + t0;
#pragma unroll 2
          for (int tl = 0; tl < nt; ++tl) {
            const float wt = wr[tl];
            if constexpr (G == 4) {
              const float4 t4 = *reinterpret_cast<const float4*>(vc + tl * p.C + 4 * cgi);
              cacc[0] = fmaf(wt, t4.x, cacc[0]); cacc[1] = fmaf(wt, t4.y, cacc[1]);
              cacc[2] = fmaf(wt, t4.z, cacc[2]); cacc[3] = fmaf(wt, t4.w, cacc[3]);
            } else {
              cacc[0] = fmaf(wt, vc[tl * p.C + cgi], cacc[0]);
            }
          }
        }
        __syncthreads();
        if (TMA) {
          if (tid == 0 && tile + DS_SLOTS < ntiles) issue_tile(tile + DS_SLOTS);
          ++tile;
        }
      }
      if (cact) {   // broadcast the context of (row, column group) to the cluster
        const int rl = rank * rpc + j0 + cj;               // row index inside the cluster
#pragma unroll
        for (int c = 0; c < G; ++c) {
          const int col = cgi * G + c;
          if (col < p.C) {
#pragma unroll 1
            for (int cc = 0; cc < CL; ++cc) cluster.map_shared_rank(ctxT, cc)[col * DS_R + rl] = cacc[c];
            if (p.ctx_out) p.ctx_out[(int64_t)(my0 + j0 + cj) * p.C + col] = cacc[c];
          }
        }
      }
    }
    // rows beyond `rows` (tail cluster): their context columns must be defined for the last product
#pragma unroll 1
    for (int jj = nmy; jj < rpc; ++jj) {
      const int rl = rank * rpc + jj;
#pragma unroll 1
      for (int col = tid; col < p.C; col += DS_THREADS)
#pragma unroll 1
        for (int cc = 0; cc < CL; ++cc) cluster.map_shared_rank(ctxT, cc)[col * DS_R + rl] = 0.f;
    }
  }
  if (prof) p.prof[5] = clock64();
  cluster.sync();
  if (prof) p.prof[6] = clock64();

  // ---- phase 5: deep output ---------------------------------------------------------------------------
  {
    int of, on;
    ds_slice((p.O + G - 1) / G, CL, rank, of, on);
    const int o0 = of * G;
    const int no = min(p.O, o0 + on * G) - o0;
    const DsSeg segs[3] = {{hnT, p.H}, {xT, p.E}, {ctxT, p.C}};
    const int ldo = (p.maxout ? 2 : 1) * p.O;
    ds_panel<G>(segs, 3, p.H + p.E + p.C, p.Wo, ldo, o0, on, p.O + o0, p.maxout ? on : 0, res, res_ld, red);
    if (row0 + r_w < p.rows) {
#pragma unroll 1
      for (int ol = lane + 32 * half_w; ol < no; ol += 32 * NHALF) {
        const int o = o0 + ol;
        float y = res[r_w * res_ld + ol] + p.bo[o];
        if (p.maxout) {
          const float y2 = res[r_w * res_ld + on * G + ol] + p.bo[p.O + o];
          y = fmaxf(y, y2);
        } else {
          y = apply_act(y, p.act);
        }
        p.out[(int64_t)(row0 + r_w) * p.O + o] = y;
      }
    }
  }
  if (prof) p.prof[7] = clock64();
}

}  // namespace nm

using namespace nm;

static long long* g_decstep_prof = nullptr;

// 227 KB per CTA minus the kernel's static shared memory (the run table), rounded up to 1 KB
constexpr int DS_MAX_DYN_SMEM = 227 * 1024 - 1024;

// The launch plan of one step: sizes, cluster size, vector or scalar variant, ring slot and tile lengths, and
// the dynamic shared memory, from the sizes, the SM count of the current device and whether every base the
// vector variant reads with 16-byte loads is 16-byte aligned.  NM_E_UNSUPPORTED (message set) for the shapes
// the kernel cannot take: nm_attn_decoder_step_supported and the launcher answer from this one function.
static int ds_plan(int64_t rows, int64_t group, int64_t E, int64_t H, int64_t A, int64_t C, int64_t Tx, int64_t O,
                   int maxout, bool aligned, DecStep& p, bool& vec, size_t& smem_bytes) {
  NM_REQUIRE(rows > 0 && group > 0 && E > 0 && H > 0 && A > 0 && C > 0 && Tx > 0 && O > 0, NM_E_INVALID,
             "nm_attn_decoder_step_fwd: bad sizes");
  NM_REQUIRE(rows < (1 << 24) && Tx < (1 << 20), NM_E_UNSUPPORTED, "nm_attn_decoder_step_fwd: too large");
  p.rows = (int)rows; p.E = (int)E; p.H = (int)H; p.A = (int)A; p.C = (int)C; p.Tx = (int)Tx; p.O = (int)O;
  p.group = (int)group; p.maxout = maxout ? 1 : 0;

  vec = (E % 4 == 0) && (H % 4 == 0) && (A % 4 == 0) && (C % 4 == 0) && (O % 4 == 0) && aligned;
  const int g = vec ? 4 : 1;
  NM_REQUIRE(ceil_div(C, g) <= DS_THREADS, NM_E_UNSUPPORTED,
             "nm_attn_decoder_step_fwd: context size %lld too large for one CTA", (long long)C);

  // cluster size: as many CTAs as fill the chip, at most 8, at least one attended row per CTA
  const int64_t clusters = ceil_div(rows, DS_R);
  int cl = 8;
  while (cl > 1 && clusters * cl > (int64_t)sm_count()) cl >>= 1;
  const char* env = getenv("NMB200_DECSTEP_CLUSTER");
  if (env && *env) {
    const int want = atoi(env);
    if (want == 1 || want == 2 || want == 4 || want == 8) cl = want;
  }
  p.cl = cl;

  // ring slots: as large as the shared memory left over allows, whole time steps of keys / values
  if (vec) {
    p.slot_floats = 0;
    const DsLayout base = ds_layout(p, true);
    const int64_t avail = (int64_t)DS_MAX_DYN_SMEM / 4 - base.total;
    int64_t slot = avail / DS_SLOTS;
    slot -= slot % 32;                                       // 128-byte granularity
    const int64_t need = (A > C ? A : C);
    NM_REQUIRE(slot >= need, NM_E_UNSUPPORTED,
               "nm_attn_decoder_step_fwd: sizes leave no room for a key/value tile in shared memory");
    int64_t cap = 8192;                                      // 32 KB per tile is plenty
    if (slot > cap) slot = cap - cap % 32;
    if (slot < need) slot = (need + 31) / 32 * 32;
    p.slot_floats = (int)slot;
    p.tck = (int)(slot / A); if (p.tck > Tx) p.tck = (int)Tx;
    p.tcv = (int)(slot / C); if (p.tcv > Tx) p.tcv = (int)Tx;
    smem_bytes = sizeof(float) * (size_t)ds_layout(p, true).total;
  } else {
    p.slot_floats = 0; p.tck = (int)Tx; p.tcv = (int)Tx;
    smem_bytes = sizeof(float) * (size_t)ds_layout(p, false).total;
  }
  NM_REQUIRE(smem_bytes <= (size_t)DS_MAX_DYN_SMEM, NM_E_UNSUPPORTED,
             "nm_attn_decoder_step_fwd: needs %zu bytes of shared memory", smem_bytes);
  return NM_OK;
}

extern "C" {

/* Diagnostic: 8 int64 device counters receiving clock64() of CTA 0 at the phase boundaries of the next
 * nm_attn_decoder_step_fwd launches (inputs staged | cluster up | gates | state | query | attention |
 * cluster joined | output done).  NULL = off. */
int nm_attn_decoder_step_debug(void* counters) {
  g_decstep_prof = reinterpret_cast<long long*>(counters);
  return NM_OK;
}

int nm_attn_decoder_step_fwd(const int64_t* symbols, const float* emb_table, const float* x_in,
                             const float* h_prev, const int32_t* parent, const float* Wg, const float* bg,
                             const float* Wc, const float* bc, const float* Wq, const float* bq,
                             const float* v, const float* att_bias, const float* keys,
                             const float* values, const float* mask, const float* Wo, const float* bo,
                             float* x_out, float* h_out, float* ctx_out, float* weights_out, float* out,
                             int64_t rows, int64_t group, int64_t E, int64_t H, int64_t A, int64_t C,
                             int64_t Tx, int64_t O, int act, int maxout, void* stream) {
  NM_REQUIRE((symbols && emb_table) || x_in, NM_E_INVALID,
             "nm_attn_decoder_step_fwd: need symbols + emb_table, or x_in");
  NM_REQUIRE(h_prev && Wg && bg && Wc && bc && Wq && bq && v && att_bias && keys && values && Wo && bo &&
                 h_out && out,
             NM_E_INVALID, "nm_attn_decoder_step_fwd: null pointer");
  NM_REQUIRE(h_prev != h_out, NM_E_INVALID, "nm_attn_decoder_step_fwd: h_out must not alias h_prev");
  // vector path: every row the kernel reads with 16-byte loads is 16-byte aligned
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  const bool aligned = al16(Wg) && al16(Wc) && al16(Wq) && al16(Wo) && al16(keys) && al16(values);
  DecStep p{};
  bool vec = false;
  size_t smem_bytes = 0;
  const int rc = ds_plan(rows, group, E, H, A, C, Tx, O, maxout, aligned, p, vec, smem_bytes);
  if (rc != NM_OK) return rc;
  p.act = act;
  p.symbols = x_in ? nullptr : symbols; p.table = emb_table; p.x_in = x_in; p.h_prev = h_prev; p.parent = parent;
  p.Wg = Wg; p.bg = bg; p.Wc = Wc; p.bc = bc; p.Wq = Wq; p.bq = bq; p.v = v; p.abias = att_bias;
  p.keys = keys; p.values = values; p.mask = mask; p.Wo = Wo; p.bo = bo;
  p.x_out = x_out; p.h_out = h_out; p.ctx_out = ctx_out; p.w_out = weights_out; p.out = out;
  p.prof = g_decstep_prof;

  auto kern = vec ? attn_decoder_step_kernel<4> : attn_decoder_step_kernel<1>;
  static bool attr_done[2] = {false, false};
  if (!attr_done[vec]) {
    NM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, DS_MAX_DYN_SMEM));
    attr_done[vec] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(ceil_div(rows, DS_R) * p.cl));
  cfg.blockDim = dim3(DS_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)p.cl;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  NM_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, p));
  NM_LAUNCH_CHECK("nm_attn_decoder_step_fwd");
  return NM_OK;
}

int nm_attn_decoder_step_supported(int64_t rows, int64_t group, int64_t E, int64_t H, int64_t A, int64_t C,
                                   int64_t Tx, int64_t O, int maxout, int aligned) {
  DecStep p{};
  bool vec = false;
  size_t smem_bytes = 0;
  return ds_plan(rows, group, E, H, A, C, Tx, O, maxout, aligned != 0, p, vec, smem_bytes) == NM_OK;
}

}  // extern "C"
