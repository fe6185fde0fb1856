// Persistent GRU sequence kernels for thread-block clusters (sm_90a).
//
// One launch runs the whole time loop.  A cluster of 8 CTAs owns a slice of the batch
// (Bc sentences); inside it, CTA r owns hidden units [r*UW, (r+1)*UW), UW = ceil(H/8).
// The recurrent weights never leave the SM: a warp owns 4 hidden units, and each of its
// 32 lanes keeps, in REGISTERS, the three weight vectors of those 4 units restricted to
// ONE of 32 reduction slices (3 * 4 * 4*CH floats per thread).  The inner product then
// streams only the state vector from shared memory - one conflict-free 16-byte load
// feeds 32 (gates) or 16 (candidate) FMAs - and is FMA-issue bound.  The 32 partial sums
// of a (row, unit) pair are combined with five shuffle steps.
//
// The two matmuls of a TF GRUCell step are dependent (the candidate needs r*h for ALL
// units), so a step has two phases separated by hardware cluster barriers; the vectors
// exchanged between the phases (h, r*h; backward: dz_c, dz_u, dz_r) are exactly the
// tensors the backward pass / the weight-gradient GEMMs need in HBM anyway, so the
// exchange costs only an L2 read of Bc*H floats per CTA per phase.  Element-wise gate
// math runs as a separate pass with threads along the hidden axis (coalesced HBM access).
#pragma once
#include "common.cuh"

namespace nm {

constexpr int GC_CLUSTER = 8;   // CTAs per cluster = slices of the hidden axis
constexpr int GC_SLICES = 32;   // reduction slices = lanes
constexpr int GC_UPW = 4;       // hidden units per warp
constexpr int GC_WARPS = 10;    // -> up to 40 units per CTA (H <= 320); 3 warps on an SMSP cap
                                // the kernel at 16384/96 = 168 registers per thread
constexpr int GC_THREADS = GC_WARPS * 32;
constexpr int GC_MAX_UNITS = GC_WARPS * GC_UPW;
constexpr int GC_RB = 2;        // batch rows per inner iteration

__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::
                   : "memory");
}
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ float reduce32(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum N values across the 32 lanes with N-1+log2(32/N)... shuffles instead of 5N: each
// butterfly level halves the number of live values (lanes whose bit `o` is set keep the
// upper half and send the lower, and vice versa).  On return v[0] of lane L is the full
// sum of the value with index (L >> (5 - log2 N)) & (N-1); lanes differing only in the
// low bits hold copies.
template <int N>
__device__ __forceinline__ void gc_reduce_scatter(float (&v)[N], int lane) {
  int o = 16;
#pragma unroll
  for (int n = N; n > 1; n >>= 1) {
    const bool upper = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float keep = upper ? v[i + n / 2] : v[i];
      const float send = upper ? v[i] : v[i + n / 2];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
    o >>= 1;
  }
  for (; o > 0; o >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
}

// Geometry: SL32 = ceil(H/32) reduction-slice length (<= 4*CH); SLP = slice pitch in the
// smem vector buffer: an odd number of 16-byte chunks so the 32 lanes of a 16-byte load
// fall into 4 conflict-free quarter-warp wavefronts; ROW = 32*SLP floats per batch row.
template <int CH>
struct GcGeom {
  static constexpr int SLP = 4 * (CH | 1);
  static constexpr int ROW = GC_SLICES * SLP;
};

// Stage H contiguous floats per row into the sliced layout.  Thread t owns columns
// t, t+GC_THREADS, ... (coalesced along the hidden axis); rows >= nrows are zero-filled.
// Per-thread constants of the loader: thread t owns the 16-byte column group k4 = t % QL
// (QL = ceil(H/4) rounded so that GC_THREADS % QL rows are handled in parallel) and the
// row lane t / QL; the four smem offsets of its columns are computed once per kernel.
struct GcLoader {
  int k, row_lane, row_lanes, off[4];
  bool active, vec4;
};

template <int CH>
__device__ __forceinline__ GcLoader gc_make_loader(int H, int SL32) {
  GcLoader L;
  const int q = (H + 3) >> 2;
  L.row_lanes = GC_THREADS / q > 0 ? GC_THREADS / q : 1;
  L.row_lane = threadIdx.x / q;
  L.k = (threadIdx.x % q) * 4;
  L.active = (threadIdx.x < q * L.row_lanes);
  L.vec4 = (H & 3) == 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = L.k + i;
    L.off[i] = (k < H) ? (k / SL32) * GcGeom<CH>::SLP + (k % SL32) : -1;
  }
  return L;
}

template <int CH>
__device__ __forceinline__ void gc_load_vec(float* __restrict__ vec, const float* __restrict__ src,
                                            int64_t pitch, int nrows, int Bc, const GcLoader& L) {
  constexpr int NB = 8;  // loads in flight per thread: issue all, then store (in-order issue
                         // would otherwise serialise one L2 round trip per load)
  constexpr int ROW = GcGeom<CH>::ROW;
  if (!L.active) return;
  const bool vec4 = L.vec4 && ((pitch & 3) == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  for (int b0 = L.row_lane; b0 < Bc; b0 += NB * L.row_lanes) {
    float4 v[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int b = b0 + i * L.row_lanes;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b < nrows) {
        const float* p = src + (int64_t)b * pitch + L.k;
        if (vec4) {
          v[i] = __ldcg(reinterpret_cast<const float4*>(p));
        } else {
          if (L.off[0] >= 0) v[i].x = __ldcg(p);
          if (L.off[1] >= 0) v[i].y = __ldcg(p + 1);
          if (L.off[2] >= 0) v[i].z = __ldcg(p + 2);
          if (L.off[3] >= 0) v[i].w = __ldcg(p + 3);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int b = b0 + i * L.row_lanes;
      if (b < Bc) {
        float* row = vec + b * ROW;
        if (L.off[0] >= 0) row[L.off[0]] = v[i].x;
        if (L.off[1] >= 0) row[L.off[1]] = v[i].y;
        if (L.off[2] >= 0) row[L.off[2]] = v[i].z;
        if (L.off[3] >= 0) row[L.off[3]] = v[i].w;
      }
    }
  }
}

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_all;" ::: "memory");
}

// acc[r][u] = partial (this lane's slice) of sum_k vec[row0+r][k] * w[u][k]
template <int CH>
__device__ __forceinline__ void gc_dot(const float* __restrict__ vec, int row0, int lane,
                                       const float (&w)[GC_UPW][4 * CH], float (&acc)[GC_RB][GC_UPW]) {
#pragma unroll
  for (int r = 0; r < GC_RB; ++r)
#pragma unroll
    for (int u = 0; u < GC_UPW; ++u) acc[r][u] = 0.f;
  const float* base = vec + row0 * GcGeom<CH>::ROW + lane * GcGeom<CH>::SLP;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
#pragma unroll
    for (int r = 0; r < GC_RB; ++r) {
      const float4 v = *reinterpret_cast<const float4*>(base + r * GcGeom<CH>::ROW + 4 * c);
#pragma unroll
      for (int u = 0; u < GC_UPW; ++u) {
        acc[r][u] = fmaf(v.x, w[u][4 * c], acc[r][u]);
        acc[r][u] = fmaf(v.y, w[u][4 * c + 1], acc[r][u]);
        acc[r][u] = fmaf(v.z, w[u][4 * c + 2], acc[r][u]);
        acc[r][u] = fmaf(v.w, w[u][4 * c + 3], acc[r][u]);
      }
    }
  }
}

// Load this lane's slice of column (or row) vectors of a weight matrix for the warp's 4
// units: w[u][i] = W[(k0+i)*sk + unit(u)*su] for i < SL32, zero elsewhere.
template <int CH>
__device__ __forceinline__ void gc_load_w(float (&w)[GC_UPW][4 * CH], const float* __restrict__ W,
                                          int64_t sk, int64_t su, int unit0, int nunits_total,
                                          int unit_limit, int k0, int SL32, int H) {
#pragma unroll
  for (int u = 0; u < GC_UPW; ++u)
#pragma unroll
    for (int i = 0; i < 4 * CH; ++i) {
      const int unit = unit0 + u, k = k0 + i;
      const bool ok = (unit < unit_limit) && (unit < nunits_total) && (i < SL32) && (k < H);
      w[u][i] = ok ? W[(int64_t)k * sk + (int64_t)unit * su] : 0.f;
    }
}

// ---------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------
struct GcFwdArgs {
  const float* xproj;   // [B,T,3H]
  const float* Wgh;     // [H,2H]
  const float* Wch;     // [H,H]
  const float* h0;      // [B,H] or null
  const int32_t* lengths;
  const float* drop_mask;
  float* states;        // [B,T,H]
  float* raw_states;    // or null
  float* final_state;   // [B,H]
  float* gates;         // [B,T,3H]
  float* hprev;         // [B,T,H]
  float* rh;            // [B,T,H]
  int B, T, H, Bc, reverse;
  long long* prof;      // optional [8] cycle counters of CTA 0 (diagnostics), or null
};

template <int CH>
__global__ void __launch_bounds__(GC_THREADS, 1) gru_seq_fwd_cluster_kernel(GcFwdArgs a) {
  extern __shared__ __align__(16) float gc_smem[];
  constexpr int ROW = GcGeom<CH>::ROW;
  float* vec = gc_smem;                 // [Bc][ROW]
  float* pre = vec + a.Bc * ROW;        // [Bc][GC_MAX_UNITS][2] pre-activations
  float* own = pre + a.Bc * GC_MAX_UNITS * 2;  // [Bc][GC_MAX_UNITS][2]: (h, u) of own units
  float* xs = own + a.Bc * GC_MAX_UNITS * 2;   // [Bc][GC_MAX_UNITS][3]: this step's xproj
  const int H = a.H, T = a.T, Bc = a.Bc;
  const int UW = (H + GC_CLUSTER - 1) / GC_CLUSTER;   // units per CTA
  const int SL32 = (H + GC_SLICES - 1) / GC_SLICES;   // reduction slice length
  const int rank = (int)cluster_rank();
  const int b0 = (blockIdx.x / GC_CLUSTER) * Bc;
  const int nrows = min(Bc, a.B - b0);
  const GcLoader loader = gc_make_loader<CH>(H, SL32);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int unit0_local = warp * GC_UPW;
  const int unit0 = rank * UW + unit0_local;          // first hidden unit of this warp
  const int unit_limit = min(H, (rank + 1) * UW);

  float wr[GC_UPW][4 * CH], wu[GC_UPW][4 * CH], wc[GC_UPW][4 * CH];
  gc_load_w<CH>(wr, a.Wgh, 2 * H, 1, unit0, H, unit_limit, lane * SL32, SL32, H);
  gc_load_w<CH>(wu, a.Wgh + H, 2 * H, 1, unit0, H, unit_limit, lane * SL32, SL32, H);
  gc_load_w<CH>(wc, a.Wch, H, 1, unit0, H, unit_limit, lane * SL32, SL32, H);

  // the slice padding of the vector buffer is never written again: it must be 0, not
  // stale shared memory (NaN * 0-weight would poison the sums)
  for (int i = threadIdx.x; i < Bc * ROW; i += GC_THREADS) vec[i] = 0.f;
  // seed the state history slot of the first step with h0 (own units, own rows)
  const int t_first = a.reverse ? T - 1 : 0;
  for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
    const int b = idx / UW, j = rank * UW + (idx - b * UW);
    if (b < nrows && j < H)
      a.hprev[((int64_t)(b0 + b) * T + t_first) * H + j] = a.h0 ? a.h0[(int64_t)(b0 + b) * H + j] : 0.f;
  }
  cluster_barrier();

  for (int step = 0; step < T; ++step) {
    const int t = a.reverse ? T - 1 - step : step;
    const bool last = (step == T - 1);
    const int t_next = a.reverse ? t - 1 : t + 1;
    const int64_t row0 = (int64_t)b0 * T + t;  // row index of batch row b0 at time t; +b*T per row

    // ---- phase 1: [r,u] = sigmoid(xg + h.Wgh), rh = r*h ----
    long long tp0 = 0, tp1 = 0;
    const bool profiling = a.prof != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
#define GC_PROF(slot) do { if (profiling) { tp1 = clock64(); a.prof[slot] += tp1 - tp0; tp0 = tp1; } } while (0)
    if (profiling) tp0 = clock64();
    // issue this step's xproj reads now (cold HBM lines) as asynchronous copies into smem:
    // they land while the dot products run and cost no registers
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, ul = idx - b * UW, j = rank * UW + ul;
      if (b < nrows && j < H) {
        const float* xp = a.xproj + (row0 + (int64_t)b * T) * 3 * H + j;
        float* xd = xs + (b * GC_MAX_UNITS + ul) * 3;
        cp_async4(xd, xp);
        cp_async4(xd + 1, xp + H);
        cp_async4(xd + 2, xp + 2 * H);
      }
    }
    gc_load_vec<CH>(vec, a.hprev + row0 * H, (int64_t)T * H, nrows, Bc, loader);
    __syncthreads();
    GC_PROF(0);
    // (no branch around the shuffles: warps past the last unit run on zero weights, which
    //  keeps every shuffle convergent and free of WARPSYNC.COLLECTIVE wrappers)
    for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
      float ar[GC_RB][GC_UPW], au[GC_RB][GC_UPW];
      gc_dot<CH>(vec, r0, lane, wr, ar);
      gc_dot<CH>(vec, r0, lane, wu, au);
      float v[2 * GC_RB * GC_UPW];  // index = gate*8 + row*4 + unit
#pragma unroll
      for (int r = 0; r < GC_RB; ++r)
#pragma unroll
        for (int u = 0; u < GC_UPW; ++u) {
          v[r * GC_UPW + u] = ar[r][u];
          v[GC_RB * GC_UPW + r * GC_UPW + u] = au[r][u];
        }
      gc_reduce_scatter<2 * GC_RB * GC_UPW>(v, lane);
      if ((lane & 1) == 0) {
        const int idx = lane >> 1, gate = idx >> 3, r = (idx >> 2) & 1, u = idx & 3;
        pre[((r0 + r) * GC_MAX_UNITS + unit0_local + u) * 2 + gate] = v[0];
      }
    }
    cp_async_commit_wait_all();
    __syncthreads();
    GC_PROF(1);
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, ul = idx - b * UW, j = rank * UW + ul;
      if (b >= nrows || j >= H) continue;
      const int64_t row = row0 + (int64_t)b * T;
      const float* xd = xs + (b * GC_MAX_UNITS + ul) * 3;
      const float rr = sigmoidf_(pre[(b * GC_MAX_UNITS + ul) * 2] + xd[0]);
      const float uu = sigmoidf_(pre[(b * GC_MAX_UNITS + ul) * 2 + 1] + xd[1]);
      const float hv = vec[b * ROW + (j / SL32) * GcGeom<CH>::SLP + (j % SL32)];
      a.gates[row * 3 * H + j] = rr;
      a.gates[row * 3 * H + H + j] = uu;
      a.rh[row * H + j] = rr * hv;
      own[(b * GC_MAX_UNITS + ul) * 2] = hv;
      own[(b * GC_MAX_UNITS + ul) * 2 + 1] = uu;
    }
    GC_PROF(2);
    cluster_barrier();
    GC_PROF(3);

    // ---- phase 2: c = tanh(xc + rh.Wch), h' = u*h + (1-u)*c ----
    gc_load_vec<CH>(vec, a.rh + row0 * H, (int64_t)T * H, nrows, Bc, loader);
    __syncthreads();
    GC_PROF(4);
    for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
      float ac[GC_RB][GC_UPW];
      gc_dot<CH>(vec, r0, lane, wc, ac);
      float v[GC_RB * GC_UPW];  // index = row*4 + unit
#pragma unroll
      for (int r = 0; r < GC_RB; ++r)
#pragma unroll
        for (int u = 0; u < GC_UPW; ++u) v[r * GC_UPW + u] = ac[r][u];
      gc_reduce_scatter<GC_RB * GC_UPW>(v, lane);
      if ((lane & 3) == 0) {
        const int idx = lane >> 2, r = idx >> 2, u = idx & 3;
        pre[((r0 + r) * GC_MAX_UNITS + unit0_local + u) * 2] = v[0];
      }
    }
    __syncthreads();
    GC_PROF(5);
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, ul = idx - b * UW, j = rank * UW + ul;
      if (b >= nrows || j >= H) continue;
      const int64_t row = row0 + (int64_t)b * T;
      const float c = tanhf(pre[(b * GC_MAX_UNITS + ul) * 2] + xs[(b * GC_MAX_UNITS + ul) * 3 + 2]);
      a.gates[row * 3 * H + 2 * H + j] = c;
      const float hv = own[(b * GC_MAX_UNITS + ul) * 2];
      const float uu = own[(b * GC_MAX_UNITS + ul) * 2 + 1];
      const bool live = (a.lengths == nullptr) || (t < a.lengths[b0 + b]);
      float hn = live ? (uu * hv + (1.f - uu) * c) : hv;
      if (a.raw_states) a.raw_states[row * H + j] = live ? hn : 0.f;
      if (a.drop_mask && live) hn *= a.drop_mask[row * H + j];
      a.states[row * H + j] = live ? hn : 0.f;
      if (last) a.final_state[(int64_t)(b0 + b) * H + j] = hn;
      else a.hprev[((int64_t)(b0 + b) * T + t_next) * H + j] = hn;
    }
    GC_PROF(6);
    cluster_barrier();
    GC_PROF(7);
#undef GC_PROF
  }
}

// ---------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------
struct GcBwdArgs {
  const float* Wgh;
  const float* Wch;
  const int32_t* lengths;
  const float* drop_mask;
  const float* gates;
  const float* hprev;
  const float* dstates;  // or null
  const float* draw;     // or null
  const float* dfinal;   // or null
  float* dxproj;         // [B,T,3H]
  float* dh0;            // or null
  int B, T, H, Bc, reverse;
};

template <int CH>
__global__ void __launch_bounds__(GC_THREADS, 1) gru_seq_bwd_cluster_kernel(GcBwdArgs a) {
  extern __shared__ __align__(16) float gc_smem[];
  constexpr int ROW = GcGeom<CH>::ROW;
  const int H = a.H, T = a.T, Bc = a.Bc;
  float* vec = gc_smem;                        // [Bc][ROW]  dz_c, then dz_r
  float* vec2 = vec + Bc * ROW;                // [Bc][ROW]  dz_u
  float* dcarry = vec2 + Bc * ROW;             // [Bc][GC_MAX_UNITS] grad of h'_t (own units)
  float* dhp = dcarry + Bc * GC_MAX_UNITS;     // [Bc][GC_MAX_UNITS]
  float* pre = dhp + Bc * GC_MAX_UNITS;        // [Bc][GC_MAX_UNITS] matmul results
  const int UW = (H + GC_CLUSTER - 1) / GC_CLUSTER;
  const int SL32 = (H + GC_SLICES - 1) / GC_SLICES;
  const int rank = (int)cluster_rank();
  const int b0 = (blockIdx.x / GC_CLUSTER) * Bc;
  const int nrows = min(Bc, a.B - b0);
  const GcLoader loader = gc_make_loader<CH>(H, SL32);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int unit0_local = warp * GC_UPW;
  const int unit0 = rank * UW + unit0_local;   // first OUTPUT unit i of this warp
  const int unit_limit = min(H, (rank + 1) * UW);

  // rows i of Wch / Wgh restricted to this lane's slice of the reduction index j
  float w1[GC_UPW][4 * CH], w2r[GC_UPW][4 * CH], w2u[GC_UPW][4 * CH];
  gc_load_w<CH>(w1, a.Wch, 1, H, unit0, H, unit_limit, lane * SL32, SL32, H);
  gc_load_w<CH>(w2r, a.Wgh, 1, 2 * H, unit0, H, unit_limit, lane * SL32, SL32, H);
  gc_load_w<CH>(w2u, a.Wgh + H, 1, 2 * H, unit0, H, unit_limit, lane * SL32, SL32, H);

  for (int i = threadIdx.x; i < 2 * Bc * ROW; i += GC_THREADS) vec[i] = 0.f;  // incl. vec2; see fwd
  for (int idx = threadIdx.x; idx < Bc * GC_MAX_UNITS; idx += GC_THREADS) {
    const int b = idx / GC_MAX_UNITS, ul = idx - b * GC_MAX_UNITS, j = rank * UW + ul;
    dcarry[idx] = (a.dfinal && b < nrows && ul < UW && j < H) ? a.dfinal[(int64_t)(b0 + b) * H + j] : 0.f;
  }
  __syncthreads();

  for (int step = T - 1; step >= 0; --step) {
    const int t = a.reverse ? T - 1 - step : step;
    const int64_t row0 = (int64_t)b0 * T + t;
    // ---- E1: gate gradients that need no matmul (own units) ----
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, ul = idx - b * UW, j = rank * UW + ul;
      if (b >= nrows || j >= H) continue;
      const int64_t row = row0 + (int64_t)b * T;
      const bool live = (a.lengths == nullptr) || (t < a.lengths[b0 + b]);
      float dh = dcarry[b * GC_MAX_UNITS + ul];
      if (!live) {
        a.dxproj[row * 3 * H + j] = 0.f;
        a.dxproj[row * 3 * H + H + j] = 0.f;
        a.dxproj[row * 3 * H + 2 * H + j] = 0.f;
        dhp[b * GC_MAX_UNITS + ul] = dh;
        continue;
      }
      const float uu = a.gates[row * 3 * H + H + j], c = a.gates[row * 3 * H + 2 * H + j];
      const float hv = a.hprev[row * H + j];
      if (a.dstates) dh += a.dstates[row * H + j];
      if (a.drop_mask) dh *= a.drop_mask[row * H + j];
      if (a.draw) dh += a.draw[row * H + j];
      const float du = dh * (hv - c);
      const float dc = dh * (1.f - uu);
      a.dxproj[row * 3 * H + 2 * H + j] = dc * (1.f - c * c);
      a.dxproj[row * 3 * H + H + j] = du * uu * (1.f - uu);
      dhp[b * GC_MAX_UNITS + ul] = dh * uu;
    }
    cluster_barrier();
    // ---- G1: drh = dz_c . Wch^T ; dz_r = drh*h*r*(1-r) ; dhp += drh*r ----
    gc_load_vec<CH>(vec, a.dxproj + row0 * 3 * H + 2 * H, (int64_t)T * 3 * H, nrows, Bc, loader);
    gc_load_vec<CH>(vec2, a.dxproj + row0 * 3 * H + H, (int64_t)T * 3 * H, nrows, Bc, loader);
    __syncthreads();
    for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
      float acc[GC_RB][GC_UPW];
      gc_dot<CH>(vec, r0, lane, w1, acc);
      float v[GC_RB * GC_UPW];
#pragma unroll
      for (int r = 0; r < GC_RB; ++r)
#pragma unroll
        for (int u = 0; u < GC_UPW; ++u) v[r * GC_UPW + u] = acc[r][u];
      gc_reduce_scatter<GC_RB * GC_UPW>(v, lane);
      if ((lane & 3) == 0) {
        const int idx = lane >> 2, r = idx >> 2, u = idx & 3;
        pre[(r0 + r) * GC_MAX_UNITS + unit0_local + u] = v[0];
      }
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, ul = idx - b * UW, i = rank * UW + ul;
      if (b >= nrows || i >= H) continue;
      const bool live = (a.lengths == nullptr) || (t < a.lengths[b0 + b]);
      if (!live) continue;
      const int64_t row = row0 + (int64_t)b * T;
      const float drh = pre[b * GC_MAX_UNITS + ul];
      const float rr = a.gates[row * 3 * H + i];
      const float hv = a.hprev[row * H + i];
      a.dxproj[row * 3 * H + i] = drh * hv * rr * (1.f - rr);
      dhp[b * GC_MAX_UNITS + ul] += drh * rr;
    }
    cluster_barrier();
    // ---- G2: dcarry = dhp + [dz_r, dz_u] . Wgh^T ----
    gc_load_vec<CH>(vec, a.dxproj + row0 * 3 * H, (int64_t)T * 3 * H, nrows, Bc, loader);
    __syncthreads();
    for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
      float accr[GC_RB][GC_UPW], accu[GC_RB][GC_UPW];
      gc_dot<CH>(vec, r0, lane, w2r, accr);
      gc_dot<CH>(vec2, r0, lane, w2u, accu);
      float v[GC_RB * GC_UPW];
#pragma unroll
      for (int r = 0; r < GC_RB; ++r)
#pragma unroll
        for (int u = 0; u < GC_UPW; ++u) v[r * GC_UPW + u] = accr[r][u] + accu[r][u];
      gc_reduce_scatter<GC_RB * GC_UPW>(v, lane);
      if ((lane & 3) == 0) {
        const int idx = lane >> 2, r = idx >> 2, u = idx & 3;
        pre[(r0 + r) * GC_MAX_UNITS + unit0_local + u] = v[0];
      }
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, ul = idx - b * UW;
      dcarry[b * GC_MAX_UNITS + ul] = dhp[b * GC_MAX_UNITS + ul] + pre[b * GC_MAX_UNITS + ul];
    }
    __syncthreads();  // dcarry/dhp/pre/vec are CTA-private: no cluster barrier needed here
  }
  if (a.dh0) {
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, ul = idx - b * UW, j = rank * UW + ul;
      if (b < nrows && j < H) a.dh0[(int64_t)(b0 + b) * H + j] = dcarry[b * GC_MAX_UNITS + ul];
    }
  }
}

}  // namespace nm
