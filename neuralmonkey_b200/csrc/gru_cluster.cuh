// Persistent GRU sequence kernels for thread-block clusters (sm_90a).
//
// One launch runs the whole time loop.  A cluster of 8 CTAs owns a slice of the batch
// (Bc sentences); inside it, CTA r owns hidden units [r*H/8, (r+1)*H/8): at least one each
// (H >= 8), at most ceil(H/8) <= 40, so every CTA sends its share of every exchanged vector.
// The recurrent weights never leave the SM: a warp owns 4 hidden units, and each of its
// 32 lanes keeps, in REGISTERS, the three weight vectors of those 4 units restricted to
// ONE of 32 reduction slices of SL = ceil(H/32) elements (3 * 4 * SL floats per thread, 120
// at H = 300).  The inner product streams only the state vector from shared memory in 16-,
// 8- or 4-byte pieces of exactly SL elements and is FMA-issue bound.  The 32 partial sums
// of a (row, unit) pair are combined with a reduce-scatter over shuffles.
//
// The two matmuls of a TF GRUCell step are dependent (the candidate needs r*h for ALL
// units).  The lanes that end up holding a reduced sum apply the gate math themselves; the
// four results of a warp's units in one row - r*h or h' forward, dz_c / dz_u / dz_r backward -
// are gathered into one lane per destination and written straight into the vector buffer of
// every CTA of the cluster as ONE 16-byte st.async, whose bytes are counted on a transaction
// mbarrier of the receiving CTA.  A CTA starts a phase as soon as its barrier has counted the
// whole Bc x H vector: no cluster-wide barrier and no L2 round trip in the loop.
// Write-after-read hazards are ordered by the dataflow itself: a peer can only send the next
// value of a buffer after it has received this CTA's contribution to the phase that follows
// the last read of that buffer; the buffers for which that is not enough (forward h,
// backward dz_u) alternate by step parity.  The saved activations (states, gates, hprev, rh,
// dxproj) go to global memory off the critical path.
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
constexpr int GC_MAX_SL = 10;   // ceil(320 / 32)
constexpr int GC_SMEM_CAP = 200 * 1024;  // dynamic shared memory a launch may plan for
constexpr int GC_BAR_BYTES = 64;  // transaction barriers at the start of dynamic shared memory
constexpr int GC_XS = 4;        // forward prefetch per (row, unit): xproj r, u, c and the dropout mask
constexpr int GC_PF = 8;        // backward prefetch per (row, unit): r, u, c, h, dstates, drop mask, draw

// Row pitch of the smem vector buffers in floats: 32 * 4 * (ceil(SL/4) | 1) >= the 32 * SL floats a
// row of the layout below uses.  The shared-memory plan, and with it the rows a cluster may take,
// is sized from it.
__host__ __device__ constexpr int gc_row(int SL) { return GC_SLICES * 4 * (((SL + 3) / 4) | 1); }
// floats of dynamic shared memory per batch row, after the barrier block
__host__ __device__ constexpr int gc_fwd_row_floats(int SL) {
  return 3 * gc_row(SL) + GC_MAX_UNITS * (1 + 2 * GC_XS) + 1;
}
__host__ __device__ constexpr int gc_bwd_row_floats(int SL) {
  return 4 * gc_row(SL) + GC_MAX_UNITS * (1 + 2 * GC_PF) + 1;
}

// Layout of an exchanged vector in a row: 8 rank regions of UP = 4*SL floats (UP >= ceil(H/8), a
// multiple of 4), local unit i of CTA r at r*UP + i, so the 4 units of warp w are the 16-byte aligned
// quad at r*UP + 4w.  Lane l's reduction slice is the SL consecutive floats at l*SL; positions past a
// CTA's units hold 0 in the buffers and in the weights.
// Slices are read in pieces of V floats, as wide as their alignment allows.  At SL = 8 the 16-byte
// pieces of lanes 4 apart fall on the same banks, so lanes with bit 2 set read their two pieces in
// the other order (the weights are loaded in the same order); every other SL is conflict-free as is.
template <int SL>
struct GcGeom {
  static constexpr int UP = 4 * SL;
  static constexpr int ROW = gc_row(SL);
  static constexpr int V = SL % 4 == 0 ? 4 : SL % 2 == 0 ? 2 : 1;
  // row offset of element e of lane `lane`'s slice
  static __device__ __forceinline__ int slice_pos(int lane, int e) {
    const int swz = SL == 8 ? ((lane >> 2) & 1) * 4 : 0;
    return lane * SL + (e ^ swz);
  }
};

__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::
                   : "memory");
}
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

// --- transaction barriers and distributed shared memory --------------------------------
__device__ __forceinline__ uint32_t gc_smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void gc_mbar_init(uint32_t bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// One local arrival that also expects `bytes` of st.async data for the barrier's current phase.
// Data may arrive before it (the transaction count goes negative); the phase completes when both
// the arrival and all the bytes are in.
__device__ __forceinline__ void gc_mbar_arm(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gc_mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
// Store v at shared-memory address `addr` of CTA `dst` of the cluster (the same layout in every
// CTA); the 4 bytes are counted on that CTA's barrier at `bar`.
__device__ __forceinline__ void gc_send(uint32_t addr, uint32_t bar, uint32_t dst, float v) {
  uint32_t ra, rb;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(addr), "r"(dst));
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(bar), "r"(dst));
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(ra),
               "r"(__float_as_uint(v)), "r"(rb)
               : "memory");
}
// The same for the 16-byte aligned quad v at `addr`: one message of 16 bytes.
__device__ __forceinline__ void gc_send4(uint32_t addr, uint32_t bar, uint32_t dst, const float (&v)[4]) {
  uint32_t ra, rb;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(addr), "r"(dst));
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(bar), "r"(dst));
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::
                   "r"(ra), "r"(__float_as_uint(v[0])), "r"(__float_as_uint(v[1])), "r"(__float_as_uint(v[2])),
               "r"(__float_as_uint(v[3])), "r"(rb)
               : "memory");
}
// q[u] = x of lane (L & KEEP) | (STRIDE * u), u = 0..3, for the calling lane L: the quad a sending lane
// passes to gc_send4.  KEEP is the segment mask of shfl.sync, which may be any set of lane bits; with
// the source lane an immediate, the shuffles hold no index registers.
template <int KEEP, int SRC>
__device__ __forceinline__ float gc_shfl_keep(float x) {
  uint32_t o;
  asm volatile("shfl.sync.idx.b32 %0, %1, %2, %3, 0xffffffff;"
               : "=r"(o)
               : "r"(__float_as_uint(x)), "n"(SRC), "n"((KEEP << 8) | 0x1f));
  return __uint_as_float(o);
}
template <int KEEP, int STRIDE>
__device__ __forceinline__ void gc_gather4(float (&q)[4], float x) {
  static_assert((KEEP & (3 * STRIDE)) == 0, "the unit bits of the source lane come from STRIDE * u");
  q[0] = gc_shfl_keep<KEEP, 0>(x);
  q[1] = gc_shfl_keep<KEEP, STRIDE>(x);
  q[2] = gc_shfl_keep<KEEP, 2 * STRIDE>(x);
  q[3] = gc_shfl_keep<KEEP, 3 * STRIDE>(x);
}
// Bytes of one exchanged Bc x H vector as the live warps of the 8 CTAs send it: per row, one quad
// per live warp, ceil(UW_r / 4) of them in CTA r.  Recomputed from the kernel parameters where it is
// used, so that it holds no register across the step loop (the SL = 10 instance is at the
// 168-register cap).
__device__ __forceinline__ uint32_t gc_quad_bytes(int H, int Bc) {
  int quads = 0;
#pragma unroll
  for (int r = 0; r < GC_CLUSTER; ++r) quads += ((r + 1) * H / GC_CLUSTER - r * H / GC_CLUSTER + 3) / 4;
  return (uint32_t)(Bc * 16 * quads);
}

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
  const uint32_t d = gc_smem_u32(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Sum N values (index = gate*8 + row*4 + unit) across the 32 lanes with N-1+log2(32/N)...
// shuffles instead of 5N: each butterfly level halves the number of live values.  On return v[0]
// of lane L is the full sum of the value with index (L >> (5 - log2 N)) & (N-1); lanes differing
// only in the low bits hold copies.  At the row level, lanes whose bit `O` is set keep the upper
// half and send the lower, and vice versa.  At the gate and unit levels every lane keeps the lower
// half: that sums matching values because the caller permutes the slots there - slot g*8 + r*4 + u
// holds gate g ^ g_L and unit u ^ u_L, the ones lane L ends up with - where the weights are loaded,
// so those levels cost no select.
// One butterfly level per instantiation, O = shuffle distance (a loop over the levels is not
// always unrolled, and a rolled loop indexes v at run time, which puts v in local memory).
template <int N, int O>
__device__ __forceinline__ void gc_reduce_level(float (&v)[N], int lane) {
  constexpr int n = N * O / 16;  // values still live at this level
  if constexpr (n == 2 * GC_UPW) {  // the row level
    const bool upper = (lane & O) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float keep = upper ? v[i + n / 2] : v[i];
      const float send = upper ? v[i] : v[i + n / 2];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
    }
  } else if constexpr (n > 1) {
#pragma unroll
    for (int i = 0; i < n / 2; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i + n / 2], O);
  } else {
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], O);
  }
  if constexpr (O > 1) gc_reduce_level<N, O / 2>(v, lane);
}
template <int N>
__device__ __forceinline__ void gc_reduce_scatter(float (&v)[N], int lane) {
  static_assert(N == GC_RB * GC_UPW || N == 2 * GC_RB * GC_UPW, "gate, row and unit index bits");
  gc_reduce_level<N, 16>(v, lane);
}

// acc[r][u] = partial (this lane's slice) of sum_k vec[row0+r][k] * w[u][k], over exactly the SL
// elements of the slice, in pieces of GcGeom<SL>::V floats
template <int SL>
__device__ __forceinline__ void gc_dot(const float* __restrict__ vec, int row0, int lane,
                                       const float (&w)[GC_UPW][SL], float (&acc)[GC_RB][GC_UPW]) {
  constexpr int V = GcGeom<SL>::V;
#pragma unroll
  for (int r = 0; r < GC_RB; ++r)
#pragma unroll
    for (int u = 0; u < GC_UPW; ++u) acc[r][u] = 0.f;
  const float* base = vec + row0 * GcGeom<SL>::ROW;
#pragma unroll
  for (int c = 0; c < SL; c += V) {
#pragma unroll
    for (int r = 0; r < GC_RB; ++r) {
      const float* p = base + r * GcGeom<SL>::ROW + GcGeom<SL>::slice_pos(lane, c);
      float x[V];
      if constexpr (V == 4) {
        const float4 q = *reinterpret_cast<const float4*>(p);
        x[0] = q.x; x[1] = q.y; x[2] = q.z; x[3] = q.w;
      } else if constexpr (V == 2) {
        const float2 q = *reinterpret_cast<const float2*>(p);
        x[0] = q.x; x[1] = q.y;
      } else {
        x[0] = p[0];
      }
#pragma unroll
      for (int u = 0; u < GC_UPW; ++u)
#pragma unroll
        for (int i = 0; i < V; ++i) acc[r][u] = fmaf(x[i], w[u][c + i], acc[r][u]);
    }
  }
}

// Load this lane's slice of column (or row) vectors of a weight matrix for the warp's 4
// units: w[u][e] = W[k*sk + (unit0 + (u ^ usw))*su] with k the hidden unit at slice position e of
// the vector layout, zero at padding positions or past the CTA's units (usw permutes the units:
// see gc_reduce_scatter).
template <int SL>
__device__ __forceinline__ void gc_load_w(float (&w)[GC_UPW][SL], const float* __restrict__ W,
                                          int64_t sk, int64_t su, int unit0, int usw, int unit_limit, int lane,
                                          int H) {
  const int r = lane >> 2;  // UP = 4 * SL: the slice lies inside the region of CTA lane / 4
  const int k0 = r * H / GC_CLUSTER - r * GcGeom<SL>::UP, k_end = (r + 1) * H / GC_CLUSTER;
#pragma unroll
  for (int e = 0; e < SL; ++e) {
    const int k = k0 + GcGeom<SL>::slice_pos(lane, e);
    const bool k_ok = k < k_end;
#pragma unroll
    for (int u = 0; u < GC_UPW; ++u) {
      const int unit = unit0 + (u ^ usw);
      w[u][e] = (k_ok && unit < unit_limit) ? W[(int64_t)k * sk + (int64_t)unit * su] : 0.f;
    }
  }
}

// Per-phase cycle counters of thread 0 of CTA 0 (diagnostics; see nm_gru_debug_profile).  The
// running timestamp is a 32-bit clock() (differences are exact across a wrap) and the counters
// are read from the kernel parameters, so profiling costs two registers in the step loop.
struct GcProf {
  bool on;
  unsigned t0;
  __device__ __forceinline__ explicit GcProf(const long long* out)
      : on(out != nullptr && blockIdx.x == 0 && threadIdx.x == 0), t0(on ? (unsigned)clock() : 0u) {}
  __device__ __forceinline__ void lap(long long* out, int slot) {
    if (on) {
      const unsigned t1 = (unsigned)clock();
      out[slot] += (long long)(t1 - t0);
      t0 = t1;
    }
  }
};

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

// Asynchronous copies of step t's xproj (and dropout mask) of the own units into the prefetch slot
// `dst` ([Bc][GC_MAX_UNITS][GC_XS]); they land while the previous step computes.
__device__ __forceinline__ void gc_fwd_prefetch(const GcFwdArgs& a, int t, float* dst, int b0, int nrows,
                                                int ubeg, int UW) {
  const int H = a.H, T = a.T;
  for (int idx = threadIdx.x; idx < a.Bc * UW; idx += GC_THREADS) {
    const int b = idx / UW, ul = idx - b * UW, j = ubeg + ul;
    if (b < nrows && j < H) {
      const int64_t row = ((int64_t)(b0 + b) * T + t);
      const float* xp = a.xproj + row * 3 * H + j;
      float* xd = dst + (b * GC_MAX_UNITS + ul) * GC_XS;
      cp_async4(xd, xp);
      cp_async4(xd + 1, xp + H);
      cp_async4(xd + 2, xp + 2 * H);
      if (a.drop_mask) cp_async4(xd + 3, a.drop_mask + row * H + j);
    }
  }
  cp_async_commit();
}

template <int SL>
__global__ void __launch_bounds__(GC_THREADS, 1) gru_seq_fwd_cluster_kernel(GcFwdArgs a) {
  extern __shared__ __align__(16) float gc_smem[];
  constexpr int ROW = GcGeom<SL>::ROW;
  const int H = a.H, T = a.T, Bc = a.Bc;
  float* hbuf = gc_smem + GC_BAR_BYTES / 4;          // [2][Bc][ROW]: h by step parity
  float* rhbuf = hbuf + 2 * Bc * ROW;                // [Bc][ROW]: r*h
  float* us = rhbuf + Bc * ROW;                      // [Bc][GC_MAX_UNITS]: update gate of own units
  float* xs = us + Bc * GC_MAX_UNITS;                // [2][Bc][GC_MAX_UNITS][GC_XS] by step parity
  int* lens = reinterpret_cast<int*>(xs + 2 * Bc * GC_MAX_UNITS * GC_XS);  // [Bc]; 0 for padding rows
  const uint32_t bar_h = gc_smem_u32(gc_smem), bar_rh = bar_h + 16;      // bar_h + 8*parity

  const int rank = (int)cluster_rank();
  const int ubeg = rank * H / GC_CLUSTER;             // first hidden unit of this CTA
  const int unit_limit = (rank + 1) * H / GC_CLUSTER;
  const int UW = unit_limit - ubeg;                   // units of this CTA
  const int b0 = (blockIdx.x / GC_CLUSTER) * Bc;
  const int nrows = min(Bc, a.B - b0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int unit0_local = warp * GC_UPW;
  const int unit0 = ubeg + unit0_local;               // first hidden unit of this warp
  const bool warp_live = unit0 < unit_limit;

  // The (row, unit) result this lane holds after each reduce-scatter, fixed for the kernel.
  // Phase 1: 16 values (gate, row, unit), 2 copies; phase 2: 8 values (row, unit), 4 copies.
  const int g1 = lane >> 4, r1 = (lane >> 3) & 1, u1 = (lane >> 1) & 3;
  const int r2 = (lane >> 4) & 1, u2 = (lane >> 2) & 3, copy2 = lane & 3;
  // the slot order gc_reduce_scatter needs: gate g1 first, units permuted by the held ones
  float wg[2][GC_UPW][SL], wc[GC_UPW][SL];
  gc_load_w<SL>(wg[0], a.Wgh + g1 * H, 2 * H, 1, unit0, u1, unit_limit, lane, H);
  gc_load_w<SL>(wg[1], a.Wgh + (g1 ^ 1) * H, 2 * H, 1, unit0, u1, unit_limit, lane, H);
  gc_load_w<SL>(wc, a.Wch, H, 1, unit0, u2, unit_limit, lane, H);
  const bool ok1 = unit0 + u1 < unit_limit, ok2 = unit0 + u2 < unit_limit;
  const int j1 = unit0 + u1, j2 = unit0 + u2;
  // the own unit in a row of every CTA; pos & ~3 is the warp's quad
  const int pos1 = rank * GcGeom<SL>::UP + unit0_local + u1, pos2 = rank * GcGeom<SL>::UP + unit0_local + u2;

  if (threadIdx.x == 0) {
    gc_mbar_init(bar_h);
    gc_mbar_init(bar_h + 8);
    gc_mbar_init(bar_rh);
    gc_mbar_arm(bar_h, (uint32_t)(Bc * H * 4));  // the h0 seed below comes in 4-byte messages
    gc_mbar_arm(bar_h + 8, gc_quad_bytes(H, Bc));
    gc_mbar_arm(bar_rh, gc_quad_bytes(H, Bc));
  }
  // Positions past a CTA's units are only written as 0 (or not at all): they must be 0, not stale
  // shared memory; padding rows (and units of the prefetch that are never loaded) stay 0 as well.
  for (int i = threadIdx.x; i < 3 * Bc * ROW; i += GC_THREADS) hbuf[i] = 0.f;
  for (int i = threadIdx.x; i < 2 * Bc * GC_MAX_UNITS * GC_XS; i += GC_THREADS) xs[i] = 0.f;
  for (int b = threadIdx.x; b < Bc; b += GC_THREADS)
    lens[b] = b < nrows ? (a.lengths ? a.lengths[b0 + b] : T) : 0;


  __syncthreads();
  cluster_barrier();  // every CTA's barriers are initialised and its buffers zeroed before anyone sends
  // seed: the state history slot of the first step gets h0, and the h0 slice of the own units goes
  // to h buffer 0 of every CTA
  const int t_first = a.reverse ? T - 1 : 0;
  for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
    const int b = idx / UW, ul = idx - b * UW, j = ubeg + ul;
    const float hv = (b < nrows && a.h0) ? a.h0[(int64_t)(b0 + b) * H + j] : 0.f;
    if (b < nrows) a.hprev[((int64_t)(b0 + b) * T + t_first) * H + j] = hv;
    const uint32_t addr = gc_smem_u32(hbuf + b * ROW + rank * GcGeom<SL>::UP + ul);
    for (int d = 0; d < GC_CLUSTER; ++d) gc_send(addr, bar_h, d, hv);
  }
  gc_fwd_prefetch(a, t_first, xs, b0, nrows, ubeg, UW);

  GcProf prof(a.prof);
  for (int step = 0; step < T; ++step) {
    const int t = a.reverse ? T - 1 - step : step;
    const bool last = (step == T - 1);
    const int t_next = a.reverse ? t - 1 : t + 1;
    const int64_t row0 = (int64_t)b0 * T + t;  // row index of batch row b0 at time t; +b*T per row
    const int par = step & 1;
    const float* hb = hbuf + par * Bc * ROW;
    const float* xc = xs + par * Bc * GC_MAX_UNITS * GC_XS;

    gc_mbar_wait(bar_h + 8 * par, (step >> 1) & 1);
    if (threadIdx.x == 0 && step + 2 < T) gc_mbar_arm(bar_h + 8 * par, gc_quad_bytes(H, Bc));
    prof.lap(a.prof, 0);
    cp_async_wait_all();
    __syncthreads();  // this step's xproj is in; every warp is done with the previous step
    if (!last) gc_fwd_prefetch(a, t_next, xs + (par ^ 1) * Bc * GC_MAX_UNITS * GC_XS, b0, nrows, ubeg, UW);
    prof.lap(a.prof, 1);

    // ---- phase 1: [r,u] = sigmoid(xg + h.Wgh), r*h -> every CTA ----
    // (warps past the last unit skip the loop as a whole, which keeps every shuffle convergent)
    if (warp_live) {
      for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
        float a0[GC_RB][GC_UPW], a1[GC_RB][GC_UPW];
        gc_dot<SL>(hb, r0, lane, wg[0], a0);
        gc_dot<SL>(hb, r0, lane, wg[1], a1);
        float v[2 * GC_RB * GC_UPW];  // slot = gate*8 + row*4 + unit, gate and unit ^ the held ones
#pragma unroll
        for (int r = 0; r < GC_RB; ++r)
#pragma unroll
          for (int u = 0; u < GC_UPW; ++u) {
            v[r * GC_UPW + u] = a0[r][u];
            v[GC_RB * GC_UPW + r * GC_UPW + u] = a1[r][u];
          }
        gc_reduce_scatter<2 * GC_RB * GC_UPW>(v, lane);
        const int b = r0 + r1, ul = unit0_local + u1;
        const float g = sigmoidf_(v[0] + xc[(b * GC_MAX_UNITS + ul) * GC_XS + g1]);
        const float rhv = ok1 ? g * hb[b * ROW + pos1] : 0.f;  // 0 in the quad's padding slots
        // lane L < 16 sends the r*h quad of row r1 (lanes (L & 8) | 2u hold it) to CTA L & 7, before the
        // stores that nothing in the cluster waits for
        // (the shuffles run on every lane: a shuffle skipped by some lanes of its mask never completes)
        float q[4];
        gc_gather4<0x18, 2>(q, rhv);
        if (lane < 16) gc_send4(gc_smem_u32(rhbuf + b * ROW + (pos1 & ~3)), bar_rh, lane & 7, q);
        if (ok1 && (lane & 1) == 0) {
          if (b < nrows) {
            const int64_t row = row0 + (int64_t)b * T;
            a.gates[row * 3 * H + g1 * H + j1] = g;
            if (g1 == 0) a.rh[row * H + j1] = rhv;
          }
          if (g1 == 1) us[b * GC_MAX_UNITS + ul] = g;
        }
      }
      __syncwarp();
    }
    prof.lap(a.prof, 2);
    gc_mbar_wait(bar_rh, step & 1);
    if (threadIdx.x == 0 && !last) gc_mbar_arm(bar_rh, gc_quad_bytes(H, Bc));
    prof.lap(a.prof, 3);

    // ---- phase 2: c = tanh(xc + rh.Wch), h' = u*h + (1-u)*c -> every CTA ----
    if (warp_live) {
      const uint32_t bar_next = bar_h + 8 * (par ^ 1);
      float* hn_buf = hbuf + (par ^ 1) * Bc * ROW;
      // the four copies of a (row, unit) share its stores: copy 0 the candidate gate, 1 the state, 2 the raw
      // state, 3 the next state; `out` is the copy's element for row b0, `out_step` the step between rows
      float* out;
      int64_t out_step = (int64_t)T * H;
      if (copy2 == 0) {
        out = a.gates + row0 * 3 * H + 2 * H + j2;
        out_step = (int64_t)T * 3 * H;
      } else if (copy2 == 1) {
        out = a.states + row0 * H + j2;
      } else if (copy2 == 2) {
        out = a.raw_states ? a.raw_states + row0 * H + j2 : nullptr;
      } else if (last) {
        out = a.final_state + (int64_t)b0 * H + j2;
        out_step = H;
      } else {
        out = a.hprev + ((int64_t)b0 * T + t_next) * H + j2;
      }
      for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
        float ac[GC_RB][GC_UPW];
        gc_dot<SL>(rhbuf, r0, lane, wc, ac);
        float v[GC_RB * GC_UPW];  // slot = row*4 + unit, unit ^ the held one
#pragma unroll
        for (int r = 0; r < GC_RB; ++r)
#pragma unroll
          for (int u = 0; u < GC_UPW; ++u) v[r * GC_UPW + u] = ac[r][u];
        gc_reduce_scatter<GC_RB * GC_UPW>(v, lane);
        const int b = r0 + r2, ul = unit0_local + u2;
        const float* xd = xc + (b * GC_MAX_UNITS + ul) * GC_XS;
        const float c = tanhf(v[0] + xd[2]);
        const float hv = hb[b * ROW + pos2];
        const float uu = us[b * GC_MAX_UNITS + ul];
        const bool live = t < lens[b];
        float hn = live ? (uu * hv + (1.f - uu) * c) : hv;
        const float raw = live ? hn : 0.f;
        // the decoder feeds the DROPPED-OUT cell output back as the next state
        if (a.drop_mask && live) hn *= xd[3];
        if (!last) {  // lane L with bit 3 clear sends the h' quad of row r2 (lanes (L & 16) | 4u) to CTA L & 7
          float q[4];
          gc_gather4<0x10, 4>(q, ok2 ? hn : 0.f);
          if ((lane & 8) == 0) gc_send4(gc_smem_u32(hn_buf + b * ROW + (pos2 & ~3)), bar_next, lane & 7, q);
        }
        if (ok2 && b < nrows && out) {
          const float val = copy2 == 0 ? c : copy2 == 1 ? (live ? hn : 0.f) : copy2 == 2 ? raw : hn;
          out[b * out_step] = val;
        }
      }
    }
    prof.lap(a.prof, 4);
  }
  cluster_barrier();  // no CTA leaves while a peer may still address its shared memory
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
  long long* prof;       // optional [8] cycle counters of CTA 0 (diagnostics), or null
};

// E1: gate gradients that need no matmul, for one (row, unit): dh = carry (+ dstates, dropout,
// + draw on live rows); returns the part of dh_prev that bypasses the matmuls (dh*u).
// pf = the prefetched (r, u, c, h, dstates, drop mask, draw) of the item.
__device__ __forceinline__ float gc_bwd_e1(const GcBwdArgs& a, const float* pf, float dh, bool live,
                                           float& zc, float& zu) {
  if (!live) {
    zc = zu = 0.f;
    return dh;
  }
  const float uu = pf[1], c = pf[2], hv = pf[3];
  if (a.dstates) dh += pf[4];
  if (a.drop_mask) dh *= pf[5];
  if (a.draw) dh += pf[6];
  const float du = dh * (hv - c);
  const float dc = dh * (1.f - uu);
  zc = dc * (1.f - c * c);
  zu = du * uu * (1.f - uu);
  return dh * uu;
}

// Asynchronous copies of step t's gates, hprev and incoming gradients of the own units, live rows
// only, into the prefetch slot `dst` ([Bc][GC_MAX_UNITS][GC_PF]).
__device__ __forceinline__ void gc_bwd_prefetch(const GcBwdArgs& a, int t, float* dst, const int* lens, int b0,
                                                int ubeg, int UW) {
  const int H = a.H, T = a.T;
  for (int idx = threadIdx.x; idx < a.Bc * UW; idx += GC_THREADS) {
    const int b = idx / UW, u = idx - b * UW, j = ubeg + u;
    if (t >= lens[b]) continue;
    const int64_t row = (int64_t)(b0 + b) * T + t;
    float* d = dst + (b * GC_MAX_UNITS + u) * GC_PF;
    const float* g = a.gates + row * 3 * H + j;
    cp_async4(d, g);
    cp_async4(d + 1, g + H);
    cp_async4(d + 2, g + 2 * H);
    cp_async4(d + 3, a.hprev + row * H + j);
    if (a.dstates) cp_async4(d + 4, a.dstates + row * H + j);
    if (a.drop_mask) cp_async4(d + 5, a.drop_mask + row * H + j);
    if (a.draw) cp_async4(d + 6, a.draw + row * H + j);
  }
  cp_async_commit();
}

template <int SL>
__global__ void __launch_bounds__(GC_THREADS, 1) gru_seq_bwd_cluster_kernel(GcBwdArgs a) {
  extern __shared__ __align__(16) float gc_smem[];
  constexpr int ROW = GcGeom<SL>::ROW;
  const int H = a.H, T = a.T, Bc = a.Bc;
  float* vc = gc_smem + GC_BAR_BYTES / 4;       // [Bc][ROW]     dz_c
  float* vu = vc + Bc * ROW;                    // [2][Bc][ROW]  dz_u by step parity
  float* vr = vu + 2 * Bc * ROW;                // [Bc][ROW]     dz_r
  float* dhp = vr + Bc * ROW;                   // [Bc][GC_MAX_UNITS] part of dh_prev that bypasses the matmuls
  float* pf = dhp + Bc * GC_MAX_UNITS;          // [2][Bc][GC_MAX_UNITS][GC_PF] by step parity
  int* lens = reinterpret_cast<int*>(pf + 2 * Bc * GC_MAX_UNITS * GC_PF);  // [Bc]; 0 for padding rows
  const uint32_t bar_a = gc_smem_u32(gc_smem), bar_b = bar_a + 16;     // bar_a + 8*parity: dz_c + dz_u

  const int rank = (int)cluster_rank();
  const int ubeg = rank * H / GC_CLUSTER;      // first hidden unit of this CTA
  const int unit_limit = (rank + 1) * H / GC_CLUSTER;
  const int UW = unit_limit - ubeg;
  const int b0 = (blockIdx.x / GC_CLUSTER) * Bc;
  const int nrows = min(Bc, a.B - b0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int unit0_local = warp * GC_UPW;
  const int unit0 = ubeg + unit0_local;        // first OUTPUT unit i of this warp
  const bool warp_live = unit0 < unit_limit;

  // the (row, unit) this lane holds after a reduce-scatter of 8 values, and its copy index
  const int rr_ = (lane >> 4) & 1, uq = (lane >> 2) & 3, copy = lane & 3;
  // rows i of Wch / Wgh restricted to this lane's slice of the reduction index j, the units in the
  // slot order of gc_reduce_scatter
  float w1[GC_UPW][SL], w2r[GC_UPW][SL], w2u[GC_UPW][SL];
  gc_load_w<SL>(w1, a.Wch, 1, H, unit0, uq, unit_limit, lane, H);
  gc_load_w<SL>(w2r, a.Wgh, 1, 2 * H, unit0, uq, unit_limit, lane, H);
  gc_load_w<SL>(w2u, a.Wgh + H, 1, 2 * H, unit0, uq, unit_limit, lane, H);
  const bool ok = unit0 + uq < unit_limit;
  const int ji = unit0 + uq, ul = unit0_local + uq;
  const int quad = rank * GcGeom<SL>::UP + unit0_local;  // the warp's units in a row of every CTA
  // time of the k-th step processed
  auto time_of = [reverse = a.reverse, T](int k) { return reverse ? k : T - 1 - k; };

  if (threadIdx.x == 0) {
    gc_mbar_init(bar_a);
    gc_mbar_init(bar_a + 8);
    gc_mbar_init(bar_b);
    gc_mbar_arm(bar_a, (uint32_t)(2 * Bc * H * 4));  // the E1 seed below comes in 4-byte messages
    gc_mbar_arm(bar_a + 8, 2 * gc_quad_bytes(H, Bc));
    gc_mbar_arm(bar_b, gc_quad_bytes(H, Bc));
  }
  for (int i = threadIdx.x; i < 4 * Bc * ROW; i += GC_THREADS) vc[i] = 0.f;  // vc, vu, vr; see fwd
  for (int i = threadIdx.x; i < 2 * Bc * GC_MAX_UNITS * GC_PF; i += GC_THREADS) pf[i] = 0.f;
  for (int b = threadIdx.x; b < Bc; b += GC_THREADS)
    lens[b] = b < nrows ? (a.lengths ? a.lengths[b0 + b] : T) : 0;
  __syncthreads();


  gc_bwd_prefetch(a, time_of(0), pf, lens, b0, ubeg, UW);
  cp_async_wait_all();
  __syncthreads();
  cluster_barrier();  // every CTA's barriers are initialised and its buffers zeroed before anyone sends
  {  // E1 of the first step processed, from dfinal
    const int t = time_of(0);
    for (int idx = threadIdx.x; idx < Bc * UW; idx += GC_THREADS) {
      const int b = idx / UW, u = idx - b * UW, j = ubeg + u;
      const bool live = t < lens[b];
      const float dh = (a.dfinal && b < nrows) ? a.dfinal[(int64_t)(b0 + b) * H + j] : 0.f;
      float zc, zu;
      dhp[b * GC_MAX_UNITS + u] = gc_bwd_e1(a, pf + (b * GC_MAX_UNITS + u) * GC_PF, dh, live, zc, zu);
      if (b < nrows) {
        const int64_t row = (int64_t)(b0 + b) * T + t;
        a.dxproj[row * 3 * H + H + j] = zu;
        a.dxproj[row * 3 * H + 2 * H + j] = zc;
      }
      const int p = rank * GcGeom<SL>::UP + u;
      const uint32_t ac = gc_smem_u32(vc + b * ROW + p), au = gc_smem_u32(vu + b * ROW + p);
      for (int d = 0; d < GC_CLUSTER; ++d) {
        gc_send(ac, bar_a, d, zc);
        gc_send(au, bar_a, d, zu);
      }
    }
  }

  GcProf prof(a.prof);
  for (int k = 0; k < T; ++k) {
    const int t = time_of(k);
    const bool last = (k == T - 1);
    const int64_t row0 = (int64_t)b0 * T + t;
    const int par = k & 1;
    const float* pfc = pf + par * Bc * GC_MAX_UNITS * GC_PF;
    float* pfn = pf + (par ^ 1) * Bc * GC_MAX_UNITS * GC_PF;

    gc_mbar_wait(bar_a + 8 * par, (k >> 1) & 1);
    if (threadIdx.x == 0 && k + 2 < T) gc_mbar_arm(bar_a + 8 * par, 2 * gc_quad_bytes(H, Bc));
    prof.lap(a.prof, 0);
    __syncthreads();  // every warp is done with the previous step (and its prefetch slot)
    if (!last) gc_bwd_prefetch(a, time_of(k + 1), pfn, lens, b0, ubeg, UW);
    prof.lap(a.prof, 1);

    // ---- G1: drh = dz_c . Wch^T ; dz_r = drh*h*r*(1-r) ; dhp += drh*r -> dz_r to every CTA ----
    if (warp_live) {
      for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
        float acc[GC_RB][GC_UPW];
        gc_dot<SL>(vc, r0, lane, w1, acc);
        float v[GC_RB * GC_UPW];
#pragma unroll
        for (int r = 0; r < GC_RB; ++r)
#pragma unroll
          for (int u = 0; u < GC_UPW; ++u) v[r * GC_UPW + u] = acc[r][u];
        gc_reduce_scatter<GC_RB * GC_UPW>(v, lane);
        const int b = r0 + rr_;
        const float drh = v[0];
        const bool live = t < lens[b];
        const float* s = pfc + (b * GC_MAX_UNITS + ul) * GC_PF;
        const float rg = s[0], hv = s[3];
        const float zr = (ok && live) ? drh * hv * rg * (1.f - rg) : 0.f;  // 0 in the quad's padding slots
        if (ok && copy == 0) {
          if (b < nrows) a.dxproj[(row0 + (int64_t)b * T) * 3 * H + ji] = zr;
          if (live) dhp[b * GC_MAX_UNITS + ul] += drh * rg;
        }
        // lane L with bit 3 clear sends the dz_r quad of row rr_ (lanes (L & 16) | 4u) to CTA L & 7
        float q[4];
        gc_gather4<0x10, 4>(q, zr);
        if ((lane & 8) == 0) gc_send4(gc_smem_u32(vr + b * ROW + quad), bar_b, lane & 7, q);
      }
      __syncwarp();
    }
    prof.lap(a.prof, 2);
    gc_mbar_wait(bar_b, k & 1);
    if (threadIdx.x == 0 && !last) gc_mbar_arm(bar_b, gc_quad_bytes(H, Bc));
    prof.lap(a.prof, 3);
    cp_async_wait_all();
    __syncthreads();  // the next step's prefetch is in
    prof.lap(a.prof, 4);

    // ---- G2: dcarry = dhp + [dz_r, dz_u] . Wgh^T, then E1 of the next step -> dz_c, dz_u ----
    if (warp_live) {
      const float* vuc = vu + par * Bc * ROW;
      float* const send_buf = (lane & 2) ? vu + (par ^ 1) * Bc * ROW : vc;  // dz_u or dz_c (see below)
      const int tn = last ? t : time_of(k + 1);
      for (int r0 = 0; r0 < Bc; r0 += GC_RB) {
        float accr[GC_RB][GC_UPW], accu[GC_RB][GC_UPW];
        gc_dot<SL>(vr, r0, lane, w2r, accr);
        gc_dot<SL>(vuc, r0, lane, w2u, accu);
        float v[GC_RB * GC_UPW];
#pragma unroll
        for (int r = 0; r < GC_RB; ++r)
#pragma unroll
          for (int u = 0; u < GC_UPW; ++u) v[r * GC_UPW + u] = accr[r][u] + accu[r][u];
        gc_reduce_scatter<GC_RB * GC_UPW>(v, lane);
        const int b = r0 + rr_;
        const float dcarry = ok ? dhp[b * GC_MAX_UNITS + ul] + v[0] : 0.f;
        __syncwarp();  // every copy has read dhp before copy 0 replaces it
        if (last) {
          if (ok && a.dh0 && copy == 0 && b < nrows) a.dh0[(int64_t)(b0 + b) * H + ji] = dcarry;
          continue;
        }
        float zc, zu;
        const float d = gc_bwd_e1(a, pfn + (b * GC_MAX_UNITS + ul) * GC_PF, dcarry, tn < lens[b], zc, zu);
        if (ok) {
          if (b < nrows) {
            const int64_t row = (int64_t)(b0 + b) * T + tn;
            if (copy == 1) a.dxproj[row * 3 * H + H + ji] = zu;
            else if (copy == 2) a.dxproj[row * 3 * H + 2 * H + ji] = zc;
          }
          if (copy == 0) dhp[b * GC_MAX_UNITS + ul] = d;
        }
        // copies 0, 1 pass on dz_c and copies 2, 3 dz_u; lane L sends the dz_c (bit 1 clear) or dz_u quad
        // of row rr_ (lanes (L & 18) | 4u) to CTA ((L >> 1) & 6) | (L & 1): all 32 lanes one message each
        float q[4];
        gc_gather4<0x12, 4>(q, ok ? (copy & 2 ? zu : zc) : 0.f);
        gc_send4(gc_smem_u32(send_buf + b * ROW + quad), bar_a + 8 * (par ^ 1), ((lane >> 1) & 6) | (lane & 1), q);
      }
    }
    prof.lap(a.prof, 5);
  }
  cluster_barrier();  // no CTA leaves while a peer may still address its shared memory
}

}  // namespace nm
