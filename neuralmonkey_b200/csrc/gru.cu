// K2: TF-1.12 GRUCell over a whole sequence (forward and backward through time).
//
// The input half of both cell matmuls is hoisted out of the recurrence by the
// host (one tensor-core GEMM over all B*T rows, see nm_gemm); what remains per
// step is the recurrent half, which is kept in exact fp32 on the CUDA cores:
//     [r,u] = sigmoid(xg_t + h.Wgh) ; c = tanh(xc_t + (r*h).Wch) ; h' = u*h + (1-u)*c
// (reference: tf.contrib.rnn.GRUCell as used by nn/ortho_gru_cell.py:44-53,
//  encoders/recurrent.py:82-95, decoders/decoder.py:283-289).
// Each step is two fused GEMM+gate kernels forward and one gate kernel plus two
// fused GEMM kernels backward; the state the step consumed is read from / written
// to the `hprev` history directly, so no state copy kernels are launched.
#include "gemm_simt.cuh"
#include "gru_cluster.cuh"

namespace nm {

// --- forward epilogues -------------------------------------------------------
struct GruGatesEpi {
  const float* xproj;  // [B,T,3H]
  const float* hprev;  // [B,T,H]
  float* gates;        // [B,T,3H]
  float* rh;           // [B,T,H]: r*h, A operand of the candidate matmul
  int64_t T, H, t;
  __device__ void operator()(int64_t b, int64_t n, float acc) const {
    const int64_t base3 = (b * T + t) * 3 * H;
    const float g = sigmoidf_(acc + xproj[base3 + n]);
    gates[base3 + n] = g;
    if (n < H) rh[(b * T + t) * H + n] = g * hprev[(b * T + t) * H + n];
  }
};

struct GruCandEpi {
  const float* xproj;
  const float* hprev;
  float* gates;
  float* states;       // [B,T,H]
  float* hnext;        // &hprev[0, t_next, 0] or final_state
  int64_t hnext_stride;  // T*H or H
  const int32_t* lengths;
  const float* drop_mask;  // [B,T,H] (already scaled by 1/keep_prob) or null
  float* raw_states;       // [B,T,H] cell outputs before dropout, or null
  int64_t T, H, t;
  __device__ void operator()(int64_t b, int64_t n, float acc) const {
    const int64_t base3 = (b * T + t) * 3 * H;
    const float c = tanhf(acc + xproj[base3 + 2 * H + n]);
    gates[base3 + 2 * H + n] = c;
    const float u = gates[base3 + H + n];
    const float h = hprev[(b * T + t) * H + n];
    const bool live = (lengths == nullptr) || (t < (int64_t)lengths[b]);
    float hn = live ? (u * h + (1.f - u) * c) : h;
    // the decoder feeds the DROPPED-OUT cell output back as the next state
    // (decoders/decoder.py:288-289,333-334,351 of the reference)
    if (raw_states) raw_states[(b * T + t) * H + n] = live ? hn : 0.f;
    if (drop_mask && live) hn *= drop_mask[(b * T + t) * H + n];
    states[(b * T + t) * H + n] = live ? hn : 0.f;
    hnext[b * hnext_stride + n] = hn;
  }
};

// --- backward ----------------------------------------------------------------
// E1: gate gradients that need no matmul.  dh_in = carry (+ dstates[t] on live rows).
__global__ void gru_bwd_gate_kernel(const float* __restrict__ gates, const float* __restrict__ hprev,
                                    const float* __restrict__ dstates, const float* __restrict__ dcarry,
                                    const int32_t* __restrict__ lengths,
                                    const float* __restrict__ drop_mask,
                                    const float* __restrict__ draw, float* __restrict__ dxproj,
                                    float* __restrict__ dhp, int64_t B, int64_t T, int64_t H,
                                    int64_t t) {
  const int64_t total = B * H;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / H, n = i - b * H;
    const int64_t base3 = (b * T + t) * 3 * H, base1 = (b * T + t) * H;
    const bool live = (lengths == nullptr) || (t < (int64_t)lengths[b]);
    const float u = gates[base3 + H + n], c = gates[base3 + 2 * H + n];
    const float h = hprev[base1 + n];
    float dh = dcarry ? dcarry[i] : 0.f;
    if (!live) {
      dxproj[base3 + n] = 0.f;  // dz_r is overwritten by the Wch kernel for live rows only
      dxproj[base3 + H + n] = 0.f;
      dxproj[base3 + 2 * H + n] = 0.f;
      dhp[i] = dh;
      continue;
    }
    if (dstates) dh += dstates[base1 + n];
    if (drop_mask) dh *= drop_mask[base1 + n];
    if (draw) dh += draw[base1 + n];  // gradient of the pre-dropout cell output
    const float du = dh * (h - c);
    const float dc = dh * (1.f - u);
    dxproj[base3 + 2 * H + n] = dc * (1.f - c * c);
    dxproj[base3 + H + n] = du * u * (1.f - u);
    dhp[i] = dh * u;
  }
}

// G1: drh = dzc . Wch^T ; dz_r = drh*h*r*(1-r) ; dhp += drh*r      (live rows only)
struct GruBwdCandEpi {
  const float* gates;
  const float* hprev;
  const int32_t* lengths;
  float* dxproj;
  float* dhp;
  int64_t T, H, t;
  __device__ void operator()(int64_t b, int64_t n, float drh) const {
    const bool live = (lengths == nullptr) || (t < (int64_t)lengths[b]);
    if (!live) return;
    const int64_t base3 = (b * T + t) * 3 * H;
    const float r = gates[base3 + n];
    const float h = hprev[(b * T + t) * H + n];
    dxproj[base3 + n] = drh * h * r * (1.f - r);
    dhp[b * H + n] += drh * r;
  }
};

// G2: dcarry = dhp + [dz_r, dz_u] . Wgh^T
struct GruBwdGatesEpi {
  const float* dhp;
  float* dcarry;
  int64_t H;
  __device__ void operator()(int64_t b, int64_t n, float acc) const {
    dcarry[b * H + n] = dhp[b * H + n] + acc;
  }
};

}  // namespace nm

using namespace nm;

namespace {

// Persistent cluster kernels need the three weight vectors of a unit slice in registers:
// H <= 320.  Other widths run on the per-step kernels.
bool cluster_path_ok(int64_t H) { return H >= 8 && H <= 320; }

struct ClusterPlan {
  int Bc, nclusters, sl;
  size_t smem;
};

// Clusters of 8 must fit inside one GPC: fewer than sm_count()/8 of them are co-resident.
// Measured once per kernel with cudaOccupancyMaxActiveClusters; a second wave would double
// the time of the whole sequence, so the batch slice per cluster is sized for ONE wave.
template <class Kern>
int max_active_clusters(Kern kern, size_t smem) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(GC_CLUSTER * 64);
  cfg.blockDim = dim3(GC_THREADS);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = GC_CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GC_SMEM_CAP) != cudaSuccess ||
      cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n < 1) {
    cudaGetLastError();
    n = sm_count() / GC_CLUSTER / 2;
  }
  return n;
}

// One CTA per SM whatever the shared-memory footprint (the register file is the limit), so the
// widest instance at a typical footprint stands for all of them.
int resident_clusters(bool backward) {
  static int cached[2] = {0, 0};
  if (cached[backward] == 0)
    cached[backward] = backward ? max_active_clusters(gru_seq_bwd_cluster_kernel<GC_MAX_SL>, 128 * 1024)
                                : max_active_clusters(gru_seq_fwd_cluster_kernel<GC_MAX_SL>, 128 * 1024);
  return cached[backward];
}

ClusterPlan plan_clusters(int64_t B, int64_t H, int sm_budget, bool backward) {
  ClusterPlan p;
  p.sl = (int)((H + GC_SLICES - 1) / GC_SLICES);  // 1..10 for H <= 320
  int max_clusters = resident_clusters(backward);
  if (sm_budget > 0 && sm_budget / GC_CLUSTER < max_clusters) max_clusters = sm_budget / GC_CLUSTER;
  if (max_clusters < 1) max_clusters = 1;
  // The kernels walk their rows GC_RB at a time, so Bc only needs to be a multiple of GC_RB: rounding it
  // further (to 4, say) would take B = 256 on 15 clusters from 18 rows to 20, leaving two clusters idle.
  int Bc = (int)((B + max_clusters - 1) / max_clusters);
  Bc = (Bc + GC_RB - 1) / GC_RB * GC_RB;
  const size_t per_row = (size_t)(backward ? gc_bwd_row_floats(p.sl) : gc_fwd_row_floats(p.sl)) * 4;
  const int cap = (int)((GC_SMEM_CAP - GC_BAR_BYTES) / per_row) / GC_RB * GC_RB;
  if (Bc > cap) Bc = cap;
  if (Bc < GC_RB) Bc = GC_RB;
  p.Bc = Bc;
  p.nclusters = (int)((B + Bc - 1) / Bc);
  p.smem = GC_BAR_BYTES + per_row * Bc;
  return p;
}

template <class Args, class Kern>
int launch_cluster(Kern kern, const Args& args, const ClusterPlan& p, cudaStream_t s, const char* name) {
  NM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(p.nclusters * GC_CLUSTER));
  cfg.blockDim = dim3(GC_THREADS);
  cfg.dynamicSmemBytes = p.smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = GC_CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  NM_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, args));
  NM_LAUNCH_CHECK(name);
  return NM_OK;
}

#define NM_GC_DISPATCH(KERN, args, plan, s, name)                  \
  switch ((plan).sl) {                                             \
    case 1: return launch_cluster(KERN<1>, args, plan, s, name);   \
    case 2: return launch_cluster(KERN<2>, args, plan, s, name);   \
    case 3: return launch_cluster(KERN<3>, args, plan, s, name);   \
    case 4: return launch_cluster(KERN<4>, args, plan, s, name);   \
    case 5: return launch_cluster(KERN<5>, args, plan, s, name);   \
    case 6: return launch_cluster(KERN<6>, args, plan, s, name);   \
    case 7: return launch_cluster(KERN<7>, args, plan, s, name);   \
    case 8: return launch_cluster(KERN<8>, args, plan, s, name);   \
    case 9: return launch_cluster(KERN<9>, args, plan, s, name);   \
    default: return launch_cluster(KERN<10>, args, plan, s, name); \
  }

}  // namespace

extern "C" {

int nm_gru_resident_clusters(int backward) { return resident_clusters(backward != 0); }

static long long* g_gru_prof = nullptr;
/* Diagnostic: device buffer of 8 int64 cycle counters accumulated by thread 0 of CTA 0 of the next
 * cluster launches, forward and backward alike (the slots are listed in tools/gru_probe.py); NULL
 * disables. */
int nm_gru_debug_profile(void* counters) {
  g_gru_prof = reinterpret_cast<long long*>(counters);
  return NM_OK;
}

int nm_gru_seq_fwd(const float* xproj, const float* Wgh, const float* Wch, const float* h0,
                   const int32_t* lengths, const float* drop_mask, int reverse, float* states,
                   float* raw_states, float* final_state, float* gates, float* hprev, float* rh,
                   int64_t B, int64_t T, int64_t H, int sm_budget, void* stream) {
  NM_REQUIRE(xproj && Wgh && Wch && states && final_state && gates && hprev && rh, NM_E_INVALID,
             "nm_gru_seq_fwd: null pointer");
  NM_REQUIRE(B > 0 && T > 0 && H > 0, NM_E_INVALID, "nm_gru_seq_fwd: bad sizes B=%lld T=%lld H=%lld",
             (long long)B, (long long)T, (long long)H);
  cudaStream_t s = (cudaStream_t)stream;
  if (cluster_path_ok(H)) {
    GcFwdArgs a{xproj, Wgh, Wch, h0, lengths, drop_mask, states, raw_states, final_state, gates,
                hprev, rh, (int)B, (int)T, (int)H, 0, reverse, g_gru_prof};
    const ClusterPlan p = plan_clusters(B, H, sm_budget, false);
    a.Bc = p.Bc;
    NM_GC_DISPATCH(gru_seq_fwd_cluster_kernel, a, p, s, "nm_gru_seq_fwd(cluster)");
  }
  const int64_t t_first = reverse ? T - 1 : 0;
  // seed the state history with h0 (or zeros): hprev[:, t_first, :]
  if (h0)
    NM_CUDA_TRY(cudaMemcpy2DAsync(hprev + t_first * H, sizeof(float) * T * H, h0, sizeof(float) * H,
                                  sizeof(float) * H, B, cudaMemcpyDeviceToDevice, s));
  else
    NM_CUDA_TRY(cudaMemset2DAsync(hprev + t_first * H, sizeof(float) * T * H, 0, sizeof(float) * H, B, s));
  for (int64_t step = 0; step < T; ++step) {
    const int64_t t = reverse ? T - 1 - step : step;
    // [r,u] = sigmoid(xg_t + h.Wgh);  rh = r*h
    GruGatesEpi e1{xproj, hprev, gates, rh, T, H, t};
    simt_gemm_launch(hprev + t * H, T * H, 1, Wgh, 2 * H, 1, B, 2 * H, H, e1, s);
    // c = tanh(xc_t + rh.Wch);  h' = u*h + (1-u)*c  -> next slot of the history / final state
    const bool last = (step == T - 1);
    const int64_t t_next = reverse ? t - 1 : t + 1;
    GruCandEpi e2{xproj, hprev, gates, states, last ? final_state : hprev + t_next * H,
                  last ? H : T * H, lengths, drop_mask, raw_states, T, H, t};
    simt_gemm_launch(rh + t * H, T * H, 1, Wch, H, 1, B, H, H, e2, s);
  }
  count_launches(2 * T - 1);  // 2 kernels per step; NM_LAUNCH_CHECK counts the last one
  NM_LAUNCH_CHECK("nm_gru_seq_fwd");
  return NM_OK;
}

int nm_gru_seq_bwd(const float* Wgh, const float* Wch, const int32_t* lengths,
                   const float* drop_mask, int reverse, const float* gates, const float* hprev,
                   const float* dstates, const float* draw, const float* dfinal,
                   float* dxproj, float* dh0, float* work, int64_t B, int64_t T, int64_t H,
                   int sm_budget, void* stream) {
  NM_REQUIRE(Wgh && Wch && gates && hprev && dxproj && work, NM_E_INVALID,
             "nm_gru_seq_bwd: null pointer");
  NM_REQUIRE(B > 0 && T > 0 && H > 0, NM_E_INVALID, "nm_gru_seq_bwd: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  if (cluster_path_ok(H)) {
    GcBwdArgs a{Wgh, Wch, lengths, drop_mask, gates, hprev, dstates, draw, dfinal, dxproj, dh0,
                (int)B, (int)T, (int)H, 0, reverse, g_gru_prof};
    const ClusterPlan p = plan_clusters(B, H, sm_budget, true);
    a.Bc = p.Bc;
    NM_GC_DISPATCH(gru_seq_bwd_cluster_kernel, a, p, s, "nm_gru_seq_bwd(cluster)");
  }
  float* dcarry = work;
  float* dhp = work + B * H;
  if (dfinal)
    NM_CUDA_TRY(cudaMemcpyAsync(dcarry, dfinal, sizeof(float) * B * H, cudaMemcpyDeviceToDevice, s));
  else
    NM_CUDA_TRY(cudaMemsetAsync(dcarry, 0, sizeof(float) * B * H, s));
  const int threads = 256;
  int64_t blocks = ceil_div(B * H, threads);
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  for (int64_t step = T - 1; step >= 0; --step) {
    const int64_t t = reverse ? T - 1 - step : step;
    gru_bwd_gate_kernel<<<(unsigned)blocks, threads, 0, s>>>(gates, hprev, dstates, dcarry, lengths,
                                                            drop_mask, draw, dxproj, dhp, B, T, H, t);
    // drh = dz_c . Wch^T   (op(B)(k=j, n=i) = Wch[i*H + j])
    GruBwdCandEpi g1{gates, hprev, lengths, dxproj, dhp, T, H, t};
    simt_gemm_launch(dxproj + t * 3 * H + 2 * H, T * 3 * H, 1, Wch, 1, H, B, H, H, g1, s);
    // dcarry = dhp + [dz_r, dz_u] . Wgh^T   (op(B)(k=j, n=i) = Wgh[i*2H + j])
    GruBwdGatesEpi g2{dhp, dcarry, H};
    simt_gemm_launch(dxproj + t * 3 * H, T * 3 * H, 1, Wgh, 1, 2 * H, B, H, 2 * H, g2, s);
  }
  if (dh0)
    NM_CUDA_TRY(cudaMemcpyAsync(dh0, dcarry, sizeof(float) * B * H, cudaMemcpyDeviceToDevice, s));
  count_launches(3 * T - 1);
  NM_LAUNCH_CHECK("nm_gru_seq_bwd");
  return NM_OK;
}


/* ---- both directions of a bidirectional layer: one sequence after the other ------------------------ */
int nm_gru_seq_fwd_pair(const float* xproj_a, const float* Wgh_a, const float* Wch_a, int reverse_a,
                        float* states_a, float* final_a, float* gates_a, float* hprev_a, float* rh_a,
                        const float* xproj_b, const float* Wgh_b, const float* Wch_b, int reverse_b,
                        float* states_b, float* final_b, float* gates_b, float* hprev_b, float* rh_b,
                        const int32_t* lengths, int64_t B, int64_t T, int64_t H, void* stream) {
  NM_REQUIRE(xproj_a && Wgh_a && Wch_a && states_a && final_a && gates_a && hprev_a && rh_a && xproj_b &&
                 Wgh_b && Wch_b && states_b && final_b && gates_b && hprev_b && rh_b,
             NM_E_INVALID, "nm_gru_seq_fwd_pair: null pointer");
  NM_REQUIRE(B > 0 && T > 0 && H > 0, NM_E_INVALID, "nm_gru_seq_fwd_pair: bad sizes");
  int rc = nm_gru_seq_fwd(xproj_a, Wgh_a, Wch_a, nullptr, lengths, nullptr, reverse_a, states_a, nullptr, final_a,
                          gates_a, hprev_a, rh_a, B, T, H, 0, stream);
  if (rc) return rc;
  return nm_gru_seq_fwd(xproj_b, Wgh_b, Wch_b, nullptr, lengths, nullptr, reverse_b, states_b, nullptr, final_b,
                        gates_b, hprev_b, rh_b, B, T, H, 0, stream);
}

int nm_gru_seq_bwd_pair(const float* Wgh_a, const float* Wch_a, int reverse_a, const float* gates_a,
                        const float* hprev_a, const float* dstates_a, const float* dfinal_a, float* dxproj_a,
                        const float* Wgh_b, const float* Wch_b, int reverse_b, const float* gates_b,
                        const float* hprev_b, const float* dstates_b, const float* dfinal_b, float* dxproj_b,
                        const int32_t* lengths, float* work, int64_t B, int64_t T, int64_t H, void* stream) {
  NM_REQUIRE(Wgh_a && Wch_a && gates_a && hprev_a && dxproj_a && Wgh_b && Wch_b && gates_b && hprev_b &&
                 dxproj_b && work,
             NM_E_INVALID, "nm_gru_seq_bwd_pair: null pointer");
  NM_REQUIRE(B > 0 && T > 0 && H > 0, NM_E_INVALID, "nm_gru_seq_bwd_pair: bad sizes");
  int rc = nm_gru_seq_bwd(Wgh_a, Wch_a, lengths, nullptr, reverse_a, gates_a, hprev_a, dstates_a, nullptr, dfinal_a,
                          dxproj_a, nullptr, work, B, T, H, 0, stream);
  if (rc) return rc;
  return nm_gru_seq_bwd(Wgh_b, Wch_b, lengths, nullptr, reverse_b, gates_b, hprev_b, dstates_b, nullptr, dfinal_b,
                        dxproj_b, nullptr, work, B, T, H, 0, stream);
}

}  // extern "C"
