// K22: the character-level sentence encoder (encoders/sentence_cnn_encoder.py, Lee, Cho & Hofmann 2017).
//
// One-row convolution, tf.nn.conv1d at stride 1 with SAME padding, + bias and an optional ReLU:
//   y = act(conv1d_same(x, W) + b)        x [B,T,Cin], W [k,Cin,Cout], b [Cout], y [B,T,Cout]
// (k-1)/2 zeros before each sequence and k-1-(k-1)/2 after; positions inside [0, T) always take part, padded batch
// positions included.  These are the one-row (1 x k window over [B, 1, T, Cin]) instantiations of the implicit-GEMM
// kernels of conv_igemm.cuh with the BiasAct epilogue: the forward, the data gradient (the same product over dY with
// W's taps reversed and its channel axes swapped, k-1-pb zeros before) and the weight gradient.
//
// Highway gate (nn/highway.py) over the outputs of its two dense products zh = x W_H + b_H, zt = x W_T + b_T:
//   t = sigmoid(zt), h = relu(zh), y = h t + x (1 - t)
// and its backward: dzh = dy t [zh > 0], dzt = dy (h - x) t (1 - t), dx = dy (1 - t) (the carry term; the
// products' data gradients add the rest).  Every output element is computed by itself, so repeat calls give
// identical bits.
#include "conv_igemm.cuh"

namespace nm {

// the wgmma tile width of the one-row convolutions
constexpr int C1D_BN = 128;

// The forward's geometry (x [B,T,Cin] -> y [B,T,Cout]) or the data gradient's (dY [B,T,Cout] -> dX [B,T,Cin],
// k-1-pb zeros before).
static int conv1d_geom(ConvGeom& g, int64_t B, int64_t T, int64_t Cin, int64_t Cout, int64_t k, bool dgrad,
                       const char* name) {
  NM_REQUIRE(B > 0 && T > 0 && Cin > 0 && Cout > 0 && k > 0, NM_E_INVALID, "%s: bad sizes", name);
  NM_REQUIRE(k * Cin < (1LL << 30) && k * Cout < (1LL << 30) && T < (1LL << 30) && B * T < (1LL << 40) &&
                 B * T * Cin < (1LL << 46) && B * T * Cout < (1LL << 46),
             NM_E_UNSUPPORTED, "%s: sizes out of range", name);
  const int64_t pb = (k - 1) / 2;
  g = dgrad ? conv_geom_of(B, 1, T, Cout, Cin, 1, k, 0, k - 1 - pb, 1, T)
            : conv_geom_of(B, 1, T, Cin, Cout, 1, k, 0, pb, 1, T);
  return NM_OK;
}

__global__ void highway_fwd_kernel(const float* __restrict__ zh, const float* __restrict__ zt,
                                   const float* __restrict__ x, float* __restrict__ y, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float t = sigmoidf_(zt[i]), h = fmaxf(zh[i], 0.f), xi = x[i];
    y[i] = h * t + xi * (1.f - t);
  }
}

__global__ void highway_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ zh,
                                   const float* __restrict__ zt, const float* __restrict__ x, float* __restrict__ dzh,
                                   float* __restrict__ dzt, float* __restrict__ dx, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float t = sigmoidf_(zt[i]), z = zh[i], d = dy[i];
    const float h = fmaxf(z, 0.f);
    dzh[i] = z > 0.f ? d * t : 0.f;
    dzt[i] = d * (h - x[i]) * t * (1.f - t);
    dx[i] = d * (1.f - t);
  }
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_conv1d_fwd(const float* x, const float* w, const float* bias, float* y, int64_t B, int64_t T, int64_t Cin,
                  int64_t Cout, int64_t k, int act, int backend, void* stream) {
  static const char* name = "nm_conv1d_fwd";
  NM_REQUIRE(x && w && y, NM_E_INVALID, "%s: null pointer", name);
  NM_REQUIRE(act == NM_ACT_NONE || act == NM_ACT_RELU, NM_E_INVALID, "%s: act must be none or relu", name);
  ConvGeom g;
  const int rc = conv1d_geom(g, B, T, Cin, Cout, k, false, name);
  if (rc) return rc;
  return conv_fwd_launch<C1D_BN, false, true>(x, w, g, BiasAct{bias, y, act}, backend, (cudaStream_t)stream, name);
}

int nm_conv1d_dgrad(const float* dy, const float* w, float* dx, int64_t B, int64_t T, int64_t Cin, int64_t Cout,
                    int64_t k, int backend, void* stream) {
  static const char* name = "nm_conv1d_dgrad";
  NM_REQUIRE(dy && w && dx, NM_E_INVALID, "%s: null pointer", name);
  ConvGeom g;
  const int rc = conv1d_geom(g, B, T, Cin, Cout, k, true, name);
  if (rc) return rc;
  return conv_fwd_launch<C1D_BN, true, true>(dy, w, g, BiasAct{nullptr, dx, NM_ACT_NONE}, backend,
                                             (cudaStream_t)stream, name);
}

int64_t nm_conv1d_wgrad_workspace(int64_t B, int64_t T, int64_t Cin, int64_t Cout, int64_t k, int backend) {
  ConvGeom g;
  if (conv1d_geom(g, B, T, Cin, Cout, k, false, "nm_conv1d_wgrad_workspace")) return -1;
  const WgradPlan p = wgrad_plan<C1D_BN>(g, backend, -1);
  return p.splits * p.part;
}

int nm_conv1d_wgrad(const float* x, const float* dy, float* dw, float* db, float* workspace, int64_t workspace_floats,
                    int64_t B, int64_t T, int64_t Cin, int64_t Cout, int64_t k, int backend, void* stream) {
  static const char* name = "nm_conv1d_wgrad";
  NM_REQUIRE(x && dy && dw && workspace, NM_E_INVALID, "%s: null pointer", name);
  ConvGeom g;
  const int rc = conv1d_geom(g, B, T, Cin, Cout, k, false, name);
  if (rc) return rc;
  return conv_wgrad_launch<C1D_BN, true>(x, dy, dw, db, workspace, workspace_floats, g, backend, (cudaStream_t)stream,
                                         name);
}

int nm_highway_fwd(const float* zh, const float* zt, const float* x, float* y, int64_t n, void* stream) {
  NM_REQUIRE(zh && zt && x && y, NM_E_INVALID, "nm_highway_fwd: null pointer");
  NM_REQUIRE(n >= 0, NM_E_INVALID, "nm_highway_fwd: negative size");
  if (n == 0) return NM_OK;
  highway_fwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(zh, zt, x, y, n);
  NM_LAUNCH_CHECK("nm_highway_fwd");
  return NM_OK;
}

int nm_highway_bwd(const float* dy, const float* zh, const float* zt, const float* x, float* dzh, float* dzt,
                   float* dx, int64_t n, void* stream) {
  NM_REQUIRE(dy && zh && zt && x && dzh && dzt && dx, NM_E_INVALID, "nm_highway_bwd: null pointer");
  NM_REQUIRE(n >= 0, NM_E_INVALID, "nm_highway_bwd: negative size");
  if (n == 0) return NM_OK;
  highway_bwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(dy, zh, zt, x, dzh, dzt, dx, n);
  NM_LAUNCH_CHECK("nm_highway_bwd");
  return NM_OK;
}

}  // extern "C"
