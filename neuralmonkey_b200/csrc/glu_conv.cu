// One layer of the convolutional seq2seq encoder (encoders/facebook_conv.py, Gehring et al. 2017): a 1-D convolution
// over time with 2F output channels, the gated linear unit and the residual add,
//   z = conv1d_same(x, W) + b            x [B,T,F], W [k,F,2F], b [2F], z [B,T,2F]
//   y = z[..., :F] * sigmoid(z[..., F:]) + x
// TF's SAME padding at stride 1: pb = (k-1)/2 zeros before, k-1-pb after, and zeros only outside [0, T) of each
// sequence (padded positions inside the batch take part).
//
// The convolution is the one-row case of conv_igemm.cuh: a 1 x k window over [B, 1, T, Cin], pads (0, 0, pb,
// k-1-pb), 128 x 128 wgmma tiles.  The forward's tile holds output column f and its gate column F + f together, so
// the bias, the GLU and the residual run in its epilogue (the Glu policy).  The data gradient is the same product
// over dZ with W's taps reversed and its channel axes swapped (pads k-1-pb before), plus dY in the epilogue.
#include "conv_igemm.cuh"

namespace nm {

// dZ = [dY * s, dY * a * s * (1 - s)], s = sigmoid(gate), a = the linear half
__global__ void glu_dz_kernel(const float* __restrict__ dy, const float* __restrict__ z, float* __restrict__ dz,
                              int64_t M, int64_t F) {
  const int64_t total = M * F;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / F, f = i - m * F;
    const float a = z[m * 2 * F + f], s = sigmoidf_(z[m * 2 * F + F + f]), d = dy[i];
    dz[m * 2 * F + f] = d * s;
    dz[m * 2 * F + F + f] = d * a * s * (1.f - s);
  }
}

// The forward's geometry (x [B,T,F] -> z [B,T,2F]) or the data gradient's (dZ [B,T,2F] -> dX [B,T,F], pads k-1-pb
// before).
static int glu_geom(ConvGeom& g, int64_t B, int64_t T, int64_t F, int64_t k, bool dgrad, const char* name) {
  NM_REQUIRE(B > 0 && T > 0 && F > 0 && k > 0, NM_E_INVALID, "%s: bad sizes", name);
  NM_REQUIRE(k * 2 * F < (1LL << 30) && T < (1LL << 30) && B * T < (1LL << 40) && B * T * 2 * F < (1LL << 46),
             NM_E_UNSUPPORTED, "%s: sizes out of range", name);
  const int64_t pb = (k - 1) / 2;
  g = conv_geom_of(B, 1, T, dgrad ? 2 * F : F, dgrad ? F : 2 * F, 1, k, 0, dgrad ? k - 1 - pb : pb, 1, T);
  return NM_OK;
}

// the wgmma tile width of the GLU convolution
constexpr int GLU_BN = 128;

}  // namespace nm

using namespace nm;

extern "C" {

int nm_glu_conv1d_fwd(const float* x, const float* w, const float* bias, float* y, float* z, int64_t B, int64_t T,
                      int64_t F, int64_t k, int backend, void* stream) {
  NM_REQUIRE(x && w && bias && y, NM_E_INVALID, "nm_glu_conv1d_fwd: null pointer");
  ConvGeom g;
  const int rc = glu_geom(g, B, T, F, k, false, "nm_glu_conv1d_fwd");
  if (rc) return rc;
  return conv_fwd_launch<GLU_BN, false, true>(x, w, g, Glu{bias, x, y, z, F}, backend, (cudaStream_t)stream,
                                              "nm_glu_conv1d_fwd");
}

int nm_glu_conv1d_dz(const float* dy, const float* z, float* dz, int64_t M, int64_t F, void* stream) {
  NM_REQUIRE(dy && z && dz, NM_E_INVALID, "nm_glu_conv1d_dz: null pointer");
  NM_REQUIRE(M > 0 && F > 0 && M * 2 * F < (1LL << 46), NM_E_INVALID, "nm_glu_conv1d_dz: bad sizes");
  glu_dz_kernel<<<grid_for(M * F), 256, 0, (cudaStream_t)stream>>>(dy, z, dz, M, F);
  NM_LAUNCH_CHECK("nm_glu_conv1d_dz");
  return NM_OK;
}

int nm_glu_conv1d_dgrad(const float* dz, const float* w, const float* dy, float* dx, int64_t B, int64_t T, int64_t F,
                        int64_t k, int backend, void* stream) {
  NM_REQUIRE(dz && w && dy && dx, NM_E_INVALID, "nm_glu_conv1d_dgrad: null pointer");
  ConvGeom g;
  const int rc = glu_geom(g, B, T, F, k, true, "nm_glu_conv1d_dgrad");
  if (rc) return rc;
  return conv_fwd_launch<GLU_BN, true, true>(dz, w, g, AddRes{dy, dx}, backend, (cudaStream_t)stream,
                                             "nm_glu_conv1d_dgrad");
}

int64_t nm_glu_conv1d_wgrad_workspace(int64_t B, int64_t T, int64_t F, int64_t k, int backend) {
  ConvGeom g;
  if (glu_geom(g, B, T, F, k, false, "nm_glu_conv1d_wgrad_workspace")) return -1;
  const WgradPlan p = wgrad_plan<GLU_BN>(g, backend, -1);
  return p.splits * p.part;
}

int nm_glu_conv1d_wgrad(const float* x, const float* dz, float* dw, float* db, float* workspace,
                        int64_t workspace_floats, int64_t B, int64_t T, int64_t F, int64_t k, int backend,
                        void* stream) {
  NM_REQUIRE(x && dz && dw && db && workspace, NM_E_INVALID, "nm_glu_conv1d_wgrad: null pointer");
  ConvGeom g;
  const int rc = glu_geom(g, B, T, F, k, false, "nm_glu_conv1d_wgrad");
  if (rc) return rc;
  return conv_wgrad_launch<GLU_BN, true>(x, dz, dw, db, workspace, workspace_floats, g, backend, (cudaStream_t)stream,
                                         "nm_glu_conv1d_wgrad");
}

}  // extern "C"
