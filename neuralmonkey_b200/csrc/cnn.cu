// Trainable CNN layers of encoders/cnn_encoder.py (reference :209-320): k x k convolution (stride 1) with its data
// and weight gradients, batch normalization with the ReLU after it, max / average pooling.  NHWC fp32, HWIO filters.
//
// The convolution runs on the implicit-GEMM kernels of conv_igemm.cuh with a k x k window and 128 x 64 wgmma tiles;
// the data gradient is the forward call with `flip` on the forward filter.
#include "conv_igemm.cuh"

namespace nm {

// ------------------------------------------------------------------------------------------------------------
// Batch normalization over P = N*H*W rows of C channels.  Per-channel sums are accumulated in fp64: grid
// (ceil(C/32), S) partial blocks of 32 channels x 8 row lanes, then one thread per channel adds the S partials in
// index order, so the statistics do not depend on scheduling.
// ------------------------------------------------------------------------------------------------------------
constexpr int BN_SPLITS = 64;      // NM_BN_WS_DOUBLES_PER_CHANNEL = 2 * BN_SPLITS + 2

// mode 0: (sum x, sum x^2); mode 1: (sum dy', sum dy' * xhat), dy' = dy masked by the fused ReLU
__global__ void __launch_bounds__(256)
bn_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ gamma,
                  const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ invstd,
                  double* __restrict__ part, int64_t P, int C, int relu, int mode) {
  __shared__ double red[2][8][32];
  const int lc = threadIdx.x & 31, lr = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lc;
  double s0 = 0.0, s1 = 0.0;
  if (c < C) {
    float mu = 0.f, is = 0.f, ga = 0.f, be = 0.f;
    if (mode == 1) { mu = mean[c]; is = invstd[c]; ga = gamma[c]; be = beta[c]; }
    for (int64_t r = (int64_t)blockIdx.y * 8 + lr; r < P; r += (int64_t)gridDim.y * 8) {
      const float v = x[r * C + c];
      if (mode == 0) {
        s0 += v;
        s1 += (double)v * v;
      } else {
        const float xh = (v - mu) * is;
        float d = dy[r * C + c];
        if (relu && fmaf(ga, xh, be) <= 0.f) d = 0.f;
        s0 += d;
        s1 += (double)d * xh;
      }
    }
  }
  red[0][lr][lc] = s0;
  red[1][lr][lc] = s1;
  __syncthreads();
  if (lr == 0 && c < C) {
    for (int i = 1; i < 8; ++i) { s0 += red[0][i][lc]; s1 += red[1][i][lc]; }
    part[((int64_t)blockIdx.y * C + c) * 2] = s0;
    part[((int64_t)blockIdx.y * C + c) * 2 + 1] = s1;
  }
}

__global__ void bn_fwd_finalize_kernel(const double* __restrict__ part, int splits, float* __restrict__ moving_mean,
                                       float* __restrict__ moving_var, float* __restrict__ save_mean,
                                       float* __restrict__ save_invstd, int64_t P, int C, float momentum, float eps,
                                       int training) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (!training) {
    save_mean[c] = moving_mean[c];
    save_invstd[c] = (float)(1.0 / sqrt((double)moving_var[c] + (double)eps));
    return;
  }
  double s0 = 0.0, s1 = 0.0;
  for (int j = 0; j < splits; ++j) {
    s0 += part[((int64_t)j * C + c) * 2];
    s1 += part[((int64_t)j * C + c) * 2 + 1];
  }
  const double mu = s0 / (double)P;
  const double var = fmax(s1 / (double)P - mu * mu, 0.0);
  save_mean[c] = (float)mu;
  save_invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (moving_mean) {
    // moving statistics: the Bessel-corrected batch variance, as TF's fused batch norm returns it
    const double unbiased = P > 1 ? var * (double)P / (double)(P - 1) : var;
    moving_mean[c] = (float)((double)momentum * moving_mean[c] + (1.0 - momentum) * mu);
    moving_var[c] = (float)((double)momentum * moving_var[c] + (1.0 - momentum) * unbiased);
  }
}

__global__ void bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ mean,
                                const float* __restrict__ invstd, float* __restrict__ y, int64_t total, int C,
                                int relu) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float v = fmaf(gamma[c], (x[i] - mean[c]) * invstd[c], beta[c]);
    y[i] = relu ? fmaxf(v, 0.f) : v;
  }
}

// one thread per channel: the two sums of the backward pass; dgamma / dbeta accumulate
__global__ void bn_bwd_finalize_kernel(const double* __restrict__ part, int splits, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, double* __restrict__ sums, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s0 = 0.0, s1 = 0.0;
  for (int j = 0; j < splits; ++j) {
    s0 += part[((int64_t)j * C + c) * 2];
    s1 += part[((int64_t)j * C + c) * 2 + 1];
  }
  sums[2 * c] = s0;
  sums[2 * c + 1] = s1;
  if (dbeta) dbeta[c] += (float)s0;
  if (dgamma) dgamma[c] += (float)s1;
}

__global__ void bn_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ mean, const float* __restrict__ invstd,
                                 const double* __restrict__ sums, float* __restrict__ dx, int64_t total, int64_t P,
                                 int C, int relu, int training) {
  const float inv_p = 1.f / (float)P;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const float is = invstd[c], ga = gamma[c];
    const float xh = (x[i] - mean[c]) * is;
    float d = dy[i];
    if (relu && fmaf(ga, xh, beta[c]) <= 0.f) d = 0.f;
    if (training) d = d - (float)sums[2 * c] * inv_p - xh * ((float)sums[2 * c + 1] * inv_p);
    dx[i] = ga * is * d;
  }
}

// ------------------------------------------------------------------------------------------------------------
// Pooling (tf.layers.max_pooling2d / average_pooling2d): k x k window, stride s; `same` pads TF's way (odd pixel
// at the bottom / right) and averages over the pixels inside the image.
// ------------------------------------------------------------------------------------------------------------
struct PoolGeom {
  int N, H, W, C, k, s, pt, pl, Ho, Wo;
};

__global__ void pool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, PoolGeom g, int is_max) {
  const int64_t total = (int64_t)g.N * g.Ho * g.Wo * g.C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    int64_t r = i / g.C;
    const int ox = (int)(r % g.Wo);
    r /= g.Wo;
    const int oy = (int)(r % g.Ho);
    const int64_t n = r / g.Ho;
    const int y0 = oy * g.s - g.pt, x0 = ox * g.s - g.pl;
    float best = -INFINITY, sum = 0.f;
    int cnt = 0;
    for (int dy = 0; dy < g.k; ++dy) {
      const int iy = y0 + dy;
      if (iy < 0 || iy >= g.H) continue;
      for (int dx = 0; dx < g.k; ++dx) {
        const int ix = x0 + dx;
        if (ix < 0 || ix >= g.W) continue;
        const float v = x[((n * g.H + iy) * g.W + ix) * g.C + c];
        if (v > best) best = v;
        sum += v;
        ++cnt;
      }
    }
    y[i] = is_max ? best : sum / (float)cnt;
  }
}

// Gradient gathered per input pixel from every window that contains it (no atomics: same bits every call).  Max
// pooling routes a window's gradient to its first maximal pixel in row-major order.
__global__ void pool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx,
                                PoolGeom g, int is_max) {
  const int64_t total = (int64_t)g.N * g.H * g.W * g.C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    int64_t r = i / g.C;
    const int ix = (int)(r % g.W);
    r /= g.W;
    const int iy = (int)(r % g.H);
    const int64_t n = r / g.H;
    // windows oy with oy*s - pt <= iy < oy*s - pt + k
    const int oy_lo = max(0, (iy + g.pt - g.k + g.s) / g.s), oy_hi = min(g.Ho - 1, (iy + g.pt) / g.s);
    const int ox_lo = max(0, (ix + g.pl - g.k + g.s) / g.s), ox_hi = min(g.Wo - 1, (ix + g.pl) / g.s);
    float acc = 0.f;
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        const int y0 = oy * g.s - g.pt, x0 = ox * g.s - g.pl;
        if (iy < y0 || ix < x0) continue;    // (iy + pt - k + s) / s rounds toward zero for negative values
        const float d = dy[((n * g.Ho + oy) * g.Wo + ox) * g.C + c];
        if (is_max) {
          float best = -INFINITY;
          int by = -1, bx = -1;
          for (int yy = max(y0, 0); yy < min(y0 + g.k, g.H); ++yy)
            for (int xx = max(x0, 0); xx < min(x0 + g.k, g.W); ++xx) {
              const float v = x[((n * g.H + yy) * g.W + xx) * g.C + c];
              if (v > best || by < 0) { best = v; by = yy; bx = xx; }
            }
          if (by == iy && bx == ix) acc += d;
        } else {
          const int cy = min(y0 + g.k, g.H) - max(y0, 0), cx = min(x0 + g.k, g.W) - max(x0, 0);
          acc += d / (float)(cy * cx);
        }
      }
    }
    dx[i] = acc;
  }
}

static int conv_geom(ConvGeom& g, int64_t N, int64_t H, int64_t W, int64_t C, int64_t K, int64_t k, int64_t pad_top,
                     int64_t pad_bottom, int64_t pad_left, int64_t pad_right, const char* name) {
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && K > 0 && k > 0 && pad_top >= 0 && pad_bottom >= 0 &&
                 pad_left >= 0 && pad_right >= 0 && pad_top < k && pad_bottom < k && pad_left < k && pad_right < k,
             NM_E_INVALID, "%s: bad sizes", name);
  const int64_t Ho = H + pad_top + pad_bottom - k + 1, Wo = W + pad_left + pad_right - k + 1;
  NM_REQUIRE(Ho > 0 && Wo > 0, NM_E_INVALID, "%s: window larger than the padded image", name);
  NM_REQUIRE(k * k * C < (1LL << 30) && K < (1LL << 24) && N * H * W * C < (1LL << 40) && H < (1 << 20) &&
                 W < (1 << 20),
             NM_E_UNSUPPORTED, "%s: sizes out of range", name);
  g = conv_geom_of(N, H, W, C, K, k, k, pad_top, pad_left, Ho, Wo);
  return NM_OK;
}

// the wgmma tile width of the convolutions here
constexpr int CONV_BN = 64;

static int pool_geom(PoolGeom& g, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k, int64_t s, int same,
                     const char* name) {
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && k > 0 && s > 0 && H < (1 << 20) && W < (1 << 20),
             NM_E_INVALID, "%s: bad sizes", name);
  int64_t Ho, Wo, pt = 0, pl = 0;
  if (same) {
    Ho = ceil_div(H, s);
    Wo = ceil_div(W, s);
    const int64_t ph = (Ho - 1) * s + k - H, pw = (Wo - 1) * s + k - W;
    pt = ph > 0 ? ph / 2 : 0;
    pl = pw > 0 ? pw / 2 : 0;
  } else {
    NM_REQUIRE(H >= k && W >= k, NM_E_INVALID, "%s: window larger than the image", name);
    Ho = (H - k) / s + 1;
    Wo = (W - k) / s + 1;
  }
  g.N = (int)N; g.H = (int)H; g.W = (int)W; g.C = (int)C; g.k = (int)k; g.s = (int)s;
  g.pt = (int)pt; g.pl = (int)pl; g.Ho = (int)Ho; g.Wo = (int)Wo;
  return NM_OK;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_conv2d_fwd(const float* x, const float* w, const float* bias, float* y, int64_t N, int64_t H, int64_t W,
                  int64_t Cin, int64_t Cout, int64_t k, int64_t pad_top, int64_t pad_bottom, int64_t pad_left,
                  int64_t pad_right, int flip, int act, int backend, void* stream) {
  NM_REQUIRE(x && w && y, NM_E_INVALID, "nm_conv2d_fwd: null pointer");
  NM_REQUIRE(act == NM_ACT_NONE || act == NM_ACT_RELU, NM_E_INVALID, "nm_conv2d_fwd: act must be none or relu");
  ConvGeom g;
  const int rc = conv_geom(g, N, H, W, Cin, Cout, k, pad_top, pad_bottom, pad_left, pad_right, "nm_conv2d_fwd");
  if (rc) return rc;
  const BiasAct epi{bias, y, act};
  cudaStream_t s = (cudaStream_t)stream;
  return flip ? conv_fwd_launch<CONV_BN, true, false>(x, w, g, epi, backend, s, "nm_conv2d_fwd")
              : conv_fwd_launch<CONV_BN, false, false>(x, w, g, epi, backend, s, "nm_conv2d_fwd");
}

int64_t nm_conv2d_wgrad_workspace(int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t k,
                                  int64_t pad_top, int64_t pad_bottom, int64_t pad_left, int64_t pad_right,
                                  int backend) {
  ConvGeom g;
  if (conv_geom(g, N, H, W, Cin, Cout, k, pad_top, pad_bottom, pad_left, pad_right, "nm_conv2d_wgrad_workspace"))
    return -1;
  const WgradPlan p = wgrad_plan<CONV_BN>(g, backend, -1);
  return p.splits * p.part;
}

int nm_conv2d_wgrad(const float* x, const float* dy, float* dw, float* db, float* workspace, int64_t workspace_floats,
                    int64_t N, int64_t H, int64_t W, int64_t Cin, int64_t Cout, int64_t k, int64_t pad_top,
                    int64_t pad_bottom, int64_t pad_left, int64_t pad_right, int backend, void* stream) {
  NM_REQUIRE(x && dy && dw && workspace, NM_E_INVALID, "nm_conv2d_wgrad: null pointer");
  ConvGeom g;
  const int rc = conv_geom(g, N, H, W, Cin, Cout, k, pad_top, pad_bottom, pad_left, pad_right, "nm_conv2d_wgrad");
  if (rc) return rc;
  return conv_wgrad_launch<CONV_BN, false>(x, dy, dw, db, workspace, workspace_floats, g, backend,
                                           (cudaStream_t)stream, "nm_conv2d_wgrad");
}

int nm_batchnorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* moving_mean,
                     float* moving_var, float* save_mean, float* save_invstd, double* workspace, int64_t P, int64_t C,
                     float momentum, float eps, int training, int relu, void* stream) {
  NM_REQUIRE(x && gamma && beta && y && moving_mean && moving_var && save_mean && save_invstd, NM_E_INVALID,
             "nm_batchnorm_fwd: null pointer");
  NM_REQUIRE(P > 0 && C > 0 && C < (1 << 24), NM_E_INVALID, "nm_batchnorm_fwd: bad sizes");
  NM_REQUIRE(!training || workspace, NM_E_INVALID, "nm_batchnorm_fwd: training needs the workspace");
  cudaStream_t s = (cudaStream_t)stream;
  const int splits = (int)(ceil_div(P, 8) < BN_SPLITS ? ceil_div(P, 8) : BN_SPLITS);
  if (training) {
    bn_partial_kernel<<<dim3((unsigned)ceil_div(C, 32), splits), 256, 0, s>>>(x, nullptr, nullptr, nullptr, nullptr,
                                                                              nullptr, workspace, P, (int)C, 0, 0);
    NM_LAUNCH_CHECK("nm_batchnorm_fwd(stats)");
  }
  bn_fwd_finalize_kernel<<<(unsigned)ceil_div(C, 128), 128, 0, s>>>(workspace, splits, moving_mean, moving_var,
                                                                      save_mean, save_invstd, P, (int)C, momentum, eps,
                                                                      training);
  NM_LAUNCH_CHECK("nm_batchnorm_fwd(finalize)");
  bn_apply_kernel<<<grid_for(P * C), 256, 0, s>>>(x, gamma, beta, save_mean, save_invstd, y, P * C, (int)C, relu);
  NM_LAUNCH_CHECK("nm_batchnorm_fwd(apply)");
  return NM_OK;
}

int nm_batchnorm_bwd(const float* x, const float* dy, const float* gamma, const float* beta, const float* save_mean,
                     const float* save_invstd, float* dx, float* dgamma, float* dbeta, double* workspace, int64_t P,
                     int64_t C, int training, int relu, void* stream) {
  NM_REQUIRE(x && dy && gamma && beta && save_mean && save_invstd && workspace, NM_E_INVALID,
             "nm_batchnorm_bwd: null pointer");
  NM_REQUIRE(P > 0 && C > 0 && C < (1 << 24), NM_E_INVALID, "nm_batchnorm_bwd: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  const int splits = (int)(ceil_div(P, 8) < BN_SPLITS ? ceil_div(P, 8) : BN_SPLITS);
  double* sums = workspace + 2 * BN_SPLITS * C;
  bn_partial_kernel<<<dim3((unsigned)ceil_div(C, 32), splits), 256, 0, s>>>(x, dy, gamma, beta, save_mean,
                                                                            save_invstd, workspace, P, (int)C, relu, 1);
  NM_LAUNCH_CHECK("nm_batchnorm_bwd(sums)");
  bn_bwd_finalize_kernel<<<(unsigned)ceil_div(C, 128), 128, 0, s>>>(workspace, splits, dgamma, dbeta, sums, (int)C);
  NM_LAUNCH_CHECK("nm_batchnorm_bwd(finalize)");
  if (dx) {
    bn_bwd_dx_kernel<<<grid_for(P * C), 256, 0, s>>>(x, dy, gamma, beta, save_mean, save_invstd, sums, dx, P * C, P,
                                                     (int)C, relu, training);
    NM_LAUNCH_CHECK("nm_batchnorm_bwd(dx)");
  }
  return NM_OK;
}

int nm_pool2d_fwd(const float* x, float* y, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k, int64_t stride,
                  int same, int is_max, void* stream) {
  NM_REQUIRE(x && y, NM_E_INVALID, "nm_pool2d_fwd: null pointer");
  PoolGeom g;
  const int rc = pool_geom(g, N, H, W, C, k, stride, same, "nm_pool2d_fwd");
  if (rc) return rc;
  pool_fwd_kernel<<<grid_for((int64_t)N * g.Ho * g.Wo * C), 256, 0, (cudaStream_t)stream>>>(x, y, g, is_max);
  NM_LAUNCH_CHECK("nm_pool2d_fwd");
  return NM_OK;
}

int nm_pool2d_bwd(const float* x, const float* dy, float* dx, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k,
                  int64_t stride, int same, int is_max, void* stream) {
  NM_REQUIRE(dy && dx && (x || !is_max), NM_E_INVALID, "nm_pool2d_bwd: null pointer");
  PoolGeom g;
  const int rc = pool_geom(g, N, H, W, C, k, stride, same, "nm_pool2d_bwd");
  if (rc) return rc;
  pool_bwd_kernel<<<grid_for(N * H * W * C), 256, 0, (cudaStream_t)stream>>>(x, dy, dx, g, is_max);
  NM_LAUNCH_CHECK("nm_pool2d_bwd");
  return NM_OK;
}

}  // extern "C"
