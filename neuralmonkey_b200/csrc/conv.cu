// K12: slim VGG-16 building blocks, forward only (the ImageNet encoder is frozen:
// encoders/imagenet_encoder.py:212,234 of the reference).  NHWC fp32.
//   conv3x3, stride 1, SAME, + bias + ReLU  (vgg_arg_scope of tensorflow/models slim nets/vgg.py)
//   max-pool 2x2 / 2
// The convolution is an implicit GEMM: M = N*H*W output pixels, N = Cout, K = 9*Cin,
// A(m, (dy,dx,c)) gathered on the fly from the input (zero outside the image), B = the
// HWIO filter viewed as [9*Cin, Cout].  Round 1 runs the tile on the CUDA cores in exact
// fp32; a TMA-im2col tensor-core mainloop is listed under "what comes next" in DESIGN.md.
#include "gemm_simt.cuh"

namespace nm {

constexpr int CV_BM = 64, CV_BN = 64, CV_TM = 4, CV_TN = 4;

__global__ void __launch_bounds__(SIMT_THREADS)
conv3x3_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
               float* __restrict__ y, int64_t NB, int H, int W, int Cin, int Cout) {
  __shared__ SimtSmem<CV_BM, CV_BN, CV_TM, CV_TN> sm;
  const int64_t M = NB * H * W;
  const int K = 9 * Cin;
  const int64_t m0 = (int64_t)blockIdx.y * CV_BM;
  const int n0 = blockIdx.x * CV_BN;
  const int t = threadIdx.x;
  const int tx = t % (CV_BN / CV_TN), ty = t / (CV_BN / CV_TN);
  float acc[CV_TM][CV_TN];
#pragma unroll
  for (int i = 0; i < CV_TM; ++i)
#pragma unroll
    for (int j = 0; j < CV_TN; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += SIMT_BK) {
    // A tile: element (m, k): k fastest across threads (c is contiguous in NHWC)
#pragma unroll
    for (int i = 0; i < (CV_BM * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int m = idx / SIMT_BK, k = idx % SIMT_BK;
      const int64_t gm = m0 + m;
      const int gk = k0 + k;
      float val = 0.f;
      if (gm < M && gk < K) {
        const int tap = gk / Cin, c = gk - tap * Cin;
        const int dy = tap / 3 - 1, dx = tap % 3 - 1;
        const int64_t n = gm / ((int64_t)H * W);
        const int rem = (int)(gm - n * (int64_t)H * W);
        const int yy = rem / W + dy, xx = rem % W + dx;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W)
          val = x[((n * H + yy) * W + xx) * Cin + c];
      }
      sm.a[k][m] = val;
    }
#pragma unroll
    for (int i = 0; i < (CV_BN * SIMT_BK) / SIMT_THREADS; ++i) {
      const int idx = t + i * SIMT_THREADS;
      const int k = idx / CV_BN, n = idx % CV_BN;
      const int gk = k0 + k, gn = n0 + n;
      sm.b[k][n] = (gk < K && gn < Cout) ? w[(int64_t)gk * Cout + gn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SIMT_BK; ++k) {
      float av[CV_TM], bv[CV_TN];
#pragma unroll
      for (int i = 0; i < CV_TM; ++i) av[i] = sm.a[k][ty * CV_TM + i];
#pragma unroll
      for (int j = 0; j < CV_TN; ++j) bv[j] = sm.b[k][tx * CV_TN + j];
#pragma unroll
      for (int i = 0; i < CV_TM; ++i)
#pragma unroll
        for (int j = 0; j < CV_TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < CV_TM; ++i) {
    const int64_t m = m0 + ty * CV_TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < CV_TN; ++j) {
      const int n = n0 + tx * CV_TN + j;
      if (n < Cout) y[m * Cout + n] = fmaxf(acc[i][j] + bias[n], 0.f);
    }
  }
}

// im2col for the tensor-core path: cols[m][tap*Cin + c] = x[n, y+dy, x+dx, c] (zero outside the
// image), row pitch `ldc` floats.  One thread per (pixel, tap, 4-channel group).
__global__ void im2col3x3_kernel(const float* __restrict__ x, float* __restrict__ cols, int64_t NB, int H,
                                 int W, int Cin, int64_t ldc) {
  const int groups = (Cin + 3) / 4;
  const int64_t total = NB * H * W * 9 * groups;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    int64_t r = i / groups;
    const int tap = (int)(r % 9);
    const int64_t m = r / 9;
    const int xx0 = (int)(m % W);
    const int yy0 = (int)((m / W) % H);
    const int64_t n = m / ((int64_t)W * H);
    const int yy = yy0 + tap / 3 - 1, xx = xx0 + tap % 3 - 1;
    const bool inside = yy >= 0 && yy < H && xx >= 0 && xx < W;
    const float* src = x + ((n * H + yy) * W + xx) * Cin + 4 * g;
    float* dst = cols + m * ldc + tap * Cin + 4 * g;
    if ((Cin & 3) == 0) {
      const float4 v = inside ? *reinterpret_cast<const float4*>(src) : make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(dst) = v;
    } else {
      for (int c = 0; c < 4 && 4 * g + c < Cin; ++c) dst[c] = inside ? src[c] : 0.f;
    }
  }
}

__global__ void maxpool2x2_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t NB, int H,
                                  int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t total = NB * Ho * Wo * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t r = i / C;
    const int xo = (int)(r % Wo);
    r /= Wo;
    const int yo = (int)(r % Ho);
    const int64_t n = r / Ho;
    const float* p = x + ((n * H + 2 * yo) * W + 2 * xo) * C + c;
    const float a = p[0], b = p[C], d = p[(int64_t)W * C], e = p[(int64_t)W * C + C];
    y[i] = fmaxf(fmaxf(a, b), fmaxf(d, e));
  }
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_conv3x3_bias_relu_fwd(const float* x, const float* w, const float* bias, float* y, int64_t N,
                             int64_t H, int64_t W, int64_t Cin, int64_t Cout, void* stream) {
  NM_REQUIRE(x && w && bias && y, NM_E_INVALID, "nm_conv3x3_bias_relu_fwd: null pointer");
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, NM_E_INVALID,
             "nm_conv3x3_bias_relu_fwd: bad sizes");
  const int64_t M = N * H * W;
  NM_REQUIRE(ceil_div(M, CV_BM) <= 0x7fffffffLL && ceil_div(Cout, CV_BN) <= 65535, NM_E_UNSUPPORTED,
             "nm_conv3x3_bias_relu_fwd: grid too large");
  dim3 grid((unsigned)ceil_div(Cout, CV_BN), (unsigned)ceil_div(M, CV_BM));
  NM_REQUIRE(grid.y <= 65535u * 16u, NM_E_UNSUPPORTED, "nm_conv3x3_bias_relu_fwd: too many pixels");
  if (grid.y > 65535u) {
    // split the batch so grid.y stays within the launch limit
    const int64_t per = (65535LL * CV_BM) / (H * W);
    NM_REQUIRE(per >= 1, NM_E_UNSUPPORTED, "nm_conv3x3_bias_relu_fwd: image too large");
    for (int64_t n0 = 0; n0 < N; n0 += per) {
      const int64_t nb = (N - n0 < per) ? N - n0 : per;
      const int rc = nm_conv3x3_bias_relu_fwd(x + n0 * H * W * Cin, w, bias, y + n0 * H * W * Cout, nb,
                                              H, W, Cin, Cout, stream);
      if (rc) return rc;
    }
    return NM_OK;
  }
  conv3x3_kernel<<<grid, SIMT_THREADS, 0, (cudaStream_t)stream>>>(x, w, bias, y, N, (int)H, (int)W,
                                                                  (int)Cin, (int)Cout);
  NM_LAUNCH_CHECK("nm_conv3x3_bias_relu_fwd");
  return NM_OK;
}

int nm_im2col3x3(const float* x, float* cols, int64_t N, int64_t H, int64_t W, int64_t Cin,
                 int64_t ldc, void* stream) {
  NM_REQUIRE(x && cols, NM_E_INVALID, "nm_im2col3x3: null pointer");
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && Cin > 0 && ldc >= 9 * Cin, NM_E_INVALID, "nm_im2col3x3: bad sizes");
  const int64_t total = N * H * W * 9 * ((Cin + 3) / 4);
  int64_t blocks = ceil_div(total, 256);
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  im2col3x3_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, cols, N, (int)H, (int)W, (int)Cin,
                                                                      ldc);
  NM_LAUNCH_CHECK("nm_im2col3x3");
  return NM_OK;
}

int nm_maxpool2x2_fwd(const float* x, float* y, int64_t N, int64_t H, int64_t W, int64_t C,
                      void* stream) {
  NM_REQUIRE(x && y, NM_E_INVALID, "nm_maxpool2x2_fwd: null pointer");
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && H % 2 == 0 && W % 2 == 0, NM_E_INVALID,
             "nm_maxpool2x2_fwd: bad sizes (H, W must be even)");
  const int64_t total = N * (H / 2) * (W / 2) * C;
  int64_t blocks = ceil_div(total, 256);
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  maxpool2x2_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, y, N, (int)H, (int)W, (int)C);
  NM_LAUNCH_CHECK("nm_maxpool2x2_fwd");
  return NM_OK;
}

}  // extern "C"
