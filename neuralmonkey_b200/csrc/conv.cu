// K12: slim VGG and ResNet-v2 building blocks, forward only (the ImageNet encoder is frozen:
// encoders/imagenet_encoder.py:212,234 of the reference).  NHWC fp32.
//   conv3x3, stride 1, SAME, + bias + ReLU  (vgg_arg_scope of tensorflow/models slim nets/vgg.py)
//   max-pool 2x2 / 2
//   nm_conv2d_bn_fwd: a k x k convolution at stride s with explicit pads, an optional batch-norm + ReLU prologue on
//   its input, and an inference-mode batch norm or bias, an optional (subsampled) residual and ReLU on its output -
//   every convolution of a ResNet-v2 bottleneck unit in one launch
// The 3x3 convolution runs on the exact fp32 CUDA-core kernel of conv_igemm.cuh (k = 3, pads 1, ReLU);
// nm_im2col3x3 builds the patch matrix for the tensor-core path through nm_gemm.  nm_conv2d_bn_fwd runs on either
// engine of conv_igemm.cuh.
#include "conv_igemm.cuh"

namespace nm {

// im2col for the tensor-core path: cols[m][tap*Cin + c] = x[n, y+dy, x+dx, c] (zero outside the
// image), row pitch `ldc` floats.  One thread per (pixel, tap, 4-channel group); the group moves as one
// float4 when Cin, ldc and both pointers keep it 16-byte aligned.
__global__ void im2col3x3_kernel(const float* __restrict__ x, float* __restrict__ cols, int64_t NB, int H,
                                 int W, int Cin, int64_t ldc) {
  const int groups = (Cin + 3) / 4;
  const bool vec = (Cin & 3) == 0 && (ldc & 3) == 0 &&
                   ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(cols)) & 15) == 0;
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
    if (vec) {
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
  const ConvGeom g = conv_geom_of(N, H, W, Cin, Cout, 3, 3, 1, 1, H, W);
  return conv_fwd_launch<CS_BN, false, false>(x, w, g, BiasAct{bias, y, NM_ACT_RELU}, NM_GEMM_SIMT,
                                              (cudaStream_t)stream, "nm_conv3x3_bias_relu_fwd");
}

int nm_conv2d_bn_fwd(const float* x, const float* w, const float* in_scale, const float* in_shift,
                     const float* out_scale, const float* out_shift, const float* bias, const float* res,
                     int64_t res_H, int64_t res_W, int64_t res_stride, float* y, int64_t N, int64_t H, int64_t W,
                     int64_t Cin, int64_t Cout, int64_t k, int64_t stride, int64_t pad_top, int64_t pad_bottom,
                     int64_t pad_left, int64_t pad_right, int act, int backend, void* stream) {
  static const char* name = "nm_conv2d_bn_fwd";
  NM_REQUIRE(x && w && y, NM_E_INVALID, "%s: null pointer", name);
  NM_REQUIRE(!in_scale == !in_shift, NM_E_INVALID, "%s: in_scale and in_shift go together", name);
  NM_REQUIRE(!out_scale == !out_shift, NM_E_INVALID, "%s: out_scale and out_shift go together", name);
  NM_REQUIRE(!(out_scale && bias), NM_E_INVALID, "%s: out_scale/out_shift and bias exclude each other", name);
  NM_REQUIRE(act == NM_ACT_NONE || act == NM_ACT_RELU, NM_E_INVALID, "%s: act must be none or relu", name);
  NM_REQUIRE(backend == NM_GEMM_AUTO || backend == NM_GEMM_TC || backend == NM_GEMM_SIMT, NM_E_INVALID,
             "%s: bad backend", name);
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && k > 0 && stride > 0, NM_E_INVALID, "%s: bad sizes",
             name);
  NM_REQUIRE(pad_top >= 0 && pad_bottom >= 0 && pad_left >= 0 && pad_right >= 0 && pad_top < k && pad_bottom < k &&
                 pad_left < k && pad_right < k,
             NM_E_INVALID, "%s: pads must lie in [0, k)", name);
  NM_REQUIRE(H + pad_top + pad_bottom >= k && W + pad_left + pad_right >= k, NM_E_INVALID,
             "%s: window larger than the padded image", name);
  const int64_t Ho = (H + pad_top + pad_bottom - k) / stride + 1, Wo = (W + pad_left + pad_right - k) / stride + 1;
  NM_REQUIRE(k * k * Cin < (1LL << 30) && Cout < (1LL << 24) && N * H * W * Cin < (1LL << 40) && H < (1 << 20) &&
                 W < (1 << 20) && stride < (1 << 10),
             NM_E_UNSUPPORTED, "%s: sizes out of range", name);
  int rs = 1;
  if (res) {
    NM_REQUIRE(res_stride == 1 || res_stride == 2, NM_E_UNSUPPORTED, "%s: res_stride must be 1 or 2", name);
    rs = (int)res_stride;
    NM_REQUIRE(res_H > 0 && res_W > 0 && ceil_div(res_H, res_stride) == Ho && ceil_div(res_W, res_stride) == Wo &&
                   res_H < (1 << 20) && res_W < (1 << 20),
               NM_E_INVALID, "%s: residual [N,%lld,%lld,Cout] at stride %lld does not match the %lldx%lld output",
               name, (long long)res_H, (long long)res_W, (long long)res_stride, (long long)Ho, (long long)Wo);
  }
  const ConvGeom g = conv_geom_of(N, H, W, Cin, Cout, k, k, pad_top, pad_left, Ho, Wo);
  const BnRes epi{out_scale, out_shift, bias, res, y, act, rs, (int)(res ? res_H : 0), (int)(res ? res_W : 0)};
  const BnReluIn in{in_scale, in_shift, (int)stride};
  return conv_fwd_launch<CS_BN, false, false>(x, w, g, epi, backend, (cudaStream_t)stream, name, in);
}

int nm_im2col3x3(const float* x, float* cols, int64_t N, int64_t H, int64_t W, int64_t Cin,
                 int64_t ldc, void* stream) {
  NM_REQUIRE(x && cols, NM_E_INVALID, "nm_im2col3x3: null pointer");
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && Cin > 0 && ldc >= 9 * Cin, NM_E_INVALID, "nm_im2col3x3: bad sizes");
  im2col3x3_kernel<<<grid_for(N * H * W * 9 * ((Cin + 3) / 4)), 256, 0, (cudaStream_t)stream>>>(
      x, cols, N, (int)H, (int)W, (int)Cin, ldc);
  NM_LAUNCH_CHECK("nm_im2col3x3");
  return NM_OK;
}

int nm_maxpool2x2_fwd(const float* x, float* y, int64_t N, int64_t H, int64_t W, int64_t C,
                      void* stream) {
  NM_REQUIRE(x && y, NM_E_INVALID, "nm_maxpool2x2_fwd: null pointer");
  NM_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && H % 2 == 0 && W % 2 == 0, NM_E_INVALID,
             "nm_maxpool2x2_fwd: bad sizes (H, W must be even)");
  maxpool2x2_kernel<<<grid_for(N * (H / 2) * (W / 2) * C), 256, 0, (cudaStream_t)stream>>>(x, y, N, (int)H, (int)W,
                                                                                           (int)C);
  NM_LAUNCH_CHECK("nm_maxpool2x2_fwd");
  return NM_OK;
}

}  // extern "C"
