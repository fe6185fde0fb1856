// Speech features of processors/speech.py: the mfcc, fbank, logfbank and ssc functions of python_speech_features
// 0.6.1 and its delta, restated in fp64 (the library computes in float64, and the log band powers span many
// decades, so fp32 would lose the quiet bands).
//
// speech_frames_kernel   a CTA walks frames f = blockIdx.x, blockIdx.x + gridDim.x, ... and for each one, in
//                        shared memory: the pre-emphasised samples (y[n] = x[n] - p*x[n-1], y[0] = x[0], the
//                        previous sample read across the frame boundary) times the window, truncated or zero-padded
//                        to nfft, in bit-reversed order; an iterative radix-2 complex FFT over a twiddle table built
//                        once per CTA; the power spectrum |X|^2/nfft of the nfft/2+1 bins; the frame energy (a
//                        fixed-order block sum); one warp per filter over the filter's nonzero bin range only; and
//                        the epilogue of the feature type: eps for zeros, log, DCT-II (ortho) + lifter + the energy
//                        column for mfcc, or the spectral-centroid ratio for ssc.
// speech_delta_kernel    one thread per output element: d[t] = sum_{n=-N..N} n*x[clamp(t+n)] / (2*sum n^2),
//                        column block k -> block k+1.
#include <float.h>

#include <algorithm>

#include "common.cuh"

namespace nm {

constexpr int SPEECH_THREADS = 256;
constexpr int SPEECH_MAX_NFFT = 8192;
constexpr int SPEECH_MAX_FILTERS = 1024;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Fixed-order block sum (so two calls give identical bits); `red` is >= 32 doubles of shared memory.
__device__ __forceinline__ double block_sum_d(double v, double* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum_d(v);
  if (lane == 0) red[w] = v;
  __syncthreads();
  double r = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.0;
  if (w == 0) r = warp_sum_d(r);
  if (threadIdx.x == 0) red[32] = r;
  __syncthreads();
  return red[32];
}

struct SpeechArgs {
  const double* signal;
  int64_t samples;
  const double* window;
  int64_t frame_len, frame_step;
  int nfft, log2n;
  double preemph;
  const double* fbank;     // [nfilt, nfft/2+1]
  const int32_t* fb_first;  // [nfilt] first nonzero bin of each filter
  const int32_t* fb_last;   // [nfilt] one past the last
  int nfilt, kind, ncoef, append_energy;
  double ceplifter, rate;
  double* out;
  int64_t frames, out_stride;
};

// Shared memory (doubles): re [nfft] | im [nfft] | cos, sin twiddles [nfft/2 each] | feat [nfilt] | num [nfilt] |
// red [33].
__global__ void __launch_bounds__(SPEECH_THREADS) speech_frames_kernel(const SpeechArgs a) {
  extern __shared__ double sm[];
  const int n = a.nfft, half = n >> 1, nbins = half + 1;
  double* re = sm;
  double* im = re + n;
  double* twc = im + n;
  double* tws = twc + half;
  double* feat = tws + half;
  double* num = feat + a.nfilt;
  double* red = num + a.nfilt;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;

  for (int j = tid; j < half; j += blockDim.x) sincospi(-2.0 * j / n, &tws[j], &twc[j]);  // exp(-2 pi i j / n)
  const int64_t used = a.frame_len < n ? a.frame_len : n;        // a frame longer than nfft is truncated
  const double step = (a.rate / 2.0 - 1.0) / (double)(nbins - 1);  // ssc: bin centre i -> linspace(1, rate/2)

  for (int64_t f = blockIdx.x; f < a.frames; f += gridDim.x) {
    const int64_t base = f * a.frame_step;
    for (int i = tid; i < n; i += blockDim.x) {
      double v = 0.0;
      const int64_t s = base + i;
      if (i < used && s < a.samples) {
        v = a.signal[s];
        if (s > 0) v = __dsub_rn(v, __dmul_rn(a.preemph, a.signal[s - 1]));
        v = __dmul_rn(v, a.window[i]);
      }
      const int r = (int)(__brev((unsigned)i) >> (32 - a.log2n));
      re[r] = v;
      im[r] = 0.0;
    }
    __syncthreads();
    for (int s = 0; s < a.log2n; ++s) {
      const int h = 1 << s, stride = half >> s;  // butterflies of span 2h use twiddles j*stride
      for (int b = tid; b < half; b += blockDim.x) {
        const int j = b & (h - 1);
        const int i0 = ((b >> s) << (s + 1)) + j, i1 = i0 + h;
        const double wr = twc[j * stride], wi = tws[j * stride];
        const double xr = re[i1], xi = im[i1];
        const double tr = wr * xr - wi * xi, ti = wr * xi + wi * xr;
        const double ur = re[i0], ui = im[i0];
        re[i0] = ur + tr;
        im[i0] = ui + ti;
        re[i1] = ur - tr;
        im[i1] = ui - ti;
      }
      __syncthreads();
    }
    double e = 0.0;
    for (int k = tid; k < nbins; k += blockDim.x) {
      const double p = (re[k] * re[k] + im[k] * im[k]) / (double)n;
      re[k] = p;  // the power spectrum replaces the real part
      e += p;
    }
    const double energy = block_sum_d(e, red);  // its barrier also publishes re[0, nbins)

    const bool ssc = a.kind == NM_SPEECH_SSC;
    for (int j = warp; j < a.nfilt; j += nwarps) {
      const double* row = a.fbank + (int64_t)j * nbins;
      double acc = 0.0, acc_r = 0.0;
      for (int k = a.fb_first[j] + lane; k < a.fb_last[j]; k += 32) {
        double p = re[k];
        if (ssc) {
          if (p == 0.0) p = DBL_EPSILON;
          const double r = (k == nbins - 1) ? a.rate / 2.0 : k * step + 1.0;
          acc_r += p * r * row[k];
        }
        acc += p * row[k];
      }
      acc = warp_sum_d(acc);
      if (ssc) acc_r = warp_sum_d(acc_r);
      if (lane == 0) {
        feat[j] = acc;
        num[j] = acc_r;
      }
    }
    __syncthreads();

    double* o = a.out + f * a.out_stride;
    if (a.kind == NM_SPEECH_SSC) {
      for (int j = tid; j < a.nfilt; j += blockDim.x) o[j] = num[j] / feat[j];  // an empty filter gives 0/0 = NaN
    } else if (a.kind != NM_SPEECH_MFCC) {
      for (int j = tid; j < a.nfilt; j += blockDim.x) {
        const double v = feat[j] == 0.0 ? DBL_EPSILON : feat[j];
        o[j] = a.kind == NM_SPEECH_LOGFBANK ? log(v) : v;
      }
    } else {
      for (int j = tid; j < a.nfilt; j += blockDim.x) num[j] = log(feat[j] == 0.0 ? DBL_EPSILON : feat[j]);
      __syncthreads();
      // DCT-II, ortho: c_k = s_k * sum_m x_m cos(pi k (2m+1) / (2 nfilt)), s_0 = sqrt(1/nfilt), else sqrt(2/nfilt)
      for (int k = warp; k < a.ncoef; k += nwarps) {
        double acc = 0.0;
        for (int m = lane; m < a.nfilt; m += 32) acc += num[m] * cospi((double)((2 * m + 1) * k) / (2.0 * a.nfilt));
        acc = warp_sum_d(acc);
        if (lane == 0) {
          double c = acc * sqrt((k == 0 ? 1.0 : 2.0) / a.nfilt);
          if (a.ceplifter > 0.0) c *= 1.0 + (a.ceplifter / 2.0) * sinpi(k / a.ceplifter);
          if (k == 0 && a.append_energy) c = log(energy == 0.0 ? DBL_EPSILON : energy);
          o[k] = c;
        }
      }
    }
    __syncthreads();  // re, im, feat and num are rewritten by the next frame
  }
}

__global__ void speech_delta_kernel(double* __restrict__ out, int64_t frames, int64_t width, int64_t out_stride,
                                    int64_t block, int N, double denom) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= frames * width) return;
  const int64_t t = idx / width, c = idx % width;
  const double* x = out + block * width + c;
  double acc = 0.0;
  for (int n = -N; n <= N; ++n) {
    const int64_t s = t + n < 0 ? 0 : (t + n >= frames ? frames - 1 : t + n);
    acc += (double)n * x[s * out_stride];
  }
  out[t * out_stride + (block + 1) * width + c] = acc / denom;
}

}  // namespace nm

using namespace nm;

extern "C" {

int nm_speech_features(const double* signal, int64_t samples, const double* window, int64_t frame_len,
                       int64_t frame_step, int64_t nfft, double preemph, const double* fbank,
                       const int32_t* fb_first, const int32_t* fb_last, int64_t nfilt, int kind, int64_t numcep,
                       double ceplifter, int append_energy, double rate, double* out, int64_t frames,
                       int64_t out_stride, void* stream) {
  NM_REQUIRE(signal && window && fbank && fb_first && fb_last && out, NM_E_INVALID,
             "nm_speech_features: null pointer");
  NM_REQUIRE(samples > 0 && frame_len > 0 && frame_step > 0 && frames > 0 && nfilt > 0 && rate > 0.0,
             NM_E_INVALID, "nm_speech_features: bad sizes samples=%lld frame_len=%lld frame_step=%lld "
             "frames=%lld nfilt=%lld", (long long)samples, (long long)frame_len, (long long)frame_step,
             (long long)frames, (long long)nfilt);
  NM_REQUIRE(nfft >= 2 && nfft <= SPEECH_MAX_NFFT && (nfft & (nfft - 1)) == 0, NM_E_INVALID,
             "nm_speech_features: nfft=%lld is not a power of two in [2, %d]", (long long)nfft, SPEECH_MAX_NFFT);
  NM_REQUIRE(kind >= NM_SPEECH_MFCC && kind <= NM_SPEECH_SSC, NM_E_INVALID, "nm_speech_features: kind %d", kind);
  NM_REQUIRE(nfilt <= SPEECH_MAX_FILTERS, NM_E_UNSUPPORTED, "nm_speech_features: %lld filters, at most %d",
             (long long)nfilt, SPEECH_MAX_FILTERS);
  NM_REQUIRE(kind != NM_SPEECH_MFCC || numcep > 0, NM_E_INVALID, "nm_speech_features: numcep=%lld",
             (long long)numcep);
  const int64_t width = kind == NM_SPEECH_MFCC ? std::min(numcep, nfilt) : nfilt;
  NM_REQUIRE(out_stride >= width, NM_E_INVALID, "nm_speech_features: out_stride %lld < width %lld",
             (long long)out_stride, (long long)width);
  int log2n = 0;
  while ((1LL << log2n) < nfft) ++log2n;
  SpeechArgs a{signal, samples, window, frame_len, frame_step, (int)nfft, log2n, preemph, fbank, fb_first, fb_last,
               (int)nfilt, kind, (int)width, append_energy, ceplifter, rate, out, frames, out_stride};
  const size_t smem = (size_t)(3 * nfft + 2 * nfilt + 33) * sizeof(double);
  NM_CUDA_TRY(cudaFuncSetAttribute(speech_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  NM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, speech_frames_kernel, SPEECH_THREADS, smem));
  const int64_t grid = std::min<int64_t>(frames, (int64_t)std::max(per_sm, 1) * sm_count());
  speech_frames_kernel<<<(unsigned)grid, SPEECH_THREADS, smem, (cudaStream_t)stream>>>(a);
  NM_LAUNCH_CHECK("nm_speech_features");
  return NM_OK;
}

int nm_speech_deltas(double* out, int64_t frames, int64_t width, int64_t out_stride, int64_t block, int64_t window,
                     void* stream) {
  NM_REQUIRE(out, NM_E_INVALID, "nm_speech_deltas: null pointer");
  NM_REQUIRE(frames > 0 && width > 0 && block >= 0 && window >= 1 && window <= 1024, NM_E_INVALID,
             "nm_speech_deltas: bad sizes frames=%lld width=%lld block=%lld window=%lld", (long long)frames,
             (long long)width, (long long)block, (long long)window);
  NM_REQUIRE(out_stride >= (block + 2) * width, NM_E_INVALID, "nm_speech_deltas: out_stride %lld < %lld",
             (long long)out_stride, (long long)((block + 2) * width));
  const double denom = 2.0 * (double)(window * (window + 1) * (2 * window + 1) / 6);  // 2 * sum_{n=1..N} n^2
  speech_delta_kernel<<<(unsigned)ceil_div(frames * width, 256), 256, 0, (cudaStream_t)stream>>>(
      out, frames, width, out_stride, block, (int)window, denom);
  NM_LAUNCH_CHECK("nm_speech_deltas");
  return NM_OK;
}

}  // extern "C"
