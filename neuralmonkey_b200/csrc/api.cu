// Library bookkeeping: version, thread-local error message, device info.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace nm {

static thread_local char g_err[512] = "";
static unsigned long long g_launches = 0;

void count_launches(int64_t n) { __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 1;   // no device: the launch reports it
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 1;
    cached[dev] = n;
  }
  return cached[dev];
}

}  // namespace nm

extern "C" {

int nm_version(void) { return NM_ABI_VERSION; }

const char* nm_last_error(void) { return nm::g_err; }

int64_t nm_launch_count(void) { return (int64_t)__atomic_load_n(&nm::g_launches, __ATOMIC_RELAXED); }

int nm_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  NM_REQUIRE(sm_count && cc_major && cc_minor, NM_E_INVALID, "nm_device_info: null output");
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    nm::set_error("nm_device_info: %s", cudaGetErrorString(e));
    return NM_E_NO_DEVICE;
  }
  NM_CUDA_TRY(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
  NM_CUDA_TRY(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
  NM_CUDA_TRY(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
  return NM_OK;
}

}  // extern "C"
