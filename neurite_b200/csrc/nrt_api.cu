// nrt_api.cu -- status strings, thread-local error detail, device queries.
#include "nrt_common.cuh"

#include <string.h>

namespace nrt {

static thread_local char g_err[512] = "";

int set_error(int status, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return status;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return set_error(NRT_E_LAUNCH, "%s: %s", what, cudaGetErrorString(e));
  return NRT_OK;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

}  // namespace nrt

extern "C" {

int nrt_version(void) { return NRT_ABI_VERSION; }

const char* nrt_last_error_string(void) { return nrt::g_err; }

const char* nrt_status_string(int status) {
  switch (status) {
    case NRT_OK: return "ok";
    case NRT_E_ARG: return "bad argument";
    case NRT_E_SIZE: return "size out of range";
    case NRT_E_LAUNCH: return "CUDA launch/runtime error";
    case NRT_E_ALIGN: return "misaligned pointer";
    case NRT_E_NODEV: return "no usable device";
    default: return "unknown status";
  }
}

}  // extern "C"
