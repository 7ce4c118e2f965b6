// Diagnostics of libtfimm_b200.so (declared in include/tfimm_b200.h) plus the error-reporting plumbing shared by every
// translation unit.  Each kernel entry point is defined in the file of its kernel.
#include <stdarg.h>

#include "common.cuh"

namespace tfimm {

namespace {
thread_local char g_last_error[1024] = "";
}

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_last_error("CUDA error in %s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return kCudaError;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  if (dev >= 0 && dev < 64 && cached[dev] > 0) return cached[dev];
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  if (dev >= 0 && dev < 64) cached[dev] = n;
  return n;
}

}  // namespace tfimm

extern "C" {

const char* tfimm_b200_version(void) { return "tfimm_b200 0.1.0 (sm_90a)"; }
const char* tfimm_b200_last_error(void) { return tfimm::g_last_error; }
int tfimm_b200_sm_count(void) { return tfimm::sm_count(); }

}  // extern "C"
