// common.cu -- what belongs to the whole library rather than to one module: the thread-local error message behind
// set_error / b200orb_last_error, the device check of every *_create, and the library-level C-ABI queries.
#include <cstdarg>

#include "common.cuh"

namespace b200 {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_device(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device available (%s); libb200orb has no CPU fallback",
              e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    cudaGetLastError();
    return B200ORB_ENOGPU;
  }
  if (device < 0 || device >= n) {
    set_error("device %d out of range (0..%d)", device, n - 1);
    return B200ORB_EINVAL;
  }
  return B200ORB_OK;
}

}  // namespace b200

extern "C" {

const char* b200orb_last_error(void) { return b200::g_err; }
const char* b200orb_version(void) { return "b200orb 0.1 (sm_90a)"; }
int b200orb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

}  // extern "C"
