// Error plumbing + trivial entry points of the C-ABI (include/ttb.h).
#include "common.cuh"
#include "ttb_internal.h"
#include <cstdarg>
#include <cstdio>

namespace ttb {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return -2;
}
}  // namespace ttb

extern "C" const char* ttb_last_error(void) { return ttb::g_err; }
extern "C" int ttb_version(void) { return 100; }
extern "C" int ttb_device_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 0;
  return (p.major == 9 && p.minor == 0) ? 1 : 0;
}
