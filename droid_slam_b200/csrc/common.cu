#include "common.cuh"
#include <stdarg.h>
#include <string.h>

namespace dba {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error in %s: %s", what, cudaGetErrorString(e));
  return DBA_ERR_CUDA;
}
}  // namespace dba

extern "C" const char* dba_last_error(void) { return dba::g_err; }
extern "C" int dba_version(void) { return 100; }

// L2 fetch granularity (cudaLimitMaxL2FetchGranularity: 32, 64 or 128 bytes; device-wide hint).  The corr_index gather
// touches 16-32 byte runs at arbitrary alignment; with the default 64-byte granularity every touched 32-byte sector drags
// its neighbour out of HBM (5.4x read amplification at pyramid level 0, measured on B200, not re-measured on H100).  Callers
// that own the device may lower it to 32.
extern "C" int dba_set_l2_fetch_granularity(int bytes) {
  if (bytes != 32 && bytes != 64 && bytes != 128) { dba::set_error("invalid argument: granularity must be 32, 64 or 128"); return DBA_ERR_INVALID; }
  cudaError_t e = cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)bytes);
  if (e != cudaSuccess) return dba::cuda_fail(e, "cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity)");
  return DBA_OK;
}
extern "C" int dba_get_l2_fetch_granularity(void) {
  size_t v = 0;
  if (cudaDeviceGetLimit(&v, cudaLimitMaxL2FetchGranularity) != cudaSuccess) { cudaGetLastError(); return -1; }
  return (int)v;
}
