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
extern "C" int dba_version(void) { return 200; }
