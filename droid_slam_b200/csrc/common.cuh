// Shared device helpers for the sm_90a kernels of the dense-BA update path.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/droid_b200.h"

namespace dba {

void set_error(const char* fmt, ...);
// chol.cu: damped SPD solve (fp64, one thread-block cluster)
size_t chol_workspace_bytes(int n);
struct CholPeers {            // fused peer-to-peer reduction (world > 1): H/b are summed over peer copies in rank order
  int world;
  const double* sys[8];       // peer-mapped pointers to each rank's [n*n + n] system for this epoch
  const unsigned long long* flags;   // this rank's flag array [world], flag[p] >= epoch when rank p has published
  unsigned long long epoch;
  const unsigned long long* epoch_dev;   // when set, the awaited value is read from this rank-local device counter (CUDA-graph replay)
};
int chol_solve_launch(const double* H, const double* b, int n, double lm, double ep, void* workspace, int* fail, float* x, cudaStream_t st,
                      const CholPeers* peers = nullptr);
int cuda_fail(cudaError_t e, const char* what);
// corr_lookup_rows.cu: dba_corr_lookup_pyramid for level rows that are not whole 16-byte chunks (arguments checked by the caller)
int corr_lookup_pyramid_rows_launch(const __half* v0, const __half* v1, const __half* v2, const __half* v3, const float* coords, __half* out,
                                    long long total, int h1, int w1, cudaStream_t st);

#define DBA_CHECK_ARG(cond, msg)                                   \
  do { if (!(cond)) { dba::set_error("invalid argument: %s", msg); return DBA_ERR_INVALID; } } while (0)
#define DBA_CHECK_LAUNCH(what)                                     \
  do { cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) return dba::cuda_fail(e__, what); } while (0)
#define DBA_CHECK_CUDA(expr, what)                                 \
  do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return dba::cuda_fail(e__, what); } while (0)

constexpr float kMinDepth = 0.25f;   // reference MIN_DEPTH, src/droid_kernels.cu:35

__device__ __forceinline__ int floor_to_int_sat(float f) {
  // static_cast<int>(floor(f)) as the GPU evaluates it: saturating, NaN -> 0; then kept away from INT limits
  int i = __float2int_rd(f);
  return max(-(1 << 30), min(1 << 30, i));
}

// ---- 128-bit streaming loads / stores -----------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// same, allocated in L1: another load of the same 32-byte sector by the SM is served from L1 instead of L2
__device__ __forceinline__ uint4 ldg_nc_v4_l1(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace dba
