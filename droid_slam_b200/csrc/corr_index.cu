// corr_index_forward / corr_index_backward for sm_90a.
//
// Replaces reference src/correlation_kernels.cu:20-185.  Semantics (checked against oracle/corr.py):
//   out[n][i][j][y][x] = bilinear sample of volume[n][y][x][.][.] at (y0-r+j, x0-r+i), taps outside the plane
//   contribute nothing; per output the four taps are combined in the volume dtype in the reference order
//   (i,j),(i,j+1),(i+1,j),(i+1,j+1)  (x-index first), weights rounded to the volume dtype:
//     f32/f64: one FMA per tap (nvcc contracts the reference's `+= s*w`),  f16: product and sum rounded separately.
//
// Design (HBM-bound gather, see DESIGN.md "corr_index"):
//   * one thread per (edge, pixel); consecutive threads = consecutive x  => the 49 stores per thread are
//     warp-coalesced rows of the [n][i][j][y][x] output, coords loads are coalesced;
//   * the 8x8 tap window is fetched as 16-byte aligned vector loads (2 per window row for f16, 3 for f32),
//     all 16/24 loads of a pixel issued before first use (memory-level parallelism), streamed past L1
//     (ld.global.nc.L1::no_allocate), except in the fused lookup on tiled volumes, where the two loads that share a 32-byte
//     sector meet in L1 (corr_lookup_pyramid_f16_kernel);  window alignment inside the vectors is resolved in registers with a
//     3-level select / funnel-shift network (no local memory, no shared memory);
//   * out-of-plane rows / 16-byte chunks are predicated off and zero filled: for finite coordinates a zero tap
//     contributes exactly +-0, identical to the reference's skip.  Non-finite coordinates take the exact
//     skip-semantics slow path.
//   * no memset of the output (the reference needs torch::zeros + 4 global RMWs per element).
#include "corr_pixel.cuh"

namespace dba {

// ------------------------------------------------------------------------------------------------------
// generic kernels: any radius, any extents, exact skip semantics.  One thread per pixel.
// ------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) corr_index_fwd_generic_kernel(const T* __restrict__ vol, const float* __restrict__ coords,
                                                                     T* __restrict__ out, long long total, int hw1, int h2, int w2, int r) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  const float x0 = coords[((size_t)n * 2 + 0) * hw1 + pin];
  const float y0 = coords[((size_t)n * 2 + 1) * hw1 + pin];
  const int rd = 2 * r + 1;
  corr_pixel_generic<T>(vol + (size_t)p * h2 * w2, out + (size_t)n * rd * rd * hw1 + pin, (size_t)hw1, x0, y0, h2, w2, r);
}

// backward: volume_grad[n][y][x][y1][x1] = g  (planes are private to a pixel -> plain stores after a memset)
template <typename T> struct GradMath;
template <> struct GradMath<float> {
  static __device__ __forceinline__ float w(float v) { return v; }
  static __device__ __forceinline__ float mac(float g, float cg, float w) { return fmaf(cg, w, g); }
  static __device__ __forceinline__ float zero() { return 0.f; }
};
template <> struct GradMath<double> {
  static __device__ __forceinline__ double w(float v) { return (double)v; }
  static __device__ __forceinline__ double mac(double g, double cg, double w) { return fma(cg, w, g); }
  static __device__ __forceinline__ double zero() { return 0.0; }
};
template <> struct GradMath<__half> {
  static __device__ __forceinline__ __half w(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ __half mac(__half g, __half cg, __half w) { return __hadd_rn(g, __hmul_rn(cg, w)); }
  static __device__ __forceinline__ __half zero() { return __float2half_rn(0.f); }
};
template <> struct GradMath<__nv_bfloat16> {   // extension: bf16 rounding per op, like the f16 path
  static __device__ __forceinline__ __nv_bfloat16 w(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ __nv_bfloat16 mac(__nv_bfloat16 g, __nv_bfloat16 cg, __nv_bfloat16 w) {
    float p = __bfloat162float(__float2bfloat16_rn(__bfloat162float(cg) * __bfloat162float(w)));
    return __float2bfloat16_rn(__bfloat162float(g) + p);
  }
  static __device__ __forceinline__ __nv_bfloat16 zero() { return __float2bfloat16_rn(0.f); }
};

template <typename T>
__global__ void __launch_bounds__(128) corr_index_bwd_kernel(const float* __restrict__ coords, const T* __restrict__ cg,
                                                             T* __restrict__ vg, long long total, int hw1, int h2, int w2, int r) {
  typedef GradMath<T> M;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  const float x0 = coords[((size_t)n * 2 + 0) * hw1 + pin];
  const float y0 = coords[((size_t)n * 2 + 1) * hw1 + pin];
  const float fxf = floorf(x0), fyf = floorf(y0);
  const float dx = x0 - fxf, dy = y0 - fyf;
  const int fx = floor_to_int_sat(fxf), fy = floor_to_int_sat(fyf);
  const T w11 = M::w(dx * dy), w10 = M::w(dx * (1.0f - dy)), w01 = M::w((1.0f - dx) * dy), w00 = M::w((1.0f - dx) * (1.0f - dy));
  const int rd = 2 * r + 1;
  const T* g_in = cg + (size_t)n * rd * rd * hw1 + pin;
  T* plane = vg + (size_t)p * h2 * w2;
  for (int i = 0; i < rd + 1; i++) {
    for (int j = 0; j < rd + 1; j++) {
      const int x1 = fx - r + i, y1 = fy - r + j;
      if ((unsigned)x1 < (unsigned)w2 && (unsigned)y1 < (unsigned)h2) {
        T g = M::zero();
        if (i > 0 && j > 0) g = M::mac(g, g_in[(size_t)((i - 1) * rd + (j - 1)) * hw1], w11);
        if (i > 0 && j < rd) g = M::mac(g, g_in[(size_t)((i - 1) * rd + j) * hw1], w10);
        if (i < rd && j > 0) g = M::mac(g, g_in[(size_t)(i * rd + (j - 1)) * hw1], w01);
        if (i < rd && j < rd) g = M::mac(g, g_in[(size_t)(i * rd + j) * hw1], w00);
        plane[(size_t)y1 * w2 + x1] = g;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// fast path, radius 3: f16 (w2 % 8 == 0) and f32 (w2 % 4 == 0), 16-byte aligned base pointers
// ------------------------------------------------------------------------------------------------------
// chunk (y1, cx) of a plane in global memory, row-major or 4x8-tiled
template <bool TILED, typename T16>
__device__ __forceinline__ const T16* plane_chunk(const T16* plane, int y1, int cx, int w2) {
  return TILED ? plane + ((size_t)(y1 >> 2) * (w2 >> 3) + cx) * 32 + (y1 & 3) * 8 : plane + (size_t)y1 * w2 + cx * 8;
}

template <bool TILED, typename T16 = __half, bool L1 = false>
__device__ __forceinline__ void corr_pixel_f16_r3(const T16* __restrict__ plane, T16* __restrict__ out_px, size_t out_stride,
                                                  float x0, float y0, int h2, int w2) {
  auto fetch = [&](int y1, int cx) {
    const T16* chunk = plane_chunk<TILED>(plane, y1, cx, w2);
    return L1 ? ldg_nc_v4_l1(chunk) : ldg_nc_v4(chunk);
  };
  corr_pixel_f16_r3_from<TILED, T16>(fetch, plane, out_px, out_stride, x0, y0, h2, w2);
}

template <typename T16>
__global__ void __launch_bounds__(128) corr_index_fwd_f16_r3_kernel(const T16* __restrict__ vol, const float* __restrict__ coords,
                                                                    T16* __restrict__ out, long long total, int hw1, int h2, int w2) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  const float x0 = coords[((size_t)n * 2 + 0) * hw1 + pin];
  const float y0 = coords[((size_t)n * 2 + 1) * hw1 + pin];
  corr_pixel_f16_r3<false, T16>(vol + (size_t)p * h2 * w2, out + (size_t)n * 49 * hw1 + pin, (size_t)hw1, x0, y0, h2, w2);
}

// CorrBlock.__call__ (reference modules/corr.py:40-50) in ONE launch: all four pyramid levels of a pixel by one thread -- the
// coordinates are read once, the level-l lookup uses coords / 2^l (exact in fp32, like the reference's `coords/2**i`), and the four
// [49,H,W] results land directly in the concatenated [E,196,H,W] tensor the update operator consumes (the reference allocates four
// tensors and copies them with torch.cat).  tiled_levels: bit l set = level l is stored in the 4x8-tile layout.
// L1: window loads allocate in L1.  A 32-byte sector holds two rows of a 4x8 tile (levels 0-1), one whole 16-wide row (level 2, both
// chunks A and B) or two 8-wide rows (level 3); the pixel loads each row separately, so without L1 every sector crosses L2 -> SM twice.
// With L1 the second load of a sector hits: on an H100 SXM (400 W) the tiled lookup at 512 edges, 48x64 goes from 1.214 to 0.706 ms.
// It is compiled with minBlocks = 1 (136 registers, 3 CTAs per SM, no spills); capping it at 80 registers for 6 CTAs measured ~9 % slower.
template <int TILED_MASK, bool L1>
__global__ void __launch_bounds__(128, L1 ? 1 : 0) corr_lookup_pyramid_f16_kernel(const __half* __restrict__ v0, const __half* __restrict__ v1,
                                                                      const __half* __restrict__ v2, const __half* __restrict__ v3,
                                                                      const float* __restrict__ coords, __half* __restrict__ out,
                                                                      long long total, int hw1, int h1, int w1) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  const float x0 = coords[((size_t)n * 2 + 0) * hw1 + pin];
  const float y0 = coords[((size_t)n * 2 + 1) * hw1 + pin];
  __half* o = out + (size_t)n * 196 * hw1 + pin;
  // coarse levels first: their planes are small and their loads return while the level-0 window (the expensive one) is being issued
  corr_pixel_f16_r3<(TILED_MASK & 8) != 0, __half, L1>(v3 + (size_t)p * (h1 >> 3) * (w1 >> 3), o + (size_t)147 * hw1, (size_t)hw1, x0 * 0.125f, y0 * 0.125f, h1 >> 3, w1 >> 3);
  corr_pixel_f16_r3<(TILED_MASK & 4) != 0, __half, L1>(v2 + (size_t)p * (h1 >> 2) * (w1 >> 2), o + (size_t)98 * hw1, (size_t)hw1, x0 * 0.25f, y0 * 0.25f, h1 >> 2, w1 >> 2);
  corr_pixel_f16_r3<(TILED_MASK & 2) != 0, __half, L1>(v1 + (size_t)p * (h1 >> 1) * (w1 >> 1), o + (size_t)49 * hw1, (size_t)hw1, x0 * 0.5f, y0 * 0.5f, h1 >> 1, w1 >> 1);
  corr_pixel_f16_r3<(TILED_MASK & 1) != 0, __half, L1>(v0 + (size_t)p * h1 * w1, o, (size_t)hw1, x0, y0, h1, w1);
}

// one pixel, one level, f32, radius 3, w2 % 4 == 0 and a 16-byte aligned plane: the 8x8 tap window from 16-byte chunks
__device__ __forceinline__ void corr_pixel_f32_r3(const float* __restrict__ plane, float* __restrict__ out_px, size_t hw1, float x0, float y0,
                                                  int h2, int w2) {
  if (!(isfinite(x0) && isfinite(y0))) {
    corr_pixel_generic<float>(plane, out_px, (size_t)hw1, x0, y0, h2, w2, 3);
    return;
  }
  const float fxf = floorf(x0), fyf = floorf(y0);
  const float dx = x0 - fxf, dy = y0 - fyf;
  const int x1s = floor_to_int_sat(fxf) - 3, y1s = floor_to_int_sat(fyf) - 3;
  const int a0 = x1s & ~3;
  const int o = x1s - a0;   // 0..3
  const bool ok0 = (unsigned)a0 < (unsigned)w2, ok1 = (unsigned)(a0 + 4) < (unsigned)w2, ok2 = (unsigned)(a0 + 8) < (unsigned)w2;
  const float w00 = (1.0f - dx) * (1.0f - dy), w01 = (1.0f - dx) * dy, w10 = dx * (1.0f - dy), w11 = dx * dy;

  float prev[8], cur[8];
  // two rows in flight at a time would starve the memory system; issue all 24 loads first
  uint4 C0[8], C1[8], C2[8];
#pragma unroll
  for (int b = 0; b < 8; b++) {
    const int y1 = y1s + b;
    const bool rowok = (unsigned)y1 < (unsigned)h2;
    const float* row = plane + (size_t)y1 * w2 + a0;
    C0[b] = make_uint4(0, 0, 0, 0); C1[b] = make_uint4(0, 0, 0, 0); C2[b] = make_uint4(0, 0, 0, 0);
    if (rowok && ok0) C0[b] = ldg_nc_v4(row);
    if (rowok && ok1) C1[b] = ldg_nc_v4(row + 4);
    if (rowok && ok2) C2[b] = ldg_nc_v4(row + 8);
  }
  auto align_row = [&](int b, float* t) {
    uint32_t f0 = C0[b].x, f1 = C0[b].y, f2 = C0[b].z, f3 = C0[b].w, f4 = C1[b].x, f5 = C1[b].y, f6 = C1[b].z, f7 = C1[b].w,
             f8 = C2[b].x, f9 = C2[b].y, f10 = C2[b].z;
    if (o & 2) { f0 = f2; f1 = f3; f2 = f4; f3 = f5; f4 = f6; f5 = f7; f6 = f8; f7 = f9; f8 = f10; }
    if (o & 1) { f0 = f1; f1 = f2; f2 = f3; f3 = f4; f4 = f5; f5 = f6; f6 = f7; f7 = f8; }
    t[0] = __uint_as_float(f0); t[1] = __uint_as_float(f1); t[2] = __uint_as_float(f2); t[3] = __uint_as_float(f3);
    t[4] = __uint_as_float(f4); t[5] = __uint_as_float(f5); t[6] = __uint_as_float(f6); t[7] = __uint_as_float(f7);
  };
  align_row(0, prev);
#pragma unroll
  for (int j = 0; j < 7; j++) {
    align_row(j + 1, cur);
#pragma unroll
    for (int i = 0; i < 7; i++) {
      float t = fmaf(prev[i], w00, 0.f);
      t = fmaf(cur[i], w01, t);
      t = fmaf(prev[i + 1], w10, t);
      t = fmaf(cur[i + 1], w11, t);
      out_px[(size_t)(i * 7 + j) * hw1] = t;
    }
#pragma unroll
    for (int i = 0; i < 8; i++) prev[i] = cur[i];
  }
}

__global__ void __launch_bounds__(128) corr_index_fwd_f32_r3_kernel(const float* __restrict__ vol, const float* __restrict__ coords,
                                                                    float* __restrict__ out, long long total, int hw1, int h2, int w2) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  corr_pixel_f32_r3(vol + (size_t)p * h2 * w2, out + (size_t)n * 49 * hw1 + pin, (size_t)hw1, coords[((size_t)n * 2 + 0) * hw1 + pin],
                    coords[((size_t)n * 2 + 1) * hw1 + pin], h2, w2);
}

// the fused 4-level lookup on f32 volumes in the reference layout: per level the path corr_index_forward takes for that plane (the
// chunked one where level rows are whole 16-byte chunks, else the generic one), so the result is that of 4 x corr_index_forward + cat
__global__ void __launch_bounds__(128) corr_lookup_pyramid_f32_kernel(const float* __restrict__ v0, const float* __restrict__ v1,
                                                                      const float* __restrict__ v2, const float* __restrict__ v3,
                                                                      const float* __restrict__ coords, float* __restrict__ out,
                                                                      long long total, int hw1, int h1, int w1) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  const float x0 = coords[((size_t)n * 2 + 0) * hw1 + pin];
  const float y0 = coords[((size_t)n * 2 + 1) * hw1 + pin];
#pragma unroll 1
  for (int l = 3; l >= 0; l--) {
    const int h2 = h1 >> l, w2 = w1 >> l;
    const float s = 1.0f / (float)(1 << l);
    const float* plane = (l == 0 ? v0 : l == 1 ? v1 : l == 2 ? v2 : v3) + (size_t)p * h2 * w2;
    float* o = out + ((size_t)n * 196 + 49 * l) * hw1 + pin;
    if (w2 % 4 == 0) corr_pixel_f32_r3(plane, o, (size_t)hw1, x0 * s, y0 * s, h2, w2);
    else corr_pixel_generic<float>(plane, o, (size_t)hw1, x0 * s, y0 * s, h2, w2, 3);
  }
}

template <typename T>
static int launch_generic_fwd(const void* vol, const float* coords, void* out, long long total, int hw1, int h2, int w2, int r,
                              cudaStream_t st) {
  const int threads = 128;
  const long long blocks = (total + threads - 1) / threads;
  corr_index_fwd_generic_kernel<T><<<(unsigned)blocks, threads, 0, st>>>((const T*)vol, coords, (T*)out, total, hw1, h2, w2, r);
  DBA_CHECK_LAUNCH("corr_index_forward(generic)");
  return DBA_OK;
}

template <typename T>
static int launch_bwd(const float* coords, const void* cg, void* vg, long long total, int hw1, int h2, int w2, int r, cudaStream_t st) {
  DBA_CHECK_CUDA(cudaMemsetAsync(vg, 0, (size_t)total * h2 * w2 * sizeof(T), st), "corr_index_backward memset");
  const int threads = 128;
  const long long blocks = (total + threads - 1) / threads;
  corr_index_bwd_kernel<T><<<(unsigned)blocks, threads, 0, st>>>(coords, (const T*)cg, (T*)vg, total, hw1, h2, w2, r);
  DBA_CHECK_LAUNCH("corr_index_backward");
  return DBA_OK;
}

}  // namespace dba

using namespace dba;

static int check_corr_args(const void* a, const void* b, const void* c, int n, int h1, int w1, int h2, int w2, int radius, int dtype) {
  DBA_CHECK_ARG(n >= 0 && h1 >= 0 && w1 >= 0 && h2 >= 0 && w2 >= 0, "negative extent");
  DBA_CHECK_ARG(radius >= 0 && radius <= 64, "radius out of range");
  DBA_CHECK_ARG(dtype == DBA_F32 || dtype == DBA_F16 || dtype == DBA_F64 || dtype == DBA_BF16, "unsupported dtype");
  const long long total = (long long)n * h1 * w1;
  if (total > 0) DBA_CHECK_ARG(a && b && c, "null pointer");
  DBA_CHECK_ARG((total + 127) / 128 < 0x7fffffffLL, "too many pixels for one launch");
  return DBA_OK;
}

extern "C" int dba_corr_index_forward(const void* volume, const float* coords, void* corr, int n, int h1, int w1, int h2, int w2,
                                      int radius, int dtype, dba_stream_t stream) {
  int rc = check_corr_args(volume, coords, corr, n, h1, w1, h2, w2, radius, dtype);
  if (rc) return rc;
  const long long total = (long long)n * h1 * w1;
  if (total == 0) return DBA_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int hw1 = h1 * w1;
  const bool aligned = (((uintptr_t)volume) & 15) == 0;
  const int threads = 128;
  const unsigned blocks = (unsigned)((total + threads - 1) / threads);
  if (radius == 3 && dtype == DBA_F16 && aligned && (w2 % 8) == 0 && h2 > 0) {
    corr_index_fwd_f16_r3_kernel<__half><<<blocks, threads, 0, st>>>((const __half*)volume, coords, (__half*)corr, total, hw1, h2, w2);
    DBA_CHECK_LAUNCH("corr_index_forward(f16,r3)");
    return DBA_OK;
  }
  if (radius == 3 && dtype == DBA_BF16 && aligned && (w2 % 8) == 0 && h2 > 0) {
    corr_index_fwd_f16_r3_kernel<__nv_bfloat16><<<blocks, threads, 0, st>>>((const __nv_bfloat16*)volume, coords, (__nv_bfloat16*)corr, total, hw1, h2, w2);
    DBA_CHECK_LAUNCH("corr_index_forward(bf16,r3)");
    return DBA_OK;
  }
  if (radius == 3 && dtype == DBA_F32 && aligned && (w2 % 4) == 0 && h2 > 0) {
    corr_index_fwd_f32_r3_kernel<<<blocks, threads, 0, st>>>((const float*)volume, coords, (float*)corr, total, hw1, h2, w2);
    DBA_CHECK_LAUNCH("corr_index_forward(f32,r3)");
    return DBA_OK;
  }
  switch (dtype) {
    case DBA_F32: return launch_generic_fwd<float>(volume, coords, corr, total, hw1, h2, w2, radius, st);
    case DBA_F16: return launch_generic_fwd<__half>(volume, coords, corr, total, hw1, h2, w2, radius, st);
    case DBA_F64: return launch_generic_fwd<double>(volume, coords, corr, total, hw1, h2, w2, radius, st);
    default: return launch_generic_fwd<__nv_bfloat16>(volume, coords, corr, total, hw1, h2, w2, radius, st);
  }
}

extern "C" int dba_corr_index_backward(const float* coords, const void* corr_grad, void* volume_grad, int n, int h1, int w1, int h2,
                                       int w2, int radius, int dtype, dba_stream_t stream) {
  int rc = check_corr_args(coords, corr_grad, volume_grad, n, h1, w1, h2, w2, radius, dtype);
  if (rc) return rc;
  const long long total = (long long)n * h1 * w1;
  if (total == 0 || h2 == 0 || w2 == 0) return DBA_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int hw1 = h1 * w1;
  switch (dtype) {
    case DBA_F32: return launch_bwd<float>(coords, corr_grad, volume_grad, total, hw1, h2, w2, radius, st);
    case DBA_F16: return launch_bwd<__half>(coords, corr_grad, volume_grad, total, hw1, h2, w2, radius, st);
    case DBA_F64: return launch_bwd<double>(coords, corr_grad, volume_grad, total, hw1, h2, w2, radius, st);
    default: return launch_bwd<__nv_bfloat16>(coords, corr_grad, volume_grad, total, hw1, h2, w2, radius, st);
  }
}

// fused 4-level lookup (f16 or f32, radius 3): out [n,196,h1,w1] = cat over levels of corr_index_forward(volume_l, coords / 2^l).
// tiled_mask bit l: level l is in the 4x8-tile layout of dba_corr_volume_pyramid(..., tiled = 1) (levels 0 and 1 there).
// w1 % 64 == 0 and h1 % 8 == 0 (every level's rows are whole 16-byte chunks): corr_lookup_pyramid_f16_kernel; any other h1, w1 >= 8
// (reference layout only): corr_lookup_pyramid_rows_f16_kernel.  f32 (reference layout): corr_lookup_pyramid_f32_kernel.
extern "C" int dba_corr_lookup_pyramid(const void* v0, const void* v1, const void* v2, const void* v3, const float* coords, void* out,
                                       int n, int h1, int w1, int tiled_mask, int dtype, dba_stream_t stream) {
  DBA_CHECK_ARG(n >= 0 && h1 > 0 && w1 > 0, "bad extents");
  DBA_CHECK_ARG(dtype == DBA_F16 || dtype == DBA_F32, "corr_lookup_pyramid: f16 or f32 volumes only; use corr_index_forward per level otherwise");
  DBA_CHECK_ARG(h1 >= 8 && w1 >= 8, "corr_lookup_pyramid: h1 and w1 must be at least 8 (level 3 must have at least one pixel)");
  const bool chunk_rows = h1 % 8 == 0 && w1 % 64 == 0;
  DBA_CHECK_ARG(tiled_mask == 0 || (tiled_mask == 3 && chunk_rows), "tiled_mask must be 0, or 3 (levels 0 and 1 tiled) with w1 % 64 == 0 and h1 % 8 == 0");
  DBA_CHECK_ARG(dtype == DBA_F16 || tiled_mask == 0, "corr_lookup_pyramid: f32 volumes are in the reference layout (tiled_mask 0)");
  const long long total = (long long)n * h1 * w1;
  if (total == 0) return DBA_OK;
  DBA_CHECK_ARG(v0 && v1 && v2 && v3 && coords && out, "null pointer");
  DBA_CHECK_ARG(((((uintptr_t)v0) | ((uintptr_t)v1) | ((uintptr_t)v2) | ((uintptr_t)v3)) & 15) == 0, "volumes must be 16-byte aligned");
  DBA_CHECK_ARG((total + 127) / 128 < 0x7fffffffLL, "too many pixels for one launch");
  const unsigned blocks = (unsigned)((total + 127) / 128);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DBA_F32) {
    corr_lookup_pyramid_f32_kernel<<<blocks, 128, 0, st>>>((const float*)v0, (const float*)v1, (const float*)v2, (const float*)v3, coords, (float*)out, total, h1 * w1, h1, w1);
    DBA_CHECK_LAUNCH("corr_lookup_pyramid(f32)");
    return DBA_OK;
  }
  if (!chunk_rows)
    return corr_lookup_pyramid_rows_launch((const __half*)v0, (const __half*)v1, (const __half*)v2, (const __half*)v3, coords, (__half*)out, total, h1, w1, st);
  if (tiled_mask == 3)
    corr_lookup_pyramid_f16_kernel<3, true><<<blocks, 128, 0, st>>>((const __half*)v0, (const __half*)v1, (const __half*)v2, (const __half*)v3, coords, (__half*)out, total, h1 * w1, h1, w1);
  else
    corr_lookup_pyramid_f16_kernel<0, false><<<blocks, 128, 0, st>>>((const __half*)v0, (const __half*)v1, (const __half*)v2, (const __half*)v3, coords, (__half*)out, total, h1 * w1, h1, w1);
  DBA_CHECK_LAUNCH("corr_lookup_pyramid");
  return DBA_OK;
}

