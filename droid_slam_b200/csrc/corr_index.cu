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
#include "common.cuh"
#include <type_traits>

namespace dba {

// ------------------------------------------------------------------------------------------------------
// dtype traits: reference rounding behaviour of `acc += s * T(w)`
// ------------------------------------------------------------------------------------------------------
template <typename T> struct CorrMath;
template <> struct CorrMath<float> {
  typedef float W;
  static __device__ __forceinline__ W weight(float w) { return w; }
  static __device__ __forceinline__ float zero() { return 0.f; }
  static __device__ __forceinline__ float mac(float s, W w, float acc) { return fmaf(s, w, acc); }
};
template <> struct CorrMath<double> {
  typedef double W;
  static __device__ __forceinline__ W weight(float w) { return (double)w; }
  static __device__ __forceinline__ double zero() { return 0.0; }
  static __device__ __forceinline__ double mac(double s, W w, double acc) { return fma(s, w, acc); }
};
template <> struct CorrMath<__half> {
  typedef __half W;
  static __device__ __forceinline__ W weight(float w) { return __float2half_rn(w); }
  static __device__ __forceinline__ __half zero() { return __float2half_rn(0.f); }
  static __device__ __forceinline__ __half mac(__half s, W w, __half acc) { return __hadd_rn(acc, __hmul_rn(s, w)); }
};
// bf16 is not dispatched by the reference; defined here as fp32 FMA chain on bf16 inputs, rounded once.
template <> struct CorrMath<__nv_bfloat16> {
  typedef float W;
  static __device__ __forceinline__ W weight(float w) { return w; }
};

// ------------------------------------------------------------------------------------------------------
// generic kernels: any radius, any extents, exact skip semantics.  One thread per pixel.
// ------------------------------------------------------------------------------------------------------
// element (y1, x1) of a plane: row-major, or the 4x8-tile layout [h2/4][w2/8][4][8] of corr_volume_pyramid's tiled mode
template <bool TILED>
__device__ __forceinline__ size_t plane_index(int y1, int x1, int w2) {
  return TILED ? ((size_t)(y1 >> 2) * (w2 >> 3) + (x1 >> 3)) * 32 + (y1 & 3) * 8 + (x1 & 7) : (size_t)y1 * w2 + x1;
}

template <typename T, bool TILED = false>
__device__ __forceinline__ void corr_pixel_generic(const T* __restrict__ plane, T* __restrict__ out_px, size_t out_stride,
                                                   float x0, float y0, int h2, int w2, int r) {
  typedef CorrMath<T> M;
  const float fxf = floorf(x0), fyf = floorf(y0);
  const float dx = x0 - fxf, dy = y0 - fyf;
  const int fx = floor_to_int_sat(fxf), fy = floor_to_int_sat(fyf);
  const typename M::W w00 = M::weight((1.0f - dx) * (1.0f - dy));
  const typename M::W w01 = M::weight((1.0f - dx) * dy);
  const typename M::W w10 = M::weight(dx * (1.0f - dy));
  const typename M::W w11 = M::weight(dx * dy);
  const int rd = 2 * r + 1;
  for (int i = 0; i < rd; i++) {
    for (int j = 0; j < rd; j++) {
      const int x1 = fx - r + i, y1 = fy - r + j;
      T acc = M::zero();
      const bool xa = (unsigned)x1 < (unsigned)w2, xb = (unsigned)(x1 + 1) < (unsigned)w2;
      const bool ya = (unsigned)y1 < (unsigned)h2, yb = (unsigned)(y1 + 1) < (unsigned)h2;
      if (xa && ya) acc = M::mac(plane[plane_index<TILED>(y1, x1, w2)], w00, acc);
      if (xa && yb) acc = M::mac(plane[plane_index<TILED>(y1 + 1, x1, w2)], w01, acc);
      if (xb && ya) acc = M::mac(plane[plane_index<TILED>(y1, x1 + 1, w2)], w10, acc);
      if (xb && yb) acc = M::mac(plane[plane_index<TILED>(y1 + 1, x1 + 1, w2)], w11, acc);
      out_px[(size_t)(i * rd + j) * out_stride] = acc;
    }
  }
}

template <>
__device__ __forceinline__ void corr_pixel_generic<__nv_bfloat16, false>(const __nv_bfloat16* __restrict__ plane,
                                                                  __nv_bfloat16* __restrict__ out_px, size_t out_stride,
                                                                  float x0, float y0, int h2, int w2, int r) {
  const float fxf = floorf(x0), fyf = floorf(y0);
  const float dx = x0 - fxf, dy = y0 - fyf;
  const int fx = floor_to_int_sat(fxf), fy = floor_to_int_sat(fyf);
  const float w00 = (1.0f - dx) * (1.0f - dy), w01 = (1.0f - dx) * dy, w10 = dx * (1.0f - dy), w11 = dx * dy;
  const int rd = 2 * r + 1;
  for (int i = 0; i < rd; i++) {
    for (int j = 0; j < rd; j++) {
      const int x1 = fx - r + i, y1 = fy - r + j;
      float acc = 0.f;
      const bool xa = (unsigned)x1 < (unsigned)w2, xb = (unsigned)(x1 + 1) < (unsigned)w2;
      const bool ya = (unsigned)y1 < (unsigned)h2, yb = (unsigned)(y1 + 1) < (unsigned)h2;
      if (xa && ya) acc = fmaf(__bfloat162float(plane[(size_t)y1 * w2 + x1]), w00, acc);
      if (xa && yb) acc = fmaf(__bfloat162float(plane[(size_t)(y1 + 1) * w2 + x1]), w01, acc);
      if (xb && ya) acc = fmaf(__bfloat162float(plane[(size_t)y1 * w2 + x1 + 1]), w10, acc);
      if (xb && yb) acc = fmaf(__bfloat162float(plane[(size_t)(y1 + 1) * w2 + x1 + 1]), w11, acc);
      out_px[(size_t)(i * rd + j) * out_stride] = __float2bfloat16_rn(acc);
    }
  }
}

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
__device__ __forceinline__ uint32_t h2_as_u32(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ __half2 u32_as_h2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }

// window row -> 4 aligned half2 words (taps 0..7) from two 16-byte chunks and the tap offset o in [0,7]
__device__ __forceinline__ void align_row_f16(const uint4& A, const uint4& B, int o, uint32_t* t /*[4]*/, uint32_t& t4) {
  uint32_t w0 = A.x, w1 = A.y, w2 = A.z, w3 = A.w, w4 = B.x, w5 = B.y, w6 = B.z, w7 = B.w;
  if (o & 4) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; w5 = w7; }
  if (o & 2) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; }
  if (o & 1) {
    w0 = __funnelshift_r(w0, w1, 16); w1 = __funnelshift_r(w1, w2, 16);
    w2 = __funnelshift_r(w2, w3, 16); w3 = __funnelshift_r(w3, w4, 16);
  }
  t[0] = w0; t[1] = w1; t[2] = w2; t[3] = w3; t4 = 0;
}

// one pixel, one level, f16, radius 3: out_px[(i*7+j) * out_stride] for the 49 taps.  TILED: the plane is stored as 4x8-element
// tiles ([h2/4][w2/8][4][8], one 64-byte DRAM atom per tile, written by corr_volume_pyramid's tiled mode): the 8x8 window then
// touches 5.2 atoms on average instead of 8-10 (a 16-byte window row at arbitrary alignment costs a whole atom in the row-major
// plane); the arithmetic and therefore every output bit is the same.
// T16 = __half (reference arithmetic: product and sum rounded in f16, two taps per half2 instruction) or __nv_bfloat16 (extension:
// fp32 FMA chain on the bf16 inputs, rounded once -- the same function as the generic bf16 path, with the vector loads of the f16 one)
//
// The window comes from fetch(y1, cx): the 16-byte chunk holding taps (y1, 8cx .. 8cx+7) of the plane, called only for chunks
// inside the plane (the others are zero).  Chunk B (taps a0+8 ..) is not fetched when the window starts on a chunk boundary (o == 0):
// all 8 taps are then in chunk A.  `plane` (global memory, layout TILED) is read only by the slow path for non-finite coordinates.
template <bool TILED, typename T16, typename Fetch>
__device__ __forceinline__ void corr_pixel_f16_r3_from(Fetch fetch, const T16* __restrict__ plane, T16* __restrict__ out_px,
                                                       size_t out_stride, float x0, float y0, int h2, int w2) {
  constexpr bool kHalf = sizeof(T16) == 2 && std::is_same<T16, __half>::value;
  if (!(isfinite(x0) && isfinite(y0))) {   // exact reference semantics for NaN/inf coordinates (slow path)
    if constexpr (TILED && !kHalf) return;                                       // (tiled planes exist for f16 only)
    else corr_pixel_generic<T16, TILED>(plane, out_px, out_stride, x0, y0, h2, w2, 3);
    return;
  }
  const float fxf = floorf(x0), fyf = floorf(y0);
  const float dx = x0 - fxf, dy = y0 - fyf;
  const int x1s = floor_to_int_sat(fxf) - 3, y1s = floor_to_int_sat(fyf) - 3;
  const int a0 = x1s & ~7;
  const int o = x1s - a0;
  const bool okA = (unsigned)a0 < (unsigned)w2, okB = o != 0 && (unsigned)(a0 + 8) < (unsigned)w2;
  const int cx = a0 >> 3;

  uint4 A[8], B[8];
#pragma unroll
  for (int b = 0; b < 8; b++) {
    const int y1 = y1s + b;
    const bool rowok = (unsigned)y1 < (unsigned)h2;
    A[b] = make_uint4(0, 0, 0, 0); B[b] = make_uint4(0, 0, 0, 0);
    if (rowok && okA) A[b] = fetch(y1, cx);
    if (rowok && okB) B[b] = fetch(y1, cx + 1);
  }
  const float f00 = (1.0f - dx) * (1.0f - dy), f01 = (1.0f - dx) * dy, f10 = dx * (1.0f - dy), f11 = dx * dy;
  const __half2 w00 = __half2half2(__float2half_rn(f00));
  const __half2 w01 = __half2half2(__float2half_rn(f01));
  const __half2 w10 = __half2half2(__float2half_rn(f10));
  const __half2 w11 = __half2half2(__float2half_rn(f11));
  const __half2 zero2 = __half2half2(__float2half_rn(0.f));

  uint32_t pa[4], ps[4], ca[4], cs[4], dummy;   // aligned / shifted-by-one-tap words of previous and current row
  align_row_f16(A[0], B[0], o, pa, dummy);
  ps[0] = __funnelshift_r(pa[0], pa[1], 16); ps[1] = __funnelshift_r(pa[1], pa[2], 16);
  ps[2] = __funnelshift_r(pa[2], pa[3], 16); ps[3] = pa[3] >> 16;
#pragma unroll
  for (int j = 0; j < 7; j++) {
    align_row_f16(A[j + 1], B[j + 1], o, ca, dummy);
    cs[0] = __funnelshift_r(ca[0], ca[1], 16); cs[1] = __funnelshift_r(ca[1], ca[2], 16);
    cs[2] = __funnelshift_r(ca[2], ca[3], 16); cs[3] = ca[3] >> 16;
#pragma unroll
    for (int k = 0; k < 4; k++) {   // lanes (i=2k, i=2k+1)
      if constexpr (kHalf) {
        __half2 t = __hadd2_rn(zero2, __hmul2_rn(u32_as_h2(pa[k]), w00));   // tap (i  , j  )
        t = __hadd2_rn(t, __hmul2_rn(u32_as_h2(ca[k]), w01));               // tap (i  , j+1)
        t = __hadd2_rn(t, __hmul2_rn(u32_as_h2(ps[k]), w10));               // tap (i+1, j  )
        t = __hadd2_rn(t, __hmul2_rn(u32_as_h2(cs[k]), w11));               // tap (i+1, j+1)
        out_px[(size_t)((2 * k) * 7 + j) * out_stride] = __low2half(t);
        if (k < 3) out_px[(size_t)((2 * k + 1) * 7 + j) * out_stride] = __high2half(t);
      } else {                         // bf16 -> fp32 is a 16-bit shift; same tap order as the generic path
        float lo = fmaf(__uint_as_float(pa[k] << 16), f00, 0.f), hi = fmaf(__uint_as_float(pa[k] & 0xffff0000u), f00, 0.f);
        lo = fmaf(__uint_as_float(ca[k] << 16), f01, lo); hi = fmaf(__uint_as_float(ca[k] & 0xffff0000u), f01, hi);
        lo = fmaf(__uint_as_float(ps[k] << 16), f10, lo); hi = fmaf(__uint_as_float(ps[k] & 0xffff0000u), f10, hi);
        lo = fmaf(__uint_as_float(cs[k] << 16), f11, lo); hi = fmaf(__uint_as_float(cs[k] & 0xffff0000u), f11, hi);
        out_px[(size_t)((2 * k) * 7 + j) * out_stride] = __float2bfloat16_rn(lo);
        if (k < 3) out_px[(size_t)((2 * k + 1) * 7 + j) * out_stride] = __float2bfloat16_rn(hi);
      }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) { pa[k] = ca[k]; ps[k] = cs[k]; }
  }
}

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

__global__ void __launch_bounds__(128) corr_index_fwd_f32_r3_kernel(const float* __restrict__ vol, const float* __restrict__ coords,
                                                                    float* __restrict__ out, long long total, int hw1, int h2, int w2) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  const float x0 = coords[((size_t)n * 2 + 0) * hw1 + pin];
  const float y0 = coords[((size_t)n * 2 + 1) * hw1 + pin];
  const float* plane = vol + (size_t)p * h2 * w2;
  float* out_px = out + (size_t)n * 49 * hw1 + pin;
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

// fused 4-level lookup (f16, radius 3): out [n,196,h1,w1] = cat over levels of corr_index_forward(volume_l, coords / 2^l).
// tiled_mask bit l: level l is in the 4x8-tile layout of dba_corr_volume_pyramid(..., tiled = 1) (levels 0 and 1 there).
extern "C" int dba_corr_lookup_pyramid(const void* v0, const void* v1, const void* v2, const void* v3, const float* coords, void* out,
                                       int n, int h1, int w1, int tiled_mask, int dtype, dba_stream_t stream) {
  DBA_CHECK_ARG(n >= 0 && h1 > 0 && w1 > 0, "bad extents");
  DBA_CHECK_ARG(dtype == DBA_F16, "corr_lookup_pyramid: f16 volumes (the live system's autocast dtype) only; use corr_index_forward per level otherwise");
  DBA_CHECK_ARG(h1 % 8 == 0 && w1 % 64 == 0, "corr_lookup_pyramid: needs w1 % 64 == 0 (every level's rows are whole 16-byte chunks) and h1 % 8 == 0");
  DBA_CHECK_ARG(tiled_mask == 0 || (tiled_mask == 3 && h1 % 8 == 0), "tiled_mask must be 0 or 3 (levels 0 and 1 tiled)");
  const long long total = (long long)n * h1 * w1;
  if (total == 0) return DBA_OK;
  DBA_CHECK_ARG(v0 && v1 && v2 && v3 && coords && out, "null pointer");
  DBA_CHECK_ARG(((((uintptr_t)v0) | ((uintptr_t)v1) | ((uintptr_t)v2) | ((uintptr_t)v3)) & 15) == 0, "volumes must be 16-byte aligned");
  DBA_CHECK_ARG((total + 127) / 128 < 0x7fffffffLL, "too many pixels for one launch");
  const unsigned blocks = (unsigned)((total + 127) / 128);
  cudaStream_t st = (cudaStream_t)stream;
  if (tiled_mask == 3)
    corr_lookup_pyramid_f16_kernel<3, true><<<blocks, 128, 0, st>>>((const __half*)v0, (const __half*)v1, (const __half*)v2, (const __half*)v3, coords, (__half*)out, total, h1 * w1, h1, w1);
  else
    corr_lookup_pyramid_f16_kernel<0, false><<<blocks, 128, 0, st>>>((const __half*)v0, (const __half*)v1, (const __half*)v2, (const __half*)v3, coords, (__half*)out, total, h1 * w1, h1, w1);
  DBA_CHECK_LAUNCH("corr_lookup_pyramid");
  return DBA_OK;
}

