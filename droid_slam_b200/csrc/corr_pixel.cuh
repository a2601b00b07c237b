// Per-pixel arithmetic of corr_index_forward shared by corr_index.cu and corr_lookup_rows.cu (device functions only).
#pragma once
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
// one pixel, any radius, any extents, exact skip semantics
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

// ------------------------------------------------------------------------------------------------------
// radius 3, f16 / bf16: the 8x8 tap window from 16-byte chunks
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

}  // namespace dba
