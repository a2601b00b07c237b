// Fused 4-level radius-3 lookup (dba_corr_lookup_pyramid, reference layout) for volumes whose level rows are not whole 16-byte chunks:
// every h1, w1 >= 8 other than w1 % 64 == 0 with h1 % 8 == 0, which corr_index.cu serves.  Kept in its own translation unit: the
// non-finite slow path calls corr_pixel_generic as a subroutine, and a second caller in corr_index.cu would change the register
// allocation (and SASS) of the kernels there.
#include "corr_pixel.cuh"

namespace dba {

// chunk (y1, cx) of a row-major plane of any width w2 and any 2-byte alignment: taps (y1, 8cx .. 8cx+7), those at x >= w2 zero.  Built
// from the (one or two) 16-byte aligned vectors that hold the taps inside the row, shifted into place with align_row_f16.  A vector that
// reaches past `end` (the end of the level tensor) is read element by element instead, so no load leaves the tensor; bytes of a vector
// outside the row are loaded but never used.  Called for 0 <= 8cx < w2 only.
__device__ __forceinline__ uint4 plane_chunk_rows(const __half* plane, const __half* end, int y1, int cx, int w2) {
  const __half* a = plane + (size_t)y1 * w2 + cx * 8;
  const int nv = min(8, w2 - cx * 8);                                   // taps inside the row
  const uintptr_t ua = reinterpret_cast<uintptr_t>(a);
  const int o = (int)(ua & 15) >> 1;                                    // first tap's element offset in its vector
  const __half* v0 = reinterpret_cast<const __half*>(ua & ~(uintptr_t)15);
  const bool need1 = o + nv > 8;
  uint4 A, B = make_uint4(0, 0, 0, 0);
  if (v0 + 8 <= end) {
    A = ldg_nc_v4_l1(v0);
  } else {                                                             // the tensor ends inside this vector: taps o .. o + nv - 1 only
    uint32_t w[4] = {0, 0, 0, 0};
    const unsigned short* e16 = reinterpret_cast<const unsigned short*>(v0);
#pragma unroll
    for (int k = 0; k < 8; k++)
      if (k >= o && k < o + nv) w[k >> 1] |= (uint32_t)__ldg(e16 + k) << (16 * (k & 1));
    A = make_uint4(w[0], w[1], w[2], w[3]);
  }
  if (need1) {
    const __half* v1 = v0 + 8;
    if (v1 + 8 <= end) {
      B = ldg_nc_v4_l1(v1);
    } else {
      uint32_t w[4] = {0, 0, 0, 0};
      const unsigned short* e16 = reinterpret_cast<const unsigned short*>(v1);
#pragma unroll
      for (int k = 0; k < 8; k++)
        if (k < o + nv - 8) w[k >> 1] |= (uint32_t)__ldg(e16 + k) << (16 * (k & 1));
      B = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
  uint32_t t[4], dummy;
  align_row_f16(A, B, o, t, dummy);
#pragma unroll
  for (int k = 0; k < 4; k++) {                                        // taps 2k, 2k + 1 at or beyond w2 -> 0
    if (2 * k >= nv) t[k] = 0;
    else if (2 * k + 1 >= nv) t[k] &= 0xffffu;
  }
  return make_uint4(t[0], t[1], t[2], t[3]);
}

// the fused lookup of corr_lookup_pyramid_f16_kernel for every h1, w1 >= 8 (reference layout): level planes of any width and alignment,
// read through plane_chunk_rows.  Same per-pixel arithmetic (corr_pixel_f16_r3_from), so every output bit is the same function of the
// window; only the way a 16-byte tap chunk is assembled differs.
__global__ void __launch_bounds__(128) corr_lookup_pyramid_rows_f16_kernel(const __half* __restrict__ v0, const __half* __restrict__ v1,
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
  const __half* vl[4] = {v0, v1, v2, v3};
#pragma unroll
  for (int l = 3; l >= 0; l--) {                                       // coarse levels first, as in corr_lookup_pyramid_f16_kernel
    const int h2 = h1 >> l, w2 = w1 >> l;
    const size_t plane_elems = (size_t)h2 * w2;
    const __half* plane = vl[l] + (size_t)p * plane_elems;
    const __half* end = vl[l] + (size_t)total * plane_elems;
    auto fetch = [&](int y1, int cx) { return plane_chunk_rows(plane, end, y1, cx, w2); };
    const float s = 1.0f / (float)(1 << l);
    corr_pixel_f16_r3_from<false, __half>(fetch, plane, o + (size_t)(49 * l) * hw1, (size_t)hw1, x0 * s, y0 * s, h2, w2);
  }
}

int corr_lookup_pyramid_rows_launch(const __half* v0, const __half* v1, const __half* v2, const __half* v3, const float* coords, __half* out,
                                    long long total, int h1, int w1, cudaStream_t st) {
  corr_lookup_pyramid_rows_f16_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(v0, v1, v2, v3, coords, out, total, h1 * w1, h1, w1);
  DBA_CHECK_LAUNCH("corr_lookup_pyramid(rows)");
  return DBA_OK;
}

}  // namespace dba
