// Device code shared by the dense BA build (ba.cu) and the motion-only filler BA (filler.cu): the per-pixel residual and
// Jacobian of K1 (reference src/droid_kernels.cu:185-433) and the reductions of its sums.
#pragma once
#include "droid_se3.cuh"

namespace dba {

// Residual, weights and Jacobians of one pixel of edge i -> j under the edge transform (t, q), single camera (fx, fy, cx, cy).
// Reference quirks kept: the weights are `.001 * weight` (an fp64 product rounded to fp32, :314-315); d = 0 and w = 0 where the
// transformed depth is below MIN_DEPTH (a double literal, :35).  Ju / Jv: pose Jacobian w.r.t. frame j; Jzu / Jzv: inverse depth.
struct PixelTerms {
  float wu, wv, ru, rv, Jzu, Jzv;
  float Ju[6], Jv[6];
};

__device__ __forceinline__ void ba_pixel_terms(const float* t, const float* q, float xi0, float xi1, float disp, float w_u, float w_v,
                                               float tgt_u, float tgt_v, float fx, float fy, float cx, float cy, PixelTerms& o) {
  float Xi[4] = {xi0, xi1, 1.f, disp}, Xj[4];
  act_se3(t, q, Xi, Xj);
  const float x = Xj[0], y = Xj[1], h = Xj[3];
  const bool close = (double)Xj[2] < 0.25;   // MIN_DEPTH is a double literal in the reference
  const float d = close ? 0.f : 1.0f / Xj[2];
  const float d2 = d * d;
  o.wu = close ? 0.f : (float)(.001 * (double)w_u);
  o.wv = close ? 0.f : (float)(.001 * (double)w_v);
  o.ru = tgt_u - (fx * d * x + cx);
  o.rv = tgt_v - (fy * d * y + cy);
  o.Ju[0] = fx * (h * d); o.Ju[1] = fx * 0; o.Ju[2] = fx * (-x * h * d2);
  o.Ju[3] = fx * (-x * y * d2); o.Ju[4] = fx * (1 + x * x * d2); o.Ju[5] = fx * (-y * d);
  o.Jv[0] = fy * 0; o.Jv[1] = fy * (h * d); o.Jv[2] = fy * (-y * h * d2);
  o.Jv[3] = fy * (-1 - y * y * d2); o.Jv[4] = fy * (x * y * d2); o.Jv[5] = fy * (x * d);
  o.Jzu = fx * (t[0] * d - t[2] * (x * d2));
  o.Jzv = fy * (t[1] * d - t[2] * (y * d2));
}

// Hjj (lower triangle, 21 entries, row-major a >= c) and vj of one pixel, added to the running fp32 sums
__device__ __forceinline__ void ba_pose_accum(const PixelTerms& o, float (&Hjj)[21], float (&vj)[6]) {
  const float wru = o.wu * o.ru, wrv = o.wv * o.rv;
  int l = 0;
#pragma unroll
  for (int a = 0; a < 6; a++) {
    vj[a] += wru * o.Ju[a] + wrv * o.Jv[a];
    const float wa_u = o.wu * o.Ju[a], wa_v = o.wv * o.Jv[a];
#pragma unroll
    for (int c = 0; c <= a; c++) { Hjj[l] += wa_u * o.Ju[c] + wa_v * o.Jv[c]; l++; }
  }
}

// total of value i ends up in lane i  (v[0] on return), 31 shuffles
__device__ __forceinline__ float transpose_reduce32(float (&v)[32], int lane) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; i++) {
      const float send = up ? v[i] : v[i + off];
      const float keep = up ? v[i + off] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  return v[0];
}

}  // namespace dba
