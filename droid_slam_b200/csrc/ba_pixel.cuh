// Device code shared by the dense BA build (ba.cu) and the motion-only filler BA (filler.cu): the per-pixel residual and
// Jacobian of K1 (reference src/droid_kernels.cu:185-433) and the left-multiplicative pose retraction (K8, :942-955).
#pragma once
#include "common.cuh"

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

// ---- retraction: poses <- Exp(dx) * poses, no renormalisation (reference :942-955 with its expSE3, :120-160) ----
__device__ __forceinline__ void exp_so3(const float* phi, float* q) {
  const float theta_sq = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
  const float theta_p4 = theta_sq * theta_sq;
  const float theta = sqrtf(theta_sq);
  float imag, real;
  if ((double)theta_sq < 1e-8) {        // double literal comparison in the reference (:128)
    imag = (float)(0.5 - (1.0 / 48.0) * (double)theta_sq + (1.0 / 3840.0) * (double)theta_p4);
    real = (float)(1.0 - (1.0 / 8.0) * (double)theta_sq + (1.0 / 384.0) * (double)theta_p4);
  } else {
    imag = (float)((double)sinf((float)(0.5 * (double)theta)) / (double)theta);
    real = cosf((float)(0.5 * (double)theta));
  }
  q[0] = imag * phi[0]; q[1] = imag * phi[1]; q[2] = imag * phi[2]; q[3] = real;
}

__device__ __forceinline__ void cross_inplace(const float* a, float* b) {
  const float x0 = a[1] * b[2] - a[2] * b[1], x1 = a[2] * b[0] - a[0] * b[2], x2 = a[0] * b[1] - a[1] * b[0];
  b[0] = x0; b[1] = x1; b[2] = x2;
}

__device__ __forceinline__ void exp_se3(const float* xi, float* t, float* q) {
  exp_so3(xi + 3, q);
  float tau[3] = {xi[0], xi[1], xi[2]};
  const float phi[3] = {xi[3], xi[4], xi[5]};
  const float theta_sq = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
  const float theta = sqrtf(theta_sq);
  t[0] = tau[0]; t[1] = tau[1]; t[2] = tau[2];
  if ((double)theta > 1e-4) {
    const float a = (1 - cosf(theta)) / theta_sq;
    cross_inplace(phi, tau);
    t[0] += a * tau[0]; t[1] += a * tau[1]; t[2] += a * tau[2];
    const float b = (theta - sinf(theta)) / (theta * theta_sq);
    cross_inplace(phi, tau);
    t[0] += b * tau[0]; t[1] += b * tau[1]; t[2] += b * tau[2];
  }
}

// ps [7] (tx,ty,tz,qx,qy,qz,qw) <- Exp(xi) * ps
__device__ __forceinline__ void retract_pose(const float* xi, float* ps) {
  float t[3], q[4], dt[3] = {0, 0, 0}, dq[4] = {0, 0, 0, 1}, t1[3], q1[4];
  t[0] = ps[0]; t[1] = ps[1]; t[2] = ps[2];
  q[0] = ps[3]; q[1] = ps[4]; q[2] = ps[5]; q[3] = ps[6];
  exp_se3(xi, dt, dq);
  q1[0] = dq[3] * q[0] + dq[0] * q[3] + dq[1] * q[2] - dq[2] * q[1];
  q1[1] = dq[3] * q[1] + dq[1] * q[3] + dq[2] * q[0] - dq[0] * q[2];
  q1[2] = dq[3] * q[2] + dq[2] * q[3] + dq[0] * q[1] - dq[1] * q[0];
  q1[3] = dq[3] * q[3] - dq[0] * q[0] - dq[1] * q[1] - dq[2] * q[2];
  act_so3(dq, t, t1);
  ps[0] = t1[0] + dt[0]; ps[1] = t1[1] + dt[1]; ps[2] = t1[2] + dt[2];
  ps[3] = q1[0]; ps[4] = q1[1]; ps[5] = q1[2]; ps[6] = q1[3];
}

}  // namespace dba
