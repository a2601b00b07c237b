// The SE3 arithmetic of the reference kernels (reference src/droid_kernels.cu:67-160), which ba_cuda, the geometry ops and the BA
// retraction compute in: quaternions are not renormalised, and the branches and constants keep the reference's double literals.  This
// is a different convention from lietorch's (lie_math.cuh); oracle/se3.py restates this one.
#pragma once
#include "common.cuh"

namespace dba {

// (reference src/droid_kernels.cu:67-116; double-literal `2.0 *` there promotes to fp64 and rounds once, which
//  is the same value as the fp32 product because multiplying by 2 is exact)
__device__ __forceinline__ void act_so3(const float* q, const float* X, float* Y) {
  float uv0 = 2.0f * (q[1] * X[2] - q[2] * X[1]);
  float uv1 = 2.0f * (q[2] * X[0] - q[0] * X[2]);
  float uv2 = 2.0f * (q[0] * X[1] - q[1] * X[0]);
  Y[0] = X[0] + q[3] * uv0 + (q[1] * uv2 - q[2] * uv1);
  Y[1] = X[1] + q[3] * uv1 + (q[2] * uv0 - q[0] * uv2);
  Y[2] = X[2] + q[3] * uv2 + (q[0] * uv1 - q[1] * uv0);
}

__device__ __forceinline__ void act_se3(const float* t, const float* q, const float* X, float* Y) {
  act_so3(q, X, Y);
  Y[3] = X[3];
  Y[0] += X[3] * t[0];
  Y[1] += X[3] * t[1];
  Y[2] += X[3] * t[2];
}

__device__ __forceinline__ void rel_se3(const float* ti, const float* qi, const float* tj, const float* qj,
                                        float* tij, float* qij) {
  qij[0] = -qj[3] * qi[0] + qj[0] * qi[3] - qj[1] * qi[2] + qj[2] * qi[1];
  qij[1] = -qj[3] * qi[1] + qj[1] * qi[3] - qj[2] * qi[0] + qj[0] * qi[2];
  qij[2] = -qj[3] * qi[2] + qj[2] * qi[3] - qj[0] * qi[1] + qj[1] * qi[0];
  qij[3] = qj[3] * qi[3] + qj[0] * qi[0] + qj[1] * qi[1] + qj[2] * qi[2];
  act_so3(qij, ti, tij);
  tij[0] = tj[0] - tij[0];
  tij[1] = tj[1] - tij[1];
  tij[2] = tj[2] - tij[2];
}

// relative transform of an edge; stereo edges (ix==jx) get the fixed baseline when `stereo_quirk`
__device__ __forceinline__ void edge_transform(const float* __restrict__ poses, int ix, int jx, bool stereo_quirk,
                                               float* tij, float* qij) {
  if (stereo_quirk && ix == jx) {
    tij[0] = -0.1f; tij[1] = 0.f; tij[2] = 0.f;
    qij[0] = 0.f; qij[1] = 0.f; qij[2] = 0.f; qij[3] = 1.f;
    return;
  }
  float ti[3], tj[3], qi[4], qj[4];
#pragma unroll
  for (int k = 0; k < 3; k++) { ti[k] = __ldg(poses + 7 * (size_t)ix + k); tj[k] = __ldg(poses + 7 * (size_t)jx + k); }
#pragma unroll
  for (int k = 0; k < 4; k++) { qi[k] = __ldg(poses + 7 * (size_t)ix + 3 + k); qj[k] = __ldg(poses + 7 * (size_t)jx + 3 + k); }
  rel_se3(ti, qi, tj, qj, tij, qij);
}

// Y = adjSE3(t,q,X)  (reference src/droid_kernels.cu:88-103)
__device__ __forceinline__ void adj_se3(const float* t, const float* q, const float* X, float* Y) {
  float qinv[4] = {-q[0], -q[1], -q[2], q[3]};
  act_so3(qinv, X, Y);
  act_so3(qinv, X + 3, Y + 3);
  float u[3], v[3];
  u[0] = t[2] * X[1] - t[1] * X[2];
  u[1] = t[0] * X[2] - t[2] * X[0];
  u[2] = t[1] * X[0] - t[0] * X[1];
  act_so3(qinv, u, v);
  Y[3] += v[0]; Y[4] += v[1]; Y[5] += v[2];
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
