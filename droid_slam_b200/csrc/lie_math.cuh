// lie_math.cuh -- the SO3 / SE3 arithmetic of lietorch's convention (quaternion normalised on load, small-angle branches at EPS = 1e-6;
// details in lie.cu's header), for every kernel that computes in it: the group ops and their gradients (lie.cu), the dense BA layer
// (ba_layer.cu), the trajectory filler's interpolation (filler.cu) and DroidAsync's hand-over (handover.cu).  Templated on the scalar
// type.  The reference kernels' convention (no renormalisation, their own branch thresholds) is droid_se3.cuh's.
#pragma once
#include "common.cuh"

namespace dba_lie {

struct SO3g { static constexpr int N = 4, K = 3; };
struct SE3g { static constexpr int N = 7, K = 6; };

// ---- 3-vector / quaternion helpers -------------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ void cross(const T* a, const T* b, T* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
template <typename T> __device__ __forceinline__ T dot3(const T* a, const T* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// R(q) p = p + w uv + qv x uv, uv = 2 qv x p (unit q)
template <typename T> __device__ __forceinline__ void rot(const T* q, const T* p, T* out) {
  T uv[3], c[3];
  cross(q, p, uv);
  uv[0] *= T(2); uv[1] *= T(2); uv[2] *= T(2);
  cross(q, uv, c);
  for (int k = 0; k < 3; k++) out[k] = p[k] + q[3] * uv[k] + c[k];
}
// R(q)^T p = R(conj q) p
template <typename T> __device__ __forceinline__ void rot_t(const T* q, const T* p, T* out) {
  const T qc[4] = {-q[0], -q[1], -q[2], q[3]};
  rot(qc, p, out);
}
// Hamilton product (x,y,z,w layout)
template <typename T> __device__ __forceinline__ void qmul(const T* a, const T* b, T* c) {
  c[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  c[1] = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  c[2] = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
  c[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}
template <typename T> __device__ __forceinline__ void qnormalize(T* q) {
  const T s = T(1) / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] *= s; q[1] *= s; q[2] *= s; q[3] *= s;
}

// ---- SO3 maps ------------------------------------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ void so3_exp(const T* phi, T* q) {
  const T eps = T(1e-6);
  const T th2 = dot3(phi, phi), th = sqrt(th2);
  T imag, real;
  if (th < eps) {
    imag = T(0.5) - th2 / T(48) + th2 * th2 / T(3840);
    real = T(1) - th2 / T(8) + th2 * th2 / T(384);
  } else {
    imag = sin(T(0.5) * th) / th;
    real = cos(T(0.5) * th);
  }
  q[0] = imag * phi[0]; q[1] = imag * phi[1]; q[2] = imag * phi[2]; q[3] = real;
  qnormalize(q);
}
// atan-based log of a unit quaternion; keeps the n^2 < EPS^2 and |w| < EPS branches
template <typename T> __device__ __forceinline__ void so3_log(const T* q, T* phi) {
  const T eps = T(1e-6);
  const T n2 = dot3(q, q), w = q[3];
  T f;
  if (n2 < eps * eps) {
    const T iw = T(1) / w;
    f = iw * (T(2) - (T(2) / T(3)) * n2 * iw * iw);
  }
  else {
    const T n = sqrt(n2);
    if (fabs(w) < eps) f = (w > T(0) ? T(3.141592653589793) : T(-3.141592653589793)) / n;
    else f = T(2) * atan(n / w) / n;
  }
  phi[0] = f * q[0]; phi[1] = f * q[1]; phi[2] = f * q[2];
}

// M = I + c1 hat(phi) + c2 hat(phi)^2 (row-major 3x3), hat(phi)^2 = phi phi^T - |phi|^2 I
template <typename T> __device__ __forceinline__ void i_hat_hat2(const T* phi, T c0, T c1, T c2, T* M) {
  const T th2 = dot3(phi, phi);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) M[3 * r + c] = (r == c ? c0 - c2 * th2 : T(0)) + c2 * phi[r] * phi[c];
  M[1] -= c1 * phi[2]; M[2] += c1 * phi[1]; M[3] += c1 * phi[2];
  M[5] -= c1 * phi[0]; M[6] -= c1 * phi[1]; M[7] += c1 * phi[0];
}
template <typename T> __device__ __forceinline__ void so3_jl(const T* phi, T* J) {
  const T eps = T(1e-6);
  const T th2 = dot3(phi, phi), th = sqrt(th2);
  const bool small = th < eps;
  const T c1 = small ? T(0.5) - th2 / T(24) : (T(1) - cos(th)) / (th * th);
  const T c2 = small ? T(1) / T(6) - th2 / T(120) : (th - sin(th)) / (th * th * th);
  i_hat_hat2(phi, T(1), c1, c2, J);
}
template <typename T> __device__ __forceinline__ void so3_jl_inv(const T* phi, T* J) {
  const T eps = T(1e-6);
  const T th2 = dot3(phi, phi), th = sqrt(th2);
  // (1 - t cos(t/2) / (2 sin(t/2))) / t^2 over one denominator: one division (a double division's slow path is a call that spills)
  const T s2 = T(2) * sin(T(0.5) * th);
  const T c2 = th < eps ? T(1) / T(12) : (s2 - th * cos(T(0.5) * th)) / (s2 * th * th);
  i_hat_hat2(phi, T(1), T(-0.5), c2, J);
}
template <typename T> __device__ __forceinline__ void mat3_mul(const T* A, const T* B, T* C) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) C[3 * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
}
template <typename T> __device__ __forceinline__ void hat(const T* v, T* M) {
  M[0] = T(0); M[1] = -v[2]; M[2] = v[1];
  M[3] = v[2]; M[4] = T(0); M[5] = -v[0];
  M[6] = -v[1]; M[7] = v[0]; M[8] = T(0);
}
// the upper-right block Q(tau, phi) of SE3's left Jacobian
template <typename T> __device__ void se3_q(const T* tau, const T* phi, T* Q) {
  const T eps = T(1e-6);
  const T th2 = dot3(phi, phi), th = sqrt(th2), th4 = th2 * th2;
  const bool small = th < eps;
  const T c1 = small ? T(1) / T(6) - th2 / T(120) : (th - sin(th)) / (th2 * th);
  const T c2 = small ? T(1) / T(24) - th2 / T(720) : (th2 + T(2) * cos(th) - T(2)) / (T(2) * th4);
  const T c3 = small ? T(1) / T(120) - th2 / T(2520) : (T(2) * th - T(3) * sin(th) + th * cos(th)) / (T(2) * th4 * th);
  T P[9], U[9], A[9], B[9], C[9];
  hat(phi, P); hat(tau, U);
  mat3_mul(P, U, A);                                             // PU
  mat3_mul(U, P, B);                                             // UP
  for (int k = 0; k < 9; k++) Q[k] = T(0.5) * U[k] + c1 * (A[k] + B[k]);
  mat3_mul(P, A, C);                                             // PPU
  for (int k = 0; k < 9; k++) Q[k] += c2 * C[k];
  mat3_mul(B, P, C);                                             // UPP
  for (int k = 0; k < 9; k++) Q[k] += c2 * C[k];
  mat3_mul(A, P, B);                                             // PUP
  for (int k = 0; k < 9; k++) Q[k] += (c1 - T(3) * c2) * B[k];
  mat3_mul(B, P, A);                                             // PUPP
  mat3_mul(P, B, C);                                             // PPUP
  for (int k = 0; k < 9; k++) Q[k] += c3 * (A[k] + C[k]);
}
template <typename T> __device__ __forceinline__ void mv3(const T* M, const T* v, T* o) {   // o = M v
  for (int r = 0; r < 3; r++) o[r] = M[3 * r] * v[0] + M[3 * r + 1] * v[1] + M[3 * r + 2] * v[2];
}
template <typename T> __device__ __forceinline__ void mtv3(const T* M, const T* v, T* o) {  // o = M^T v
  for (int c = 0; c < 3; c++) o[c] = M[c] * v[0] + M[3 + c] * v[1] + M[6 + c] * v[2];
}

// ---- a group element, quaternion normalised on load ------------------------------------------------------------------------------------
template <class G, typename T> struct Elem {
  T t[3], q[4];
  // from data of any scalar type S (fp64 elements from fp32 poses), converted before the normalisation
  template <typename S> __device__ __forceinline__ void load(const S* d) {
    if constexpr (G::N == 7) { t[0] = T(d[0]); t[1] = T(d[1]); t[2] = T(d[2]); d += 3; }
    else { t[0] = t[1] = t[2] = T(0); }
    q[0] = T(d[0]); q[1] = T(d[1]); q[2] = T(d[2]); q[3] = T(d[3]);
    qnormalize(q);
  }
  __device__ __forceinline__ void store(T* d) const {
    if constexpr (G::N == 7) { d[0] = t[0]; d[1] = t[1]; d[2] = t[2]; d += 3; }
    d[0] = q[0]; d[1] = q[1]; d[2] = q[2]; d[3] = q[3];
  }
};

template <class G, typename T> __device__ __forceinline__ Elem<G, T> g_inv(const Elem<G, T>& X) {
  Elem<G, T> Y;
  Y.q[0] = -X.q[0]; Y.q[1] = -X.q[1]; Y.q[2] = -X.q[2]; Y.q[3] = X.q[3];
  T r[3];
  rot(Y.q, X.t, r);
  Y.t[0] = -r[0]; Y.t[1] = -r[1]; Y.t[2] = -r[2];
  return Y;
}
// X Y = (R_X t_Y + t_X, q_X q_Y normalised)
template <class G, typename T> __device__ __forceinline__ Elem<G, T> g_mul(const Elem<G, T>& X, const Elem<G, T>& Y) {
  Elem<G, T> Z;
  T r[3];
  rot(X.q, Y.t, r);
  for (int k = 0; k < 3; k++) Z.t[k] = X.t[k] + r[k];
  qmul(X.q, Y.q, Z.q);
  qnormalize(Z.q);
  return Z;
}
// Adj(X) a: SE3 (R a_tau + t x R a_phi, R a_phi); SO3 R a
template <class G, typename T> __device__ __forceinline__ void g_adj(const Elem<G, T>& X, const T* a, T* b) {
  if constexpr (G::K == 6) {
    T ra[3], rp[3], c[3];
    rot(X.q, a, ra); rot(X.q, a + 3, rp); cross(X.t, rp, c);
    for (int k = 0; k < 3; k++) { b[k] = ra[k] + c[k]; b[3 + k] = rp[k]; }
  } else {
    rot(X.q, a, b);
  }
}
// Adj(X)^T a: SE3 (R^T a_tau, R^T (a_phi - t x a_tau)); SO3 R^T a
template <class G, typename T> __device__ __forceinline__ void g_adjT(const Elem<G, T>& X, const T* a, T* b) {
  if constexpr (G::K == 6) {
    T c[3], v[3];
    rot_t(X.q, a, b);
    cross(X.t, a, c);
    for (int k = 0; k < 3; k++) v[k] = a[3 + k] - c[k];
    rot_t(X.q, v, b + 3);
  } else {
    rot_t(X.q, a, b);
  }
}
// g ad(b) for a row g: SE3 (g1 x b_phi, g1 x b_tau + g2 x b_phi); SO3 g x b
template <class G, typename T> __device__ __forceinline__ void row_ad(const T* g, const T* b, T* o) {
  if constexpr (G::K == 6) {
    T c1[3], c2[3];
    cross(g, b + 3, o);
    cross(g, b, c1); cross(g + 3, b + 3, c2);
    for (int k = 0; k < 3; k++) o[3 + k] = c1[k] + c2[k];
  } else {
    cross(g, b, o);
  }
}
// log of X into a[K]
template <class G, typename T> __device__ __forceinline__ void g_log(const Elem<G, T>& X, T* a) {
  if constexpr (G::K == 6) {
    T Ji[9];
    so3_log(X.q, a + 3);
    so3_jl_inv(a + 3, Ji);
    mv3(Ji, X.t, a);
  } else {
    so3_log(X.q, a);
  }
}
template <class G, typename T> __device__ __forceinline__ Elem<G, T> g_exp(const T* a) {
  Elem<G, T> X;
  if constexpr (G::K == 6) {
    T J[9];
    so3_exp(a + 3, X.q);
    so3_jl(a + 3, J);
    mv3(J, a, X.t);
  } else {
    so3_exp(a, X.q);
    X.t[0] = X.t[1] = X.t[2] = T(0);
  }
  return X;
}
// the SO3 part of the projector applied to a row: 0.5 (w g - g x v - g_w v) for the quaternion's row gradient g (4)
template <typename T> __device__ __forceinline__ void so3_row_proj(const T* q, const T* g, T* o) {
  T c[3];
  cross(g, q, c);
  for (int k = 0; k < 3; k++) o[k] = T(0.5) * (q[3] * g[k] - c[k] - g[3] * q[k]);
}
// 4 A g for A the projector's 4x3 block: (2 (w g - v x g), -2 v.g)
template <typename T> __device__ __forceinline__ void so3_pinv_col(const T* q, const T* g, T* o) {
  T c[3];
  cross(q, g, c);
  for (int k = 0; k < 3; k++) o[k] = T(2) * (q[3] * g[k] - c[k]);
  o[3] = T(-2) * dot3(q, g);
}

}  // namespace dba_lie
