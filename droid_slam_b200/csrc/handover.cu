// DroidAsync's frontend -> backend fragment hand-over (reference droid_slam/droid_async.py:54-119, droid_slam/align.py) for sm_90a.
//
//   * handover_align_kernel: every CTA ORs `disps_sens1 != 0` over its slice of the frontend's disps_sens into its own flag (no
//     initialisation, no atomics); CTA 0 also computes align_pose_fragements in fp64 (81 relative translations, one per thread, summed
//     in a fixed order by thread 0; the 3 log-mean-exp refinements with one thread per pose).
//   * handover_apply_kernel: each CTA folds the flags into align_scale, then re-anchors its frame's pose (chunk 0, one thread) and
//     divides its chunk of the frame's inverse depths by s.
// The SE3 arithmetic is lietorch's (thirdparty/lietorch/lietorch/include/so3.h, se3.h; restated in oracle/shims/lietorch) in fp64.
// The fp32 lie_* helpers of filler.cu reproduce lietorch's fp32 roundings; these are a separate fp64 set on purpose.
#include "common.cuh"
#include <math.h>

namespace dba {

namespace {

constexpr int kAlignThreads = 128;
constexpr int kApplyThreads = 256;
constexpr int kApplyChunk = 4 * kApplyThreads;                // inverse depths per CTA of the apply kernel
constexpr int kSensPerCta = 16384;                             // disps_sens floats per CTA of the align kernel (at least)
constexpr int kAlignPoses = 9;                                 // poses [t0-10, t0-1)
constexpr int kMaxSlices = (DBA_HANDOVER_WORKSPACE_BYTES - 8 * sizeof(double)) / sizeof(int);
constexpr double kEps = 1e-6;                                  // lietorch include/common.h: EPS

struct G64 { double t[3], q[4]; };

__device__ void cross3(const double* a, const double* b, double* r) {
  r[0] = a[1] * b[2] - a[2] * b[1]; r[1] = a[2] * b[0] - a[0] * b[2]; r[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ void qnorm(double* q) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
__device__ void rot(const double* q, const double* p, double* r) {        // so3.h:55-60
  double uv[3], c[3];
  cross3(q, p, uv);
  uv[0] *= 2.0; uv[1] *= 2.0; uv[2] *= 2.0;
  cross3(q, uv, c);
  for (int k = 0; k < 3; k++) r[k] = p[k] + q[3] * uv[k] + c[k];
}
__device__ G64 load(const float* p) {                                      // quaternion normalised on load (so3.h:35-37)
  G64 g;
  for (int k = 0; k < 3; k++) g.t[k] = p[k];
  for (int k = 0; k < 4; k++) g.q[k] = p[3 + k];
  qnorm(g.q);
  return g;
}
__device__ G64 inv(const G64& g) {                                         // se3.h:36-38
  G64 r;
  r.q[0] = -g.q[0]; r.q[1] = -g.q[1]; r.q[2] = -g.q[2]; r.q[3] = g.q[3];
  rot(r.q, g.t, r.t);
  r.t[0] = -r.t[0]; r.t[1] = -r.t[1]; r.t[2] = -r.t[2];
  return r;
}
__device__ G64 mul(const G64& a, const G64& b) {                           // se3.h:45-47
  G64 r;
  rot(a.q, b.t, r.t);
  for (int k = 0; k < 3; k++) r.t[k] += a.t[k];
  r.q[0] = a.q[3] * b.q[0] + a.q[0] * b.q[3] + a.q[1] * b.q[2] - a.q[2] * b.q[1];
  r.q[1] = a.q[3] * b.q[1] - a.q[0] * b.q[2] + a.q[1] * b.q[3] + a.q[2] * b.q[0];
  r.q[2] = a.q[3] * b.q[2] + a.q[0] * b.q[1] - a.q[1] * b.q[0] + a.q[2] * b.q[3];
  r.q[3] = a.q[3] * b.q[3] - a.q[0] * b.q[0] - a.q[1] * b.q[1] - a.q[2] * b.q[2];
  qnorm(r.q);
  return r;
}
// v + c1 phi x v + c2 phi x (phi x v)
__device__ void jac_apply(const double* phi, double c1, double c2, const double* v, double* r) {
  double a[3], b[3];
  cross3(phi, v, a);
  cross3(phi, a, b);
  for (int k = 0; k < 3; k++) r[k] = v[k] + c1 * a[k] + c2 * b[k];
}
__device__ void se3_log(const G64& g, double* xi) {                            // se3.h:124-132, so3.h:111-147, 188-206
  const double* v = g.q;
  const double w = g.q[3];
  const double n2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  const double n = sqrt(n2);
  double f;
  if (n2 < kEps * kEps) f = 2.0 / w - (2.0 / 3.0) * n2 / (w * w * w);
  else if (fabs(w) < kEps) f = w > 0.0 ? M_PI / n : -M_PI / n;
  else f = 2.0 * atan(n / w) / n;
  const double phi[3] = {f * v[0], f * v[1], f * v[2]};
  const double th = sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
  const double c2 = th < kEps ? 1.0 / 12.0 : (1.0 - th * cos(0.5 * th) / (2.0 * sin(0.5 * th))) / (th * th);
  jac_apply(phi, -0.5, c2, g.t, xi);
  xi[3] = phi[0]; xi[4] = phi[1]; xi[5] = phi[2];
}
__device__ G64 se3_exp(const double* xi) {                                     // se3.h:134-142, so3.h:149-186
  const double* phi = xi + 3;
  const double th2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
  const double th = sqrt(th2);
  const bool small = th < kEps;
  G64 g;
  const double imag = small ? 0.5 - th2 / 48.0 + th2 * th2 / 3840.0 : sin(0.5 * th) / th;
  g.q[3] = small ? 1.0 - th2 / 8.0 + th2 * th2 / 384.0 : cos(0.5 * th);
  g.q[0] = imag * phi[0]; g.q[1] = imag * phi[1]; g.q[2] = imag * phi[2];
  qnorm(g.q);
  const double c1 = small ? 0.5 - th2 / 24.0 : (1.0 - cos(th)) / th2;
  const double c2 = small ? 1.0 / 6.0 - th2 / 120.0 : (th - sin(th)) / (th2 * th);
  jac_apply(phi, c1, c2, xi, g.t);
  return g;
}

// workspace: [0] s, [1..7] dG (fp64), then one int flag per align-kernel CTA
__global__ void __launch_bounds__(kAlignThreads) handover_align_kernel(const float* __restrict__ p_front, const float* __restrict__ p_back,
                                                                       const float* __restrict__ sens, long long n_sens, int per_cta,
                                                                       bool vec4, double* __restrict__ ws) {
  const int tid = threadIdx.x;
  const long long lo = (long long)blockIdx.x * per_cta;
  const long long hi = min(n_sens, lo + per_cta);
  bool nz = false;
  if (vec4) {
    const float4* s4 = reinterpret_cast<const float4*>(sens);
    for (long long k = lo / 4 + tid; k < hi / 4; k += kAlignThreads) {
      const float4 v = __ldg(s4 + k);
      nz |= v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f;       // NaN != 0: torch.any counts it
    }
  } else {
    for (long long k = lo + tid; k < hi; k += kAlignThreads) nz |= __ldg(sens + k) != 0.f;
  }
  nz = __syncthreads_or(nz);
  int* flags = reinterpret_cast<int*>(ws + 8);
  if (tid == 0) flags[blockIdx.x] = nz ? 1 : 0;
  if (blockIdx.x != 0) return;

  __shared__ G64 P0[kAlignPoses], P1[kAlignPoses];
  __shared__ double s_dot[kAlignPoses * kAlignPoses][2];
  __shared__ double s_e[kAlignPoses][6];
  __shared__ G64 s_dG;
  __shared__ double s_s;
  if (p_front == nullptr) {                                                // t0 == 0: identity, s = 1
    if (tid < 8) ws[tid] = tid == 0 || tid == 7 ? 1.0 : 0.0;
    return;
  }
  if (tid < kAlignPoses) { P0[tid] = load(p_front + 7 * tid); P1[tid] = load(p_back + 7 * tid); }
  __syncthreads();
  if (tid < kAlignPoses * kAlignPoses) {                                  // dP[i][j] = P[j]^-1 P[i]: its translation
    const int i = tid / kAlignPoses, j = tid % kAlignPoses;
    const G64 d1 = mul(inv(P0[j]), P0[i]), d2 = mul(inv(P1[j]), P1[i]);
    s_dot[tid][0] = d1.t[0] * d2.t[0] + d1.t[1] * d2.t[1] + d1.t[2] * d2.t[2];
    s_dot[tid][1] = d1.t[0] * d1.t[0] + d1.t[1] * d1.t[1] + d1.t[2] * d1.t[2];
  }
  __syncthreads();
  if (tid == 0) {
    double num = 0.0, den = 0.0;
    for (int k = 0; k < kAlignPoses * kAlignPoses; k++) { num += s_dot[k][0]; den += s_dot[k][1]; }
    s_s = num / den;
  }
  __syncthreads();
  if (tid < kAlignPoses) for (int k = 0; k < 3; k++) P0[tid].t[k] *= s_s;
  __syncthreads();
  if (tid == 0) s_dG = mul(P1[0], inv(P0[0]));
  __syncthreads();
  for (int it = 0; it < 3; it++) {
    if (tid < kAlignPoses) se3_log(mul(P1[tid], inv(mul(s_dG, P0[tid]))), s_e[tid]);
    __syncthreads();
    if (tid == 0) {
      double m[6];
      for (int c = 0; c < 6; c++) {
        double a = 0.0;
        for (int k = 0; k < kAlignPoses; k++) a += s_e[k][c];
        m[c] = a / kAlignPoses;
      }
      s_dG = mul(se3_exp(m), s_dG);
    }
    __syncthreads();
  }
  if (tid == 0) {
    ws[0] = s_s;
    for (int k = 0; k < 3; k++) ws[1 + k] = s_dG.t[k];
    for (int k = 0; k < 4; k++) ws[4 + k] = s_dG.q[k];
  }
}

__global__ void __launch_bounds__(kApplyThreads) handover_apply_kernel(float* __restrict__ poses2, float* __restrict__ disps2, int t0, int n_frames,
                                                                       int hw, int n_flags, bool stereo, const double* __restrict__ ws,
                                                                       double* __restrict__ diag) {
  const int tid = threadIdx.x;
  const int* flags = reinterpret_cast<const int*>(ws + 8);
  bool any = false;
  for (int k = tid; k < n_flags; k += kApplyThreads) any |= flags[k] != 0;
  any = __syncthreads_or(any);
  const bool align_scale = !stereo && !any;
  const double s = align_scale ? ws[0] : 1.0;
  const float s_f = (float)s;
  if (blockIdx.x == 0 && blockIdx.y == 0 && tid < 9 && diag) diag[tid] = tid == 0 ? s : tid == 8 ? (align_scale ? 1.0 : 0.0) : ws[tid];
  if ((int)blockIdx.x >= n_frames) return;                                 // the one CTA of an empty [t0,t1)
  const size_t f = (size_t)t0 + blockIdx.x;
  if (blockIdx.y == 0 && tid == 0) {
    float* p = poses2 + 7 * f;
    float ps[7];
    for (int k = 0; k < 7; k++) ps[k] = p[k];
    for (int k = 0; k < 3; k++) ps[k] = __fmul_rn(ps[k], s_f);             // the reference's `pose1_copy[..., :3] *= s` in fp32
    G64 dG;
    for (int k = 0; k < 3; k++) dG.t[k] = ws[1 + k];
    for (int k = 0; k < 4; k++) dG.q[k] = ws[4 + k];
    const G64 g = mul(dG, load(ps));
    for (int k = 0; k < 3; k++) p[k] = (float)g.t[k];
    for (int k = 0; k < 4; k++) p[3 + k] = (float)g.q[k];
  }
  float* d = disps2 + f * hw;
  const int lo = blockIdx.y * kApplyChunk, hi = min(hw, lo + kApplyChunk);
  for (int k = lo + tid; k < hi; k += kApplyThreads) d[k] = __fdiv_rn(d[k], s_f);
}

}  // namespace
}  // namespace dba
using namespace dba;

extern "C" int dba_fragment_handover(const float* poses1_align, float* poses2, float* disps2, const float* disps_sens1, long long n_sens, int t0,
                                     int t1, int hw, int stereo, void* workspace, double* diagnostics, dba_stream_t stream) {
  DBA_CHECK_ARG(t0 == 0 || t0 >= 10, "t0 must be 0 or at least 10 (the frames [t0-10, t0-1) are aligned)");
  DBA_CHECK_ARG(n_sens >= 0 && hw > 0 && t1 >= 0, "negative extent");
  DBA_CHECK_ARG(poses2 && disps2 && workspace, "null pointer");
  DBA_CHECK_ARG(n_sens == 0 || disps_sens1, "null disps_sens1");
  DBA_CHECK_ARG(t0 == 0 || poses1_align, "null poses1_align (t0 > 0)");
  DBA_CHECK_ARG(((uintptr_t)workspace & 7) == 0, "workspace must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long slices = (n_sens + kSensPerCta - 1) / kSensPerCta;
  const int n_cta = (int)max(1LL, min((long long)kMaxSlices, slices));
  long long per = (n_sens + n_cta - 1) / n_cta;
  per = (per + 3) / 4 * 4;
  DBA_CHECK_ARG(per <= INT32_MAX, "disps_sens1 too large");
  const bool vec4 = ((uintptr_t)disps_sens1 & 15) == 0 && n_sens % 4 == 0;
  handover_align_kernel<<<n_cta, kAlignThreads, 0, st>>>(t0 > 0 ? poses1_align : nullptr, poses2 + 7 * (size_t)(t0 > 0 ? t0 - 10 : 0),
                                                         disps_sens1, n_sens, (int)per, vec4, (double*)workspace);
  DBA_CHECK_LAUNCH("fragment_handover (align)");
  const int n_frames = max(0, t1 - t0);
  dim3 grid(max(1, n_frames), (hw + kApplyChunk - 1) / kApplyChunk);
  handover_apply_kernel<<<grid, kApplyThreads, 0, st>>>(poses2, disps2, t0, n_frames, hw, n_cta, stereo != 0, (const double*)workspace,
                                                        diagnostics);
  DBA_CHECK_LAUNCH("fragment_handover (apply)");
  return DBA_OK;
}
