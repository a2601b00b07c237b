// DroidAsync's frontend -> backend fragment hand-over (reference droid_slam/droid_async.py:54-119, droid_slam/align.py) for sm_90a.
//
//   * handover_align_kernel: every CTA ORs `disps_sens1 != 0` over its slice of the frontend's disps_sens into its own flag (no
//     initialisation, no atomics); CTA 0 also computes align_pose_fragements in fp64 (81 relative translations, one per thread, summed
//     in a fixed order by thread 0; the 3 log-mean-exp refinements with one thread per pose).
//   * handover_apply_kernel: each CTA folds the flags into align_scale, then re-anchors its frame's pose (chunk 0, one thread) and
//     divides its chunk of the frame's inverse depths by s.
// The SE3 arithmetic is lietorch's (lie_math.cuh; thirdparty/lietorch/lietorch/include/so3.h, se3.h, restated in oracle/shims/lietorch)
// in fp64, on poses converted from fp32 on load.
#include "common.cuh"
#include "lie_math.cuh"
#include <math.h>

namespace dba {

namespace {

using dba_lie::Elem;
using dba_lie::SE3g;
using dba_lie::g_exp;
using dba_lie::g_inv;
using dba_lie::g_log;
using dba_lie::g_mul;

constexpr int kAlignThreads = 128;
constexpr int kApplyThreads = 256;
constexpr int kApplyChunk = 4 * kApplyThreads;                // inverse depths per CTA of the apply kernel
constexpr int kSensPerCta = 16384;                             // disps_sens floats per CTA of the align kernel (at least)
constexpr int kAlignPoses = 9;                                 // poses [t0-10, t0-1)
constexpr int kMaxSlices = (DBA_HANDOVER_WORKSPACE_BYTES - 8 * sizeof(double)) / sizeof(int);

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

  __shared__ Elem<SE3g, double> P0[kAlignPoses], P1[kAlignPoses];
  __shared__ double s_dot[kAlignPoses * kAlignPoses][2];
  __shared__ double s_e[kAlignPoses][6];
  __shared__ Elem<SE3g, double> s_dG;
  __shared__ double s_s;
  if (p_front == nullptr) {                                                // t0 == 0: identity, s = 1
    if (tid < 8) ws[tid] = tid == 0 || tid == 7 ? 1.0 : 0.0;
    return;
  }
  if (tid < kAlignPoses) { P0[tid].load(p_front + 7 * tid); P1[tid].load(p_back + 7 * tid); }
  __syncthreads();
  if (tid < kAlignPoses * kAlignPoses) {                                  // dP[i][j] = P[j]^-1 P[i]: its translation
    const int i = tid / kAlignPoses, j = tid % kAlignPoses;
    const Elem<SE3g, double> d1 = g_mul(g_inv(P0[j]), P0[i]), d2 = g_mul(g_inv(P1[j]), P1[i]);
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
  if (tid == 0) s_dG = g_mul(P1[0], g_inv(P0[0]));
  __syncthreads();
  for (int it = 0; it < 3; it++) {
    if (tid < kAlignPoses) g_log(g_mul(P1[tid], g_inv(g_mul(s_dG, P0[tid]))), s_e[tid]);
    __syncthreads();
    if (tid == 0) {
      double m[6];
      for (int c = 0; c < 6; c++) {
        double a = 0.0;
        for (int k = 0; k < kAlignPoses; k++) a += s_e[k][c];
        m[c] = a / kAlignPoses;
      }
      s_dG = g_mul(g_exp<SE3g, double>(m), s_dG);
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
    Elem<SE3g, double> dG, P;
    for (int k = 0; k < 3; k++) dG.t[k] = ws[1 + k];
    for (int k = 0; k < 4; k++) dG.q[k] = ws[4 + k];
    P.load(ps);
    const Elem<SE3g, double> g = g_mul(dG, P);
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
