// Non-keyframe pose filling (PoseTrajectoryFiller, reference droid_slam/trajectory_filler.py) for sm_90a.
//
//   * fill_interpolate_kernel: the linear pose interpolation of `__fill` (:51-65), one thread per frame: the bracket search
//     t0 = #{k < N : ts[k] <= t} - 1 over an unsorted ts, then G = Exp(Log(P[t1] P[t0]^-1) / dt * (t - ts[t0])) P[t0] in fp32 with
//     lietorch's SE3 arithmetic (lie_math.cuh; thirdparty/lietorch/lietorch/include/so3.h, se3.h, restated in oracle/shims/lietorch).
//   * pose_only_ba_kernel: every Gauss-Newton iteration of one motion-only BA call of the filler's graph in a single launch.  Every edge
//     goes from a fixed frame (ii < t0) to one optimised frame (t0 <= jj < t1), so the pose system is block diagonal: a CTA owns one
//     optimised frame, sums the per-pixel Hjj / vj of K1 (the device code of ba_build_kernel, ba_pixel.cuh) over that frame's edges in
//     ascending edge order, damps the 6x6 block, solves it in fp64 and retracts the pose with the reference kernels' SE3 arithmetic
//     (droid_se3.cuh).  Fixed reduction order and no atomics: the result of a frame does not depend on which other frames share the launch.
#include "common.cuh"
#include "ba_pixel.cuh"
#include "droid_se3.cuh"
#include "lie_math.cuh"
#include <math.h>

namespace dba {

using dba_lie::Elem;
using dba_lie::SE3g;
using dba_lie::g_exp;
using dba_lie::g_inv;
using dba_lie::g_log;
using dba_lie::g_mul;

// t0 / t1 / interpolated pose of frame f (reference trajectory_filler.py:57-65).  t0 = -1 (a frame stamped before every keyframe) is
// kept as the reference computes it; Python's negative indexing then reads keyframe N-1 for P[t0] and ts[t0].
__global__ void __launch_bounds__(128) fill_interpolate_kernel(const float* __restrict__ poses, const float* __restrict__ ts, int N,
                                                               const float* __restrict__ tt, int F, int64_t* __restrict__ t0_out,
                                                               int64_t* __restrict__ t1_out, float* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const float t = tt[f];
  int cnt = 0;
  for (int k = 0; k < N; k++) cnt += (ts[k] <= t) ? 1 : 0;
  const int t0 = cnt - 1;
  const int t1 = t0 < N - 1 ? t0 + 1 : t0;
  const int i0 = t0 < 0 ? t0 + N : t0;
  const float dt = __fadd_rn(__fsub_rn(ts[t1], ts[i0]), 1e-3f);
  Elem<SE3g, float> P0, P1;
  P0.load(poses + 7 * (size_t)i0); P1.load(poses + 7 * (size_t)t1);
  float xi[6];
  g_log(g_mul(P1, g_inv(P0)), xi);
  const float s = __fsub_rn(t, ts[i0]);
#pragma unroll
  for (int c = 0; c < 6; c++) xi[c] = __fmul_rn(__fdiv_rn(xi[c], dt), s);
  g_mul(g_exp<SE3g, float>(xi), P0).store(out + 7 * (size_t)f);
  t0_out[f] = t0;
  t1_out[f] = t1;
}

// ---- motion-only BA of the filler graph ----
constexpr int kPoseThreads = 256;
enum { POSE_ST_STRUCTURE = 1, POSE_ST_NOT_SPD = 2 };

// status = 0, then POSE_ST_STRUCTURE when an edge is not (0 <= ii < min(t0, n_disps), t0 <= jj < t1).  Runs before the BA kernel on the
// same stream, which leaves every pose untouched when the bit is set.
__global__ void __launch_bounds__(256) pose_ba_check_kernel(const int64_t* __restrict__ ii, const int64_t* __restrict__ jj, int E, int n_disps,
                                                            int t0, int t1, int* __restrict__ status) {
  __shared__ int s_bad;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const long long i = ii[e], j = jj[e];
    if (i < 0 || i >= t0 || i >= n_disps || j < t0 || j >= t1) s_bad = 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) *status = s_bad ? POSE_ST_STRUCTURE : 0;
}

// Damped 6x6 solve in fp64: (H + diag(ep + lm diag(H))) x = b by LLT; a non-positive pivot gives x = 0 (reference :1216-1219).
__device__ bool solve6_damped(const double* Hl, const double* b, double lm, double ep, float* x) {
  double L[6][6], y[6];
  for (int r = 0; r < 6; r++)
    for (int c = 0; c <= r; c++) {
      double v = Hl[r * (r + 1) / 2 + c];
      if (r == c) v += ep + lm * v;
      for (int k = 0; k < c; k++) v -= L[r][k] * L[c][k];
      if (r == c) {
        if (!(v > 0.0)) { for (int k = 0; k < 6; k++) x[k] = 0.f; return false; }
        L[r][r] = sqrt(v);
      } else {
        L[r][c] = v / L[c][c];
      }
    }
  for (int r = 0; r < 6; r++) { double v = b[r]; for (int k = 0; k < r; k++) v -= L[r][k] * y[k]; y[r] = v / L[r][r]; }
  for (int r = 5; r >= 0; r--) { double v = y[r]; for (int k = r + 1; k < 6; k++) v -= L[k][r] * y[k]; y[r] = v / L[r][r]; }
  bool finite = true;
  for (int k = 0; k < 6; k++) finite = finite && isfinite(y[k]);
  for (int k = 0; k < 6; k++) x[k] = finite ? (float)y[k] : 0.f;
  return finite;
}

// CTA = optimised frame t0 + blockIdx.x.  Per iteration: the frame's edges in ascending edge order (ballot compaction of the edge list,
// 256 edges at a time); per edge, each thread sums its pixels' Hjj / vj in fp32, a warp transpose-reduction and an fp64 sum over the
// warps (fixed order) give the edge's 27 sums, added in fp64 to the frame's block.  Thread 0 damps, solves and retracts.  The frame's
// pose lives in shared memory during the call (fixed poses are read with __ldg: this kernel never writes them).
__global__ void __launch_bounds__(kPoseThreads) pose_only_ba_kernel(
    float* __restrict__ poses, const float* __restrict__ disps, const float* __restrict__ intr, const float* __restrict__ targets,
    const float* __restrict__ weights, const int64_t* __restrict__ ii, const int64_t* __restrict__ jj, int E, int HW, int wd, int t0,
    int iterations, double lm, double ep, int* __restrict__ status, double* __restrict__ sys_out, float* __restrict__ dx_out) {
  if (*reinterpret_cast<volatile int*>(status) & POSE_ST_STRUCTURE) return;
  constexpr int NW = kPoseThreads / 32;
  const int k = blockIdx.x, fj = t0 + k;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ float s_pose[7];
  __shared__ float s_T[7];
  __shared__ int s_edges[kPoseThreads];
  __shared__ int s_wcount[NW];
  __shared__ int s_ix;
  __shared__ float s_part[NW][27];
  __shared__ double s_sum[27];
  if (tid < 7) s_pose[tid] = poses[7 * (size_t)fj + tid];
  const float fx = __ldg(intr), fy = __ldg(intr + 1), cx = __ldg(intr + 2), cy = __ldg(intr + 3);

  for (int it = 0; it < iterations; it++) {
    if (tid < 27) s_sum[tid] = 0.0;
    for (int base = 0; base < E; base += kPoseThreads) {
      const int e = base + tid;
      const bool mine = e < E && jj[e] == fj;
      const unsigned bal = __ballot_sync(0xffffffffu, mine);
      __syncthreads();                                  // the previous chunk's edge list is consumed
      if (lane == 0) s_wcount[warp] = __popc(bal);
      __syncthreads();
      int pos = 0, n = 0;
      for (int w = 0; w < NW; w++) { pos += w < warp ? s_wcount[w] : 0; n += s_wcount[w]; }
      if (mine) s_edges[pos + __popc(bal & ((1u << lane) - 1u))] = e;
      __syncthreads();
      for (int a = 0; a < n; a++) {
        const int ea = s_edges[a];
        if (tid == 0) {
          const int ix = (int)ii[ea];
          float ti[3], qi[4];
#pragma unroll
          for (int c = 0; c < 3; c++) ti[c] = __ldg(poses + 7 * (size_t)ix + c);
#pragma unroll
          for (int c = 0; c < 4; c++) qi[c] = __ldg(poses + 7 * (size_t)ix + 3 + c);
          rel_se3(ti, qi, s_pose, s_pose + 3, s_T, s_T + 3);       // the edge transform of ba_build_kernel (edge_transform)
          s_ix = ix;
        }
        __syncthreads();
        const int ix = s_ix;
        float Hjj[21], vj[6];
#pragma unroll
        for (int c = 0; c < 21; c++) Hjj[c] = 0.f;
#pragma unroll
        for (int c = 0; c < 6; c++) vj[c] = 0.f;
        const float* tg = targets + (size_t)ea * 2 * HW;
        const float* wg = weights + (size_t)ea * 2 * HW;
        for (int p = tid; p < HW; p += kPoseThreads) {
          const int i = p / wd, j = p - i * wd;
          PixelTerms P;
          ba_pixel_terms(s_T, s_T + 3, ((float)j - cx) / fx, ((float)i - cy) / fy, __ldg(disps + (size_t)ix * HW + p), __ldg(wg + p),
                         __ldg(wg + HW + p), __ldg(tg + p), __ldg(tg + HW + p), fx, fy, cx, cy, P);
          ba_pose_accum(P, Hjj, vj);
        }
        float v32[32];
#pragma unroll
        for (int c = 0; c < 21; c++) v32[c] = Hjj[c];
#pragma unroll
        for (int c = 0; c < 6; c++) v32[21 + c] = vj[c];
#pragma unroll
        for (int c = 27; c < 32; c++) v32[c] = 0.f;
        const float tot = transpose_reduce32(v32, lane);
        if (lane < 27) s_part[warp][lane] = tot;
        __syncthreads();
        if (tid < 27) {
          double s = 0.0;
#pragma unroll
          for (int w = 0; w < NW; w++) s += (double)s_part[w][tid];
          s_sum[tid] += s;
        }
        __syncthreads();                                // s_T, s_part free for the next edge
      }
    }
    __syncthreads();
    if (tid == 0) {
      float dx[6];
      const bool ok = solve6_damped(s_sum, s_sum + 21, lm, ep, dx);
      if (!ok) atomicOr(status, POSE_ST_NOT_SPD);
      if (it == iterations - 1) {
        if (sys_out) {
          double* so = sys_out + 42 * (size_t)k;
          for (int r = 0; r < 6; r++)
            for (int c = 0; c < 6; c++) so[r * 6 + c] = s_sum[r >= c ? r * (r + 1) / 2 + c : c * (c + 1) / 2 + r];
          for (int r = 0; r < 6; r++) so[36 + r] = s_sum[21 + r];
        }
        if (dx_out)
          for (int c = 0; c < 6; c++) dx_out[6 * (size_t)k + c] = dx[c];
      }
      retract_pose(dx, s_pose);
    }
    __syncthreads();
  }
  if (tid < 7) poses[7 * (size_t)fj + tid] = s_pose[tid];
}

}  // namespace dba
using namespace dba;

extern "C" int dba_fill_interpolate(const float* poses, const float* tstamps, int n_keyframes, const float* t, int n, int64_t* t0_out,
                                    int64_t* t1_out, float* poses_out, dba_stream_t stream) {
  DBA_CHECK_ARG(n_keyframes >= 0 && n >= 0, "negative extent");
  if (n == 0) return DBA_OK;
  DBA_CHECK_ARG(n_keyframes >= 1, "no keyframe to interpolate from");
  DBA_CHECK_ARG(poses && tstamps && t && t0_out && t1_out && poses_out, "null pointer");
  fill_interpolate_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(poses, tstamps, n_keyframes, t, n, t0_out, t1_out, poses_out);
  DBA_CHECK_LAUNCH("fill_interpolate");
  return DBA_OK;
}

extern "C" int dba_pose_only_ba(float* poses, const float* disps, const float* intrinsics, const float* targets, const float* weights,
                                const int64_t* ii, const int64_t* jj, int n_frames, int n_disps, int n_edges, int ht, int wd, int t0, int t1,
                                int iterations, float lm, float ep, int* status, double* sys_out, float* dx_out, dba_stream_t stream) {
  DBA_CHECK_ARG(n_frames >= 0 && n_disps >= 0 && n_edges >= 0 && ht > 0 && wd > 0 && iterations >= 0, "negative extent");
  DBA_CHECK_ARG(t0 >= 0 && t1 >= t0 && t1 <= n_frames, "bad window [t0,t1)");
  DBA_CHECK_ARG(status != nullptr, "null status");
  DBA_CHECK_ARG(poses && disps && intrinsics, "null state pointer");
  DBA_CHECK_ARG(n_edges == 0 || (targets && weights && ii && jj), "null edge pointer");
  cudaStream_t st = (cudaStream_t)stream;
  pose_ba_check_kernel<<<1, 256, 0, st>>>(ii, jj, n_edges, n_disps, t0, t1, status);
  DBA_CHECK_LAUNCH("pose_only_ba (check)");
  if (t1 == t0 || iterations == 0) return DBA_OK;
  pose_only_ba_kernel<<<t1 - t0, kPoseThreads, 0, st>>>(poses, disps, intrinsics, targets, weights, ii, jj, n_edges, ht * wd, wd, t0, iterations,
                                                        (double)lm, (double)ep, status, sys_out, dx_out);
  DBA_CHECK_LAUNCH("pose_only_ba");
  return DBA_OK;
}
