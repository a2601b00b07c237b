// Streaming geometry ops for sm_90a: projmap, frame_distance, depth_filter, iproj.
// Replace reference src/droid_kernels.cu:436-859 (kernels) and :1447-1550 (drivers).
// All four are HBM-streaming (4-16 B per pixel); one CTA computes the edge transform once into shared memory,
// pixels are thread-strided so every global access is warp-coalesced, outputs are written once (no memset, and
// no atomics in depth_filter: a thread owns its pixel and loops over the six neighbours).
#include "droid_se3.cuh"

namespace dba {

struct Intr { float fx, fy, cx, cy; };
__device__ __forceinline__ Intr load_intr(const float* __restrict__ k) {
  Intr r; r.fx = __ldg(k); r.fy = __ldg(k + 1); r.cx = __ldg(k + 2); r.cy = __ldg(k + 3); return r;
}

__global__ void __launch_bounds__(256) projmap_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                                                      const float* __restrict__ intr, const int64_t* __restrict__ ii,
                                                      const int64_t* __restrict__ jj, float* __restrict__ coords,
                                                      float* __restrict__ valid, int ht, int wd) {
  const int e = blockIdx.x;   // edges / frames on grid.x (2^31-1 blocks), pixel chunks on grid.y
  __shared__ float T[7];
  const int ix = (int)ii[e], jx = (int)jj[e];
  if (threadIdx.x == 0) edge_transform(poses, ix, jx, /*stereo_quirk=*/false, T, T + 3);   // no stereo branch (:475-490)
  __syncthreads();
  const Intr K = load_intr(intr);
  const int hw = ht * wd;
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= hw) return;
  const int i = k / wd, j = k - i * wd;
  const float u = (float)j, v = (float)i;
  float Xi[4] = {(u - K.cx) / K.fx, (v - K.cy) / K.fy, 1.f, __ldg(disps + (size_t)ix * hw + k)}, Xj[4];
  act_se3(T, T + 3, Xi, Xj);
  float cu = u, cv = v;
  if (Xj[2] > 0.01f) {   // literal is a double in the reference; (float)z > 0.01 (double) differs from 0.01f only for z == 0.01f exactly
    cu = K.fx * (Xj[0] / Xj[2]) + K.cx;
    cv = K.fy * (Xj[1] / Xj[2]) + K.cy;
  }
  float* c = coords + ((size_t)e * hw + k) * 3;
  c[0] = cu; c[1] = cv; c[2] = 0.f;
  valid[(size_t)e * hw + k] = ((double)Xj[2] > 0.25) ? 1.f : 0.f;
}

__global__ void __launch_bounds__(256) frame_distance_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                                                             const float* __restrict__ intr, const int64_t* __restrict__ ii,
                                                             const int64_t* __restrict__ jj, float* __restrict__ dist,
                                                             int ht, int wd, float beta) {
  const int e = blockIdx.x;
  __shared__ float T[7];
  __shared__ float red[3][8];
  const int ix = (int)ii[e], jx = (int)jj[e];
  if (threadIdx.x == 0) edge_transform(poses, ix, jx, false, T, T + 3);
  __syncthreads();
  const Intr K = load_intr(intr);
  const int hw = ht * wd;
  float accum = 0.f, vsum = 0.f, total = 0.f;
  const float* di = disps + (size_t)ix * hw;
  for (int k = threadIdx.x; k < hw; k += blockDim.x) {
    const int i = k / wd, j = k - i * wd;
    const float u = (float)j, v = (float)i;
    float Xi[4] = {(u - K.cx) / K.fx, (v - K.cy) / K.fy, 1.f, __ldg(di + k)}, Xj[4];
    act_se3(T, T + 3, Xi, Xj);
    float du = K.fx * (Xj[0] / Xj[2]) + K.cx - u;
    float dv = K.fy * (Xj[1] / Xj[2]) + K.cy - v;
    float d = sqrtf(du * du + dv * dv);
    total += beta;
    if ((double)Xj[2] > 0.25) { accum += beta * d; vsum += beta; }
    // translation only (:627-645)
    Xj[0] = Xi[0] + Xi[3] * T[0];
    Xj[1] = Xi[1] + Xi[3] * T[1];
    Xj[2] = Xi[2] + Xi[3] * T[2];
    du = K.fx * (Xj[0] / Xj[2]) + K.cx - u;
    dv = K.fy * (Xj[1] / Xj[2]) + K.cy - v;
    d = sqrtf(du * du + dv * dv);
    total += (1 - beta);
    if ((double)Xj[2] > 0.25) { accum += (1 - beta) * d; vsum += (1 - beta); }
  }
  accum = warp_sum(accum); vsum = warp_sum(vsum); total = warp_sum(total);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = accum; red[1][w] = vsum; red[2][w] = total; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, vv = 0.f, t = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); k++) { a += red[0][k]; vv += red[1][k]; t += red[2][k]; }
    dist[e] = ((double)vv / ((double)t + 1e-8) < 0.75) ? 1000.0f : a / vv;   // (:664) `total[0] + 1e-8` is fp64
  }
}

__global__ void __launch_bounds__(256) depth_filter_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                                                           const float* __restrict__ intr, const int64_t* __restrict__ inds,
                                                           const float* __restrict__ thresh, float* __restrict__ counter,
                                                           int num, int ht, int wd) {
  const int b = blockIdx.x;   // edges / frames on grid.x (2^31-1 blocks), pixel chunks on grid.y
  __shared__ float T[6][7];
  __shared__ int J[6];
  const int ix = (int)inds[b];
  if (threadIdx.x < 6) {
    const int neigh = threadIdx.x;
    const int jx = (neigh < 3) ? ix - neigh - 1 : ix + neigh;   // (:704) kept as is: -1,-2,-3,+3,+4,+5
    const bool ok = jx >= 0 && jx < num;
    J[neigh] = ok ? jx : -1;
    if (ok) edge_transform(poses, ix, jx, false, T[neigh], T[neigh] + 3);
  }
  __syncthreads();
  const Intr K = load_intr(intr);
  const int hw = ht * wd;
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= hw) return;
  const int i = k / wd, j = k - i * wd;
  const float ui = (float)j, vi = (float)i;
  const float di = __ldg(disps + (size_t)ix * hw + k);
  const double t = (double)__ldg(thresh + b);
  float Xi[4] = {(ui - K.cx) / K.fx, (vi - K.cy) / K.fy, 1.f, di}, Xj[4];
  float count = 0.f;
#pragma unroll
  for (int neigh = 0; neigh < 6; neigh++) {
    const int jx = J[neigh];
    if (jx < 0) continue;
    act_se3(T[neigh], T[neigh] + 3, Xi, Xj);
    const float uj = K.fx * (Xj[0] / Xj[2]) + K.cx;
    const float vj = K.fy * (Xj[1] / Xj[2]) + K.cy;
    const float dj = Xj[3] / Xj[2];
    const int u0 = __float2int_rd(uj), v0 = __float2int_rd(vj);   // static_cast<int>(floor(.)): saturating, NaN -> 0
    if (u0 >= 0 && v0 >= 0 && u0 < wd - 1 && v0 < ht - 1) {
      const float* dj_map = disps + (size_t)jx * hw;
      const float d00 = __ldg(dj_map + v0 * wd + u0), d01 = __ldg(dj_map + v0 * wd + u0 + 1);
      const float d10 = __ldg(dj_map + (v0 + 1) * wd + u0), d11 = __ldg(dj_map + (v0 + 1) * wd + u0 + 1);
      const double idj = 1.0 / (double)dj;   // the comparisons are fp64 in the reference (:777-781)
      if (fabs(idj - 1.0 / (double)d00) < t || fabs(idj - 1.0 / (double)d01) < t ||
          fabs(idj - 1.0 / (double)d10) < t || fabs(idj - 1.0 / (double)d11) < t)
        count += 1.0f;
    }
  }
  counter[(size_t)b * hw + k] = count;
}

__global__ void __launch_bounds__(256) iproj_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                                                    const float* __restrict__ intr, float* __restrict__ points, int ht, int wd) {
  const int n = blockIdx.x;   // edges / frames on grid.x (2^31-1 blocks), pixel chunks on grid.y
  const Intr K = load_intr(intr);
  float t[3], q[4];
#pragma unroll
  for (int k = 0; k < 3; k++) t[k] = __ldg(poses + 7 * (size_t)n + k);
#pragma unroll
  for (int k = 0; k < 4; k++) q[k] = __ldg(poses + 7 * (size_t)n + 3 + k);
  const int hw = ht * wd;
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= hw) return;
  const int i = k / wd, j = k - i * wd;
  float Xi[4] = {((float)j - K.cx) / K.fx, ((float)i - K.cy) / K.fy, 1.f, __ldg(disps + (size_t)n * hw + k)}, Xj[4];
  act_se3(t, q, Xi, Xj);
  float* p = points + ((size_t)n * hw + k) * 3;
  p[0] = Xj[0] / Xj[3]; p[1] = Xj[1] / Xj[3]; p[2] = Xj[2] / Xj[3];
}

// One pixel of the reprojection below: k = pixel index in frame ix, T = the edge transform,
// returns the coordinates in frame jx and the transformed point's depth z; X1, when given, receives the transformed point.
__device__ __forceinline__ float2 reproject_pixel(const float* T, const Intr& Ki, const Intr& Kj, const float* __restrict__ disps, int ix,
                                                  int k, int hw, int wd, float& z, float* X1 = nullptr) {
  const int i = k / wd, j = k - i * wd;
  float Xi[4] = {((float)j - Ki.cx) / Ki.fx, ((float)i - Ki.cy) / Ki.fy, 1.f, __ldg(disps + (size_t)ix * hw + k)}, Xj[4];
  act_se3(T, T + 3, Xi, Xj);
  const float Z = (Xj[2] < 0.5f * 0.2f) ? 1.f : Xj[2];
  const float d = 1.0f / Z;
  float2 c;
  c.x = Kj.fx * (Xj[0] * d) + Kj.cx;
  c.y = Kj.fy * (Xj[1] * d) + Kj.cy;
  z = Xj[2];
  if (X1) { X1[0] = Xj[0]; X1[1] = Xj[1]; X1[2] = Xj[2]; X1[3] = Xj[3]; }
  return c;
}

// Fused reprojection of the update operator's input (replaces the ~10 torch/lietorch launches of
// pops.projective_transform(..., jacobian=False), reference droid_slam/geom/projective_ops.py:165-198, called through
// DepthVideo.reproject, depth_video.py:171-179):  coords = proj(G_j G_i^-1 iproj(d_i)), valid = Z > 0.2.
// Differences from projmap that this path has in the reference and that are kept: per-frame intrinsics (iproj with frame
// ii's, proj with frame jj's), stereo edges ii == jj use the fixed baseline (-0.1,0,0 | identity) (:176-178), MIN_DEPTH is 0.2
// and depths below 0.1 are replaced by 1 before the division (:52,185)  (quirk Q3).
__global__ void __launch_bounds__(256) reproject_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                                                        const float* __restrict__ intr, const int64_t* __restrict__ ii,
                                                        const int64_t* __restrict__ jj, float* __restrict__ coords,
                                                        float* __restrict__ valid, int ht, int wd) {
  const int e = blockIdx.x;   // edges / frames on grid.x (2^31-1 blocks), pixel chunks on grid.y
  __shared__ float T[7];
  const int ix = (int)ii[e], jx = (int)jj[e];
  if (threadIdx.x == 0) edge_transform(poses, ix, jx, /*stereo_quirk=*/true, T, T + 3);
  __syncthreads();
  const Intr Ki = load_intr(intr + 4 * (size_t)ix), Kj = load_intr(intr + 4 * (size_t)jx);
  const int hw = ht * wd;
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= hw) return;
  float z;
  const float2 c = reproject_pixel(T, Ki, Kj, disps, ix, k, hw, wd, z);
  reinterpret_cast<float2*>(coords)[(size_t)e * hw + k] = c;
  valid[(size_t)e * hw + k] = (z > 0.2f) ? 1.f : 0.f;
}

// torch.clamp(v, -64, 64): NaN stays NaN (fminf / fmaxf would return the bound)
__device__ __forceinline__ float clamp64(float v) { return v < -64.f ? -64.f : (v > 64.f ? 64.f : v); }

// The motion features of FactorGraph.update / update_lowmem (reference factor_graph.py:220-222, :280-282) in one pass: the
// reprojection above (same device code, so coords are bit-identical to reproject_kernel's), written in both layouts the corr
// lookups take, and motn = clamp(cat([coords - grid, target - coords]), +-64) channel-major.  Call row r reads graph edge
// e = edge_index[r] (identity when edge_index is null): ii[e], jj[e], target[e].
__global__ void __launch_bounds__(256) motion_features_kernel(const float* __restrict__ poses, const float* __restrict__ disps,
                                                              const float* __restrict__ intr, const int64_t* __restrict__ ii,
                                                              const int64_t* __restrict__ jj, const int64_t* __restrict__ edge_index,
                                                              const float* __restrict__ target, float* __restrict__ coords,
                                                              float* __restrict__ coords_t, float* __restrict__ motn, int ht, int wd) {
  const int r = blockIdx.x;
  const size_t e = edge_index ? (size_t)edge_index[r] : (size_t)r;
  __shared__ float T[7];
  const int ix = (int)ii[e], jx = (int)jj[e];
  if (threadIdx.x == 0) edge_transform(poses, ix, jx, /*stereo_quirk=*/true, T, T + 3);
  __syncthreads();
  const Intr Ki = load_intr(intr + 4 * (size_t)ix), Kj = load_intr(intr + 4 * (size_t)jx);
  const int hw = ht * wd;
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= hw) return;
  float z;
  const float2 c = reproject_pixel(T, Ki, Kj, disps, ix, k, hw, wd, z);
  const int i = k / wd, j = k - i * wd;
  const float2 t = reinterpret_cast<const float2*>(target)[e * hw + k];
  reinterpret_cast<float2*>(coords)[(size_t)r * hw + k] = c;
  coords_t[(size_t)r * 2 * hw + k] = c.x;
  coords_t[((size_t)r * 2 + 1) * hw + k] = c.y;
  float* m = motn + (size_t)r * 4 * hw + k;
  m[0] = clamp64(__fsub_rn(c.x, (float)j));
  m[hw] = clamp64(__fsub_rn(c.y, (float)i));
  m[2 * hw] = clamp64(__fsub_rn(t.x, c.x));
  m[3 * hw] = clamp64(__fsub_rn(t.y, c.y));
}

// Write-back of one update-operator call into the factor graph (reference factor_graph.py:234-238, :304-307):
// rows r < n: target = coords + delta, weight, at graph edge e = edge_index[r] of the graph's [E,ht,wd,2] tensors and at row
// n_inactive + e of BA's channel-major [E_ba,2,ht,wd] inputs; rows n + m: damping[src_frames[m]] = eta[m].
__global__ void __launch_bounds__(256) graph_writeback_kernel(const float* __restrict__ delta, const float* __restrict__ weight,
                                                              const float* __restrict__ coords, const int64_t* __restrict__ edge_index, int n,
                                                              float* __restrict__ g_target, float* __restrict__ g_weight,
                                                              float* __restrict__ ba_target, float* __restrict__ ba_weight, int n_inactive,
                                                              const float* __restrict__ eta, const int64_t* __restrict__ src_frames,
                                                              float* __restrict__ damping, int hw) {
  const int r = blockIdx.x;
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= hw) return;
  if (r >= n) {
    const int m = r - n;
    damping[(size_t)src_frames[m] * hw + k] = eta[(size_t)m * hw + k];
    return;
  }
  const size_t e = edge_index ? (size_t)edge_index[r] : (size_t)r;
  const float2 c = reinterpret_cast<const float2*>(coords)[(size_t)r * hw + k];
  const float2 d = reinterpret_cast<const float2*>(delta)[(size_t)r * hw + k];
  const float2 w = reinterpret_cast<const float2*>(weight)[(size_t)r * hw + k];
  const float2 t = make_float2(__fadd_rn(c.x, d.x), __fadd_rn(c.y, d.y));
  reinterpret_cast<float2*>(g_target)[e * hw + k] = t;
  reinterpret_cast<float2*>(g_weight)[e * hw + k] = w;
  const size_t b = (size_t)n_inactive + e;
  ba_target[b * 2 * hw + k] = t.x; ba_target[(b * 2 + 1) * hw + k] = t.y;
  ba_weight[b * 2 * hw + k] = w.x; ba_weight[(b * 2 + 1) * hw + k] = w.y;
}

// BA's damping input: out[r] = .2 * damping[frames[r]] + ep with the reference's two roundings (factor_graph.py:251, :320)
__global__ void __launch_bounds__(256) damping_gather_kernel(const float* __restrict__ damping, const int64_t* __restrict__ frames,
                                                             float* __restrict__ out, float ep, int hw) {
  const int r = blockIdx.x;
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= hw) return;
  out[(size_t)r * hw + k] = __fadd_rn(__fmul_rn(damping[(size_t)frames[r] * hw + k], 0.2f), ep);
}

}  // namespace dba
using namespace dba;

extern "C" int dba_reproject(const float* poses, const float* disps, const float* intrinsics_per_frame, const int64_t* ii, const int64_t* jj,
                             float* coords, float* valid, int n_edges, int ht, int wd, dba_stream_t stream) {
  DBA_CHECK_ARG(n_edges >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (n_edges == 0 || ht * wd == 0) return DBA_OK;
  DBA_CHECK_ARG(poses && disps && intrinsics_per_frame && ii && jj && coords && valid, "null pointer");
  DBA_CHECK_ARG((ht * wd + 255) / 256 <= 65535, "image too large");
  dim3 grid(n_edges, (ht * wd + 255) / 256);
  reproject_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics_per_frame, ii, jj, coords, valid, ht, wd);
  DBA_CHECK_LAUNCH("reproject");
  return DBA_OK;
}

extern "C" int dba_motion_features(const float* poses, const float* disps, const float* intrinsics_per_frame, const int64_t* ii,
                                   const int64_t* jj, const int64_t* edge_index, const float* target, float* coords, float* coords_t,
                                   float* motn, int n_rows, int ht, int wd, dba_stream_t stream) {
  DBA_CHECK_ARG(n_rows >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (n_rows == 0 || ht * wd == 0) return DBA_OK;
  DBA_CHECK_ARG(poses && disps && intrinsics_per_frame && ii && jj && target && coords && coords_t && motn, "null pointer");
  DBA_CHECK_ARG((ht * wd + 255) / 256 <= 65535, "image too large");
  dim3 grid(n_rows, (ht * wd + 255) / 256);
  motion_features_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics_per_frame, ii, jj, edge_index, target, coords,
                                                                 coords_t, motn, ht, wd);
  DBA_CHECK_LAUNCH("motion_features");
  return DBA_OK;
}

extern "C" int dba_graph_writeback(const float* delta, const float* weight, const float* coords, const int64_t* edge_index, int n_rows,
                                   float* target, float* weight_out, float* ba_target, float* ba_weight, int n_inactive,
                                   const float* eta, const int64_t* src_frames, int n_src, float* damping,
                                   const int64_t* ba_frames, int n_ba_frames, float* ba_damping, float ep, int ht, int wd,
                                   dba_stream_t stream) {
  DBA_CHECK_ARG(n_rows >= 0 && n_inactive >= 0 && n_src >= 0 && n_ba_frames >= 0 && ht >= 0 && wd >= 0, "negative extent");
  const int hw = ht * wd;
  if (hw == 0) return DBA_OK;
  DBA_CHECK_ARG((hw + 255) / 256 <= 65535, "image too large");
  DBA_CHECK_ARG(n_rows == 0 || (delta && weight && coords && target && weight_out && ba_target && ba_weight), "null pointer");
  DBA_CHECK_ARG(n_src == 0 || (eta && src_frames && damping), "null pointer");
  DBA_CHECK_ARG(n_ba_frames == 0 || (damping && ba_frames && ba_damping), "null pointer");
  if (n_rows + n_src > 0) {
    dim3 grid(n_rows + n_src, (hw + 255) / 256);
    graph_writeback_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(delta, weight, coords, edge_index, n_rows, target, weight_out, ba_target,
                                                                   ba_weight, n_inactive, eta, src_frames, damping, hw);
    DBA_CHECK_LAUNCH("graph_writeback");
  }
  if (n_ba_frames > 0) {
    dim3 grid(n_ba_frames, (hw + 255) / 256);
    damping_gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(damping, ba_frames, ba_damping, ep, hw);
    DBA_CHECK_LAUNCH("graph_writeback (damping gather)");
  }
  return DBA_OK;
}

extern "C" int dba_projmap(const float* poses, const float* disps, const float* intrinsics, const int64_t* ii, const int64_t* jj,
                           float* coords, float* valid, int n_edges, int ht, int wd, dba_stream_t stream) {
  DBA_CHECK_ARG(n_edges >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (n_edges == 0 || ht * wd == 0) return DBA_OK;
  DBA_CHECK_ARG(poses && disps && intrinsics && ii && jj && coords && valid, "null pointer");
  DBA_CHECK_ARG((ht * wd + 255) / 256 <= 65535, "image too large");
  dim3 grid(n_edges, (ht * wd + 255) / 256);
  projmap_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, ii, jj, coords, valid, ht, wd);
  DBA_CHECK_LAUNCH("projmap");
  return DBA_OK;
}

extern "C" int dba_frame_distance(const float* poses, const float* disps, const float* intrinsics, const int64_t* ii,
                                  const int64_t* jj, float* dist, int n_pairs, int ht, int wd, float beta, dba_stream_t stream) {
  DBA_CHECK_ARG(n_pairs >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (n_pairs == 0) return DBA_OK;
  DBA_CHECK_ARG(poses && (disps || ht * wd == 0) && intrinsics && ii && jj && dist, "null pointer");   // hw = 0: every pair is 1000
  frame_distance_kernel<<<n_pairs, 256, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, ii, jj, dist, ht, wd, beta);
  DBA_CHECK_LAUNCH("frame_distance");
  return DBA_OK;
}

extern "C" int dba_depth_filter(const float* poses, const float* disps, const float* intrinsics, const int64_t* ix,
                                const float* thresh, float* counter, int num, int n_disps, int ht, int wd, dba_stream_t stream) {
  DBA_CHECK_ARG(num >= 0 && n_disps >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (num == 0 || ht * wd == 0) return DBA_OK;
  DBA_CHECK_ARG(poses && disps && intrinsics && ix && thresh && counter, "null pointer");
  DBA_CHECK_ARG((ht * wd + 255) / 256 <= 65535, "image too large");
  dim3 grid(num, (ht * wd + 255) / 256);
  depth_filter_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, ix, thresh, counter, n_disps, ht, wd);
  DBA_CHECK_LAUNCH("depth_filter");
  return DBA_OK;
}

extern "C" int dba_iproj(const float* poses, const float* disps, const float* intrinsics, float* points, int n, int ht, int wd,
                         dba_stream_t stream) {
  DBA_CHECK_ARG(n >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (n == 0 || ht * wd == 0) return DBA_OK;
  DBA_CHECK_ARG(poses && disps && intrinsics && points, "null pointer");
  DBA_CHECK_ARG((ht * wd + 255) / 256 <= 65535, "image too large");
  dim3 grid(n, (ht * wd + 255) / 256);
  iproj_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(poses, disps, intrinsics, points, ht, wd);
  DBA_CHECK_LAUNCH("iproj");
  return DBA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------
// convex upsampling of the inverse depth maps (reference droid_slam/droid_net.py:21-42 `cvx_upsample` / `upsample_disp`, called by
// DepthVideo.upsample, depth_video.py:155-159): out[b][8y+i][8x+j] = sum_k softmax_k(mask[b][k*64 + i*8 + j][y][x]) * d[b][y+ky-1][x+kx-1],
// k = 3*ky + kx, zero padding (F.unfold).  One thread = one source pixel and one sub-row i: 72 coalesced mask loads (lanes run over x),
// softmax over the 9 taps in fp32 (autocast runs softmax in fp32 too), 8 consecutive outputs = one 32-byte sector.
// ---------------------------------------------------------------------------------------------------------------------------
namespace dba {
template <typename TM>
__global__ void __launch_bounds__(256) cvx_upsample_kernel(const float* __restrict__ disps, const TM* __restrict__ mask, float* __restrict__ out,
                                                           int n, int ht, int wd) {
  const int hw = ht * wd;
  const long long total = (long long)n * 8 * hw;
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= total) return;
  const int pin = (int)(id % hw);
  const int i = (int)((id / hw) % 8);
  const int b = (int)(id / (8LL * hw));
  const int y = pin / wd, x = pin - y * wd;
  float d[9];
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    d[k] = (yy >= 0 && yy < ht && xx >= 0 && xx < wd) ? __ldg(disps + (size_t)b * hw + (size_t)yy * wd + xx) : 0.f;
  }
  const TM* m = mask + ((size_t)b * 576 + i * 8) * hw + pin;
  float res[8];
#pragma unroll
  for (int j = 0; j < 8; j++) {
    float v[9], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 9; k++) { v[k] = (float)m[((size_t)k * 64 + j) * hw]; mx = fmaxf(mx, v[k]); }
    float den = 0.f, num = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) { const float e = __expf(v[k] - mx); den += e; num += e * d[k]; }
    res[j] = num / den;
  }
  float4* o = reinterpret_cast<float4*>(out + ((size_t)b * 8 * ht + 8 * y + i) * (size_t)(8 * wd) + 8 * x);
  o[0] = make_float4(res[0], res[1], res[2], res[3]);
  o[1] = make_float4(res[4], res[5], res[6], res[7]);
}
}  // namespace dba

extern "C" int dba_cvx_upsample(const float* disps, const void* mask, float* out, int n, int ht, int wd, int mask_dtype, dba_stream_t stream) {
  DBA_CHECK_ARG(n >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (n == 0 || ht * wd == 0) return DBA_OK;
  DBA_CHECK_ARG(disps && mask && out, "null pointer");
  DBA_CHECK_ARG(mask_dtype == DBA_F16 || mask_dtype == DBA_F32, "mask must be f16 or f32");
  DBA_CHECK_ARG((((uintptr_t)out) & 15) == 0, "out must be 16-byte aligned");
  const long long total = (long long)n * 8 * ht * wd;
  DBA_CHECK_ARG((total + 255) / 256 < 0x7fffffffLL, "too many pixels for one launch");
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (mask_dtype == DBA_F16) dba::cvx_upsample_kernel<__half><<<blocks, 256, 0, (cudaStream_t)stream>>>(disps, (const __half*)mask, out, n, ht, wd);
  else dba::cvx_upsample_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(disps, (const float*)mask, out, n, ht, wd);
  DBA_CHECK_LAUNCH("cvx_upsample");
  return DBA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------
// Training's tail: the flow loss (reference droid_slam/geom/losses.py:89-118) and the backward of upsample_disp (droid_net.py:21-42).
//
// flow_loss compares, on the chain graph of the clip (edges (0,1), (1,0), (1,2), (2,1), ... as losses.py:93-97 builds them), the
// ground-truth reprojection coords0 / val0 with each iterate's coords1 / val1, both the projective_transform of projective_ops.py:165-198
// at full resolution: loss = sum_s gamma^(n-1-s) mean(v |c1 - c0|), v = val0 val1, val0 also masked by disps > 0.  Nothing per pixel is
// stored: the forward recomputes c0 once per pixel and runs every iterate in the same pass; the backward recomputes c0 and c1.  Every
// per-pixel value is reproject_pixel's (one reprojection for the whole file); the edge transforms Gij = Pj Pi^-1 use lietorch's mul and
// inv (quaternions normalised on load), as the reference's lietorch does.  Sums go through per-block partials reduced in a fixed
// order: no atomics, bit-identical runs.
// ---------------------------------------------------------------------------------------------------------------------------
#include "lie_math.cuh"
#include "../../include/droid_b200_training.h"

namespace dba {
constexpr int kFlowThreads = 256;

// edge e of the chain graph: source i, target j
__device__ __forceinline__ void chain_edge(int e, int& i, int& j) {
  if (e == 0) { i = 0; j = 1; return; }
  i = (e + 1) >> 1;
  j = (e & 1) ? i - 1 : i + 1;
}

// the sum of v over the block (kFlowThreads threads) in a fixed order, in thread 0; red: kFlowThreads / 32 shared floats
__device__ __forceinline__ float flow_block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < kFlowThreads / 32; w++) s += red[w];
  __syncthreads();
  return s;
}

// G[b][s][e] (7 floats: t, q) = Pj Pi^-1 of edge e in slot s: 0 the ground truth Ps, 1 + k the iterate poses_est[k]
__global__ void flow_edges_kernel(const float* __restrict__ Ps, const float* const* __restrict__ poses_est, float* __restrict__ G, int B,
                                  int N, int n) {
  const int E = 2 * (N - 1);
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= B * (n + 1) * E) return;
  const int e = id % E, s = (id / E) % (n + 1), b = id / (E * (n + 1));
  const float* P = (s == 0 ? Ps : poses_est[s - 1]) + (size_t)b * N * 7;
  int i, j;
  chain_edge(e, i, j);
  dba_lie::Elem<dba_lie::SE3g, float> Pi, Pj;
  Pi.load(P + 7 * i);
  Pj.load(P + 7 * j);
  dba_lie::g_mul(Pj, dba_lie::g_inv(Pi)).store(G + (size_t)id * 7);
}

// grid (pixel chunks, E, B).  Per block: the partial sums of v |c1 - c0| for every iterate, then for the last iterate the sum of epe
// where v > 0.5, that count and the count with epe < 1: part[slot][block], n + 3 slots.  A pixel with v = 0 is not skipped: a NaN
// coordinate makes 0 * NaN, as in the reference.
__global__ void __launch_bounds__(kFlowThreads) flow_loss_kernel(const float* __restrict__ G, const float* __restrict__ disps,
                                                                 const float* const* __restrict__ disps_est, const float* __restrict__ intr,
                                                                 float* __restrict__ part, int N, int n, int ht, int wd) {
  __shared__ float red[kFlowThreads / 32];
  const int chunk = blockIdx.x, e = blockIdx.y, b = blockIdx.z, E = gridDim.y;
  const int hw = ht * wd;
  const size_t nblk = (size_t)gridDim.x * E * gridDim.z, blk = ((size_t)b * E + e) * gridDim.x + chunk;
  int i, j;
  chain_edge(e, i, j);
  const int k = chunk * kFlowThreads + threadIdx.x;
  const bool in = k < hw;
  const Intr Ki = load_intr(intr + 4 * ((size_t)b * N + i)), Kj = load_intr(intr + 4 * ((size_t)b * N + j));
  const size_t fb = (size_t)b * N * hw;
  const float* Gb = G + ((size_t)b * (n + 1) * E + e) * 7;
  float2 c0 = make_float2(0.f, 0.f);
  float v0 = 0.f;
  if (in) {
    float z0;
    c0 = reproject_pixel(Gb, Ki, Kj, disps + fb, i, k, hw, wd, z0);
    v0 = (z0 > 0.2f && __ldg(disps + fb + (size_t)i * hw + k) > 0.f) ? 1.f : 0.f;   // X0.z is 1
  }
  for (int s = 0; s < n; s++) {
    float epe = 0.f, v = 0.f;
    if (in) {
      float z1;
      const float2 c1 = reproject_pixel(Gb + (size_t)(s + 1) * E * 7, Ki, Kj, disps_est[s] + fb, i, k, hw, wd, z1);
      v = v0 * (z1 > 0.2f ? 1.f : 0.f);
      const float dx = c1.x - c0.x, dy = c1.y - c0.y;
      epe = v * sqrtf(dx * dx + dy * dy);
    }
    float t = flow_block_sum(epe, red);
    if (threadIdx.x == 0) part[(size_t)s * nblk + blk] = t;
    if (s == n - 1) {
      const bool m = v > 0.5f;
      t = flow_block_sum(m ? epe : 0.f, red);
      if (threadIdx.x == 0) part[(size_t)n * nblk + blk] = t;
      t = flow_block_sum(m ? 1.f : 0.f, red);
      if (threadIdx.x == 0) part[(size_t)(n + 1) * nblk + blk] = t;
      t = flow_block_sum(m && epe < 1.f ? 1.f : 0.f, red);
      if (threadIdx.x == 0) part[(size_t)(n + 2) * nblk + blk] = t;
    }
  }
}

// one block: each slot of part summed in fp64 in a fixed order; loss = sum_s gamma^(n-1-s) slot_s / count, metrics = the last 3 slots
__global__ void __launch_bounds__(256) flow_loss_reduce_kernel(const float* __restrict__ part, size_t nblk, int n, double gamma, double count,
                                                               float* __restrict__ loss, double* __restrict__ metrics) {
  __shared__ double red[8];
  double L = 0.0;
  for (int s = 0; s < n + 3; s++) {
    double a = 0.0;
    for (size_t q = threadIdx.x; q < nblk; q += 256) a += (double)part[(size_t)s * nblk + q];
    a = warp_sum(a);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < 8; w++) t += red[w];
      if (s < n) L += pow(gamma, (double)(n - 1 - s)) * (t / count);
      else metrics[s - n] = t;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = (float)L;
}

// grid (pixel chunks, N source frames, B).  Per pixel of frame a and iterate s: the gradient of the loss at c1 on each out-edge of a
// (to a-1, then to a+1), pulled back through proj (no gradient to Z where Z < 0.1 was replaced by 1; 0 where c1 == c0, as torch's
// norm gives) to the transformed point X1: the disparity gets X1's derivative along Gij's translation (both edges summed, written once),
// the edge the actp Jacobian's transpose, summed over the block -> gpart[s][b][e][chunk][6].
__global__ void __launch_bounds__(kFlowThreads) flow_loss_bwd_kernel(const float* __restrict__ grad, const float* __restrict__ G,
                                                                     const float* __restrict__ disps, const float* const* __restrict__ disps_est,
                                                                     const float* __restrict__ intr, float* const* __restrict__ grad_disps_est,
                                                                     float* __restrict__ gpart, int N, int n, int ht, int wd, double gamma,
                                                                     double count) {
  __shared__ float red[12][kFlowThreads / 32];
  const int chunk = blockIdx.x, a = blockIdx.y, b = blockIdx.z, nch = gridDim.x, B = gridDim.z;
  const int E = 2 * (N - 1), hw = ht * wd;
  const int k = chunk * kFlowThreads + threadIdx.x;
  const bool in = k < hw;
  int eo[2], ne = 0;
  if (a > 0) eo[ne++] = 2 * a - 1;
  if (a < N - 1) eo[ne++] = a == 0 ? 0 : 2 * a;
  const size_t fb = (size_t)b * N * hw;
  const Intr Ki = load_intr(intr + 4 * ((size_t)b * N + a));
  Intr Kj[2];
  float2 c0[2];
  float v0[2];
  for (int q = 0; q < ne; q++) {
    int i, j;
    chain_edge(eo[q], i, j);
    Kj[q] = load_intr(intr + 4 * ((size_t)b * N + j));
    c0[q] = make_float2(0.f, 0.f);
    v0[q] = 0.f;
    if (in) {
      float z0;
      c0[q] = reproject_pixel(G + ((size_t)b * (n + 1) * E + eo[q]) * 7, Ki, Kj[q], disps + fb, a, k, hw, wd, z0);
      v0[q] = (z0 > 0.2f && __ldg(disps + fb + (size_t)a * hw + k) > 0.f) ? 1.f : 0.f;
    }
  }
  const double g = (double)__ldg(grad);
  for (int s = 0; s < n; s++) {
    const float cs = (float)(g * pow(gamma, (double)(n - 1 - s)) / count);
    float gd = 0.f, g6[2][6] = {};
    for (int q = 0; q < ne && in; q++) {
      const float* T = G + (((size_t)b * (n + 1) + s + 1) * E + eo[q]) * 7;
      float X1[4], z1;
      const float2 c1 = reproject_pixel(T, Ki, Kj[q], disps_est[s] + fb, a, k, hw, wd, z1, X1);
      const float v = v0[q] * (z1 > 0.2f ? 1.f : 0.f);
      const float dx = c1.x - c0[q].x, dy = c1.y - c0[q].y;
      const float nrm = sqrtf(dx * dx + dy * dy);
      const float r = nrm == 0.f ? 0.f : (cs * v) / nrm;
      const float gcx = dx * r, gcy = dy * r;
      const bool clamped = X1[2] < 0.5f * 0.2f;
      const float id = 1.0f / (clamped ? 1.f : X1[2]);
      const float gX = gcx * Kj[q].fx * id, gY = gcy * Kj[q].fy * id;
      const float gZ = clamped ? 0.f : -((gcx * Kj[q].fx * X1[0] + gcy * Kj[q].fy * X1[1]) * id * id);
      gd += gX * T[0] + gY * T[1] + gZ * T[2];
      // actp's Jacobian rows (X1 = (X, Y, Z, W)): (W,0,0, 0,Z,-Y), (0,W,0, -Z,0,X), (0,0,W, Y,-X,0)
      g6[q][0] = gX * X1[3]; g6[q][1] = gY * X1[3]; g6[q][2] = gZ * X1[3];
      g6[q][3] = gZ * X1[1] - gY * X1[2];
      g6[q][4] = gX * X1[2] - gZ * X1[0];
      g6[q][5] = gY * X1[0] - gX * X1[1];
    }
    if (in) grad_disps_est[s][fb + (size_t)a * hw + k] = gd;
    const int w = threadIdx.x >> 5;
#pragma unroll
    for (int m = 0; m < 12; m++) {
      const float t = warp_sum(g6[m / 6][m % 6]);
      if ((threadIdx.x & 31) == 0) red[m][w] = t;
    }
    __syncthreads();
    if (threadIdx.x < 6 * ne) {
      const int q = threadIdx.x / 6, m = threadIdx.x % 6;
      float t = 0.f;
      for (int x = 0; x < kFlowThreads / 32; x++) t += red[q * 6 + m][x];
      gpart[((((size_t)s * B + b) * E + eo[q]) * nch + chunk) * 6 + m] = t;
    }
    __syncthreads();
  }
}

// grid (N, B, n), one warp: frame f's gradient for iterate s, lietorch's left-tangent convention (7th entry 0): over the edges touching
// f in edge order, + g_e where f is the target and - Adj(Gij)^T g_e where f is the source, g_e the edge's chunk partials summed in fp64
__global__ void __launch_bounds__(32) flow_pose_grad_kernel(const float* __restrict__ G, const float* __restrict__ gpart,
                                                            float* const* __restrict__ grad_poses_est, int N, int n, int nch) {
  const int f = blockIdx.x, b = blockIdx.y, s = blockIdx.z, B = gridDim.y;
  const int E = 2 * (N - 1);
  double acc[6] = {};
  for (int e = 0; e < E; e++) {
    int i, j;
    chain_edge(e, i, j);
    if (i != f && j != f) continue;
    const float* p = gpart + (((size_t)s * B + b) * E + e) * nch * 6;
    double ge[6] = {};
    for (int c = threadIdx.x; c < nch; c += 32)
      for (int m = 0; m < 6; m++) ge[m] += (double)p[(size_t)c * 6 + m];
    for (int m = 0; m < 6; m++) ge[m] = warp_sum(ge[m]);
    if (j == f) {
      for (int m = 0; m < 6; m++) acc[m] += ge[m];
    } else {
      dba_lie::Elem<dba_lie::SE3g, double> Gij;
      Gij.load(G + (((size_t)b * (n + 1) + s + 1) * E + e) * 7);
      double o[6];
      dba_lie::g_adjT(Gij, ge, o);
      for (int m = 0; m < 6; m++) acc[m] -= o[m];
    }
  }
  if (threadIdx.x == 0) {
    float* out = grad_poses_est[s] + ((size_t)b * N + f) * 7;
    for (int m = 0; m < 6; m++) out[m] = (float)acc[m];
    out[6] = 0.f;
  }
}

// the backward of cvx_upsample_kernel for fp32 masks, one thread per source pixel and sub-row i as in the forward: the softmax
// recomputed from the mask, grad_mask = p (g d - sum_l p_l g d_l) per tap, and per tap k the sum over the thread's 8 outputs of g p_k
// -> taps[b][k][i][pixel]; the disparity gradient is gathered from these below
__global__ void __launch_bounds__(256) cvx_upsample_bwd_kernel(const float* __restrict__ disps, const float* __restrict__ mask,
                                                               const float* __restrict__ gout, float* __restrict__ gmask, float* __restrict__ taps,
                                                               int n, int ht, int wd) {
  const int hw = ht * wd;
  const long long total = (long long)n * 8 * hw;
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= total) return;
  const int pin = (int)(id % hw);
  const int i = (int)((id / hw) % 8);
  const int b = (int)(id / (8LL * hw));
  const int y = pin / wd, x = pin - y * wd;
  float d[9];
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    d[k] = (yy >= 0 && yy < ht && xx >= 0 && xx < wd) ? __ldg(disps + (size_t)b * hw + (size_t)yy * wd + xx) : 0.f;
  }
  const float4* g4 = reinterpret_cast<const float4*>(gout + ((size_t)b * 8 * ht + 8 * y + i) * (size_t)(8 * wd) + 8 * x);
  const float4 ga = __ldg(g4), gb = __ldg(g4 + 1);
  const float g[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
  const size_t off = ((size_t)b * 576 + i * 8) * hw + pin;
  const float* m = mask + off;
  float* gm = gmask + off;
  float P[9] = {};
#pragma unroll
  for (int j = 0; j < 8; j++) {
    float v[9], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 9; k++) { v[k] = __ldg(m + ((size_t)k * 64 + j) * hw); mx = fmaxf(mx, v[k]); }
    float den = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) { v[k] = expf(v[k] - mx); den += v[k]; }
    float sp = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) { v[k] = v[k] / den; sp += v[k] * (g[j] * d[k]); }
#pragma unroll
    for (int k = 0; k < 9; k++) {
      gm[((size_t)k * 64 + j) * hw] = v[k] * (g[j] * d[k] - sp);
      P[k] += g[j] * v[k];
    }
  }
#pragma unroll
  for (int k = 0; k < 9; k++) taps[(((size_t)b * 9 + k) * 8 + i) * hw + pin] = P[k];
}

// grad_disps at (y, x): tap k of source pixel (y - ky + 1, x - kx + 1) read it (zero padding: sources outside the map do not exist),
// summed over k then the 8 sub-rows in a fixed order
__global__ void __launch_bounds__(256) cvx_upsample_gather_kernel(const float* __restrict__ taps, float* __restrict__ gdisps, int n, int ht, int wd) {
  const int hw = ht * wd;
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (long long)n * hw) return;
  const int pin = (int)(id % hw), b = (int)(id / hw);
  const int y = pin / wd, x = pin - y * wd;
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 9; k++) {
    const int sy = y - k / 3 + 1, sx = x - k % 3 + 1;
    if (sy < 0 || sy >= ht || sx < 0 || sx >= wd) continue;
    const float* t = taps + ((size_t)b * 9 + k) * 8 * hw + (size_t)sy * wd + sx;
#pragma unroll
    for (int i = 0; i < 8; i++) acc += __ldg(t + (size_t)i * hw);
  }
  gdisps[id] = acc;
}

static size_t flow_align(size_t b) { return (b + 255) & ~(size_t)255; }
static int flow_chunks(int ht, int wd) { return (ht * wd + kFlowThreads - 1) / kFlowThreads; }
static size_t flow_edges_bytes(int B, int N, int n) { return flow_align((size_t)B * (n + 1) * 2 * (N - 1) * 7 * sizeof(float)); }
}  // namespace dba

extern "C" size_t dba_flow_loss_workspace_bytes(int B, int N, int ht, int wd, int n) {
  if (B < 1 || N < 2 || ht < 1 || wd < 1 || n < 1) return 0;
  const size_t E = 2 * (size_t)(N - 1), nblk = (size_t)B * E * dba::flow_chunks(ht, wd);
  const size_t fwd = (size_t)(n + 3) * nblk * sizeof(float), bwd = (size_t)n * nblk * 6 * sizeof(float);
  return dba::flow_edges_bytes(B, N, n) + dba::flow_align(fwd > bwd ? fwd : bwd);
}

static int flow_loss_check(const float* Ps, const float* disps, const float* intrinsics, const float* const* poses_est,
                           const float* const* disps_est, int n, int B, int N, int ht, int wd, void* workspace, size_t workspace_bytes) {
  DBA_CHECK_ARG(B >= 1 && N >= 2 && ht >= 1 && wd >= 1 && n >= 1, "flow_loss needs B >= 1, N >= 2, a non-empty image and an iterate");
  DBA_CHECK_ARG(Ps && disps && intrinsics && poses_est && disps_est && workspace, "null pointer");
  DBA_CHECK_ARG(B <= 65535 && N <= 32768, "too many batch elements or frames for one launch");
  DBA_CHECK_ARG((long long)ht * wd <= 0x7fffffffLL - dba::kFlowThreads, "image too large");
  DBA_CHECK_ARG(workspace_bytes >= dba_flow_loss_workspace_bytes(B, N, ht, wd, n), "workspace smaller than dba_flow_loss_workspace_bytes");
  return DBA_OK;
}

static int flow_edges_launch(const float* Ps, const float* const* poses_est, float* G, int B, int N, int n, cudaStream_t st) {
  const int total = B * (n + 1) * 2 * (N - 1);
  dba::flow_edges_kernel<<<(total + 127) / 128, 128, 0, st>>>(Ps, poses_est, G, B, N, n);
  DBA_CHECK_LAUNCH("flow_loss (edge transforms)");
  return DBA_OK;
}

extern "C" int dba_flow_loss_forward(const float* Ps, const float* disps, const float* intrinsics, const float* const* poses_est,
                                     const float* const* disps_est, int n, float* loss, double* metrics, int B, int N, int ht, int wd,
                                     double gamma, void* workspace, size_t workspace_bytes, dba_stream_t stream) {
  int rc = flow_loss_check(Ps, disps, intrinsics, poses_est, disps_est, n, B, N, ht, wd, workspace, workspace_bytes);
  if (rc != DBA_OK) return rc;
  DBA_CHECK_ARG(loss && metrics, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  float* G = (float*)workspace;
  float* part = (float*)((char*)workspace + dba::flow_edges_bytes(B, N, n));
  if ((rc = flow_edges_launch(Ps, poses_est, G, B, N, n, st)) != DBA_OK) return rc;
  const int E = 2 * (N - 1), nch = dba::flow_chunks(ht, wd);
  dba::flow_loss_kernel<<<dim3(nch, E, B), dba::kFlowThreads, 0, st>>>(G, disps, disps_est, intrinsics, part, N, n, ht, wd);
  DBA_CHECK_LAUNCH("flow_loss");
  const size_t nblk = (size_t)nch * E * B;
  dba::flow_loss_reduce_kernel<<<1, 256, 0, st>>>(part, nblk, n, gamma, (double)B * E * ht * wd, loss, metrics);
  DBA_CHECK_LAUNCH("flow_loss (reduction)");
  return DBA_OK;
}

extern "C" int dba_flow_loss_backward(const float* grad_loss, const float* Ps, const float* disps, const float* intrinsics,
                                      const float* const* poses_est, const float* const* disps_est, int n, float* const* grad_poses_est,
                                      float* const* grad_disps_est, int B, int N, int ht, int wd, double gamma, void* workspace,
                                      size_t workspace_bytes, dba_stream_t stream) {
  int rc = flow_loss_check(Ps, disps, intrinsics, poses_est, disps_est, n, B, N, ht, wd, workspace, workspace_bytes);
  if (rc != DBA_OK) return rc;
  DBA_CHECK_ARG(grad_loss && grad_poses_est && grad_disps_est, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  float* G = (float*)workspace;
  float* gpart = (float*)((char*)workspace + dba::flow_edges_bytes(B, N, n));
  if ((rc = flow_edges_launch(Ps, poses_est, G, B, N, n, st)) != DBA_OK) return rc;
  const int E = 2 * (N - 1), nch = dba::flow_chunks(ht, wd);
  dba::flow_loss_bwd_kernel<<<dim3(nch, N, B), dba::kFlowThreads, 0, st>>>(grad_loss, G, disps, disps_est, intrinsics, grad_disps_est, gpart, N,
                                                                            n, ht, wd, gamma, (double)B * E * ht * wd);
  DBA_CHECK_LAUNCH("flow_loss_backward");
  dba::flow_pose_grad_kernel<<<dim3(N, B, n), 32, 0, st>>>(G, gpart, grad_poses_est, N, n, nch);
  DBA_CHECK_LAUNCH("flow_loss_backward (pose gradients)");
  return DBA_OK;
}

extern "C" int dba_cvx_upsample_backward(const float* disps, const float* mask, const float* grad_out, float* grad_disps, float* grad_mask,
                                         float* tap_partials, int n, int ht, int wd, dba_stream_t stream) {
  DBA_CHECK_ARG(n >= 0 && ht >= 0 && wd >= 0, "negative extent");
  if (n == 0 || ht * wd == 0) return DBA_OK;
  DBA_CHECK_ARG(disps && mask && grad_out && grad_disps && grad_mask && tap_partials, "null pointer");
  DBA_CHECK_ARG((((uintptr_t)grad_out) & 15) == 0, "grad_out must be 16-byte aligned");
  const long long total = (long long)n * 8 * ht * wd;
  DBA_CHECK_ARG((total + 255) / 256 < 0x7fffffffLL, "too many pixels for one launch");
  cudaStream_t st = (cudaStream_t)stream;
  dba::cvx_upsample_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(disps, mask, grad_out, grad_mask, tap_partials, n, ht, wd);
  DBA_CHECK_LAUNCH("cvx_upsample_backward");
  const long long pix = (long long)n * ht * wd;
  dba::cvx_upsample_gather_kernel<<<(unsigned)((pix + 255) / 256), 256, 0, st>>>(tap_partials, grad_disps, n, ht, wd);
  DBA_CHECK_LAUNCH("cvx_upsample_backward (gather)");
  return DBA_OK;
}
