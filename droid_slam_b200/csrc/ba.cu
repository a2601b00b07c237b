// Dense bundle adjustment (Gauss-Newton, Schur complement over per-pixel inverse depth) for sm_90a.
//
// Replaces reference src/droid_kernels.cu:185-433 (K1), :863-1124 (accum / retraction / Schur kernels),
// :1126-1320 (CPU SparseBlock + schur_block) and the driver :1323-1443.  Same maths, different machine mapping:
//
//   * everything stays on the device and on one stream: no .to(kCPU), no argsort/CSR on the host, no Eigen;
//   * edges are grouped by SOURCE frame (CSR built once per call by two small kernels).  One CTA owns
//     (depth frame k, pixel chunk): it walks the out-edges of k, so the depth-block sums C_k, w_k, Ei_k are plain
//     register accumulations (no atomics, no segmented-sum kernels, deterministic);
//   * only Hjj (21 unique) and vj (6) are accumulated per pixel.  Ji = -Adj^T(G_ij) Jj is linear in Jj, hence
//     Hii = A Hjj A^T, Hij = -A Hjj, vi = -A vj are formed once per edge from the reduced fp64 sums
//     (the reference accumulates all 78+12 sums per pixel and does 90 serial block reductions);
//   * reductions: fp32 per thread over its pixels -> warp shuffles -> fp64 across warps -> fp64 atomics into the
//     dense reduced system Hsys [6P x 6P] / bsys [6P] (this is the buffer an edge-sharded multi-GPU run all-reduces);
//   * the Schur complement S = sum_k E_k Q_k E_k^T is a per-frame SYRK over the (1+deg_k) rows of frame k on the tensor cores, all
//     frames in one launch of one CTA per SM, balanced by a work plan ba_prepare_kernel writes (the reference enumerates (i,j,k)
//     triples on the CPU, O(P^2 deg^2));
//   * solve: damping (diag += ep + lm*diag) and a tiled fp64 Cholesky on the device; a non-positive pivot gives
//     dx = 0 like the reference's `solver.info() != Success` branch;
//   * back-substitution dz = Q (w - E^T dx) keeps the reference quirk Q9 (rows whose pose index is <= 0 are skipped,
//     src/droid_kernels.cu:1114), then retraction of poses (left-multiplicative Exp, no renormalisation) and disps.
#include "common.cuh"
#include "ba_pixel.cuh"
#include "droid_se3.cuh"
#include "wgmma.cuh"
#include <math.h>
#include <algorithm>

namespace dba {

constexpr int kBuildThreads = 256;
constexpr int kEdgeBatch = 16;     // edges whose transforms / partial sums live in shared memory at once

struct Layout {
  size_t off_hdr, off_frame2k, off_kx, off_rowptr, off_edgeidx, off_plan, off_sys, off_L, off_dx, off_Eij, off_C, off_w, off_Ei, total;
  int P, n;
};

__host__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Stride of the workspace's per-pixel rows (Eij [E][6][pitch], C and w [M][pitch], Ei [M][6][pitch]): HW rounded up to 4 floats,
// so that every row starts on a 16-byte boundary for the tensor-core Schur kernel's cp.async / float4 loads.  Pixels [HW, pitch)
// are zeroed by ba_prepare_kernel and never written again.  Caller tensors (disps, targets, weights, eta, dz_out) keep the stride HW.
__host__ __device__ __forceinline__ int ba_pitch(int HW) { return (HW + 3) & ~3; }

__host__ inline Layout make_layout(int N, int E, int ht, int wd, int t0, int t1) {
  Layout L;
  const size_t pitch = (size_t)ba_pitch(ht * wd);
  L.P = t1 - t0 > 0 ? t1 - t0 : 0;
  L.n = 6 * L.P;
  size_t o = 0;
  L.off_hdr = o;      o = align_up(o + 64 * sizeof(int), 256);
  L.off_frame2k = o;  o = align_up(o + (size_t)(N + 1) * sizeof(int), 256);
  L.off_kx = o;       o = align_up(o + (size_t)(N + 1) * sizeof(int), 256);
  L.off_rowptr = o;   o = align_up(o + (size_t)(N + 2) * sizeof(int), 256);
  L.off_edgeidx = o;  o = align_up(o + (size_t)(E + 1) * sizeof(int), 256);
  L.off_plan = o;     o = align_up(o + 4 * (size_t)(N + 1) * sizeof(int), 256); // SchurPlan
  L.off_sys = o;      o = align_up(o + ((size_t)L.n * L.n + L.n) * sizeof(double), 256);
  L.off_L = o;        o = align_up(o + chol_workspace_bytes(L.n), 256);
  L.off_dx = o;       o = align_up(o + (size_t)(L.n + 6) * sizeof(float), 256);
  L.off_Eij = o;      o = align_up(o + (size_t)E * 6 * pitch * sizeof(float), 256);
  const size_t Mmax = (size_t)N;   // at most one depth frame per buffer frame
  L.off_C = o;        o = align_up(o + Mmax * pitch * sizeof(float), 256);
  L.off_w = o;        o = align_up(o + Mmax * pitch * sizeof(float), 256);
  L.off_Ei = o;       o = align_up(o + Mmax * 6 * pitch * sizeof(float), 256);
  L.total = o;
  return L;
}

// header words
enum { HDR_STATUS = 0, HDR_M = 1, HDR_CHOL_FAIL = 2, HDR_NBIG = 3, HDR_NPAIR = 4 };
enum { ST_BAD_INDEX = 1, ST_ETA_ROWS = 2, ST_CHOL_FAIL = 4, ST_DEGREE = 8 };

// Schur routes by the rows of a depth frame (see the Schur section): packed tiles up to kPackedRowsMax rows, one tile up to kTcRowsMax,
// pairs of kPairTileRows-row tiles up to kSchurMaxRows (out-degree + 1; larger frames raise ST_DEGREE)
constexpr int kPackedRowsMax = 10;
constexpr int kTcRowsMax = 21;
constexpr int kPairTileRows = 10;        // 60 lines + the w line <= 64 operand rows
constexpr int kSchurMaxRows = 255;

// The Schur launch's work plan, written by ba_prepare_kernel (four arrays of N + 1 ints at Layout::off_plan):
//   rows[m]   Schur rows of depth frame m: its own pose if it is in [t0, t1), plus one per out-edge whose target is; 0 without out-edges
//   cost[m]   exclusive prefix sum over the frames of their packed / single-tile cost (schur_cost), cost[M] = the total
//   big[i]    the depth frames above kTcRowsMax rows (pair route), ascending, i < hdr[HDR_NBIG]
//   pairs[i]  exclusive prefix sum of their tile-pair counts; hdr[HDR_NPAIR] = the total
struct SchurPlan { int *rows, *cost, *big, *pairs; };
__host__ __device__ inline SchurPlan schur_plan(void* base, int N) {
  int* p = reinterpret_cast<int*>(base);
  return SchurPlan{p, p + (N + 1), p + 2 * (N + 1), p + 3 * (N + 1)};
}
// Cost of a frame's packed or single-tile Schur work in the units the launch balances: one per 64-pixel packed chunk (an M = N = 64
// product per warpgroup), two per 32-pixel single-tile chunk (M = 64, N = 128: twice the MMA work).  0 on the pair route.
__device__ __forceinline__ int schur_cost(int rows, int HW) {
  return rows == 0 || rows > kTcRowsMax ? 0 : rows <= kPackedRowsMax ? (HW + 63) / 64 : 2 * ((HW + 31) / 32);
}
__device__ __forceinline__ int schur_pair_count(int rows) {
  const int T = (min(rows, kSchurMaxRows) + kPairTileRows - 1) / kPairTileRows;
  return T * (T - 1) / 2;
}

// ---------------------------------------------------------------------------------------------------------
// prepare: kx = sorted unique(ii U [t0,t1)), frame2k, CSR of edges by source frame (stable in edge order)
// ---------------------------------------------------------------------------------------------------------
// Exclusive prefix sum over i in [0, count) by the whole block, blockDim.x elements at a time: value(i) gives element i, and
// emit(i, v, before) receives it with the sum of the elements before it.  Every thread gets the total.  Ends with a __syncthreads().
template <class Value, class Emit>
__device__ __forceinline__ int block_exclusive_scan(int count, int* s_scan, Value value, Emit emit) {
  const int tid = threadIdx.x;
  int carry = 0;
  for (int base = 0; base < count; base += blockDim.x) {
    const int i = base + tid;
    const int v = (i < count) ? value(i) : 0;
    s_scan[tid] = v;
    __syncthreads();
    for (int off = 1; off < (int)blockDim.x; off <<= 1) {
      const int t = (tid >= off) ? s_scan[tid - off] : 0;
      __syncthreads();
      s_scan[tid] += t;
      __syncthreads();
    }
    if (i < count) emit(i, v, carry + s_scan[tid] - v);
    carry += s_scan[blockDim.x - 1];
    __syncthreads();                               // s_scan is rewritten by the next chunk
  }
  return carry;
}

__global__ void __launch_bounds__(1024) ba_prepare_kernel(const int64_t* __restrict__ ii, const int64_t* __restrict__ jj, int E, int N,
                                                          int t0, int t1, int eta_rows, int motion_only, int* __restrict__ hdr,
                                                          int* __restrict__ frame2k, int* __restrict__ kx, int* __restrict__ rowptr, SchurPlan plan,
                                                          int HW, float* __restrict__ Eij, float* __restrict__ C, float* __restrict__ w,
                                                          float* __restrict__ Ei) {
  __shared__ int s_scan[1024];
  const int tid = threadIdx.x;
  if (tid == 0) { hdr[HDR_STATUS] = 0; hdr[HDR_CHOL_FAIL] = 0; }
  // pad pixels [HW, pitch) of the per-pixel rows Eij [6E], C [N], w [N], Ei [6N]: the tensor-core Schur kernel reads them with the
  // last 16-byte piece of a row, so they must be finite, and nothing else writes them
  const int pitch = ba_pitch(HW);
  if (pitch != HW) {
    for (int r = tid; r < 6 * E + 8 * N; r += blockDim.x) {
      const int k = r - 6 * E;
      float* row = k < 0 ? Eij + (size_t)r * pitch : k < N ? C + (size_t)k * pitch : k < 2 * N ? w + (size_t)(k - N) * pitch
                 : Ei + (size_t)(k - 2 * N) * pitch;
      for (int p = HW; p < pitch; p++) row[p] = 0.f;
    }
  }
  for (int f = tid; f < N; f += blockDim.x) { frame2k[f] = (f >= t0 && f < t1) ? 1 : 0; rowptr[f] = 0; }
  if (tid == 0) { rowptr[N] = 0; rowptr[N + 1] = 0; }
  __syncthreads();
  for (int e = tid; e < E; e += blockDim.x) {
    const long long i = ii[e], j = jj[e];
    if (i < 0 || i >= N || j < 0 || j >= N) { atomicOr(&hdr[HDR_STATUS], ST_BAD_INDEX); continue; }
    frame2k[i] = 1;
  }
  __syncthreads();
  // exclusive scan of the presence flags -> dense index
  const int M = block_exclusive_scan(N, s_scan, [&](int f) { return frame2k[f]; }, [&](int f, int flag, int idx) {
    frame2k[f] = flag ? idx : -1;
    if (flag) kx[idx] = f;
  });
  if (tid == 0) {
    hdr[HDR_M] = M;
    if (eta_rows != M && eta_rows != 1) atomicOr(&hdr[HDR_STATUS], ST_ETA_ROWS);
  }
  // out-degree per depth frame -> rowptr
  for (int e = tid; e < E; e += blockDim.x) {
    const long long i = ii[e], j = jj[e];
    if (i < 0 || i >= N || j < 0 || j >= N) continue;
    atomicAdd(&rowptr[frame2k[i] + 1], 1);
  }
  __syncthreads();
  // rowptr[m] holds deg(m - 1) and rowptr[0] = 0, so the inclusive sum over [0, m] is the start of frame m's segment
  block_exclusive_scan(M + 1, s_scan, [&](int m) { return rowptr[m]; }, [&](int m, int cnt, int before) { rowptr[m] = before + cnt; });
  // the Schur kernels hold at most kSchurMaxRows rows per depth frame: flag a larger frame here, so that the caller can raise before
  // build and solve change any state (motion-only runs no Schur kernel and has no such limit)
  if (!motion_only)
    for (int m = tid; m < M; m += blockDim.x)
      if (rowptr[m + 1] - rowptr[m] > kSchurMaxRows - 1) atomicOr(&hdr[HDR_STATUS], ST_DEGREE);
  // the Schur plan: rows per depth frame, the prefix sum of the packed / single-tile costs, the pair-route frames and their tile pairs
  for (int m = tid; m < M; m += blockDim.x) plan.rows[m] = 0;
  __syncthreads();
  for (int e = tid; e < E; e += blockDim.x) {
    const long long i = ii[e], j = jj[e];
    if (i < 0 || i >= N || j < 0 || j >= N) continue;
    if (j >= t0 && j < t1) atomicAdd(&plan.rows[frame2k[i]], 1);
  }
  __syncthreads();
  for (int m = tid; m < M; m += blockDim.x)
    plan.rows[m] = rowptr[m + 1] > rowptr[m] ? plan.rows[m] + (kx[m] >= t0 && kx[m] < t1 ? 1 : 0) : 0;
  __syncthreads();
  const int total = block_exclusive_scan(M, s_scan, [&](int m) { return schur_cost(plan.rows[m], HW); },
                                         [&](int m, int, int before) { plan.cost[m] = before; });
  const int nbig = block_exclusive_scan(M, s_scan, [&](int m) { return plan.rows[m] > kTcRowsMax ? 1 : 0; },
                                        [&](int m, int flag, int idx) { if (flag) plan.big[idx] = m; });
  const int npair = block_exclusive_scan(nbig, s_scan, [&](int i) { return schur_pair_count(plan.rows[plan.big[i]]); },
                                         [&](int i, int, int before) { plan.pairs[i] = before; });
  if (tid == 0) { plan.cost[M] = total; hdr[HDR_NBIG] = nbig; hdr[HDR_NPAIR] = npair; }
}

// stable placement of every edge inside its source frame's segment: rank = #earlier edges with the same source.
// One warp per edge, lanes stride over the earlier edges (E^2/2 compares spread over E warps).
__global__ void __launch_bounds__(256) ba_fill_csr_kernel(const int64_t* __restrict__ ii, const int64_t* __restrict__ jj, int E, int N,
                                                          const int* __restrict__ frame2k, const int* __restrict__ rowptr,
                                                          int* __restrict__ edgeidx) {
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= E) return;
  const long long i = ii[e], j = jj[e];
  if (i < 0 || i >= N || j < 0 || j >= N) return;
  int rank = 0;
  for (int f = lane; f < e; f += 32) {
    const long long i2 = ii[f], j2 = jj[f];
    rank += (i2 == i && j2 >= 0 && j2 < N) ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) rank += __shfl_xor_sync(0xffffffffu, rank, o);
  if (lane == 0) edgeidx[rowptr[frame2k[i]] + rank] = e;
}

// ---------------------------------------------------------------------------------------------------------
// build: per (depth frame, pixel chunk): geometry of all out-edges, depth-block sums, per-edge pose blocks
// ---------------------------------------------------------------------------------------------------------
struct EdgeSm {
  float t[3], q[4];      // G_ij
  float A[36];           // Ji = -A Jj   (A = transposed adjoint, applied with the reference's adjSE3 arithmetic)
  int e, jx, stereo;
};

template <int kPPT>   // pixels per thread: 4 when many frames fill the GPU, fewer when a rank owns only a few source frames
__global__ void __launch_bounds__(kBuildThreads, 2) ba_build_kernel(
    const float* __restrict__ poses, const float* __restrict__ disps, const float* __restrict__ intr,
    const float* __restrict__ disps_sens, const float* __restrict__ targets, const float* __restrict__ weights,
    const float* __restrict__ eta, int eta_rows, int eta_by_frame, const int64_t* __restrict__ jj,
    const int* __restrict__ hdr, const int* __restrict__ kx, const int* __restrict__ rowptr, const int* __restrict__ edgeidx,
    int HW, int wd, int t0, int P, int motion_only,
    double* __restrict__ Hsys, double* __restrict__ bsys, float* __restrict__ Eij, float* __restrict__ Cout, float* __restrict__ wout,
    float* __restrict__ Eiout) {
  const int m = blockIdx.y;
  if (m >= hdr[HDR_M]) return;
  const int ix = kx[m];
  const int e_begin = rowptr[m], e_end = rowptr[m + 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = kBuildThreads / 32;

  __shared__ EdgeSm s_edge[kEdgeBatch];
  __shared__ float s_part[NW][kEdgeBatch][27];
  __shared__ double s_sum[kEdgeBatch][27];

  const float fx = __ldg(intr), fy = __ldg(intr + 1), cx = __ldg(intr + 2), cy = __ldg(intr + 3);
  const int n = 6 * P;
  const int pitch = ba_pitch(HW);

  // this thread's pixels
  int pix[kPPT];
  float Xi0[kPPT], Xi1[kPPT], dsp[kPPT];
  float Cacc[kPPT], wacc[kPPT], Eiacc[kPPT][6];
#pragma unroll
  for (int s = 0; s < kPPT; s++) {
    const int p = blockIdx.x * (kPPT * kBuildThreads) + s * kBuildThreads + tid;
    pix[s] = p;
    const bool ok = p < HW;
    const int i = ok ? p / wd : 0, j = ok ? p - i * wd : 0;
    Xi0[s] = ((float)j - cx) / fx;
    Xi1[s] = ((float)i - cy) / fy;
    dsp[s] = ok ? __ldg(disps + (size_t)ix * HW + p) : 1.f;
    Cacc[s] = 0.f; wacc[s] = 0.f;
#pragma unroll
    for (int c = 0; c < 6; c++) Eiacc[s][c] = 0.f;
  }

  for (int eb = e_begin; eb < e_end; eb += kEdgeBatch) {
    const int nb = min(kEdgeBatch, e_end - eb);
    __syncthreads();   // previous batch fully consumed
    // ---- edge transforms + adjoint matrices for the batch
    if (tid < nb) {
      EdgeSm& S = s_edge[tid];
      const int e = edgeidx[eb + tid];
      S.e = e; S.jx = (int)jj[e]; S.stereo = (S.jx == ix);
      edge_transform(poses, ix, S.jx, /*stereo_quirk=*/true, S.t, S.q);
    }
    __syncthreads();
    if (tid < nb * 6) {
      const int b = tid / 6, c = tid - b * 6;
      float X[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, Y[6];
      X[c] = 1.f;
      adj_se3(s_edge[b].t, s_edge[b].q, X, Y);
#pragma unroll
      for (int r = 0; r < 6; r++) s_edge[b].A[r * 6 + c] = Y[r];
    }
    __syncthreads();

    // software pipeline: the four target/weight loads of edge b+1 are in flight while edge b is computed
    float nw_u[kPPT], nw_v[kPPT], nt_u[kPPT], nt_v[kPPT];
    {
      const int e0 = s_edge[0].e;
#pragma unroll
      for (int s = 0; s < kPPT; s++) {
        const int p = pix[s];
        const bool okp = p < HW;
        nw_u[s] = okp ? __ldg(weights + ((size_t)e0 * 2 + 0) * HW + p) : 0.f;
        nw_v[s] = okp ? __ldg(weights + ((size_t)e0 * 2 + 1) * HW + p) : 0.f;
        nt_u[s] = okp ? __ldg(targets + ((size_t)e0 * 2 + 0) * HW + p) : 0.f;
        nt_v[s] = okp ? __ldg(targets + ((size_t)e0 * 2 + 1) * HW + p) : 0.f;
      }
    }
    for (int b = 0; b < nb; b++) {
      const EdgeSm& S = s_edge[b];
      const int e = S.e;
      float cw_u[kPPT], cw_v[kPPT], ct_u[kPPT], ct_v[kPPT];
#pragma unroll
      for (int s = 0; s < kPPT; s++) { cw_u[s] = nw_u[s]; cw_v[s] = nw_v[s]; ct_u[s] = nt_u[s]; ct_v[s] = nt_v[s]; }
      if (b + 1 < nb) {
        const int e1 = s_edge[b + 1].e;
#pragma unroll
        for (int s = 0; s < kPPT; s++) {
          const int p = pix[s];
          if (p < HW) {
            nw_u[s] = __ldg(weights + ((size_t)e1 * 2 + 0) * HW + p);
            nw_v[s] = __ldg(weights + ((size_t)e1 * 2 + 1) * HW + p);
            nt_u[s] = __ldg(targets + ((size_t)e1 * 2 + 0) * HW + p);
            nt_v[s] = __ldg(targets + ((size_t)e1 * 2 + 1) * HW + p);
          }
        }
      }
      const bool stereo = S.stereo != 0;
      float Hjj[21], vj[6];
#pragma unroll
      for (int k = 0; k < 21; k++) Hjj[k] = 0.f;
#pragma unroll
      for (int k = 0; k < 6; k++) vj[k] = 0.f;

#pragma unroll
      for (int s = 0; s < kPPT; s++) {
        const int p = pix[s];
        if (p < HW) {
          PixelTerms P;
          ba_pixel_terms(S.t, S.q, Xi0[s], Xi1[s], dsp[s], cw_u[s], cw_v[s], ct_u[s], ct_v[s], fx, fy, cx, cy, P);
          Cacc[s] += P.wu * P.Jzu * P.Jzu + P.wv * P.Jzv * P.Jzv;
          wacc[s] += P.wu * P.ru * P.Jzu + P.wv * P.rv * P.Jzv;
          if (stereo) { P.wu = 0.f; P.wv = 0.f; }   // pose weights vanish AFTER the depth terms (Q1)
          const float au = P.wu * P.Jzu, av = P.wv * P.Jzv;
          float Ej[6];
#pragma unroll
          for (int c = 0; c < 6; c++) Ej[c] = au * P.Ju[c] + av * P.Jv[c];
          if (!motion_only) {
#pragma unroll
            for (int c = 0; c < 6; c++) Eij[((size_t)e * 6 + c) * pitch + p] = Ej[c];
            // Eii = -A Eij, accumulated over the out-edges of this frame
#pragma unroll
            for (int r = 0; r < 6; r++) {
              float acc = 0.f;
#pragma unroll
              for (int c = 0; c < 6; c++) acc += S.A[r * 6 + c] * Ej[c];
              Eiacc[s][r] -= acc;
            }
          }
          ba_pose_accum(P, Hjj, vj);
        }
      }
      // warp reduction of the 27 sums (padded to 32): transpose-reduction, 31 shuffles; lane k ends with the total of value k
      {
        float v32[32];
#pragma unroll
        for (int k = 0; k < 21; k++) v32[k] = Hjj[k];
#pragma unroll
        for (int k = 0; k < 6; k++) v32[21 + k] = vj[k];
#pragma unroll
        for (int k = 27; k < 32; k++) v32[k] = 0.f;
        const float tot = transpose_reduce32(v32, lane);
        if (lane < 27) s_part[warp][b][lane] = tot;
      }
    }
    __syncthreads();
    // ---- cross-warp sums in fp64
    for (int k = tid; k < nb * 27; k += kBuildThreads) {
      const int b = k / 27, c = k - b * 27;
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < NW; w++) s += (double)s_part[w][b][c];
      s_sum[b][c] = s;
    }
    __syncthreads();
    // ---- per edge: Hii = A Hjj A^T, Hij = -A Hjj, Hji = Hij^T, vi = -A vj ; scatter into the reduced system
    // 156 outputs per edge: 144 matrix entries (4 blocks x 36) + 12 vector entries
    for (int k = tid; k < nb * 156; k += kBuildThreads) {
      const int b = k / 156, o = k - b * 156;
      const EdgeSm& S = s_edge[b];
      if (S.stereo) continue;                           // all-zero blocks
      const int pi = ix - t0, pj = S.jx - t0;
      const double* hs = s_sum[b];
      auto H = [&](int a, int c) -> double { return (a >= c) ? hs[a * (a + 1) / 2 + c] : hs[c * (c + 1) / 2 + a]; };
      if (o < 144) {
        const int blk = o / 36, rc = o - blk * 36, r = rc / 6, c = rc - r * 6;
        int prow, pcol; double val = 0.0;
        if (blk == 0) {          // Hii[r][c] = sum_ab A[r][a] Hjj[a][b] A[c][b]
          prow = pi; pcol = pi;
          for (int a = 0; a < 6; a++) { double t = 0.0; for (int b2 = 0; b2 < 6; b2++) t += H(a, b2) * (double)S.A[c * 6 + b2]; val += (double)S.A[r * 6 + a] * t; }
        } else if (blk == 1) {   // Hij[r][c] = -sum_a A[r][a] Hjj[a][c]
          prow = pi; pcol = pj;
          for (int a = 0; a < 6; a++) val -= (double)S.A[r * 6 + a] * H(a, c);
        } else if (blk == 2) {   // Hji[r][c] = Hij[c][r]
          prow = pj; pcol = pi;
          for (int a = 0; a < 6; a++) val -= (double)S.A[c * 6 + a] * H(a, r);
        } else {
          prow = pj; pcol = pj; val = H(r, c);
        }
        if (prow >= 0 && prow < P && pcol >= 0 && pcol < P) atomicAdd(&Hsys[(size_t)(prow * 6 + r) * n + pcol * 6 + c], val);
      } else {
        const int v = o - 144, blk = v / 6, r = v - blk * 6;
        double val = 0.0; int prow;
        if (blk == 0) { prow = pi; for (int a = 0; a < 6; a++) val -= (double)S.A[r * 6 + a] * hs[21 + a]; }
        else { prow = pj; val = hs[21 + r]; }
        if (prow >= 0 && prow < P) atomicAdd(&bsys[prow * 6 + r], val);
      }
    }
  }

  if (!motion_only) {
    // depth block:  C = sum Cii + m*alpha + (1-m)*eta ;  w = sum bz - m*alpha*(d - d_sens)   (reference :1405-1408)
    const float alpha = 0.05f;
    const int erow = (eta_rows == 1) ? 0 : min(eta_by_frame ? ix : m, eta_rows - 1);
#pragma unroll
    for (int s = 0; s < kPPT; s++) {
      const int p = pix[s];
      if (p < HW) {
        const float dsn = __ldg(disps_sens + (size_t)ix * HW + p);
        const float mk = (dsn > 0.f) ? 1.f : 0.f;
        const float C = Cacc[s] + mk * alpha + (1 - mk) * __ldg(eta + (size_t)erow * HW + p);
        const float w = wacc[s] - mk * alpha * (dsp[s] - dsn);
        Cout[(size_t)m * pitch + p] = C;
        wout[(size_t)m * pitch + p] = w;
#pragma unroll
        for (int c = 0; c < 6; c++) Eiout[((size_t)m * 6 + c) * pitch + p] = Eiacc[s][c];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Schur complement:  Hsys -= sum_k E_k Q_k E_k^T ,  bsys -= sum_k E_k Q_k w_k       (reference K9/K10 + schur_block)
// rows of frame k: (pose k, Ei_k) if k is in [t0,t1), then (pose jj[e], Eij[e]) for the out-edges e of k; rows whose pose
// is outside [t0,t1) are dropped (they contribute nothing, reference :1155,:1257).
// The rows of a frame decide its route, for every image size (the workspace rows are padded to ba_pitch, i.e. 16-byte aligned):
//   <= kPackedRowsMax rows (every frame of a sliding-window graph)   packed: two 32-pixel halves per 64-pixel chunk
//   <= kTcRowsMax rows                                               single: one row tile per 32-pixel chunk
//   kTcRowsMax+1 .. kSchurMaxRows rows (dense graphs, sharded)       pair:   pairs of row tiles over the whole pixel range
// All three run in one launch (ba_schur_tc_kernel) and flush once per pass with fp64 atomics into the LOWER triangle of the reduced
// system.
// ---------------------------------------------------------------------------------------------------------
enum SchurRoute { kPacked = 0, kSingle = 1, kPair = 2 };
constexpr int kTcThreads = 256;
// Q = 1/C of the eliminated depth block.  C <= 0 only for a pixel with eta = 0 and no weight on any edge; the reference divides
// anyway (inf -> NaN system -> zero pose update and NaN depths at that pixel).  The Schur kernel and the back-substitution here
// drop such a pixel instead (Q = 0, dz = 0): one rule on every path, documented in INTEGRATION.md.
__device__ __forceinline__ float safe_rcp(float c) { return c > 0.f ? 1.0f / c : 0.f; }

// Row list of a depth frame: (pose ix, Ei) first when ix is inside the window, then (pose jj[e], Eij[e]) for its out-edges in CSR
// order whose target pose is inside the window.  Built by the whole CTA: thread a handles out-edge a, an order-preserving
// ballot compaction keeps the reference's row order.  Ends with a __syncthreads().
__device__ __forceinline__ void build_row_list(const int64_t* __restrict__ jj, int* __restrict__ hdr, const int* __restrict__ edgeidx,
                                               int e_begin, int deg, int ix, int m, int pitch, int t0, int P, const float* __restrict__ Eij,
                                               const float* __restrict__ Eiin, int* s_pose, const float** s_ptr, int* s_nrows, int* s_wcount) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool self = (ix >= t0 && ix < t0 + P);
  int pj = -1, e = -1;
  if (tid < deg && tid < kSchurMaxRows - 1) { e = edgeidx[e_begin + tid]; pj = (int)jj[e] - t0; }
  const bool keep = (pj >= 0 && pj < P);
  const unsigned bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) s_wcount[warp] = __popc(bal);
  __syncthreads();
  int base = self ? 1 : 0;
  for (int w = 0; w < warp; w++) base += s_wcount[w];
  if (keep) {
    const int pos = base + __popc(bal & ((1u << lane) - 1u));
    s_pose[pos] = pj; s_ptr[pos] = Eij + (size_t)e * 6 * pitch;
  }
  if (tid == 0) {
    if (self) { s_pose[0] = ix - t0; s_ptr[0] = Eiin + (size_t)m * 6 * pitch; }
    int tot = self ? 1 : 0;
    for (int w = 0; w < kTcThreads / 32; w++) tot += s_wcount[w];
    *s_nrows = tot;
    if (deg > kSchurMaxRows - 1) atomicOr(&hdr[HDR_STATUS], ST_DEGREE);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------
// Schur complement on the tensor cores (packed and single routes; PAIR mode below: up to kSchurMaxRows rows):
//   S = X X^T  with  X = [ E_r / sqrt(C) ; w / sqrt(C) ]  (6R + 1 rows x pixels),  so that S[:6R,:6R] = sum E q E^T and
//   S[:6R, 6R] = sum E q w  -- one symmetric rank-K update per frame, K = pixels.
// fp32 accuracy on the tf32 pipe by operand splitting (3xTF32): x = hi + lo with hi = tf32(x), lo = x - hi (exact), and
//   S = hi hi^T + G + G^T,  G = hi lo^T   (the dropped lo lo^T term is ~2^-22 relative),
// i.e. TWO wgmma per 8-pixel K step: G is accumulated once and symmetrised in the epilogue.
// The tensor core truncates every addend to the accumulator's exponent, so a long accumulation chain drifts (one accumulator over
// the whole pixel range -> 1e-4 on the depths).  hi hi^T therefore gets a fresh register accumulator per chunk which is added into
// an fp32 running sum when the next chunk's MMAs are issued; G is 2^-11 smaller and keeps one accumulator for the whole range.
// A pass = (frame, pixel range), 256 threads = two warpgroups.  Every warp cp.asyncs its own raw rows of a chunk into a 4-deep
// warp-private raw ring and splits them into the two K-major SWIZZLE_128B operand tiles [128 rows x 32 px] of a 4-deep operand
// ring (generic-proxy stores + fence.proxy.async); after a CTA barrier warpgroup w issues the chunk's MMAs for operand rows
// 64 w .. 64 w + 63 (both operands described from the SAME tile) and splits the next chunk while they run.  Finally G goes through
// shared memory and the lower triangle is added into the reduced system with fp64 atomics.
//   single, PAIR: wgmma.m64n128k8 against all 128 operand rows (PAIR: the rows of tile a and tile b).
//   packed (6R + 2 <= 64, R <= kPackedRowsMax): the two 32-pixel halves of a 64-pixel chunk sit in operand rows 0..63 and 64..127 with
//   the same lines, and warpgroup w needs only its own half's product: wgmma.m64n64k8 of rows 64 w .. 64 w + 63 against themselves.
// The copies move whole 16-byte pieces, so the last piece of a row also carries the pad pixels [HW, pitch).  They are zero in E, w
// and C, and rsqrt(C) is taken as 0 there, so they add nothing.
// ---------------------------------------------------------------------------------------------------------
constexpr int kTcRawStages = 4;
constexpr int kTcRawBytes = 128 * 128;          // up to 128 lines (6R rows, w, C; two halves when packed) x 128 bytes
constexpr int kTcOpBytes = 128 * 128;           // one operand tile (hi or lo)
constexpr int kTcOpStages = 4;
constexpr int kTcCxStride = 129;                // floats per row of the G staging matrix (conflict-free transposed reads)
constexpr int kTcSmem = kTcRawStages * kTcRawBytes + kTcOpStages * 2 * kTcOpBytes + 1024 /*alignment*/ + 256 /*barriers*/;
static_assert(128 * kTcCxStride * 4 <= kTcOpStages * 2 * kTcOpBytes, "G staging matrix must fit the operand ring");

__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }

// One pass of the Schur complement over pixels [px_begin, px_end) of depth frame m (rows in s_pose / s_ptr): the whole frame, or in
// PAIR mode the row tiles ta < tb, whose diagonal blocks S_aa / S_bb are added only where emit_a / emit_b.  A caller that runs
// another pass must put a CTA barrier in between: the epilogue reads s_gidx and the operand ring, which the next pass rewrites.
// lane and warp come from the caller, which in PAIR mode makes warp opaque per pass (see the pair loop).
template <int MODE>
__device__ __forceinline__ void schur_tc_pass(int lane, int warp, int m, int nrows, int ta, int tb, bool emit_a, bool emit_b,
                                              int px_begin, int px_end, int pitch, int n, const float* __restrict__ Cin,
                                              const float* __restrict__ win, double* __restrict__ Hsys, double* __restrict__ bsys,
                                              const int* s_pose, const float* const* s_ptr, int* s_gidx) {
  constexpr bool PAIR = MODE == kPair;
  constexpr bool packed = MODE == kPacked;               // two PIXEL halves of a 64-pixel chunk in operand rows 0..63 / 64..127 (R6 + 2 <= 64)
  constexpr int NC = packed ? 64 : 128;                  // columns of a warpgroup's products
  const int tid = threadIdx.x;
  extern __shared__ uint8_t tc_smem_raw[];
  const int R6a = PAIR ? 6 * min(kPairTileRows, nrows - kPairTileRows * ta) : 6 * nrows;
  const int R6b = PAIR ? 6 * min(kPairTileRows, nrows - kPairTileRows * tb) : 6 * nrows;
  const int R6 = R6a;                                    // operand rows 0..R6-1: E rows, row R6: w  (PAIR: of tile a, R6b of tile b)
  constexpr bool two_halves = PAIR || packed;                // operand rows 64..127 carry a second set of lines
  constexpr int nhalf = packed ? 2 : 1;
  const int cpx = 32 * nhalf;                            // pixels per chunk
  const int nchunks = (px_end - px_begin + cpx - 1) / cpx;

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t op_base = smem_u32(smem);               // [stage][hi|lo][128 rows][128 B], 1024-byte aligned tiles
  const uint32_t raw_base = op_base + kTcOpStages * 2 * kTcOpBytes;   // [stage][row][128 B]

  if (tid < 128) {
    if (PAIR) {                                          // operand row -> index in the reduced system, per half
      const int hfx = tid >> 6, ln = tid & 63, R6x = hfx ? R6b : R6a, row0 = kPairTileRows * (hfx ? tb : ta);
      s_gidx[tid] = (ln < R6x) ? s_pose[row0 + ln / 6] * 6 + (ln % 6) : (ln == R6x ? -1 : -2);
    } else s_gidx[tid] = (tid < R6) ? s_pose[tid / 6] * 6 + (tid % 6) : (tid == R6 ? -1 : -2);
  }
  {
    // operand tiles start each pass as zeros (the previous pass's G staging overwrote them): rows that carry no line are never written
    uint4* z = reinterpret_cast<uint4*>(smem);
    for (int k = tid; k < kTcOpStages * 2 * kTcOpBytes / 16; k += kTcThreads) z[k] = make_uint4(0u, 0u, 0u, 0u);
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  // ================= raw rows -> split operands =================
  // Every warp stages and splits its OWN lines (line = warp + 8 i); the operand stage is shared by both warpgroups' MMAs.
  // Warp-private raw slab: 16 rows x 128 B per stage; slab row li = i (not packed) or hf * 8 + i (packed: half hf of the chunk).
  // A thread owns four (slab row, 16-byte piece) copy slots: li = 4 s + lane / 8, piece = lane % 8.
  const float* src[4];
  uint32_t dst[4];
  int pxo[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int li = 4 * i + (lane >> 3), piece = lane & 7;
    const int hf = two_halves ? (li >> 3) : 0, line = warp + 8 * (two_halves ? (li & 7) : li);
    const int R6x = PAIR ? (hf ? R6b : R6a) : R6, row0 = PAIR ? kPairTileRows * (hf ? tb : ta) : 0;
    // slots without a line copy zero bytes (cp.async zero-fills) into their unused slab row: no branch in the copy loop
    src[i] = Cin; pxo[i] = 1 << 30;
    dst[i] = raw_base + warp * 2048 + li * 128 + piece * 16;
    if (line <= R6x) {
      const float* base = (line < R6x) ? s_ptr[row0 + line / 6] + (size_t)(line % 6) * pitch : win + (size_t)m * pitch;
      pxo[i] = (packed ? hf * 32 : 0) + piece * 4;
      src[i] = base + pxo[i];
    }
  }
  const float* Cm = Cin + (size_t)m * pitch;
  auto issue = [&](int c) {
    if (c < nchunks) {
      const int p0 = px_begin + c * cpx;
      const uint32_t stage_off = (uint32_t)(c % kTcRawStages) * kTcRawBytes;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const bool ok = p0 + pxo[i] < px_end;            // false for slots without a line (pxo = 2^30)
        cp_async16_zfill(dst[i] + stage_off, ok ? (const void*)(src[i] + p0) : (const void*)Cin, ok ? 16u : 0u);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
#pragma unroll
  for (int s = 0; s < kTcRawStages - 1; s++) issue(s);

  // A thread splits exactly the 16-byte pieces it copied (slot i: slab row 4 i + lane / 8, pixels 4 (lane % 8) .. + 3): one
  // 128-bit shared load, four scale / round / subtract chains, two 128-bit swizzled stores per slot.  A 16-byte piece stays
  // contiguous under the 128-byte swizzle (chunk index ^ row % 8).
  const int piece = lane & 7;
  uint32_t op_off[4];                                      // byte offset of the slot's piece inside an operand tile
  bool live[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int li = 4 * i + (lane >> 3);
    const int hf = two_halves ? (li >> 3) : 0, line = warp + 8 * (two_halves ? (li & 7) : li);
    const uint32_t rr = (uint32_t)(hf * 64 + line);
    live[i] = line <= (PAIR ? (hf ? R6b : R6a) : R6);
    op_off[i] = rr * 128 + (((uint32_t)piece ^ (rr & 7u)) << 4);
  }
  auto load_c4 = [&](int c, int hf) -> float4 {          // C of this thread's four pixels in half hf of chunk c (0 beyond the range)
    const int px = px_begin + c * cpx + hf * 32 + 4 * piece;
    return (c < nchunks && px < px_end) ? __ldg(reinterpret_cast<const float4*>(Cm + px)) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  auto rsq4 = [](float4 v) -> float4 {                     // sqrt(Q); pixels beyond the range stay zero
    return make_float4(v.x > 0.f ? rsqrtf(v.x) : 0.f, v.y > 0.f ? rsqrtf(v.y) : 0.f, v.z > 0.f ? rsqrtf(v.z) : 0.f, v.w > 0.f ? rsqrtf(v.w) : 0.f);
  };
  float4 Cn0 = load_c4(0, 0), Cn1 = packed ? load_c4(0, 1) : make_float4(0.f, 0.f, 0.f, 0.f);
  const int wg = warp >> 2;
  float acc[NC / 2], D[NC / 2], G[NC / 2];                  // running hi hi^T, this chunk's hi hi^T, hi lo^T (m64nNC fragments)
#pragma unroll
  for (int j = 0; j < NC / 2; j++) acc[j] = 0.f;
  // Operand stage c % 4 is rewritten at chunk c: the MMAs of chunk c - 4 that read it are complete, because each warpgroup waits
  // for its chunk c - 2 before issuing chunk c - 1, and both passed the CTA barrier of chunk c - 1.
  for (int c = 0; c < nchunks; c++) {
    asm volatile("cp.async.wait_group %0;" ::"n"(kTcRawStages - 2) : "memory");
    __syncwarp();                                          // this warp's copies of chunk c have landed
    const int os = c % kTcOpStages;
    const uint32_t raw = raw_base + (uint32_t)(c % kTcRawStages) * kTcRawBytes + (uint32_t)warp * 2048 + (uint32_t)(lane >> 3) * 128 +
                         (uint32_t)piece * 16;
    const uint32_t ophi = op_base + (uint32_t)os * 2 * kTcOpBytes;
    const float4 sq0 = rsq4(Cn0), sq1 = rsq4(Cn1);
    Cn0 = load_c4(c + 1, 0); Cn1 = packed ? load_c4(c + 1, 1) : Cn1;      // one chunk ahead
    float4 xv[4];
#pragma unroll
    for (int i = 0; i < 4; i++)
      asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(xv[i].x), "=f"(xv[i].y), "=f"(xv[i].z), "=f"(xv[i].w) : "r"(raw + (uint32_t)i * 512) : "memory");
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float4 q = (packed && i >= 2) ? sq1 : sq0;
      const float x[4] = {xv[i].x * q.x, xv[i].y * q.y, xv[i].z * q.z, xv[i].w * q.w};
      float hi[4], lo[4];
#pragma unroll
      for (int k = 0; k < 4; k++) {                        // tf32 round-to-nearest (ties away), as cvt.rna.tf32.f32 for finite x
        hi[k] = __uint_as_float((__float_as_uint(x[k]) + 0x1000u) & 0xffffe000u);
        lo[k] = x[k] - hi[k];
      }
      if (live[i]) {
        asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(ophi + op_off[i]), "f"(hi[0]), "f"(hi[1]), "f"(hi[2]), "f"(hi[3]) : "memory");
        asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(ophi + kTcOpBytes + op_off[i]), "f"(lo[0]), "f"(lo[1]), "f"(lo[2]), "f"(lo[3]) : "memory");
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");         // generic-proxy stores -> visible to the tensor core
    __syncthreads();
    if (c > 0) {                                                         // chunk c - 1's hi hi^T into the running sum
      wgmma_wait<0>();
      wgmma_fence_regs(D);
#pragma unroll
      for (int j = 0; j < NC / 2; j++) acc[j] += D[j];
    }
    wgmma_fence();
    {
      const uint32_t hi0 = ophi, lo0 = ophi + kTcOpBytes;
      const uint32_t b0 = packed ? wg * 64 * 128 : 0;                    // first operand row of the B side
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const uint64_t da = gmma_desc_sw128(hi0 + wg * 64 * 128 + k * 32, 16, 1024);
        const uint64_t dbh = gmma_desc_sw128(hi0 + b0 + k * 32, 16, 1024), dbl = gmma_desc_sw128(lo0 + b0 + k * 32, 16, 1024);
        if constexpr (packed) {
          wgmma_tf32_n64(D, da, dbh, k > 0 ? 1 : 0);
          wgmma_tf32_n64(G, da, dbl, (c > 0 || k > 0) ? 1 : 0);
        } else {
          wgmma_tf32_n128(D, da, dbh, k > 0 ? 1 : 0);
          wgmma_tf32_n128(G, da, dbl, (c > 0 || k > 0) ? 1 : 0);
        }
      }
    }
    wgmma_commit();
    issue(c + kTcRawStages - 1);
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  wgmma_wait<0>();
  wgmma_fence_regs(D);
  wgmma_fence_regs(G);
#pragma unroll
  for (int j = 0; j < NC / 2; j++) acc[j] += D[j];

  // ================= G = hi lo^T: through shared memory (the operand ring is idle now) so that G + G^T can be formed
  __syncthreads();                                         // both warpgroups' MMAs have completed: the ring may be overwritten
  // staged as [operand row][local column]: G of operand rows (r, c) is at [r][c - cb0], cb0 the operand row of local column 0
  const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2), c_base = 2 * (lane & 3), cb0 = packed ? wg * 64 : 0;
#pragma unroll
  for (int j = 0; j < NC / 8; j++)
#pragma unroll
    for (int e = 0; e < 4; e++)
      sts_f32(op_base + (uint32_t)((r_base + 8 * (e >> 1)) * kTcCxStride + 8 * j + c_base + (e & 1)) * 4, G[4 * j + e]);
  __syncthreads();

  // ================= epilogue: lower triangle of S (and the rhs column) into the reduced system =================
#pragma unroll
  for (int ih = 0; ih < 2; ih++) {
    const int row = r_base + 8 * ih;
    const int lrow = row - cb0;                                        // line of this row (packed), operand row otherwise
    const int gr = PAIR ? s_gidx[row] : ((lrow < R6) ? s_gidx[lrow] : -2);
    if (gr < 0) continue;
    const bool rb = row >= 64;
#pragma unroll
    for (int j = 0; j < NC / 8; j++) {
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int col = 8 * j + c_base + e;
        const bool cbk = col >= 64;
        if (PAIR) {          // rows of tile a need S_aa (if this pass emits it); rows of tile b need S_ba and S_bb (if emitted)
          if (!rb && (cbk || !emit_a)) continue;
          if (rb && cbk && !emit_b) continue;
        }
        const int gc = s_gidx[col];                                    // packed: local columns are the lines of this row's half
        if (gc == -2) continue;
        const float g = lds_f32(op_base + (uint32_t)(row * kTcCxStride + col) * 4) + lds_f32(op_base + (uint32_t)((cb0 + col) * kTcCxStride + lrow) * 4);
        const double v = -(double)(acc[4 * j + 2 * ih + e] + g);
        if (PAIR && rb != cbk) {                                     // lower-left block S_ba: every unordered row pair appears once
          if (gc < 0) continue;                                      // the rhs comes from the diagonal blocks
          if (gr > gc) atomicAdd(&Hsys[(size_t)gr * n + gc], v);
          else if (gr < gc) atomicAdd(&Hsys[(size_t)gc * n + gr], v);
          else atomicAdd(&Hsys[(size_t)gr * n + gr], 2.0 * v);       // two different rows with the same pose: (r,c) and (c,r) land on one entry
        } else if (gc >= 0) {
          if (gr >= gc) atomicAdd(&Hsys[(size_t)gr * n + gc], v);
        } else {
          atomicAdd(&bsys[gr], v);
        }
      }
    }
  }
}

// The passes of one route (packed or single) over the frames m0.. whose chunks start in the cost interval [lo, hi).  Each frame part
// gets its own row list and pass.
template <int MODE>
__device__ __forceinline__ void schur_sweep(int m0, int M, int lo, int hi, const SchurPlan& plan, const int64_t* __restrict__ jj,
                                            int* __restrict__ hdr, const int* __restrict__ kx, const int* __restrict__ rowptr,
                                            const int* __restrict__ edgeidx, int HW, int t0, int P, const float* __restrict__ Eij,
                                            const float* __restrict__ Cin, const float* __restrict__ win, const float* __restrict__ Eiin,
                                            double* __restrict__ Hsys, double* __restrict__ bsys, int* s_pose, const float** s_ptr,
                                            int* s_nrows, int* s_wcount, int* s_gidx) {
  constexpr int w = MODE == kPacked ? 1 : 2, cpx = 64 / w;        // cost and pixels of one chunk (schur_cost)
  const int pitch = ba_pitch(HW);
  for (int m = m0; m < M && plan.cost[m] < hi; m++) {
    const int off = plan.cost[m], cost = plan.cost[m + 1] - off;
    if (cost == 0 || (plan.rows[m] <= kPackedRowsMax) != (MODE == kPacked)) continue;
    const int c_begin = lo > off ? (lo - off + w - 1) / w : 0;
    const int c_end = min(cost / w, (hi - off + w - 1) / w);
    if (c_begin >= c_end) continue;
    const int e_begin = rowptr[m];
    build_row_list(jj, hdr, edgeidx, e_begin, rowptr[m + 1] - e_begin, kx[m], m, pitch, t0, P, Eij, Eiin, s_pose, s_ptr, s_nrows, s_wcount);
    const int nrows = *s_nrows;
    if (nrows == 0 || nrows > (MODE == kPacked ? kPackedRowsMax : kTcRowsMax)) continue;
    // lane and warp made opaque per pass: the copy slots and swizzled offsets derived from them are then computed inside the pass.
    // Hoisted out of it, they would stay live across every pass and the kernel would spill.
    int lane_p = threadIdx.x & 31, warp_p = threadIdx.x >> 5;
    asm volatile("" : "+r"(lane_p), "+r"(warp_p));
    schur_tc_pass<MODE>(lane_p, warp_p, m, nrows, 0, 0, true, true, c_begin * cpx, min(HW, c_end * cpx), pitch, 6 * P, Cin, win, Hsys, bsys,
                        s_pose, s_ptr, s_gidx);
    __syncthreads();                              // the next pass rewrites the row list, s_gidx and the operand ring
  }
}

// PAIR mode (frames with 22..kSchurMaxRows rows: dense graphs, edge-sharded ranks): the rows are cut into T <= 26 tiles of 10, and a pass
// stacks tile a in operand rows 0..63 and tile b in rows 64..127 over the SAME 32 pixels (the packed layout with a zero pixel offset
// for the second half), so the one M = N = 128 product holds S_ba in its lower-left block and S_aa / S_bb on the diagonal (emitted
// only by the designated pair (t, t+1)); G + G^T symmetrisation unchanged.  Off-diagonal-block entries go to (max, min) of the global
// indices and count twice where two different rows share a pose.  A pass covers one tile pair over the whole pixel range.
//
// One persistent launch of one CTA per SM does every route (one CTA fits an SM: 255 registers x 256 threads, ~194 KB of shared
// memory).  The plan of ba_prepare_kernel (SchurPlan) orders the packed and single-tile work as one cost line, frame after frame;
// CTA b takes the chunks that START in [b T / grid, (b + 1) T / grid) of its total T, which may be parts of several frames, and runs
// one pass per frame part.  The tile pairs of the pair-route frames are one flat list of items after that, taken round-robin.
// The plan's row counts pick each frame's route; the row list a pass builds counts the same rows (fewer only for a frame with more
// than kSchurMaxRows - 1 out-edges, which raises ST_DEGREE), and the single-tile pass takes any count up to kTcRowsMax.
__global__ void __launch_bounds__(kTcThreads, 1) ba_schur_tc_kernel(
    const int64_t* __restrict__ jj, int* __restrict__ hdr, const int* __restrict__ kx, const int* __restrict__ rowptr,
    const int* __restrict__ edgeidx, int HW, int t0, int P, const float* __restrict__ Eij, const float* __restrict__ Cin,
    const float* __restrict__ win, const float* __restrict__ Eiin, double* __restrict__ Hsys, double* __restrict__ bsys, SchurPlan plan) {
  const int M = hdr[HDR_M];
  const int pitch = ba_pitch(HW);

  __shared__ int s_pose[kSchurMaxRows + 1];
  __shared__ const float* s_ptr[kSchurMaxRows + 1];
  __shared__ int s_nrows;
  __shared__ int s_wcount[kTcThreads / 32];
  __shared__ int s_gidx[128];                     // operand row / column -> index in the reduced system (-1: rhs, -2: padding)

  // ---- packed and single-tile routes: this CTA's interval [lo, hi) of the cost line, one sweep per route (a sweep that runs both
  // routes' passes would spill)
  const long long total = plan.cost[M];
  const int lo = (int)((long long)blockIdx.x * total / gridDim.x), hi = (int)((long long)(blockIdx.x + 1) * total / gridDim.x);
  if (lo < hi) {
    int m0 = 0;                                   // the first frame whose cost interval ends after lo
    for (int top = M - 1; m0 < top;) {
      const int mid = (m0 + top) >> 1;
      if (plan.cost[mid + 1] > lo) top = mid; else m0 = mid + 1;
    }
    schur_sweep<kPacked>(m0, M, lo, hi, plan, jj, hdr, kx, rowptr, edgeidx, HW, t0, P, Eij, Cin, win, Eiin, Hsys, bsys, s_pose, s_ptr,
                         &s_nrows, s_wcount, s_gidx);
    schur_sweep<kSingle>(m0, M, lo, hi, plan, jj, hdr, kx, rowptr, edgeidx, HW, t0, P, Eij, Cin, win, Eiin, Hsys, bsys, s_pose, s_ptr,
                         &s_nrows, s_wcount, s_gidx);
  }

  // ---- pair route: items (frame big[i], tile pair pr) numbered from plan.pairs[i]
  const int nbig = hdr[HDR_NBIG], npair = hdr[HDR_NPAIR];
  int listed = -1;                                // the frame whose rows are in s_pose / s_ptr
  for (int item = blockIdx.x; item < npair; item += gridDim.x) {
    int i = 0;                                    // the last big frame whose items start at or before this one
    for (int top = nbig - 1; i < top;) {
      const int mid = (i + top + 1) >> 1;
      if (plan.pairs[mid] <= item) i = mid; else top = mid - 1;
    }
    const int m = plan.big[i], pr = item - plan.pairs[i];
    if (m != listed) {
      const int e_begin = rowptr[m];
      build_row_list(jj, hdr, edgeidx, e_begin, rowptr[m + 1] - e_begin, kx[m], m, pitch, t0, P, Eij, Eiin, s_pose, s_ptr, &s_nrows, s_wcount);
      listed = m;
    }
    const int nrows = s_nrows;
    const int T = (nrows + kPairTileRows - 1) / kPairTileRows;         // 3 .. 26
    if (nrows <= kTcRowsMax || pr >= T * (T - 1) / 2) continue;
    int tb = (int)((sqrtf(8.f * (float)pr + 1.f) + 1.f) * 0.5f);       // the two row tiles of this pass (ta < tb)
    while (tb * (tb - 1) / 2 > pr) tb--;
    while ((tb + 1) * tb / 2 <= pr) tb++;
    const int ta = pr - tb * (tb - 1) / 2;
    int lane_p = threadIdx.x & 31, warp_p = threadIdx.x >> 5;
    asm volatile("" : "+r"(lane_p), "+r"(warp_p));
    // S_tt of tile t < T-1 comes from pair (t, t+1), of tile T-1 from pair (T-2, T-1)
    schur_tc_pass<kPair>(lane_p, warp_p, m, nrows, ta, tb, tb == ta + 1, tb == T - 1 && ta == T - 2, 0, HW, pitch, 6 * P, Cin,
                         win, Hsys, bsys, s_pose, s_ptr, s_gidx);
    __syncthreads();                              // the next pass rewrites s_gidx and the operand ring
  }
}

// ---------------------------------------------------------------------------------------------------------
// back substitution + retractions
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ba_backsub_kernel(
    const int64_t* __restrict__ jj, const int* __restrict__ hdr, const int* __restrict__ kx, const int* __restrict__ rowptr,
    const int* __restrict__ edgeidx, int HW, int t0, int P,
    const float* __restrict__ Eij, const float* __restrict__ Cin, const float* __restrict__ win, const float* __restrict__ Eiin,
    const float* __restrict__ dx, float* __restrict__ disps, float* __restrict__ dz_out, int own_lo, int own_hi) {
  const int m = blockIdx.y;
  if (m >= hdr[HDR_M]) return;
  const int ix = kx[m];
  const bool owned = ix >= own_lo && ix < own_hi;   // edge-sharded runs: other ranks hold the out-edges of the other frames
  const int e_begin = rowptr[m], e_end = rowptr[m + 1];
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const int pitch = ba_pitch(HW);
  // dw = sum over rows of frame m of  E[row,:,p] . dx[pose]   with the Q9 guard 0 < pose < P   (reference :1114)
  float dw = 0.f;
  {
    const int ps = ix - t0;
    if (ps > 0 && ps < P) {
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < 6; c++) s += __ldg(Eiin + ((size_t)m * 6 + c) * pitch + p) * __ldg(dx + ps * 6 + c);
      dw += s;
    }
  }
  for (int a = e_begin; a < e_end; a++) {
    const int e = edgeidx[a];
    const int pj = (int)jj[e] - t0;
    if (pj > 0 && pj < P) {
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < 6; c++) s += __ldg(Eij + ((size_t)e * 6 + c) * pitch + p) * __ldg(dx + pj * 6 + c);
      dw += s;
    }
  }
  const float q = safe_rcp(__ldg(Cin + (size_t)m * pitch + p));
  const float dz = q * (__ldg(win + (size_t)m * pitch + p) - dw);
  dz_out[(size_t)m * HW + p] = owned ? dz : 0.f;
  if (owned) disps[(size_t)ix * HW + p] += dz;       // K8 (:942-955)
}

__global__ void ba_pose_retr_kernel(float* __restrict__ poses, const float* __restrict__ dx, int t0, int P, float* __restrict__ dx_out,
                                    int* __restrict__ hdr) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k == 0 && hdr[HDR_CHOL_FAIL]) atomicOr(&hdr[HDR_STATUS], ST_CHOL_FAIL);   // sticky: some iteration was not SPD (its dx is 0)
  if (k >= P) return;
  float xi[6];
#pragma unroll
  for (int c = 0; c < 6; c++) { xi[c] = dx[k * 6 + c]; if (dx_out) dx_out[k * 6 + c] = xi[c]; }
  retract_pose(xi, poses + 7 * (size_t)(t0 + k));
}

}  // namespace dba
using namespace dba;

// ---------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------
extern "C" size_t dba_ba_workspace_bytes(int n_frames, int n_edges, int ht, int wd, int t0, int t1) {
  return make_layout(n_frames, n_edges, ht, wd, t0, t1).total;
}
extern "C" size_t dba_ba_system_offset(int n_frames, int n_edges, int ht, int wd, int t0, int t1) {
  return make_layout(n_frames, n_edges, ht, wd, t0, t1).off_sys;
}
extern "C" size_t dba_ba_system_bytes(int t0, int t1) {
  const size_t n = 6 * (size_t)(t1 - t0 > 0 ? t1 - t0 : 0);
  return (n * n + n) * sizeof(double);
}

static int check_ba_args(const dba_ba_args* a, Layout& L) {
  DBA_CHECK_ARG(a != nullptr, "null args");
  DBA_CHECK_ARG(a->n_frames > 0 && a->n_edges >= 0 && a->ht > 0 && a->wd > 0, "bad extents");
  DBA_CHECK_ARG(a->t0 >= 0 && a->t1 >= a->t0 && a->t1 <= a->n_frames, "bad window [t0,t1)");
  DBA_CHECK_ARG(a->poses && a->disps && a->intrinsics && a->disps_sens, "null state pointer");
  DBA_CHECK_ARG(a->n_edges == 0 || (a->targets && a->weights && a->ii && a->jj), "null edge pointer");
  DBA_CHECK_ARG(a->motion_only || (a->eta && a->eta_rows >= 1), "eta missing");
  DBA_CHECK_ARG(a->motion_only || !a->eta_by_frame || a->eta_rows >= a->n_frames, "eta_by_frame needs one eta row per frame");
  DBA_CHECK_ARG(a->own_lo >= 0 && a->own_hi >= a->own_lo, "bad ownership range");
  DBA_CHECK_ARG(a->p2p_world <= 8 && (a->p2p_world <= 1 || (a->p2p_rank >= 0 && a->p2p_rank < a->p2p_world)), "bad p2p rank/world");
  DBA_CHECK_ARG(a->workspace != nullptr, "null workspace");
  DBA_CHECK_ARG(a->n_frames <= 65535, "more than 65535 frames");
  L = make_layout(a->n_frames, a->n_edges, a->ht, a->wd, a->t0, a->t1);
  if (a->workspace_bytes < L.total) { dba::set_error("workspace too small: %zu < %zu", a->workspace_bytes, L.total); return DBA_ERR_WORKSPACE; }
  return DBA_OK;
}

#define WS(T, off) reinterpret_cast<T*>(reinterpret_cast<char*>(a->workspace) + (off))

// where the reduced pose system of this Gauss-Newton iteration is accumulated: the private workspace, or -- for the fused
// peer-to-peer reduction -- slot (epoch & 1) of this rank's peer-visible buffer
static double* system_ptr(const dba_ba_args* a, const Layout& L) {
  if (a->p2p_world > 1) return reinterpret_cast<double*>(a->p2p_system[a->p2p_rank]) + (size_t)(a->p2p_epoch & 1ull) * ((size_t)L.n * L.n + L.n);
  return reinterpret_cast<double*>(reinterpret_cast<char*>(a->workspace) + L.off_sys);
}

extern "C" int dba_ba_prepare(const dba_ba_args* a) {
  Layout L; int rc = check_ba_args(a, L); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)a->stream;
  ba_prepare_kernel<<<1, 1024, 0, st>>>(a->ii, a->jj, a->n_edges, a->n_frames, a->t0, a->t1, (a->motion_only || a->eta_by_frame) ? 1 : a->eta_rows,
                                        a->motion_only,
                                        WS(int, L.off_hdr), WS(int, L.off_frame2k), WS(int, L.off_kx), WS(int, L.off_rowptr),
                                        schur_plan(WS(void, L.off_plan), a->n_frames), a->ht * a->wd, WS(float, L.off_Eij), WS(float, L.off_C), WS(float, L.off_w), WS(float, L.off_Ei));
  DBA_CHECK_LAUNCH("ba_prepare");
  if (a->n_edges > 0) {
    ba_fill_csr_kernel<<<(a->n_edges + 7) / 8, 256, 0, st>>>(a->ii, a->jj, a->n_edges, a->n_frames, WS(int, L.off_frame2k),
                                                                  WS(int, L.off_rowptr), WS(int, L.off_edgeidx));
    DBA_CHECK_LAUNCH("ba_fill_csr");
  }
  return DBA_OK;
}

extern "C" int dba_ba_build(const dba_ba_args* a) {
  Layout L; int rc = check_ba_args(a, L); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)a->stream;
  const int HW = a->ht * a->wd;
  double* Hsys = system_ptr(a, L);
  double* bsys = Hsys + (size_t)L.n * L.n;
  DBA_CHECK_CUDA(cudaMemsetAsync(Hsys, 0, ((size_t)L.n * L.n + L.n) * sizeof(double), st), "ba_build memset");
  DBA_CHECK_CUDA(cudaMemsetAsync(WS(int, L.off_hdr) + HDR_CHOL_FAIL, 0, sizeof(int), st), "ba_build memset");
  // an empty window still has depth blocks to build (and back-substitute with dx = 0) unless the call is motion-only
  if (L.P == 0 && a->motion_only) return DBA_OK;
  // frames that can own edges on this rank (edge-sharded runs own a sub-range): size the pixel chunks so the grid fills the GPU
  const int eff_frames = std::max(1, std::min(a->n_frames, a->own_hi - a->own_lo));
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
  const int ppt = (eff_frames * ((HW + 4 * kBuildThreads - 1) / (4 * kBuildThreads)) >= sms) ? 4
                : (eff_frames * ((HW + 2 * kBuildThreads - 1) / (2 * kBuildThreads)) >= sms) ? 2 : 1;
#define LAUNCH_BUILD(PPT)                                                                                                               \
  ba_build_kernel<PPT><<<dim3((HW + PPT * kBuildThreads - 1) / (PPT * kBuildThreads), a->n_frames), kBuildThreads, 0, st>>>(             \
      a->poses, a->disps, a->intrinsics, a->disps_sens, a->targets, a->weights, a->eta, a->eta_rows, a->eta_by_frame, a->jj, WS(int, L.off_hdr),  \
      WS(int, L.off_kx), WS(int, L.off_rowptr), WS(int, L.off_edgeidx), HW, a->wd, a->t0, L.P, a->motion_only, Hsys, bsys,               \
      WS(float, L.off_Eij), WS(float, L.off_C), WS(float, L.off_w), WS(float, L.off_Ei))
  if (ppt == 4) LAUNCH_BUILD(4); else if (ppt == 2) LAUNCH_BUILD(2); else LAUNCH_BUILD(1);
#undef LAUNCH_BUILD
  DBA_CHECK_LAUNCH("ba_build");
  if (!a->motion_only && L.P > 0) {
    static bool attr_set = false;
    if (!attr_set) {
      DBA_CHECK_CUDA(cudaFuncSetAttribute(ba_schur_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmem), "schur tc smem attr");
      attr_set = true;
    }
    // one CTA per SM shares every route's work by the plan ba_prepare_kernel wrote (see ba_schur_tc_kernel)
    ba_schur_tc_kernel<<<sms, kTcThreads, kTcSmem, st>>>(a->jj, WS(int, L.off_hdr), WS(int, L.off_kx), WS(int, L.off_rowptr), WS(int, L.off_edgeidx),
                                                        HW, a->t0, L.P, WS(float, L.off_Eij), WS(float, L.off_C), WS(float, L.off_w),
                                                        WS(float, L.off_Ei), Hsys, bsys, schur_plan(WS(void, L.off_plan), a->n_frames));
    DBA_CHECK_LAUNCH("ba_schur");
  }
  return DBA_OK;
}

extern "C" int dba_ba_solve(const dba_ba_args* a) {
  Layout L; int rc = check_ba_args(a, L); if (rc) return rc;
  if (L.P == 0 && a->motion_only) return DBA_OK;
  cudaStream_t st = (cudaStream_t)a->stream;
  const int HW = a->ht * a->wd;
  double* Hsys = system_ptr(a, L);
  double* bsys = Hsys + (size_t)L.n * L.n;
  float* dx = WS(float, L.off_dx);
  if (L.P > 0) {      // an empty window has no pose system: dx = 0, which the back-substitution never reads (0 < pose < P)
    CholPeers peers; peers.world = 0;
    if (a->p2p_world > 1) {
      const size_t nd = (size_t)L.n * L.n + L.n;
      peers.world = a->p2p_world; peers.epoch = a->p2p_epoch; peers.epoch_dev = a->p2p_epoch_dev;
      for (int k = 0; k < a->p2p_world; k++) peers.sys[k] = reinterpret_cast<const double*>(a->p2p_system[k]) + (size_t)(a->p2p_epoch & 1ull) * nd;
      peers.flags = reinterpret_cast<const unsigned long long*>(reinterpret_cast<const double*>(a->p2p_system[a->p2p_rank]) + 2 * nd);
    }
    int rc2 = chol_solve_launch(Hsys, bsys, L.n, (double)a->lm, (double)a->ep, WS(void, L.off_L), WS(int, L.off_hdr) + HDR_CHOL_FAIL, dx, st,
                                a->p2p_world > 1 ? &peers : nullptr);
    if (rc2) return rc2;
  }
  if (!a->motion_only) {
    DBA_CHECK_ARG(a->dz_out != nullptr, "dz_out missing");
    dim3 grid((HW + 255) / 256, a->n_frames);
    ba_backsub_kernel<<<grid, 256, 0, st>>>(a->jj, WS(int, L.off_hdr), WS(int, L.off_kx), WS(int, L.off_rowptr), WS(int, L.off_edgeidx),
                                            HW, a->t0, L.P, WS(float, L.off_Eij), WS(float, L.off_C), WS(float, L.off_w),
                                            WS(float, L.off_Ei), dx, a->disps, a->dz_out, a->own_lo, a->own_hi);
    DBA_CHECK_LAUNCH("ba_backsub");
  }
  if (L.P > 0) {
    ba_pose_retr_kernel<<<(L.P + 127) / 128, 128, 0, st>>>(a->poses, dx, a->t0, L.P, a->dx_out, WS(int, L.off_hdr));
    DBA_CHECK_LAUNCH("ba_pose_retr");
  }
  return DBA_OK;
}

// publish this rank's partial system to every peer: release stores of the epoch into flags[rank] of each peer's buffer
namespace dba {
struct P2PSignal { unsigned long long* flag[8]; int world; unsigned long long epoch; unsigned long long* epoch_dev; };
__global__ void ba_p2p_signal_kernel2(P2PSignal s) {
  __threadfence_system();
  const int lane = threadIdx.x;
  unsigned long long e = s.epoch;
  if (s.epoch_dev) {                     // device-resident epoch: advance it here so a captured graph publishes a fresh value per replay
    if (lane == 0) { e = *s.epoch_dev + 1ull; *s.epoch_dev = e; }
    e = __shfl_sync(0xffffffffu, e, 0);
  }
  if (lane < s.world) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(s.flag[lane]), "l"(e) : "memory");
}
}  // namespace dba

extern "C" int dba_ba_p2p_signal(const dba_ba_args* a) {
  Layout L; int rc = check_ba_args(a, L); if (rc) return rc;
  if (a->p2p_world <= 1) return DBA_OK;
  const size_t nd = (size_t)L.n * L.n + L.n;
  dba::P2PSignal s; s.world = a->p2p_world; s.epoch = a->p2p_epoch; s.epoch_dev = a->p2p_epoch_dev;
  for (int k = 0; k < a->p2p_world; k++)
    s.flag[k] = reinterpret_cast<unsigned long long*>(reinterpret_cast<double*>(a->p2p_system[k]) + 2 * nd) + a->p2p_rank;
  dba::ba_p2p_signal_kernel2<<<1, 32, 0, (cudaStream_t)a->stream>>>(s);
  DBA_CHECK_LAUNCH("ba_p2p_signal");
  return DBA_OK;
}

extern "C" int dba_ba(const dba_ba_args* a, int iterations) {
  int rc = dba_ba_prepare(a);
  if (rc) return rc;
  for (int it = 0; it < iterations; it++) {
    rc = dba_ba_build(a); if (rc) return rc;
    rc = dba_ba_solve(a); if (rc) return rc;
  }
  return DBA_OK;
}

extern "C" int dba_ba_read_info(const dba_ba_args* a, int* n_depth_frames, int* device_status) {
  Layout L; int rc = check_ba_args(a, L); if (rc) return rc;
  int h[4] = {0, 0, 0, 0};
  DBA_CHECK_CUDA(cudaMemcpyAsync(h, WS(int, L.off_hdr), sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)a->stream), "read_info copy");
  DBA_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)a->stream), "read_info sync");
  if (n_depth_frames) *n_depth_frames = h[HDR_M];
  if (device_status) *device_status = h[HDR_STATUS];
  return DBA_OK;
}
