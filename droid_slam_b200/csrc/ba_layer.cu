// ba_layer.cu -- the differentiable dense bundle adjustment layer DroidNet trains through (reference droid_slam/geom/ba.py:31-106 with
// geom/chol.py:46-73 and the Jacobian path of geom/projective_ops.py), forward and backward on sm_90a.
//
// Semantics are the Python layer's, not ba_cuda's (ba_pixel.cuh): valid = X1.z > 0.2, proj replaces Z < 0.1 by 1, w = .001 valid weight,
// per-frame intrinsics (source frame for iproj, target frame for proj), Ji = -adjT(Gij, Jj), Gij = [-0.1,0,0, 0,0,0,1] on ii == jj
// edges.  Depth unknowns: the distinct source frames (ascending, k = rank among them), C = sum w Jz^2 + eta + 1e-7.  Pose unknowns: frames
// fixedp .. N-1.  Damping H + ep + lm diag(H) before the Schur complement.  Retraction Exp(dx) X for every frame (dx = 0 for fixed ones)
// with lietorch's exp and mul, disps + dz, then where(> 10, 0) and clamp(min = 0).  A failed factor anywhere in the batch gives dx = 0 for
// every batch element, and no gradient through dx (the reference's CholeskySolver).
//
// Forward (one stream, no host synchronisation):
//   prepare       one thread: the ii -> k map from a presence bitmap over the N frames; out-of-range ii / jj (and a source count other
//                 than eta's M) set the status word, and such edges are skipped everywhere
//   pixel         per edge pixel: J (2 x 13: Ji, Jj, Jz), r, w in fp32 -> workspace; Es = sum_c w_c Js_c Jz_c (12)
//   edge reduce   per edge: the 12 x 12 local pose block and the 12-vector J^T W r, fp64 sums over the pixels in a fixed order
//   depth         per (k, pixel): C and w = sum w Jz r over the out-edges of k in edge order (fp64), Q = 1 / C
//   pair          per ordered pair of edges with a common source: sum_p Es_e Q Es_f^T (12 x 12, fp64)
//   edge y        per edge: sum_p Es_e Q w
//   factor        per batch element (one CTA): S = H_damped - E Q E^T and y = v - E Q w assembled in shared memory in edge order, a fp64
//                 Cholesky, the two triangular solves -> dx; the factor is kept for the backward
//   pose retr     Exp(dx) X (dx = 0 when any batch element failed)
//   depth retr    dz = Q (w - E^T dx) and the disparity update
// Backward, with lambda = K^-1 g for the damped system K z = b and its factor from the forward:
//   the same prepare / pixel / depth passes (recomputed, nothing per pixel was kept), the retraction's backward (g Jl(dx), g Adj(Exp dx),
//   the where / clamp masks), lambda_x from the kept factor, lambda_z = Q (g_z - E^T lambda_x), then per edge pixel the local adjoint
//   dL/dr = w u, dL/dw = u (r - s) - lm T, dL/dJ = w [(r - s) lambda - u z] - lm w dT/dJ  (u = J lambda, s = J z, T the damping's
//   sum_d lambda_d z_d J_d^2 over pose dims) pulled back to Gij and the source disparity by forward-mode duals over the 7 local
//   directions; per-edge fp64 sums and per-frame gathers in edge order give the pose and disparity gradients.  No atomics anywhere.
#include "lie_math.cuh"

namespace {

using dba_lie::Elem;
using dba_lie::SE3g;

constexpr int kMaxPoses = DBA_BA_LAYER_MAX_POSES;
constexpr int kTile = 128;          // pixels staged per shared-memory tile in the reduction kernels
constexpr int kPix = 30;            // per edge pixel: J rows u (13), v (13), r (2), w (2)

// ---- forward-mode dual numbers (value, one directional derivative) ----------------------------------------------------------------
struct Df {
  float v, d;
  __device__ __forceinline__ Df(float v_ = 0.f, float d_ = 0.f) : v(v_), d(d_) {}
};
__device__ __forceinline__ Df operator+(Df a, Df b) { return Df(a.v + b.v, a.d + b.d); }
__device__ __forceinline__ Df operator-(Df a, Df b) { return Df(a.v - b.v, a.d - b.d); }
__device__ __forceinline__ Df operator-(Df a) { return Df(-a.v, -a.d); }
__device__ __forceinline__ Df operator*(Df a, Df b) { return Df(a.v * b.v, a.v * b.d + a.d * b.v); }
__device__ __forceinline__ Df operator*(float a, Df b) { return Df(a * b.v, a * b.d); }
__device__ __forceinline__ Df recip(Df a) { const float r = 1.f / a.v; return Df(r, -a.d * r * r); }
__device__ __forceinline__ float recip(float a) { return 1.f / a; }
__device__ __forceinline__ float val(float a) { return a; }
__device__ __forceinline__ float val(Df a) { return a.v; }

// proj (Z < 0.1 replaced by 1) of the transformed homogeneous point (X, Y, Z, W) with the target frame's intrinsics, and the Jacobians
// Jj = Jp Ja (actp's 4 x 6), Jz = Jp (Gij [0,0,0,1]) = Jp (t, 1).  T = float or Df.
template <class T>
__device__ __forceinline__ void proj_terms(T X, T Y, T Z, T W, T tx, T ty, T tz, float fx, float fy, float cx, float cy, T* coords,
                                           T (&Jj)[2][6], T (&Jz)[2]) {
  const T Zc = val(Z) < 0.1f ? T(1.f) : Z;
  const T d = recip(Zc);
  coords[0] = fx * (X * d) + T(cx);
  coords[1] = fy * (Y * d) + T(cy);
  const T a0 = fx * d, a2 = -(fx * (X * d * d));     // Jp row u: (a0, 0, a2, 0)
  const T b1 = fy * d, b2 = -(fy * (Y * d * d));     // Jp row v: (0, b1, b2, 0)
  // Ja rows: (W,0,0, 0,Z,-Y), (0,W,0, -Z,0,X), (0,0,W, Y,-X,0)
  Jj[0][0] = a0 * W; Jj[0][1] = T(0.f); Jj[0][2] = a2 * W; Jj[0][3] = a2 * Y; Jj[0][4] = a0 * Z - a2 * X; Jj[0][5] = -(a0 * Y);
  Jj[1][0] = T(0.f); Jj[1][1] = b1 * W; Jj[1][2] = b2 * W; Jj[1][3] = b2 * Y - b1 * Z; Jj[1][4] = -(b2 * X); Jj[1][5] = b1 * X;
  Jz[0] = a0 * tx + a2 * tz;
  Jz[1] = b1 * ty + b2 * tz;
}

// Gij = poses[jj] * poses[ii]^-1 with lietorch's inv and mul (quaternions normalised on load), or the reference's constant on ii == jj
template <typename T>
__device__ __forceinline__ Elem<SE3g, T> edge_gij(const float* __restrict__ pb, int i, int j) {
  Elem<SE3g, T> G;
  if (i == j) {
    G.t[0] = T(-0.1f); G.t[1] = G.t[2] = T(0); G.q[0] = G.q[1] = G.q[2] = T(0); G.q[3] = T(1);
    return G;
  }
  Elem<SE3g, T> Pj, Pi;
  Pj.load(pb + 7 * j); Pi.load(pb + 7 * i);
  return dba_lie::g_mul(Pj, dba_lie::g_inv(Pi));
}

// one edge pixel's primal terms
struct Pixel {
  float J[2][13];      // Ji (0-5), Jj (6-11), Jz (12)
  float r[2], w[2];
  float X1[4], valid;
};

struct LayerCtx {
  const float *target, *weight, *eta, *poses, *disps, *intr;
  const int64_t *ii, *jj;
  int B, N, E, M, ht, wd, HW, P, fixedp;
};

__device__ __forceinline__ void pixel_terms(const LayerCtx& c, const Elem<SE3g, float>& G, int b, int e, int i, int j, int p, Pixel& o) {
  const float* ki = c.intr + ((int64_t)b * c.N + i) * 4;
  const float* kj = c.intr + ((int64_t)b * c.N + j) * 4;
  const float x = (float)(p % c.wd), y = (float)(p / c.wd);
  const float disp = c.disps[((int64_t)b * c.N + i) * c.HW + p];
  const float P0[3] = {(x - ki[2]) / ki[0], (y - ki[3]) / ki[1], 1.f};
  float R[3];
  dba_lie::rot(G.q, P0, R);
  o.X1[0] = R[0] + G.t[0] * disp; o.X1[1] = R[1] + G.t[1] * disp; o.X1[2] = R[2] + G.t[2] * disp; o.X1[3] = disp;
  float coords[2], Jj[2][6], Jz[2];
  proj_terms<float>(o.X1[0], o.X1[1], o.X1[2], o.X1[3], G.t[0], G.t[1], G.t[2], kj[0], kj[1], kj[2], kj[3], coords, Jj, Jz);
  o.valid = (o.X1[2] > 0.2f && 1.f > 0.2f) ? 1.f : 0.f;          // X0.z is 1
  const int64_t pe = (((int64_t)b * c.E + e) * c.HW + p) * 2;
  for (int r = 0; r < 2; r++) {
    float Ji[6];
    dba_lie::g_adjT(G, Jj[r], Ji);
    for (int m = 0; m < 6; m++) { o.J[r][m] = -Ji[m]; o.J[r][6 + m] = Jj[r][m]; }
    o.J[r][12] = Jz[r];
    o.r[r] = c.target[pe + r] - coords[r];
    o.w[r] = .001f * (o.valid * c.weight[pe + r]);
  }
}

// ---- prepare: edge -> k map and the status word -----------------------------------------------------------------------------------
__global__ void bal_prepare_kernel(const int64_t* __restrict__ ii, const int64_t* __restrict__ jj, int E, int N, int M, int* __restrict__ kmap,
                                   int* __restrict__ ek, int* __restrict__ flags, int B, int clear_fail) {
  if (threadIdx.x != 0) return;
  int status = 0;
  for (int f = 0; f < N; f++) kmap[f] = 0;
  for (int e = 0; e < E; e++) {
    const int64_t i = ii[e], j = jj[e];
    if (i < 0 || i >= N || j < 0 || j >= N) status |= DBA_BA_LAYER_BAD_INDEX;
    else kmap[i] = 1;
  }
  int k = 0;
  for (int f = 0; f < N; f++) kmap[f] = kmap[f] ? k++ : -1;
  if (k != M) status |= DBA_BA_LAYER_BAD_M;
  for (int e = 0; e < E; e++) {
    const int64_t i = ii[e], j = jj[e];
    const bool ok = i >= 0 && i < N && j >= 0 && j < N && kmap[i] < M;
    ek[e] = ok ? kmap[i] : -1;
  }
  flags[0] = status;
  if (clear_fail)
    for (int b = 0; b < B; b++) flags[1 + b] = 0;
}

// ---- per edge pixel terms -> workspace --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) bal_pixel_kernel(LayerCtx c, const int* __restrict__ ek, float* __restrict__ pix,
                                                         float* __restrict__ es) {
  const int e = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (ek[e] < 0 || p >= c.HW) return;
  const int i = (int)c.ii[e], j = (int)c.jj[e];
  const Elem<SE3g, float> G = edge_gij<float>(c.poses + (int64_t)b * c.N * 7, i, j);
  Pixel o;
  pixel_terms(c, G, b, e, i, j, p, o);
  float* dst = pix + ((int64_t)b * c.E + e) * kPix * c.HW + p;
  for (int r = 0; r < 2; r++)
    for (int m = 0; m < 13; m++) dst[(int64_t)(13 * r + m) * c.HW] = o.J[r][m];
  dst[(int64_t)26 * c.HW] = o.r[0]; dst[(int64_t)27 * c.HW] = o.r[1];
  dst[(int64_t)28 * c.HW] = o.w[0]; dst[(int64_t)29 * c.HW] = o.w[1];
  float* de = es + ((int64_t)b * c.E + e) * 12 * c.HW + p;
  for (int s = 0; s < 12; s++) de[(int64_t)s * c.HW] = o.w[0] * o.J[0][s] * o.J[0][12] + o.w[1] * o.J[1][s] * o.J[1][12];
}

// upper-triangle index of (a, c), a <= c < 12
__host__ __device__ __forceinline__ int tri12(int a, int c) { return a * 12 - a * (a - 1) / 2 + (c - a); }

// ---- per edge: local 12 x 12 pose block (78 upper entries) and J^T W r (12), fp64 over the pixels in order --------------------------
__global__ void __launch_bounds__(96) bal_edge_reduce_kernel(const float* __restrict__ pix, const int* __restrict__ ek, int E, int HW,
                                                              double* __restrict__ eh) {
  const int e = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  if (ek[e] < 0) return;
  __shared__ float sh[28][kTile];                        // J pose rows u (12), v (12), r (2), w (2)
  int a = 0, cc = 0;
  if (t < 78) {
    int l = t;
    while (l >= 12 - a) { l -= 12 - a; a++; }
    cc = a + l;
  }
  const float* src = pix + ((int64_t)b * E + e) * kPix * HW;
  double acc = 0.0;
  for (int p0 = 0; p0 < HW; p0 += kTile) {
    const int np = min(kTile, HW - p0);
    __syncthreads();
    for (int l = t; l < 28 * kTile; l += blockDim.x) {
      const int row = l / kTile, q = l % kTile;
      const int srow = row < 12 ? row : row < 24 ? row + 1 : row + 2;   // skip Jz_u (12) and Jz_v (25)
      sh[row][q] = q < np ? src[(int64_t)srow * HW + p0 + q] : 0.f;
    }
    __syncthreads();
    if (t < 78) {
      for (int q = 0; q < np; q++)
        acc += (double)sh[26][q] * sh[a][q] * sh[cc][q] + (double)sh[27][q] * sh[12 + a][q] * sh[12 + cc][q];
    } else if (t < 90) {
      const int s = t - 78;
      for (int q = 0; q < np; q++)
        acc += (double)sh[26][q] * sh[s][q] * sh[24][q] + (double)sh[27][q] * sh[12 + s][q] * sh[25][q];
    }
  }
  if (t < 90) eh[((int64_t)b * E + e) * 90 + t] = acc;
}

// ---- per (k, pixel): C, w, Q -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bal_depth_kernel(LayerCtx c, const float* __restrict__ pix, const int* __restrict__ ek,
                                                         double* __restrict__ q_out, double* __restrict__ wz_out) {
  const int k = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.HW) return;
  double C = 0.0, w = 0.0;
  for (int e = 0; e < c.E; e++) {
    if (ek[e] != k) continue;
    const float* s = pix + ((int64_t)b * c.E + e) * kPix * c.HW + p;
    const double jzu = s[(int64_t)12 * c.HW], jzv = s[(int64_t)25 * c.HW];
    const double ru = s[(int64_t)26 * c.HW], rv = s[(int64_t)27 * c.HW], wu = s[(int64_t)28 * c.HW], wv = s[(int64_t)29 * c.HW];
    C += wu * jzu * jzu + wv * jzv * jzv;
    w += wu * ru * jzu + wv * rv * jzv;
  }
  const int64_t o = ((int64_t)b * c.M + k) * c.HW + p;
  C += (double)c.eta[o] + 1e-7;
  q_out[o] = 1.0 / C;
  if (wz_out) wz_out[o] = w;
}

// ---- per ordered pair of edges with a common source: sum_p Es_e Q Es_f^T ----------------------------------------------------------
__global__ void __launch_bounds__(160) bal_pair_kernel(const float* __restrict__ es, const double* __restrict__ q, const int* __restrict__ ek,
                                                        int E, int M, int HW, double* __restrict__ pair) {
  const int e = blockIdx.x, f = blockIdx.y, b = blockIdx.z, t = threadIdx.x;
  const int k = ek[e];
  if (k < 0 || ek[f] != k) return;
  __shared__ float se[12][kTile], sf[12][kTile];
  __shared__ double sq[kTile];
  const float* pe = es + ((int64_t)b * E + e) * 12 * HW;
  const float* pf = es + ((int64_t)b * E + f) * 12 * HW;
  const double* pq = q + ((int64_t)b * M + k) * HW;
  const int s = t / 12, u = t % 12;
  double acc = 0.0;
  for (int p0 = 0; p0 < HW; p0 += kTile) {
    const int np = min(kTile, HW - p0);
    __syncthreads();
    for (int l = t; l < 12 * kTile; l += blockDim.x) {
      const int row = l / kTile, x = l % kTile;
      se[row][x] = x < np ? pe[(int64_t)row * HW + p0 + x] : 0.f;
      sf[row][x] = x < np ? pf[(int64_t)row * HW + p0 + x] : 0.f;
    }
    for (int x = t; x < kTile; x += blockDim.x) sq[x] = x < np ? pq[p0 + x] : 0.0;
    __syncthreads();
    if (t < 144)
      for (int x = 0; x < np; x++) acc += (double)se[s][x] * sq[x] * (double)sf[u][x];
  }
  if (t < 144) pair[(((int64_t)b * E + e) * E + f) * 144 + t] = acc;
}

// ---- per edge: sum_p Es_e Q vec (vec = w in the forward, the depth part of the upstream gradient in the backward) --------------------
__global__ void __launch_bounds__(384) bal_edge_y_kernel(const float* __restrict__ es, const double* __restrict__ q,
                                                          const double* __restrict__ vec, const int* __restrict__ ek, int E, int M, int HW,
                                                          double* __restrict__ ey) {
  const int e = blockIdx.x, b = blockIdx.y, s = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int k = ek[e];
  if (k < 0) return;
  const float* pe = es + (((int64_t)b * E + e) * 12 + s) * HW;
  const int64_t o = ((int64_t)b * M + k) * HW;
  double acc = 0.0;
  for (int p = lane; p < HW; p += 32) acc += (double)pe[p] * q[o + p] * vec[o + p];
  acc = dba::warp_sum(acc);
  if (lane == 0) ey[((int64_t)b * E + e) * 12 + s] = acc;
}

__device__ __forceinline__ int pose_slot(int64_t f, int fixedp, int P) {
  const int64_t s = f - fixedp;
  return s >= 0 && s < P ? (int)s : -1;
}

// L L^T x = v in place (L lower, row-major n x n in shared memory), column-oriented so each step is one parallel update
__device__ void chol_solve_smem(const double* L, double* v, int n) {
  for (int k = 0; k < n; k++) {
    __syncthreads();
    if (threadIdx.x == 0) v[k] /= L[k * n + k];
    __syncthreads();
    for (int r = k + 1 + threadIdx.x; r < n; r += blockDim.x) v[r] -= L[r * n + k] * v[k];
  }
  for (int k = n - 1; k >= 0; k--) {
    __syncthreads();
    if (threadIdx.x == 0) v[k] /= L[k * n + k];
    __syncthreads();
    for (int r = threadIdx.x; r < k; r += blockDim.x) v[r] -= L[k * n + r] * v[k];
  }
  __syncthreads();
}

// v_a of the reduced right-hand side: sum over edges in order of the local vector's pose-a parts
__device__ __forceinline__ void gather_pose_vec(const double* __restrict__ src, int stride, int offset, const int64_t* ii, const int64_t* jj,
                                                const int* ek, int E, int fixedp, int P, int a, double (&acc)[6], double sign) {
  for (int e = 0; e < E; e++) {
    if (ek[e] < 0) continue;
    const int si = pose_slot(ii[e], fixedp, P), sj = pose_slot(jj[e], fixedp, P);
    const double* x = src + (int64_t)e * stride + offset;
    if (si == a) for (int d = 0; d < 6; d++) acc[d] += sign * x[d];
    if (sj == a) for (int d = 0; d < 6; d++) acc[d] += sign * x[6 + d];
  }
}

// ---- per batch element: assemble S and y, factor, solve -> dx; the factor goes to `factor` -----------------------------------------
__global__ void __launch_bounds__(256) bal_factor_kernel(const double* __restrict__ eh, const double* __restrict__ pair,
                                                          const double* __restrict__ ey, const int64_t* __restrict__ ii,
                                                          const int64_t* __restrict__ jj, const int* __restrict__ ek, int E, int P, int fixedp,
                                                          float ep, float lm, double* __restrict__ factor, double* __restrict__ dx,
                                                          int* __restrict__ flags) {
  extern __shared__ double S[];
  const int b = blockIdx.x, n = 6 * P;
  double* y = S + n * n;
  __shared__ int fail;
  const double* ehb = eh + (int64_t)b * E * 90;
  const double* pb = pair + (int64_t)b * E * E * 144;
  for (int blk = threadIdx.x; blk < P * P; blk += blockDim.x) {
    const int A = blk / P, Bc = blk % P;
    double acc[36];
    for (int l = 0; l < 36; l++) acc[l] = 0.0;
    for (int e = 0; e < E; e++) {
      if (ek[e] < 0) continue;
      const int sl[2] = {pose_slot(ii[e], fixedp, P), pose_slot(jj[e], fixedp, P)};
      for (int x = 0; x < 2; x++)
        for (int z = 0; z < 2; z++) {
          if (sl[x] != A || sl[z] != Bc) continue;
          for (int r = 0; r < 6; r++)
            for (int c = 0; c < 6; c++) {
              const int ra = 6 * x + r, cb = 6 * z + c;
              acc[6 * r + c] += ehb[e * 90 + (ra <= cb ? tri12(ra, cb) : tri12(cb, ra))];
            }
        }
    }
    if (A == Bc)
      for (int d = 0; d < 6; d++) acc[7 * d] += (double)ep + (double)lm * acc[7 * d];
    for (int e = 0; e < E; e++) {
      const int k = ek[e];
      if (k < 0) continue;
      const int se[2] = {pose_slot(ii[e], fixedp, P), pose_slot(jj[e], fixedp, P)};
      for (int f = 0; f < E; f++) {
        if (ek[f] != k) continue;
        const int sf[2] = {pose_slot(ii[f], fixedp, P), pose_slot(jj[f], fixedp, P)};
        const double* pr = pb + ((int64_t)e * E + f) * 144;
        for (int x = 0; x < 2; x++)
          for (int z = 0; z < 2; z++) {
            if (se[x] != A || sf[z] != Bc) continue;
            for (int r = 0; r < 6; r++)
              for (int c = 0; c < 6; c++) acc[6 * r + c] -= pr[(6 * x + r) * 12 + 6 * z + c];
          }
      }
    }
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 6; c++) S[(6 * A + r) * n + 6 * Bc + c] = acc[6 * r + c];
  }
  for (int A = threadIdx.x; A < P; A += blockDim.x) {
    double acc[6] = {0, 0, 0, 0, 0, 0};
    gather_pose_vec(ehb, 90, 78, ii, jj, ek, E, fixedp, P, A, acc, 1.0);
    gather_pose_vec(ey + (int64_t)b * E * 12, 12, 0, ii, jj, ek, E, fixedp, P, A, acc, -1.0);
    for (int d = 0; d < 6; d++) y[6 * A + d] = acc[d];
  }
  if (threadIdx.x == 0) fail = 0;
  // right-looking Cholesky, lower triangle, in shared memory
  for (int k = 0; k < n; k++) {
    __syncthreads();
    if (threadIdx.x == 0) {
      const double d = S[k * n + k];
      if (!(d > 0.0) || !(d < INFINITY)) fail = 1;
      else S[k * n + k] = sqrt(d);
    }
    __syncthreads();
    if (fail) break;
    const double lkk = S[k * n + k];
    for (int r = k + 1 + threadIdx.x; r < n; r += blockDim.x) S[r * n + k] /= lkk;
    __syncthreads();
    const int m = n - k - 1;
    for (int l = threadIdx.x; l < m * m; l += blockDim.x) {
      const int r = k + 1 + l / m, c = k + 1 + l % m;
      if (c <= r) S[r * n + c] -= S[r * n + k] * S[c * n + k];
    }
  }
  __syncthreads();
  if (!fail) chol_solve_smem(S, y, n);
  double* fo = factor + (int64_t)b * n * n;
  for (int l = threadIdx.x; l < n * n; l += blockDim.x) fo[l] = (l % n) <= (l / n) ? S[l] : 0.0;
  for (int l = threadIdx.x; l < n; l += blockDim.x) dx[(int64_t)b * n + l] = fail ? 0.0 : y[l];
  if (threadIdx.x == 0) flags[1 + b] = fail;
}

__device__ __forceinline__ bool any_failed(const int* flags, int B) {
  int f = 0;
  for (int b = 0; b < B; b++) f |= flags[1 + b];
  return f != 0;
}

// ---- retraction of the poses: Exp(dx) X with lietorch's exp and mul; dx = 0 everywhere when any batch element failed ----------------
__global__ void bal_pose_retr_kernel(const float* __restrict__ poses, double* __restrict__ dx, const int* __restrict__ flags, int B, int N,
                                     int P, int fixedp, float* __restrict__ out) {
  const int b = blockIdx.x;
  const bool failed = any_failed(flags, B);
  for (int f = threadIdx.x; f < N; f += blockDim.x) {
    float xi[6] = {0, 0, 0, 0, 0, 0};
    const int s = pose_slot(f, fixedp, P);
    if (s >= 0) {
      double* d = dx + ((int64_t)b * P + s) * 6;
      for (int k = 0; k < 6; k++) {
        if (failed) d[k] = 0.0;
        xi[k] = (float)d[k];
      }
    }
    const Elem<SE3g, float> X = dba_lie::g_exp<SE3g, float>(xi);
    Elem<SE3g, float> Y;
    Y.load(poses + ((int64_t)b * N + f) * 7);
    dba_lie::g_mul(X, Y).store(out + ((int64_t)b * N + f) * 7);
  }
}

// E^T v at (k, p): sum over the out-edges of k (edge order) of Es_e . v[pose slots of e]
__device__ __forceinline__ double et_dot(const LayerCtx& c, const float* __restrict__ es, const int* __restrict__ ek, const double* v, int b,
                                         int k, int p) {
  double acc = 0.0;
  for (int e = 0; e < c.E; e++) {
    if (ek[e] != k) continue;
    const int sl[2] = {pose_slot(c.ii[e], c.fixedp, c.P), pose_slot(c.jj[e], c.fixedp, c.P)};
    const float* s = es + ((int64_t)b * c.E + e) * 12 * c.HW + p;
    for (int x = 0; x < 2; x++) {
      if (sl[x] < 0) continue;
      const double* vv = v + ((int64_t)b * c.P + sl[x]) * 6;
      for (int d = 0; d < 6; d++) acc += (double)s[(int64_t)(6 * x + d) * c.HW] * vv[d];
    }
  }
  return acc;
}

// ---- back-substitution and the disparity update ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bal_depth_retr_kernel(LayerCtx c, const float* __restrict__ es, const int* __restrict__ ek,
                                                              const int* __restrict__ kmap, const double* __restrict__ q,
                                                              const double* __restrict__ wz, const double* __restrict__ dx,
                                                              double* __restrict__ dz, float* __restrict__ out) {
  const int f = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.HW) return;
  const int64_t o = ((int64_t)b * c.N + f) * c.HW + p;
  float v = c.disps[o];
  const int k = kmap[f];
  if (k >= 0 && k < c.M) {
    const int64_t ok = ((int64_t)b * c.M + k) * c.HW + p;
    const double z = q[ok] * (wz[ok] - et_dot(c, es, ek, dx, b, k, p));
    dz[ok] = z;
    v = v + (float)z;
  }
  v = v > 10.f ? 0.f : v;
  out[o] = v < 0.f ? 0.f : v;                // clamp(min = 0); a NaN stays NaN as in torch
}

// ================================================= backward =======================================================================

// g on the retracted poses -> grad_poses (g Adj(Exp dx)) and the pose part of g_z (g Jl(dx)) for free frames
__global__ void bal_pose_retr_bwd_kernel(const float* __restrict__ gpose, const double* __restrict__ dx, int N, int P, int fixedp,
                                         float* __restrict__ grad_poses, double* __restrict__ gx) {
  const int b = blockIdx.x;
  for (int f = threadIdx.x; f < N; f += blockDim.x) {
    float xi[6] = {0, 0, 0, 0, 0, 0}, g[6];
    const int s = pose_slot(f, fixedp, P);
    if (s >= 0)
      for (int k = 0; k < 6; k++) xi[k] = (float)dx[((int64_t)b * P + s) * 6 + k];
    for (int k = 0; k < 6; k++) g[k] = gpose[((int64_t)b * N + f) * 7 + k];
    const Elem<SE3g, float> X = dba_lie::g_exp<SE3g, float>(xi);
    float o[6];
    dba_lie::g_adjT(X, g, o);
    float* gp = grad_poses + ((int64_t)b * N + f) * 7;
    for (int k = 0; k < 6; k++) gp[k] = o[k];
    gp[6] = 0.f;
    if (s >= 0) {
      float J[9], Q[9], u[3], v[3], da[6];
      dba_lie::so3_jl(xi + 3, J);
      dba_lie::se3_q(xi, xi + 3, Q);
      dba_lie::mtv3(J, g, da);
      dba_lie::mtv3(Q, g, u); dba_lie::mtv3(J, g + 3, v);
      for (int k = 0; k < 3; k++) da[3 + k] = u[k] + v[k];
      for (int k = 0; k < 6; k++) gx[((int64_t)b * P + s) * 6 + k] = da[k];
    }
  }
}

// the where / clamp masks: grad_disps (direct part) and the depth part of g_z
__global__ void __launch_bounds__(256) bal_depth_retr_bwd_kernel(LayerCtx c, const float* __restrict__ gdisp, const int* __restrict__ kmap,
                                                                  const double* __restrict__ dz, float* __restrict__ grad_disps,
                                                                  double* __restrict__ gz) {
  const int f = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.HW) return;
  const int64_t o = ((int64_t)b * c.N + f) * c.HW + p;
  float v = c.disps[o];
  const int k = kmap[f];
  int64_t ok = -1;
  if (k >= 0 && k < c.M) {
    ok = ((int64_t)b * c.M + k) * c.HW + p;
    v = v + (float)dz[ok];
  }
  const float g = (!(v > 10.f) && v >= 0.f) ? gdisp[o] : 0.f;
  grad_disps[o] = g;
  if (ok >= 0) gz[ok] = g;
}

// lambda_x = S^-1 (g_x - E Q g_z) with the forward's factor; 0 when any batch element failed
__global__ void __launch_bounds__(256) bal_lambda_x_kernel(const double* __restrict__ factor, const double* __restrict__ gx,
                                                            const double* __restrict__ ey, const int64_t* __restrict__ ii,
                                                            const int64_t* __restrict__ jj, const int* __restrict__ ek, const int* __restrict__ flags,
                                                            int B, int E, int P, int fixedp, double* __restrict__ lamx) {
  extern __shared__ double L[];
  const int b = blockIdx.x, n = 6 * P;
  double* v = L + n * n;
  const bool failed = any_failed(flags, B);
  if (failed) {
    for (int l = threadIdx.x; l < n; l += blockDim.x) lamx[(int64_t)b * n + l] = 0.0;
    return;
  }
  for (int l = threadIdx.x; l < n * n; l += blockDim.x) L[l] = factor[(int64_t)b * n * n + l];
  for (int A = threadIdx.x; A < P; A += blockDim.x) {
    double acc[6];
    for (int d = 0; d < 6; d++) acc[d] = gx[((int64_t)b * P + A) * 6 + d];
    gather_pose_vec(ey + (int64_t)b * E * 12, 12, 0, ii, jj, ek, E, fixedp, P, A, acc, -1.0);
    for (int d = 0; d < 6; d++) v[6 * A + d] = acc[d];
  }
  __syncthreads();
  chol_solve_smem(L, v, n);
  for (int l = threadIdx.x; l < n; l += blockDim.x) lamx[(int64_t)b * n + l] = v[l];
}

// lambda_z = Q (g_z - E^T lambda_x); grad_eta = -lambda_z dz.  Frames with no out-edge in eta's k range get grad_eta from here too.
__global__ void __launch_bounds__(256) bal_lambda_z_kernel(LayerCtx c, const float* __restrict__ es, const int* __restrict__ ek,
                                                            const double* __restrict__ q, const double* __restrict__ gz,
                                                            const double* __restrict__ lamx, const double* __restrict__ dz,
                                                            double* __restrict__ lamz, float* __restrict__ grad_eta) {
  const int k = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.HW) return;
  const int64_t o = ((int64_t)b * c.M + k) * c.HW + p;
  const double l = q[o] * (gz[o] - et_dot(c, es, ek, lamx, b, k, p));
  lamz[o] = l;
  grad_eta[o] = (float)(-l * dz[o]);
}

// ---- per edge pixel: the local adjoint, pulled back to Gij (6) and the source disparity (1) -------------------------------------------
__global__ void __launch_bounds__(128) bal_pixel_bwd_kernel(LayerCtx c, const int* __restrict__ ek, const double* __restrict__ dx,
                                                             const double* __restrict__ dz, const double* __restrict__ lamx,
                                                             const double* __restrict__ lamz, float lm, float* __restrict__ grad_target,
                                                             float* __restrict__ grad_weight, float* __restrict__ gxi, float* __restrict__ gdp) {
  const int e = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.HW) return;
  const int64_t pe = (((int64_t)b * c.E + e) * c.HW + p) * 2;
  float* gx_out = gxi + ((int64_t)b * c.E + e) * 6 * c.HW + p;
  float* gd_out = gdp + ((int64_t)b * c.E + e) * c.HW + p;
  const int k = ek[e];
  if (k < 0) {
    grad_target[pe] = grad_target[pe + 1] = 0.f;
    grad_weight[pe] = grad_weight[pe + 1] = 0.f;
    for (int m = 0; m < 6; m++) gx_out[(int64_t)m * c.HW] = 0.f;
    *gd_out = 0.f;
    return;
  }
  const int i = (int)c.ii[e], j = (int)c.jj[e];
  const Elem<SE3g, float> G = edge_gij<float>(c.poses + (int64_t)b * c.N * 7, i, j);
  Pixel o;
  pixel_terms(c, G, b, e, i, j, p, o);
  // local unknowns: lambda and z over (pose i, pose j, depth)
  float lam[13], z[13];
  const int sl[2] = {pose_slot(i, c.fixedp, c.P), pose_slot(j, c.fixedp, c.P)};
  for (int x = 0; x < 2; x++)
    for (int d = 0; d < 6; d++) {
      lam[6 * x + d] = sl[x] >= 0 ? (float)lamx[((int64_t)b * c.P + sl[x]) * 6 + d] : 0.f;
      z[6 * x + d] = sl[x] >= 0 ? (float)dx[((int64_t)b * c.P + sl[x]) * 6 + d] : 0.f;
    }
  const int64_t ok = ((int64_t)b * c.M + k) * c.HW + p;
  lam[12] = (float)lamz[ok];
  z[12] = (float)dz[ok];
  const bool same = i == j;
  float gJ[2][13], gr[2];
  for (int r = 0; r < 2; r++) {
    float u = 0.f, s = 0.f;
    for (int m = 0; m < 13; m++) { u += o.J[r][m] * lam[m]; s += o.J[r][m] * z[m]; }
    // damping term T = sum_d lambda_d z_d (sum of this row's entries on frame d's slots)^2
    float T = 0.f, dT[12];
    for (int d = 0; d < 6; d++) {
      const float lz = lam[d] * z[d];               // both slots of an ii == jj edge hold the same frame's lambda, z
      if (same) {
        const float js = o.J[r][d] + o.J[r][6 + d];
        T += lz * js * js;
        dT[d] = dT[6 + d] = 2.f * lz * js;
      } else {
        const float lz2 = lam[6 + d] * z[6 + d];
        T += lz * o.J[r][d] * o.J[r][d] + lz2 * o.J[r][6 + d] * o.J[r][6 + d];
        dT[d] = 2.f * lz * o.J[r][d];
        dT[6 + d] = 2.f * lz2 * o.J[r][6 + d];
      }
    }
    const float rs = o.r[r] - s;
    gr[r] = o.w[r] * u;
    grad_target[pe + r] = gr[r];
    grad_weight[pe + r] = .001f * o.valid * (u * rs - lm * T);
    for (int m = 0; m < 13; m++) gJ[r][m] = o.w[r] * (rs * lam[m] - u * z[m]);
    for (int m = 0; m < 12; m++) gJ[r][m] -= lm * o.w[r] * dT[m];
  }
  const float* kj = c.intr + ((int64_t)b * c.N + j) * 4;
  // directions 0-5: Gij <- Exp(e_m) Gij (none on an ii == jj edge, whose Gij is a constant); 6: the source disparity
#pragma unroll
  for (int m = 0; m < 7; m++) {
    if (same && m < 6) continue;
    float dX[4], dt[3] = {0.f, 0.f, 0.f};
    if (m < 6) {
      const float X = o.X1[0], Y = o.X1[1], Z = o.X1[2], W = o.X1[3];
      const float Ja[3][6] = {{W, 0, 0, 0, Z, -Y}, {0, W, 0, -Z, 0, X}, {0, 0, W, Y, -X, 0}};
      dX[0] = Ja[0][m]; dX[1] = Ja[1][m]; dX[2] = Ja[2][m]; dX[3] = 0.f;
      if (m < 3) dt[m] = 1.f;
      else {
        float ev[3] = {0.f, 0.f, 0.f};
        ev[m - 3] = 1.f;
        dba_lie::cross(ev, G.t, dt);
      }
    } else {
      dX[0] = G.t[0]; dX[1] = G.t[1]; dX[2] = G.t[2]; dX[3] = 1.f;
    }
    Df coords[2], Jj[2][6], Jz[2];
    proj_terms<Df>(Df(o.X1[0], dX[0]), Df(o.X1[1], dX[1]), Df(o.X1[2], dX[2]), Df(o.X1[3], dX[3]), Df(G.t[0], dt[0]), Df(G.t[1], dt[1]),
                   Df(G.t[2], dt[2]), kj[0], kj[1], kj[2], kj[3], coords, Jj, Jz);
    float acc = 0.f;
    for (int r = 0; r < 2; r++) {
      acc -= gr[r] * coords[r].d;
      float dJj[6], jv[6], a[6], dJi[6];
      for (int l = 0; l < 6; l++) { dJj[l] = Jj[r][l].d; jv[l] = Jj[r][l].v; }
      if (m < 6) {
        float xi[6] = {0, 0, 0, 0, 0, 0}, ra[6];
        xi[m] = 1.f;
        dba_lie::row_ad<SE3g, float>(jv, xi, ra);
        for (int l = 0; l < 6; l++) a[l] = dJj[l] + ra[l];
      } else {
        for (int l = 0; l < 6; l++) a[l] = dJj[l];
      }
      dba_lie::g_adjT(G, a, dJi);
      for (int l = 0; l < 6; l++) acc += gJ[r][l] * (-dJi[l]) + gJ[r][6 + l] * dJj[l];
      acc += gJ[r][12] * Jz[r].d;
    }
    if (m < 6) gx_out[(int64_t)m * c.HW] = acc;
    else *gd_out = acc;
  }
  if (same)
    for (int m = 0; m < 6; m++) gx_out[(int64_t)m * c.HW] = 0.f;
}

// per edge: the Gij gradient summed over the pixels (fp64, lane-strided then a fixed shuffle tree)
__global__ void __launch_bounds__(192) bal_edge_grad_kernel(const float* __restrict__ gxi, int E, int HW, double* __restrict__ egx) {
  const int e = blockIdx.x, b = blockIdx.y, m = threadIdx.x / 32, lane = threadIdx.x % 32;
  const float* src = gxi + (((int64_t)b * E + e) * 6 + m) * HW;
  double acc = 0.0;
  for (int p = lane; p < HW; p += 32) acc += (double)src[p];
  acc = dba::warp_sum(acc);
  if (lane == 0) egx[((int64_t)b * E + e) * 6 + m] = acc;
}

// per frame: grad_poses += sum over edges in order of g_e (frame jj) and -g_e Adj(Gij) (frame ii)
__global__ void bal_pose_grad_kernel(LayerCtx c, const int* __restrict__ ek, const double* __restrict__ egx, float* __restrict__ grad_poses) {
  const int b = blockIdx.x;
  for (int f = threadIdx.x; f < c.N; f += blockDim.x) {
    double acc[6];
    float* gp = grad_poses + ((int64_t)b * c.N + f) * 7;
    for (int k = 0; k < 6; k++) acc[k] = gp[k];
    for (int e = 0; e < c.E; e++) {
      const int i = (int)c.ii[e], j = (int)c.jj[e];
      if (ek[e] < 0 || i == j || (i != f && j != f)) continue;
      const double* g = egx + ((int64_t)b * c.E + e) * 6;
      if (j == f) for (int k = 0; k < 6; k++) acc[k] += g[k];
      if (i == f) {
        const Elem<SE3g, double> G = edge_gij<double>(c.poses + (int64_t)b * c.N * 7, i, j);
        double gg[6], o[6];
        for (int k = 0; k < 6; k++) gg[k] = g[k];
        dba_lie::g_adjT(G, gg, o);
        for (int k = 0; k < 6; k++) acc[k] -= o[k];
      }
    }
    for (int k = 0; k < 6; k++) gp[k] = (float)acc[k];
  }
}

// per (frame, pixel): grad_disps += sum over the frame's out-edges in order of the per-pixel disparity gradient
__global__ void __launch_bounds__(256) bal_disp_grad_kernel(LayerCtx c, const int* __restrict__ ek, const float* __restrict__ gdp,
                                                             float* __restrict__ grad_disps) {
  const int f = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= c.HW) return;
  const int64_t o = ((int64_t)b * c.N + f) * c.HW + p;
  double acc = grad_disps[o];
  for (int e = 0; e < c.E; e++)
    if (ek[e] >= 0 && c.ii[e] == f) acc += (double)gdp[((int64_t)b * c.E + e) * c.HW + p];
  grad_disps[o] = (float)acc;
}

// ---- workspace ---------------------------------------------------------------------------------------------------------------------
struct Ws {
  int *kmap, *ek;
  float *pix, *es, *gxi, *gdp;
  double *eh, *pair, *ey, *q, *wz, *gx, *lamx, *lamz, *egx;
  size_t bytes;
};

Ws carve(const dba_ba_layer_args* a, char* base) {
  Ws w{};
  const int64_t B = a->B, E = a->E, N = a->N, M = a->M, HW = (int64_t)a->ht * a->wd, n = 6LL * (a->N - a->fixedp);
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += (bytes + 255) / 256 * 256; return p; };
  w.kmap = (int*)take(N * 4);
  w.ek = (int*)take(E * 4);
  w.pix = (float*)take(B * E * kPix * HW * 4);
  w.es = (float*)take(B * E * 12 * HW * 4);
  w.gxi = (float*)take(B * E * 6 * HW * 4);
  w.gdp = (float*)take(B * E * HW * 4);
  w.eh = (double*)take(B * E * 90 * 8);
  w.pair = (double*)take(B * E * E * 144 * 8);
  w.ey = (double*)take(B * E * 12 * 8);
  w.q = (double*)take(B * M * HW * 8);
  w.wz = (double*)take(B * M * HW * 8);
  w.gx = (double*)take(B * n * 8);
  w.lamx = (double*)take(B * n * 8);
  w.lamz = (double*)take(B * M * HW * 8);
  w.egx = (double*)take(B * E * 6 * 8);
  w.bytes = off;
  return w;
}

int check_args(const dba_ba_layer_args* a, bool backward) {
  if (!a || a->B < 1 || a->N < 1 || a->E < 1 || a->M < 1 || a->ht < 1 || a->wd < 1) return DBA_ERR_INVALID;
  if (a->fixedp < 0 || a->fixedp >= a->N || a->N - a->fixedp > kMaxPoses) return DBA_ERR_INVALID;
  if (!a->target || !a->weight || !a->eta || !a->poses || !a->disps || !a->intrinsics || !a->ii || !a->jj || !a->flags) return DBA_ERR_INVALID;
  if (!a->factor || !a->dx || !a->dz) return DBA_ERR_INVALID;
  if (!backward && (!a->poses_out || !a->disps_out)) return DBA_ERR_INVALID;
  if (backward && (!a->grad_poses_out || !a->grad_disps_out || !a->grad_target || !a->grad_weight || !a->grad_eta || !a->grad_poses ||
                   !a->grad_disps))
    return DBA_ERR_INVALID;
  if (!a->workspace || a->workspace_bytes < carve(a, nullptr).bytes) return DBA_ERR_WORKSPACE;
  return DBA_OK;
}

LayerCtx ctx_of(const dba_ba_layer_args* a) {
  LayerCtx c;
  c.target = a->target; c.weight = a->weight; c.eta = a->eta; c.poses = a->poses; c.disps = a->disps; c.intr = a->intrinsics;
  c.ii = a->ii; c.jj = a->jj;
  c.B = a->B; c.N = a->N; c.E = a->E; c.M = a->M; c.ht = a->ht; c.wd = a->wd; c.HW = a->ht * a->wd; c.P = a->N - a->fixedp;
  c.fixedp = a->fixedp;
  return c;
}

size_t solve_smem(int P) { return (size_t)(6 * P) * (6 * P + 1) * 8; }

// prepare, per-pixel terms and the depth pass: the part both directions run
void common_passes(const dba_ba_layer_args* a, const LayerCtx& c, const Ws& w, cudaStream_t st, bool forward) {
  bal_prepare_kernel<<<1, 32, 0, st>>>(c.ii, c.jj, c.E, c.N, c.M, w.kmap, w.ek, a->flags, c.B, forward ? 1 : 0);
  bal_pixel_kernel<<<dim3((c.HW + 127) / 128, c.E, c.B), 128, 0, st>>>(c, w.ek, w.pix, w.es);
  bal_depth_kernel<<<dim3((c.HW + 255) / 256, c.M, c.B), 256, 0, st>>>(c, w.pix, w.ek, w.q, forward ? w.wz : nullptr);
}

}  // namespace

extern "C" size_t dba_ba_layer_workspace_bytes(int B, int N, int E, int M, int ht, int wd, int fixedp) {
  dba_ba_layer_args a{};
  a.B = B; a.N = N; a.E = E; a.M = M; a.ht = ht; a.wd = wd; a.fixedp = fixedp;
  return carve(&a, nullptr).bytes;
}

extern "C" int dba_ba_layer_forward(const dba_ba_layer_args* a) {
  const int rc = check_args(a, false);
  if (rc != DBA_OK) return rc;
  cudaStream_t st = (cudaStream_t)a->stream;
  const LayerCtx c = ctx_of(a);
  const Ws w = carve(a, (char*)a->workspace);
  common_passes(a, c, w, st, true);
  bal_edge_reduce_kernel<<<dim3(c.E, c.B), 96, 0, st>>>(w.pix, w.ek, c.E, c.HW, w.eh);
  bal_pair_kernel<<<dim3(c.E, c.E, c.B), 160, 0, st>>>(w.es, w.q, w.ek, c.E, c.M, c.HW, w.pair);
  bal_edge_y_kernel<<<dim3(c.E, c.B), 384, 0, st>>>(w.es, w.q, w.wz, w.ek, c.E, c.M, c.HW, w.ey);
  const size_t smem = solve_smem(c.P);
  if (cudaFuncSetAttribute(bal_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return DBA_ERR_CUDA;
  bal_factor_kernel<<<c.B, 256, smem, st>>>(w.eh, w.pair, w.ey, c.ii, c.jj, w.ek, c.E, c.P, c.fixedp, a->ep, a->lm, a->factor, a->dx,
                                            a->flags);
  bal_pose_retr_kernel<<<c.B, 64, 0, st>>>(c.poses, a->dx, a->flags, c.B, c.N, c.P, c.fixedp, a->poses_out);
  bal_depth_retr_kernel<<<dim3((c.HW + 255) / 256, c.N, c.B), 256, 0, st>>>(c, w.es, w.ek, w.kmap, w.q, w.wz, a->dx, a->dz, a->disps_out);
  return cudaPeekAtLastError() == cudaSuccess ? DBA_OK : DBA_ERR_CUDA;
}

extern "C" int dba_ba_layer_backward(const dba_ba_layer_args* a) {
  const int rc = check_args(a, true);
  if (rc != DBA_OK) return rc;
  cudaStream_t st = (cudaStream_t)a->stream;
  const LayerCtx c = ctx_of(a);
  const Ws w = carve(a, (char*)a->workspace);
  common_passes(a, c, w, st, false);
  bal_pose_retr_bwd_kernel<<<c.B, 64, 0, st>>>(a->grad_poses_out, a->dx, c.N, c.P, c.fixedp, a->grad_poses, w.gx);
  bal_depth_retr_bwd_kernel<<<dim3((c.HW + 255) / 256, c.N, c.B), 256, 0, st>>>(c, a->grad_disps_out, w.kmap, a->dz, a->grad_disps, w.wz);
  bal_edge_y_kernel<<<dim3(c.E, c.B), 384, 0, st>>>(w.es, w.q, w.wz, w.ek, c.E, c.M, c.HW, w.ey);
  const size_t smem = solve_smem(c.P);
  if (cudaFuncSetAttribute(bal_lambda_x_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return DBA_ERR_CUDA;
  bal_lambda_x_kernel<<<c.B, 256, smem, st>>>(a->factor, w.gx, w.ey, c.ii, c.jj, w.ek, a->flags, c.B, c.E, c.P, c.fixedp, w.lamx);
  bal_lambda_z_kernel<<<dim3((c.HW + 255) / 256, c.M, c.B), 256, 0, st>>>(c, w.es, w.ek, w.q, w.wz, w.lamx, a->dz, w.lamz, a->grad_eta);
  bal_pixel_bwd_kernel<<<dim3((c.HW + 127) / 128, c.E, c.B), 128, 0, st>>>(c, w.ek, a->dx, a->dz, w.lamx, w.lamz, a->lm, a->grad_target,
                                                                           a->grad_weight, w.gxi, w.gdp);
  bal_edge_grad_kernel<<<dim3(c.E, c.B), 192, 0, st>>>(w.gxi, c.E, c.HW, w.egx);
  bal_pose_grad_kernel<<<c.B, 64, 0, st>>>(c, w.ek, w.egx, a->grad_poses);
  bal_disp_grad_kernel<<<dim3((c.HW + 255) / 256, c.N, c.B), 256, 0, st>>>(c, w.ek, w.gdp, a->grad_disps);
  return cudaPeekAtLastError() == cudaSuccess ? DBA_OK : DBA_ERR_CUDA;
}
