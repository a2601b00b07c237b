// lie.cu -- SO3 / SE3 group operations and their gradients: the arithmetic of the `lietorch` package (droid_slam_b200/lietorch) on sm_90a.
//
// Groups: SO3, data (qx,qy,qz,qw), tangent 3; SE3, data (tx,ty,tz,qx,qy,qz,qw), tangent (tau, phi) 6.  fp32 and fp64.  The quaternion is
// normalised on load.  The small-angle branches of exp / log / the left Jacobian and its inverse switch at EPS = 1e-6 like lietorch's.
//
// Broadcasting: the operands have the output's rank; in each batch dimension an operand has the output's size or size 1 (stride 0).
// Nothing is copied to the output's batch: every launch indexes each operand through its own strides.
//   forward   one thread per output element (grid-stride), the operands read through their strides.
//   backward  an operand broadcast over some dimensions has its gradient summed over them in the launch: one CTA per element of that
//             operand, its threads strided over the output elements that read it (the per-edge layout of geom.cu: one pose, many
//             pixels), partial sums in a fixed order (per-thread ascending, then a fixed shuffle tree and warp order), so two runs give the
//             same bits.  The other operand's gradient is written by the same pass when it is not broadcast; when both are broadcast each
//             gets a pass.  With no broadcast at all: one thread per output element.
//
// Gradient convention (lietorch's): the gradient with respect to a group input X is the left-tangent gradient d/de L(Exp(e) X) at e = 0,
// in the first K entries of an N-entry record whose other entries are 0; an upstream gradient on a group output is read the same way.
// Tangent and point inputs get their Euclidean gradient.  With Ad = Adj(X), ad(b) the small adjoint, g the upstream gradient (a row):
//   exp(a)      da = g Jl(a)                     log(X)      dX = g Jl(log X)^-1
//   inv(X)      dX = -g Adj(X^-1)                mul(X, Y)   dX = g, dY = g Adj(X)
//   adj(X, a)   da = g Ad, dX = -g ad(Ad a)      adjT(X, a)  da = Ad g^T, dX = -a^T ad(Ad g^T)
//   act(X, p)   dp = g R, dX = g [I | -hat(Xp)]  act4(X, p)  dp = g T(X), dX = g [q_w I | -hat(q_xyz)], q = X p
//   vec(X)      dX = g P(X)                      fromvec(x)  dx = g pinv(P(X)),  P = the orthogonal projector, pinv(P) in closed form
// (SO3: the translation blocks drop out.)  Jinv and the projector have no backward, as in lietorch.
#include <algorithm>
#include "lie_math.cuh"

namespace {

using namespace dba_lie;

constexpr int kMaxDims = DBA_LIE_MAX_DIMS;

// ---- record sizes of each operation --------------------------------------------------------------------------------------------------
struct Sizes { int a, b, out; };
template <class G> __host__ __device__ constexpr Sizes sizes(int op) {
  return op == DBA_LIE_EXP ? Sizes{G::K, 0, G::N}
       : op == DBA_LIE_LOG ? Sizes{G::N, 0, G::K}
       : op == DBA_LIE_INV ? Sizes{G::N, 0, G::N}
       : op == DBA_LIE_MUL ? Sizes{G::N, G::N, G::N}
       : (op == DBA_LIE_ADJ || op == DBA_LIE_ADJT || op == DBA_LIE_JINV) ? Sizes{G::N, G::K, G::K}
       : op == DBA_LIE_ACT ? Sizes{G::N, 3, 3}
       : op == DBA_LIE_ACT4 ? Sizes{G::N, 4, 4}
       : op == DBA_LIE_PROJECTOR ? Sizes{G::N, 0, G::N * G::N}
       : (op == DBA_LIE_VEC || op == DBA_LIE_FROMVEC) ? Sizes{G::N, 0, G::N}
       : Sizes{0, 0, 0};
}

// ---- forward of one element ----------------------------------------------------------------------------------------------------------
template <class G, typename T, int OP> __device__ __forceinline__ void fwd_elem(const T* pa, const T* pb, T* out) {
  if constexpr (OP == DBA_LIE_EXP) {
    T a[G::K];
    for (int k = 0; k < G::K; k++) a[k] = pa[k];
    g_exp<G, T>(a).store(out);
  } else {
    Elem<G, T> X;
    X.load(pa);
    if constexpr (OP == DBA_LIE_LOG) {
      T a[G::K];
      g_log(X, a);
      for (int k = 0; k < G::K; k++) out[k] = a[k];
    } else if constexpr (OP == DBA_LIE_INV) {
      g_inv(X).store(out);
    } else if constexpr (OP == DBA_LIE_MUL) {
      Elem<G, T> Y;
      Y.load(pb);
      g_mul(X, Y).store(out);
    } else if constexpr (OP == DBA_LIE_ADJ || OP == DBA_LIE_ADJT || OP == DBA_LIE_JINV) {
      T a[G::K], b[G::K];
      for (int k = 0; k < G::K; k++) a[k] = pb[k];
      if constexpr (OP == DBA_LIE_ADJ) g_adj(X, a, b);
      else if constexpr (OP == DBA_LIE_ADJT) g_adjT(X, a, b);
      else {                                                     // Jl(log X)^-1 a
        T x[G::K], Ji[9];
        g_log(X, x);
        if constexpr (G::K == 6) {
          T Q[9], u[3], v[3];
          so3_jl_inv(x + 3, Ji);
          se3_q(x, x + 3, Q);
          mv3(Ji, a + 3, b + 3);                                 // Ji a2
          mv3(Q, b + 3, u);
          for (int k = 0; k < 3; k++) v[k] = a[k] - u[k];
          mv3(Ji, v, b);                                         // Ji (a1 - Q Ji a2)
        } else {
          so3_jl_inv(x, Ji);
          mv3(Ji, a, b);
        }
      }
      for (int k = 0; k < G::K; k++) out[k] = b[k];
    } else if constexpr (OP == DBA_LIE_ACT || OP == DBA_LIE_ACT4) {
      const T p[3] = {pb[0], pb[1], pb[2]};
      T r[3];
      rot(X.q, p, r);
      const T w = OP == DBA_LIE_ACT4 ? pb[3] : T(1);
      for (int k = 0; k < 3; k++) out[k] = r[k] + X.t[k] * w;
      if constexpr (OP == DBA_LIE_ACT4) out[3] = w;
    } else if constexpr (OP == DBA_LIE_PROJECTOR) {
      // row-major N x N: SO3 [[0.5 (w I - hat(v)), 0], [-0.5 v^T, 0]]; SE3 [[I, -hat(t), 0], [0, that 4x4 block]]
      for (int k = 0; k < G::N * G::N; k++) out[k] = T(0);
      const int o = G::N == 7 ? 3 : 0;
      T* P = out + o * G::N + o;
      const T* q = X.q;
      for (int r = 0; r < 3; r++) P[r * G::N + r] = T(0.5) * q[3];
      P[0 * G::N + 1] = T(0.5) * q[2];  P[0 * G::N + 2] = T(-0.5) * q[1];
      P[1 * G::N + 0] = T(-0.5) * q[2]; P[1 * G::N + 2] = T(0.5) * q[0];
      P[2 * G::N + 0] = T(0.5) * q[1];  P[2 * G::N + 1] = T(-0.5) * q[0];
      for (int c = 0; c < 3; c++) P[3 * G::N + c] = T(-0.5) * q[c];
      if constexpr (G::N == 7) {
        for (int r = 0; r < 3; r++) out[r * 7 + r] = T(1);
        out[0 * 7 + 4] = X.t[2];  out[0 * 7 + 5] = -X.t[1];
        out[1 * 7 + 3] = -X.t[2]; out[1 * 7 + 5] = X.t[0];
        out[2 * 7 + 3] = X.t[1];  out[2 * 7 + 4] = -X.t[0];
      }
    }
  }
}

// ---- backward of one element: this element's contributions to da (size a) and db (size b) -------------------------------------------
template <class G, typename T, int OP> __device__ __forceinline__ void bwd_elem(const T* g, const T* pa, const T* pb, T* da, T* db) {
  constexpr Sizes S = sizes<G>(OP);
  for (int k = 0; k < S.a; k++) da[k] = T(0);
  for (int k = 0; k < S.b; k++) db[k] = T(0);
  if constexpr (OP == DBA_LIE_EXP) {                             // da = g Jl(a)
    if constexpr (G::K == 6) {
      T J[9], Q[9], u[3], v[3];
      so3_jl(pa + 3, J);
      se3_q(pa, pa + 3, Q);
      mtv3(J, g, da);                                            // J^T g1
      mtv3(Q, g, u); mtv3(J, g + 3, v);
      for (int k = 0; k < 3; k++) da[3 + k] = u[k] + v[k];      // Q^T g1 + J^T g2
    } else {
      T J[9];
      so3_jl(pa, J);
      mtv3(J, g, da);
    }
  } else if constexpr (OP == DBA_LIE_FROMVEC || OP == DBA_LIE_VEC) {
    Elem<G, T> X;
    X.load(pa);
    if constexpr (OP == DBA_LIE_VEC) {                           // g P
      if constexpr (G::N == 7) {
        T c[3], s[3];
        cross(X.t, g, c);
        so3_row_proj(X.q, g + 3, s);
        for (int k = 0; k < 3; k++) { da[k] = g[k]; da[3 + k] = c[k] + s[k]; }
      } else {
        so3_row_proj(X.q, g, da);
      }
    } else {                                                     // g pinv(P)
      if constexpr (G::N == 7) {
        T c[3], v[3];
        cross(g, X.t, c);
        for (int k = 0; k < 3; k++) { da[k] = g[k]; v[k] = c[k] + g[3 + k]; }
        so3_pinv_col(X.q, v, da + 3);
      } else {
        so3_pinv_col(X.q, g, da);
      }
    }
  } else {
    Elem<G, T> X;
    X.load(pa);
    if constexpr (OP == DBA_LIE_LOG) {                           // dX = g Jl(log X)^-1
      T x[G::K], Ji[9];
      g_log(X, x);
      if constexpr (G::K == 6) {
        T Q[9], u[3], w[3], v[3];
        so3_jl_inv(x + 3, Ji);
        se3_q(x, x + 3, Q);
        mtv3(Ji, g, da);                                         // Ji^T g1
        mtv3(Q, da, u);                                          // Q^T Ji^T g1
        for (int k = 0; k < 3; k++) w[k] = g[3 + k] - u[k];
        mtv3(Ji, w, v);
        for (int k = 0; k < 3; k++) da[3 + k] = v[k];            // Ji^T (g2 - Q^T Ji^T g1)
      } else {
        so3_jl_inv(x, Ji);
        mtv3(Ji, g, da);
      }
    } else if constexpr (OP == DBA_LIE_INV) {                    // dX = -g Adj(X^-1)
      T o[G::K];
      g_adjT(g_inv(X), g, o);
      for (int k = 0; k < G::K; k++) da[k] = -o[k];
    } else if constexpr (OP == DBA_LIE_MUL) {                    // dX = g, dY = g Adj(X)
      for (int k = 0; k < G::K; k++) da[k] = g[k];
      g_adjT(X, g, db);
    } else if constexpr (OP == DBA_LIE_ADJ) {                    // da = g Ad, dX = -g ad(Ad a)
      T a[G::K], b[G::K], o[G::K];
      for (int k = 0; k < G::K; k++) a[k] = pb[k];
      g_adjT(X, g, db);
      g_adj(X, a, b);
      row_ad<G>(g, b, o);
      for (int k = 0; k < G::K; k++) da[k] = -o[k];
    } else if constexpr (OP == DBA_LIE_ADJT) {                   // da = Ad g, dX = -a ad(Ad g)
      T a[G::K], o[G::K];
      for (int k = 0; k < G::K; k++) a[k] = pb[k];
      g_adj(X, g, db);
      row_ad<G>(a, db, o);
      for (int k = 0; k < G::K; k++) da[k] = -o[k];
    } else if constexpr (OP == DBA_LIE_ACT || OP == DBA_LIE_ACT4) {
      const T p[3] = {pb[0], pb[1], pb[2]};
      const T w = OP == DBA_LIE_ACT4 ? pb[3] : T(1);
      T r[3], q[3], c[3];
      rot(X.q, p, r);
      for (int k = 0; k < 3; k++) q[k] = r[k] + X.t[k] * w;    // the image X p
      rot_t(X.q, g, db);                                         // dp_xyz = g R
      if constexpr (OP == DBA_LIE_ACT4) db[3] = dot3(g, X.t) + g[3];
      cross(q, g, c);                                            // g hat(-q) = q x g
      if constexpr (G::K == 6) {
        for (int k = 0; k < 3; k++) { da[k] = g[k] * w; da[3 + k] = c[k]; }
      } else {
        for (int k = 0; k < 3; k++) da[k] = c[k];
      }
    }
  }
}

// ---- launches --------------------------------------------------------------------------------------------------------------------------
// Coalesced batch layout (records): size[d], the contiguous output stride, and each operand's stride (0 where it broadcasts)
struct Layout {
  int nd;
  long long size[kMaxDims], so[kMaxDims], sa[kMaxDims], sb[kMaxDims];
};

template <class G, typename T, int OP>
__global__ void __launch_bounds__(256) lie_forward_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, Layout L,
                                                          long long n) {
  constexpr Sizes S = sizes<G>(OP);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long rem = i, ia = 0, ib = 0;
    for (int d = L.nd - 1; d >= 0; d--) {
      const long long x = rem % L.size[d];
      rem /= L.size[d];
      ia += x * L.sa[d];
      ib += x * L.sb[d];
    }
    fwd_elem<G, T, OP>(a + ia * S.a, S.b ? b + ib * S.b : nullptr, out + i * S.out);
  }
}

// no gradient needs a reduction: one thread per output element writes the gradients asked for (ga / gb NULL: not asked for)
template <class G, typename T, int OP>
__global__ void __launch_bounds__(256) lie_backward_elementwise(const T* __restrict__ grad, const T* __restrict__ a, const T* __restrict__ b,
                                                                T* __restrict__ ga, T* __restrict__ gb, Layout L, long long n) {
  constexpr Sizes S = sizes<G>(OP);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long rem = i, ia = 0, ib = 0;
    for (int d = L.nd - 1; d >= 0; d--) {
      const long long x = rem % L.size[d];
      rem /= L.size[d];
      ia += x * L.sa[d];
      ib += x * L.sb[d];
    }
    T da[S.a], db[S.b > 0 ? S.b : 1];
    bwd_elem<G, T, OP>(grad + i * S.out, a + ia * S.a, S.b ? b + ib * S.b : nullptr, da, db);
    if (ga)
      for (int k = 0; k < S.a; k++) ga[ia * S.a + k] = da[k];
    if (gb)
      for (int k = 0; k < S.b; k++) gb[ib * S.b + k] = db[k];
  }
}

// One CTA per element of the reduced operand (which = 0: a, 1: b), its threads strided over the output elements that element reaches.
// kept: the dimensions the reduced operand is not broadcast over (its elements), red: those it is broadcast over (summed).
// The reduced operand's element is staged in shared memory once per CTA; every thread's per-pixel arithmetic reads it from there (and
// re-derives the unit quaternion, a few flops, so the bits are those of the elementwise kernel).
// write_other: the other operand's gradient is asked for and it is not broadcast, so it is written here element by element.
struct Split {
  int nk, nr;
  long long ksize[kMaxDims], kso[kMaxDims], ksa[kMaxDims], ksb[kMaxDims];
  long long rsize[kMaxDims], rso[kMaxDims], rsa[kMaxDims], rsb[kMaxDims];
  long long n_kept, n_red;
};

template <typename T, int D> __device__ __forceinline__ void block_sum(T (&v)[D], T* sh /* [D][32] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < D; k++)
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
  if (lane == 0)
    for (int k = 0; k < D; k++) sh[k * 32 + warp] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 0; k < D; k++) {
      T s = sh[k * 32];
      for (int w = 1; w < nw; w++) s += sh[k * 32 + w];
      v[k] = s;
    }
  __syncthreads();
}

template <class G, typename T, int OP, int WHICH>
__global__ void __launch_bounds__(256) lie_backward_reduce(const T* __restrict__ grad, const T* __restrict__ a, const T* __restrict__ b,
                                                           T* __restrict__ ga, T* __restrict__ gb, Split P, int write_other) {
  constexpr Sizes S = sizes<G>(OP);
  constexpr int DR = WHICH == 0 ? S.a : (S.b > 0 ? S.b : 1);
  __shared__ T sh[DR * 32];
  __shared__ T rec[DR];
  // index decoding in 32 bits (the host checks n_kept, n_red < 2^31): a 64-bit division is a subroutine call, and its register saves spill
  {
    const unsigned e = blockIdx.x;                             // one CTA per element: gridDim.x = n_kept
    unsigned rem = e;
    long long o0 = 0, a0 = 0, b0 = 0;
    for (int d = P.nk - 1; d > 0; d--) {
      const unsigned x = rem % (unsigned)P.ksize[d];
      rem /= (unsigned)P.ksize[d];
      o0 += x * P.kso[d]; a0 += x * P.ksa[d]; b0 += x * P.ksb[d];
    }
    o0 += rem * P.kso[0]; a0 += rem * P.ksa[0]; b0 += rem * P.ksb[0];   // nk = 0: e = 0 and the strides are 0
    if constexpr (WHICH == 0 || S.b > 0) {
      if (threadIdx.x < DR) rec[threadIdx.x] = WHICH == 0 ? a[a0 * S.a + threadIdx.x] : b[b0 * S.b + threadIdx.x];
    }
    __syncthreads();
    T acc[DR];
    for (int k = 0; k < DR; k++) acc[k] = T(0);
    const unsigned n_red = (unsigned)P.n_red;
    for (unsigned r = threadIdx.x; r < n_red; r += blockDim.x) {
      unsigned rr = r;
      long long io = o0, ia = a0, ib = b0;
      for (int d = P.nr - 1; d > 0; d--) {                       // the outermost index needs no division (one reduced dimension: none)
        const unsigned x = rr % (unsigned)P.rsize[d];
        rr /= (unsigned)P.rsize[d];
        io += x * P.rso[d]; ia += x * P.rsa[d]; ib += x * P.rsb[d];
      }
      io += rr * P.rso[0]; ia += rr * P.rsa[0]; ib += rr * P.rsb[0];
      T da[S.a], db[S.b > 0 ? S.b : 1];
      bwd_elem<G, T, OP>(grad + io * S.out, WHICH == 0 ? rec : a + ia * S.a, WHICH == 1 ? rec : (S.b ? b + ib * S.b : nullptr), da, db);
      if constexpr (WHICH == 0) {
        for (int k = 0; k < S.a; k++) acc[k] += da[k];
        if (write_other)
          for (int k = 0; k < S.b; k++) gb[ib * S.b + k] = db[k];
      } else {
        for (int k = 0; k < S.b; k++) acc[k] += db[k];
        if (write_other)
          for (int k = 0; k < S.a; k++) ga[ia * S.a + k] = da[k];
      }
    }
    block_sum<T, DR>(acc, sh);
    if (threadIdx.x == 0) {
      T* dst = WHICH == 0 ? ga + a0 * S.a : gb + b0 * S.b;
      for (int k = 0; k < DR; k++) dst[k] = acc[k];
    }
  }
}

int grid_for(long long n, int threads) {
  const long long want = (n + threads - 1) / threads;
  return (int)(want < 132LL * 64 ? (want > 0 ? want : 1) : 132LL * 64);
}

// Layout of the output batch after dropping size-1 dimensions and merging neighbours that every operand walks contiguously
Layout coalesce(int ndim, const int64_t* shape, const int64_t* sa, const int64_t* sb) {
  Layout L{};
  long long so[kMaxDims];
  long long acc = 1;
  for (int d = ndim - 1; d >= 0; d--) { so[d] = acc; acc *= shape[d]; }
  for (int d = 0; d < ndim; d++) {
    if (shape[d] == 1) continue;
    const long long a = sa ? sa[d] : 0, b = sb ? sb[d] : 0;
    if (L.nd > 0) {
      const int p = L.nd - 1;
      if (L.so[p] == so[d] * shape[d] && L.sa[p] == a * shape[d] && L.sb[p] == b * shape[d]) {
        L.size[p] *= shape[d];
        L.so[p] = so[d]; L.sa[p] = a; L.sb[p] = b;
        continue;
      }
    }
    L.size[L.nd] = shape[d]; L.so[L.nd] = so[d]; L.sa[L.nd] = a; L.sb[L.nd] = b;
    L.nd++;
  }
  return L;
}

Split split_for(const Layout& L, int which) {
  Split P{};
  P.n_kept = P.n_red = 1;
  for (int d = 0; d < L.nd; d++) {
    const bool red = (which == 0 ? L.sa[d] : L.sb[d]) == 0;
    if (red) {
      P.rsize[P.nr] = L.size[d]; P.rso[P.nr] = L.so[d]; P.rsa[P.nr] = L.sa[d]; P.rsb[P.nr] = L.sb[d]; P.nr++;
      P.n_red *= L.size[d];
    } else {
      P.ksize[P.nk] = L.size[d]; P.kso[P.nk] = L.so[d]; P.ksa[P.nk] = L.sa[d]; P.ksb[P.nk] = L.sb[d]; P.nk++;
      P.n_kept *= L.size[d];
    }
  }
  return P;
}

bool broadcasts(const Layout& L, const long long* s) {
  for (int d = 0; d < L.nd; d++)
    if (s[d] == 0) return true;
  return false;
}

template <class G, typename T, int OP>
int forward_t(const void* a, const void* b, void* out, const Layout& L, long long n, cudaStream_t st) {
  lie_forward_kernel<G, T, OP><<<grid_for(n, 256), 256, 0, st>>>((const T*)a, (const T*)b, (T*)out, L, n);
  DBA_CHECK_LAUNCH("lie_forward_kernel");
  return DBA_OK;
}

template <class G, typename T, int OP>
int backward_t(const void* grad, const void* a, const void* b, void* ga, void* gb, const Layout& L, long long n, cudaStream_t st) {
  constexpr Sizes S = sizes<G>(OP);
  const T *g_ = (const T*)grad, *a_ = (const T*)a, *b_ = (const T*)b;
  T *ga_ = (T*)ga, *gb_ = S.b > 0 ? (T*)gb : nullptr;
  // an operand's gradient is summed in a reduce pass when it is asked for and the operand is broadcast; otherwise it is written element
  // by element, by the reduce pass of the other operand when there is one, else by the elementwise kernel
  const bool ra = ga_ && broadcasts(L, L.sa), rb = gb_ && broadcasts(L, L.sb);
  if (!ra && !rb) {
    lie_backward_elementwise<G, T, OP><<<grid_for(n, 256), 256, 0, st>>>(g_, a_, b_, ga_, gb_, L, n);
    DBA_CHECK_LAUNCH("lie_backward_elementwise");
    return DBA_OK;
  }
  auto threads = [](long long r) { int t = 32; while (t < 256 && t < r) t *= 2; return t; };
  const long long lim = (1LL << 31) - 256;                     // the reduce kernel decodes its indices in 32 bits
  for (int w = 0; w < 2; w++) {
    const Split P = split_for(L, w);
    if ((w == 0 ? ra : rb) && (P.n_kept > lim || P.n_red > lim)) {
      dba::set_error("dba_lie_backward: a broadcast operand with %lld elements each reaching %lld outputs (at most 2^31 - 256 each)",
                     P.n_kept, P.n_red);
      return DBA_ERR_INVALID;
    }
  }
  if (ra) {
    const Split P = split_for(L, 0);
    lie_backward_reduce<G, T, OP, 0><<<(int)P.n_kept, threads(P.n_red), 0, st>>>(g_, a_, b_, ga_, gb_, P, gb_ && !rb);
    DBA_CHECK_LAUNCH("lie_backward_reduce");
  }
  if (rb) {
    const Split P = split_for(L, 1);
    lie_backward_reduce<G, T, OP, 1><<<(int)P.n_kept, threads(P.n_red), 0, st>>>(g_, a_, b_, ga_, gb_, P, ga_ && !ra);
    DBA_CHECK_LAUNCH("lie_backward_reduce");
  }
  return DBA_OK;
}

// dispatch over (group, dtype, op); backward = false: forward
template <class G, typename T>
int dispatch_op(bool backward, int op, const void* grad, const void* a, const void* b, void* out, void* ga, void* gb, const Layout& L,
                long long n, cudaStream_t st) {
#define DBA_LIE_CASE(OPC)                                                                                  \
  case OPC: return backward ? backward_t<G, T, OPC>(grad, a, b, ga, gb, L, n, st) : forward_t<G, T, OPC>(a, b, out, L, n, st);
#define DBA_LIE_FWD_ONLY(OPC)                                                                              \
  case OPC: return backward ? DBA_ERR_INVALID : forward_t<G, T, OPC>(a, b, out, L, n, st);
#define DBA_LIE_BWD_ONLY(OPC)                                                                              \
  case OPC: return backward ? backward_t<G, T, OPC>(grad, a, b, ga, gb, L, n, st) : DBA_ERR_INVALID;
  switch (op) {
    DBA_LIE_CASE(DBA_LIE_EXP) DBA_LIE_CASE(DBA_LIE_LOG) DBA_LIE_CASE(DBA_LIE_INV) DBA_LIE_CASE(DBA_LIE_MUL)
    DBA_LIE_CASE(DBA_LIE_ADJ) DBA_LIE_CASE(DBA_LIE_ADJT) DBA_LIE_CASE(DBA_LIE_ACT) DBA_LIE_CASE(DBA_LIE_ACT4)
    DBA_LIE_FWD_ONLY(DBA_LIE_JINV) DBA_LIE_FWD_ONLY(DBA_LIE_PROJECTOR)
    DBA_LIE_BWD_ONLY(DBA_LIE_VEC) DBA_LIE_BWD_ONLY(DBA_LIE_FROMVEC)
    default: return DBA_ERR_INVALID;
  }
#undef DBA_LIE_CASE
#undef DBA_LIE_FWD_ONLY
#undef DBA_LIE_BWD_ONLY
}

bool has_forward(int op) { return op >= 0 && op < DBA_LIE_OPS && op != DBA_LIE_VEC && op != DBA_LIE_FROMVEC; }
bool has_backward(int op) { return op >= 0 && op < DBA_LIE_OPS && op != DBA_LIE_JINV && op != DBA_LIE_PROJECTOR; }

int run(bool backward, int op, int group, int dtype, const void* grad, const void* a, const int64_t* a_strides, const void* b,
        const int64_t* b_strides, void* out, void* ga, void* gb, int ndim, const int64_t* shape, dba_stream_t stream) {
  const char* what = backward ? "dba_lie_backward" : "dba_lie_forward";
  int da = 0, db = 0, dout = 0;
  if (dba_lie_record_sizes(op, group, &da, &db, &dout) != DBA_OK) {
    dba::set_error("%s: no operation %d for group %d", what, op, group);
    return DBA_ERR_INVALID;
  }
  if (!(backward ? has_backward(op) : has_forward(op))) {
    dba::set_error("%s: operation %d has no %s", what, op, backward ? "backward" : "forward");
    return DBA_ERR_INVALID;
  }
  if (dtype != DBA_F32 && dtype != DBA_F64) {
    dba::set_error("%s: dtype %d (DBA_F32 and DBA_F64 have kernels)", what, dtype);
    return DBA_ERR_INVALID;
  }
  if (ndim < 0 || ndim > kMaxDims || (ndim > 0 && !shape)) {
    dba::set_error("%s: %d batch dimensions (0..%d)", what, ndim, kMaxDims);
    return DBA_ERR_INVALID;
  }
  long long n = 1;
  for (int d = 0; d < ndim; d++) {
    if (shape[d] < 0) { dba::set_error("%s: negative extent %lld in dimension %d", what, (long long)shape[d], d); return DBA_ERR_INVALID; }
    n *= shape[d];
  }
  if (n == 0) return DBA_OK;                                     // nothing to read or write
  if (!a || (ndim > 0 && !a_strides) || (db > 0 && (!b || (ndim > 0 && !b_strides)))) {
    dba::set_error("%s: an operand or its strides are NULL", what);
    return DBA_ERR_INVALID;
  }
  for (int d = 0; d < ndim; d++)
    if (a_strides[d] < 0 || (db > 0 && b_strides[d] < 0)) {
      dba::set_error("%s: negative stride in dimension %d", what, d);
      return DBA_ERR_INVALID;
    }
  if (backward ? (!grad || (!ga && (db == 0 || !gb))) : !out) {
    dba::set_error("%s: the output, the upstream gradient or every gradient pointer is NULL", what);
    return DBA_ERR_INVALID;
  }
  const Layout L = coalesce(ndim, shape, a_strides, db > 0 ? b_strides : nullptr);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (group == DBA_LIE_SO3)
    rc = dtype == DBA_F32 ? dispatch_op<SO3g, float>(backward, op, grad, a, b, out, ga, gb, L, n, st)
                          : dispatch_op<SO3g, double>(backward, op, grad, a, b, out, ga, gb, L, n, st);
  else
    rc = dtype == DBA_F32 ? dispatch_op<SE3g, float>(backward, op, grad, a, b, out, ga, gb, L, n, st)
                          : dispatch_op<SE3g, double>(backward, op, grad, a, b, out, ga, gb, L, n, st);
  return rc;
}

}  // namespace

extern "C" int dba_lie_record_sizes(int op, int group, int* a, int* b, int* out) {
  Sizes s{0, 0, 0};
  if (group == DBA_LIE_SO3) s = sizes<SO3g>(op);
  else if (group == DBA_LIE_SE3) s = sizes<SE3g>(op);
  if (s.a == 0) return DBA_ERR_INVALID;
  if (a) *a = s.a;
  if (b) *b = s.b;
  if (out) *out = s.out;
  return DBA_OK;
}

extern "C" int dba_lie_forward(int op, int group, int dtype, const void* a, const int64_t* a_strides, const void* b, const int64_t* b_strides,
                               void* out, int ndim, const int64_t* shape, dba_stream_t stream) {
  return run(false, op, group, dtype, nullptr, a, a_strides, b, b_strides, out, nullptr, nullptr, ndim, shape, stream);
}

extern "C" int dba_lie_backward(int op, int group, int dtype, const void* grad, const void* a, const int64_t* a_strides, const void* b,
                                const int64_t* b_strides, void* grad_a, void* grad_b, int ndim, const int64_t* shape, dba_stream_t stream) {
  return run(true, op, group, dtype, grad, a, a_strides, b, b_strides, nullptr, grad_a, grad_b, ndim, shape, stream);
}
