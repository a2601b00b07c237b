// ConvGRU of DroidNet's update operator for training (reference droid_slam/modules/gru.py:19-32, ConvGRU(128, 128+128+64)), forward
// and backward on fp32 NCHW maps.  Per edge b, with X = [net, inp, corr, flow] (448 channels) and X_q = [r * net, inp, corr, flow]:
//
//   glo  = mean_p sigmoid(W_w net + b_w) * net                            gemm<GloFwd> (into q's buffer) + gru_rowsum_kernel
//   v_j  = b_j + b_jglo + W_jglo glo  (j = z, r, q; one 128-vector each)  gru_vec_kernel
//   z, r = sigmoid(conv3x3([W_z; W_r], X) + v_z, v_r)                     gemm<ConvFwd<false>>, N = 256
//   q    = tanh(conv3x3(W_q, X_q) + v_q),  out = (1 - z) net + z q        gemm<ConvFwd<true>>, r * net formed while staging
//
// The forward keeps z, r (one [b,256,h,w] map), q ([b,128,h,w]) and glo ([b,128]): 384 channels per pixel plus a vector per edge, less
// than the 1536 new channels autograd keeps for the reference's op sequence.  Keeping them costs one write per channel; recomputing them
// would repeat both 3x3 GEMMs (93 % of the forward's work) in the backward.  The backward recomputes only W_w net (a 1x1 GEMM).
//
// Backward, from the upstream gradient g of out:
//   a_z = g (q - net) z (1 - z),  a_q = g z (1 - q^2),  g_net = g (1 - z)                          gru_gate_grad_kernel
//   D_q = conv3x3^T(W_q, a_q): g_net += D_q[:128] r, a_r = D_q[:128] net r (1 - r), g_in = D_q[128:]  gemm<ConvData<true>>
//   D_zr = conv3x3^T([W_z; W_r], [a_z; a_r]): g_net += D_zr[:128], g_in += D_zr[128:]                 gemm<ConvData<false>>
//   g_W = sum over (b, p) of a (x) the shifted sources; g_b and the per-edge sums E_j = sum_p a_j      gemm<Wgrad> + partials, rowsum
//   g_W_jglo = sum_b E_j glo^T, g_b_jglo = g_b_j = sum_b E_j, g_glo = sum_j W_jglo^T E_j               gru_glo_param_grad / glo_grad
//   s = sigmoid(W_w net + b_w):  g_net += g_glo s / hw,  a_w = g_glo / hw net s (1 - s)               gemm<GloGrad>
//   g_net += W_w^T a_w;  g_W_w, g_b_w from a_w                                                        gemm<GloData>, gemm<Wgrad>
//
// Every product of the GEMMs is 3xTF32 on mma.sync (tf32x3.cuh) with fp32 accumulation.  Sums over pixels are never atomic: the weight
// gradients reduce kWgradChunk pixels per CTA into a partial, and the partials, the per-edge sums, the per-edge 128 x 128 vector
// products and the sums over edges are accumulated in fp64 in a fixed order (the gradient of glo feeds every pixel's, so its error is
// kept below the GEMMs'), so two runs give the same bits.
#include "common.cuh"
#include "tf32x3.cuh"
#include "../../include/droid_b200_training.h"

namespace dba {

constexpr int kGruC = 128;                 // hidden channels; net, inp, corr have 128, flow 64
constexpr int kGruIn = 448;                // channels of X
constexpr int kGruK3 = kGruIn * 9;         // reduction length of a 3x3 convolution (ci * 9 + tap)
constexpr int kDa = 384;                   // channels of the backward's pre-activation gradient buffer: a_z, a_r, a_q
constexpr int kWgradChunk = 4096;          // pixels one weight-gradient partial sums
constexpr int kGruParams = 14;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// the 14 parameters in the module's order: convz, convr, convq, w, convz_glo, convr_glo, convq_glo (weight then bias each)
enum { kWz, kBz, kWr, kBr, kWq, kBq, kWw, kBw, kWzg, kBzg, kWrg, kBrg, kWqg, kBqg };
struct GruParams {
  const float* p[kGruParams];
};
struct GruGradParams {
  float* p[kGruParams];
};

// The inputs of one call and its map geometry.
struct GruMaps {
  const float *net, *inp, *corr, *flow;
  int ht, wd, hw;
  // channel ci of X at pixel p of edge b
  __device__ __forceinline__ float x(int b, int ci, int p) const {
    if (ci < 128) return net[((size_t)b * 128 + ci) * hw + p];
    if (ci < 256) return inp[((size_t)b * 128 + ci - 128) * hw + p];
    if (ci < 384) return corr[((size_t)b * 128 + ci - 256) * hw + p];
    return flow[((size_t)b * 64 + ci - 384) * hw + p];
  }
  // channel ci of X_q: r * net for the first 128 channels (r: channels 128.. of zr)
  __device__ __forceinline__ float xq(int b, int ci, int p, const float* zr) const {
    if (ci < 128) return zr[((size_t)b * 256 + 128 + ci) * hw + p] * net[((size_t)b * 128 + ci) * hw + p];
    return x(b, ci, p);
  }
  // pixel p shifted by tap (ty, tx) - 1, sign s: -1 for none outside the image
  __device__ __forceinline__ int shift(int p, int tap, int s) const {
    const int y = p / wd + s * (tap / 3 - 1), x = p % wd + s * (tap % 3 - 1);
    return (y >= 0 && y < ht && x >= 0 && x < wd) ? y * wd + x : -1;
  }
};

// ---- one GEMM engine for every product ---------------------------------------------------------------------------------------------
// C[m][n] = sum_{k in [k_begin(z), k_end(z))} A(z, k, m) B(z, k, n), a 64 x 64 tile per CTA (grid x over n, y over m, z over the
// op's z: the edge, or the weight gradient's pixel chunk).  The op gives its elements (a() / b(), never called outside [0, M) x [0, N)
// or the k range) and consumes the result (store()).  kAKFast / kBKFast: which index the staging threads walk fastest, chosen per op
// so that consecutive threads read consecutive addresses.  The next chunk is loaded into registers while the current one is multiplied.
template <class Op>
__global__ void __launch_bounds__(kCtThreads, 2) gru_gemm_kernel(const Op op) {
  __shared__ __align__(16) float sA[kCtK][kLd];
  __shared__ __align__(16) float sB[kCtK][kLd];
  const int n0 = blockIdx.x * kCtTile, m0 = blockIdx.y * kCtTile, z = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kb = op.k_begin(z), ke = op.k_end(z);
  constexpr int kPer = kCtK * kCtTile / kCtThreads;
  float ra[kPer], rb[kPer];
  auto load = [&](int k0) {
#pragma unroll
    for (int r = 0; r < kPer; r++) {
      const int idx = tid + r * kCtThreads;
      const int ka = Op::kAKFast ? idx % kCtK : idx / kCtTile, m = Op::kAKFast ? idx / kCtK : idx % kCtTile;
      const int kk = Op::kBKFast ? idx % kCtK : idx / kCtTile, n = Op::kBKFast ? idx / kCtK : idx % kCtTile;
      ra[r] = (k0 + ka < ke && m0 + m < op.M) ? op.a(z, k0 + ka, m0 + m) : 0.f;
      rb[r] = (k0 + kk < ke && n0 + n < op.N) ? op.b(z, k0 + kk, n0 + n) : 0.f;
    }
  };
  float acc[2][2][4] = {};
  if (kb < ke) load(kb);
  for (int k0 = kb; k0 < ke; k0 += kCtK) {
#pragma unroll
    for (int r = 0; r < kPer; r++) {
      const int idx = tid + r * kCtThreads;
      if (Op::kAKFast) sA[idx % kCtK][idx / kCtK] = ra[r]; else sA[idx / kCtTile][idx % kCtTile] = ra[r];
      if (Op::kBKFast) sB[idx % kCtK][idx / kCtK] = rb[r]; else sB[idx / kCtTile][idx % kCtTile] = rb[r];
    }
    __syncthreads();
    if (k0 + kCtK < ke) load(k0 + kCtK);
    chunk_mma_3xtf32(sA, sB, acc, warp & 1, warp >> 1, lane);
    __syncthreads();
  }
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int h = 0; h < 4; h++) {
        const int m = m0 + 32 * (warp & 1) + 16 * i + g + 8 * (h >> 1), n = n0 + 16 * (warp >> 1) + 8 * j + 2 * t + (h & 1);
        if (m < op.M && n < op.N) op.store(z, m, n, acc[i][j][h]);
      }
}

// ---- the ops -----------------------------------------------------------------------------------------------------------------------
// z: the edge; k over the whole reduction
struct PerEdge {
  int M, N, K;
  __device__ int k_begin(int) const { return 0; }
  __device__ int k_end(int) const { return K; }
};

// s = sigmoid(W_w net + b_w) * net -> out [b,128,hw] (the forward's glo before its mean)
struct GloFwd : PerEdge {
  static constexpr bool kAKFast = true, kBKFast = false;
  GruMaps s;
  const float *w, *bias;
  float* out;
  __device__ float a(int, int k, int m) const { return w[m * kGruC + k]; }
  __device__ float b(int z, int k, int n) const { return s.net[((size_t)z * kGruC + k) * s.hw + n]; }
  __device__ void store(int z, int m, int n, float v) const {
    const size_t i = ((size_t)z * kGruC + m) * s.hw + n;
    out[i] = sigmoidf_(v + bias[m]) * s.net[i];
  }
};

// Q = false: [z; r] = sigmoid(conv3x3([W_z; W_r], X) + v) -> zr [b,256,hw].  Q = true: q = tanh(conv3x3(W_q, X_q) + v_q) -> q, and
// out = (1 - z) net + z q.  vec [b,384]: v_z, v_r, v_q.
template <bool Q>
struct ConvFwd : PerEdge {
  static constexpr bool kAKFast = true, kBKFast = false;
  GruMaps s;
  const float *wz, *wr, *wq, *vec;
  float *zr, *q, *out;
  __device__ float a(int, int k, int m) const {
    if (Q) return wq[(size_t)m * kGruK3 + k];
    return m < kGruC ? wz[(size_t)m * kGruK3 + k] : wr[(size_t)(m - kGruC) * kGruK3 + k];
  }
  __device__ float b(int z, int k, int n) const {
    const int ci = k / 9, p = s.shift(n, k - 9 * ci, 1);
    if (p < 0) return 0.f;
    return Q ? s.xq(z, ci, p, zr) : s.x(z, ci, p);
  }
  __device__ void store(int z, int m, int n, float v) const {
    if (!Q) {
      zr[((size_t)z * 256 + m) * s.hw + n] = sigmoidf_(v + vec[z * kDa + m]);
      return;
    }
    const float qv = tanhf(v + vec[z * kDa + 256 + m]);
    const size_t i = ((size_t)z * kGruC + m) * s.hw + n;
    const float zz = zr[((size_t)z * 256 + m) * s.hw + n];
    q[i] = qv;
    out[i] = (1.f - zz) * s.net[i] + zz * qv;
  }
};

// The gradients of one backward call.
struct GruGrads {
  float *net, *inp, *corr, *flow;
  // g_in[ci - 128] of X's channel ci >= 128
  __device__ __forceinline__ float& in(int b, int ci, int p, int hw) const {
    if (ci < 256) return inp[((size_t)b * 128 + ci - 128) * hw + p];
    if (ci < 384) return corr[((size_t)b * 128 + ci - 256) * hw + p];
    return flow[((size_t)b * 64 + ci - 384) * hw + p];
  }
};

// D = conv3x3^T(W, a): m = the input channel ci, k = co * 9 + tap over the output channels.  Q = true: W_q and a_q (da channels
// 256..383); it starts g_in and forms a_r (da channels 128..255).  Q = false: [W_z; W_r] and [a_z; a_r] (da channels 0..255); it adds.
template <bool Q>
struct ConvData : PerEdge {
  static constexpr bool kAKFast = true, kBKFast = false;
  GruMaps s;
  const float *wz, *wr, *wq, *zr;
  float* da;
  GruGrads gr;
  __device__ float a(int, int k, int m) const {
    const int co = k / 9, tap = k - 9 * co;
    if (Q) return wq[((size_t)co * kGruIn + m) * 9 + tap];
    return co < kGruC ? wz[((size_t)co * kGruIn + m) * 9 + tap] : wr[((size_t)(co - kGruC) * kGruIn + m) * 9 + tap];
  }
  __device__ float b(int z, int k, int n) const {
    const int co = k / 9, p = s.shift(n, k - 9 * co, -1);
    return p < 0 ? 0.f : da[((size_t)z * kDa + (Q ? 256 : 0) + co) * s.hw + p];
  }
  __device__ void store(int z, int m, int n, float v) const {
    if (m >= kGruC) {
      float& d = gr.in(z, m, n, s.hw);
      d = Q ? v : d + v;
      return;
    }
    const size_t i = ((size_t)z * kGruC + m) * s.hw + n;
    if (!Q) {
      gr.net[i] += v;
      return;
    }
    const float r = zr[((size_t)z * 256 + kGruC + m) * s.hw + n];
    da[((size_t)z * kDa + kGruC + m) * s.hw + n] = v * s.net[i] * r * (1.f - r);
    gr.net[i] += v * r;
  }
};

// Weight gradient partials: part[z][m][n] = sum over the flattened pixels k = b hw + p of chunk z of a(b, m, p) src(b, n, p).  a: da's
// channels off..off + M.  kind 0: n = ci * 9 + tap of X (W_z, W_r), 1: of X_q (W_q), 2: n = ci of net (W_w, 1x1).
template <int kind>
struct Wgrad {
  static constexpr bool kAKFast = true, kBKFast = true;
  int M, N, total, off;
  GruMaps s;
  const float *da, *zr;
  float* part;
  __device__ int k_begin(int z) const { return z * kWgradChunk; }
  __device__ int k_end(int z) const { return min(total, (z + 1) * kWgradChunk); }
  __device__ float a(int, int k, int m) const {
    const int b = k / s.hw, p = k - b * s.hw;
    return da[((size_t)b * kDa + off + m) * s.hw + p];
  }
  __device__ float b(int, int k, int n) const {
    const int b = k / s.hw, p = k - b * s.hw;
    if (kind == 2) return s.net[((size_t)b * kGruC + n) * s.hw + p];
    const int ci = n / 9, ps = s.shift(p, n - 9 * ci, 1);
    if (ps < 0) return 0.f;
    return kind == 1 ? s.xq(b, ci, ps, zr) : s.x(b, ci, ps);
  }
  __device__ void store(int z, int m, int n, float v) const { part[((size_t)z * M + m) * N + n] = v; }
};

// The backward's recomputation of s = sigmoid(W_w net + b_w): g_net += dglo s, a_w = dglo net s (1 - s) -> da channels 0..127, with
// dglo = g_glo / hw per (edge, channel)
struct GloGrad : PerEdge {
  static constexpr bool kAKFast = true, kBKFast = false;
  GruMaps s;
  const float *w, *bias, *dglo;
  float *da, *gnet;
  __device__ float a(int, int k, int m) const { return w[m * kGruC + k]; }
  __device__ float b(int z, int k, int n) const { return s.net[((size_t)z * kGruC + k) * s.hw + n]; }
  __device__ void store(int z, int m, int n, float v) const {
    const float sg = sigmoidf_(v + bias[m]), d = dglo[z * kGruC + m];
    const size_t i = ((size_t)z * kGruC + m) * s.hw + n;
    gnet[i] += d * sg;
    da[((size_t)z * kDa + m) * s.hw + n] = d * s.net[i] * sg * (1.f - sg);
  }
};

// g_net += W_w^T a_w
struct GloData : PerEdge {
  static constexpr bool kAKFast = false, kBKFast = false;
  int hw;
  const float *w, *da;
  float* gnet;
  __device__ float a(int, int k, int m) const { return w[k * kGruC + m]; }
  __device__ float b(int z, int k, int n) const { return da[((size_t)z * kDa + k) * hw + n]; }
  __device__ void store(int z, int m, int n, float v) const { gnet[((size_t)z * kGruC + m) * hw + n] += v; }
};

// ---- reductions and the per-edge vectors -------------------------------------------------------------------------------------------
// out[e * C + c] = (sum_p x[(e * stride + c) * hw + p]) / div, one CTA per (e, c): strided partial sums, then a fixed tree, in fp64
__global__ void __launch_bounds__(256) gru_rowsum_kernel(const float* __restrict__ x, float* __restrict__ out, int C, int stride, int hw,
                                                         double div) {
  __shared__ double red[256];
  const int e = blockIdx.x / C, c = blockIdx.x - e * C;
  const float* row = x + ((size_t)e * stride + c) * hw;
  double s = 0.0;
  for (int p = threadIdx.x; p < hw; p += 256) s += row[p];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = (float)(red[0] / div);
}

// vec[b][j * 128 + c] = b_j[c] + b_jglo[c] + W_jglo[c] . glo[b]   (j = z, r, q)
__global__ void __launch_bounds__(128) gru_vec_kernel(GruParams P, const float* __restrict__ glo, float* __restrict__ vec, int B) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * kDa) return;
  const int b = t / kDa, j = (t - b * kDa) / kGruC, c = t % kGruC;
  const float* w = (j == 0 ? P.p[kWzg] : j == 1 ? P.p[kWrg] : P.p[kWqg]) + c * kGruC;
  const float* g = glo + b * kGruC;
  double s = 0.0;
  for (int i = 0; i < kGruC; i++) s = fma((double)w[i], (double)g[i], s);
  const float* bc = j == 0 ? P.p[kBz] : j == 1 ? P.p[kBr] : P.p[kBq];
  const float* bg = j == 0 ? P.p[kBzg] : j == 1 ? P.p[kBrg] : P.p[kBqg];
  vec[t] = (float)(((double)bc[c] + (double)bg[c]) + s);
}

// parameter gradients of the glo path and the biases from the per-edge sums E [B][384]:
//   g_W_jglo[c][i] = sum_b E[b][j 128 + c] glo[b][i],  g_b_jglo[c] = g_b_j[c] = sum_b E[b][j 128 + c]
__global__ void __launch_bounds__(128) gru_glo_param_grad_kernel(GruGradParams G, const float* __restrict__ E, const float* __restrict__ glo,
                                                                 int B) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * kGruC * (kGruC + 1)) return;
  const int j = t / (kGruC * (kGruC + 1)), r = t - j * kGruC * (kGruC + 1), c = r / (kGruC + 1), i = r - c * (kGruC + 1);
  double s = 0.0;
  if (i < kGruC) {
    for (int b = 0; b < B; b++) s = fma((double)E[b * kDa + j * kGruC + c], (double)glo[b * kGruC + i], s);
    (j == 0 ? G.p[kWzg] : j == 1 ? G.p[kWrg] : G.p[kWqg])[c * kGruC + i] = (float)s;
  } else {
    for (int b = 0; b < B; b++) s += E[b * kDa + j * kGruC + c];
    (j == 0 ? G.p[kBzg] : j == 1 ? G.p[kBrg] : G.p[kBqg])[c] = (float)s;
    (j == 0 ? G.p[kBz] : j == 1 ? G.p[kBr] : G.p[kBq])[c] = (float)s;
  }
}

// dglo[b][i] = sum_j sum_c W_jglo[c][i] E[b][j 128 + c] / hw   (the gradient of glo, spread over the mean's hw pixels)
__global__ void __launch_bounds__(128) gru_glo_grad_kernel(GruParams P, const float* __restrict__ E, float* __restrict__ dglo, int B, int hw) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * kGruC) return;
  const int b = t / kGruC, i = t - b * kGruC;
  double s = 0.0;
  for (int j = 0; j < 3; j++) {
    const float* w = j == 0 ? P.p[kWzg] : j == 1 ? P.p[kWrg] : P.p[kWqg];
    for (int c = 0; c < kGruC; c++) s = fma((double)w[c * kGruC + i], (double)E[b * kDa + j * kGruC + c], s);
  }
  dglo[t] = (float)(s / hw);
}

// out[i] = sum_b E[b * stride + i] over i < C (the bias gradient of W_w from its per-edge sums)
__global__ void __launch_bounds__(128) gru_sum_edges_kernel(const float* __restrict__ E, float* __restrict__ out, int B, int C, int stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C) return;
  double s = 0.0;
  for (int b = 0; b < B; b++) s += E[b * stride + i];
  out[i] = (float)s;
}

// out = the sum of S partials of n elements in partial order, in fp64; elements n0.. go to out1
__global__ void __launch_bounds__(256) gru_sum_partials_kernel(const float* __restrict__ part, int S, long long n, long long n0,
                                                               float* __restrict__ out0, float* __restrict__ out1) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int k = 0; k < S; k++) s += part[(size_t)k * n + i];
  if (i < n0) out0[i] = (float)s; else out1[i - n0] = (float)s;
}

// the gate's gradients: g_net = g (1 - z), a_z = g (q - net) z (1 - z), a_q = g z (1 - q^2)
__global__ void __launch_bounds__(256) gru_gate_grad_kernel(const float* __restrict__ g, const float* __restrict__ net,
                                                            const float* __restrict__ zr, const float* __restrict__ q,
                                                            float* __restrict__ gnet, float* __restrict__ da, long long total, int hw) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const long long bc = t / hw;
  const int b = (int)(bc / kGruC), c = (int)(bc - (long long)b * kGruC), p = (int)(t - bc * hw);
  const float gv = g[t], nv = net[t], qv = q[t], zz = zr[((size_t)b * 256 + c) * hw + p];
  gnet[t] = gv * (1.f - zz);
  da[((size_t)b * kDa + c) * hw + p] = gv * (qv - nv) * (zz * (1.f - zz));
  da[((size_t)b * kDa + 256 + c) * hw + p] = gv * zz * (1.f - qv * qv);
}

template <class Op>
static int gemm(const Op& op, int nz, cudaStream_t st, const char* what) {
  const dim3 grid((op.N + kCtTile - 1) / kCtTile, (op.M + kCtTile - 1) / kCtTile, nz);
  gru_gemm_kernel<Op><<<grid, kCtThreads, 0, st>>>(op);
  DBA_CHECK_LAUNCH(what);
  return DBA_OK;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static int wgrad_chunks(int B, int hw) { return (int)(((long long)B * hw + kWgradChunk - 1) / kWgradChunk); }

// the backward's workspace, in order: da [B,384,hw], E [B,384], dglo [B,128], Ew [B,128], the weight-gradient partials
struct BwdLayout {
  size_t da, E, dglo, Ew, part, total;
  BwdLayout(int B, int hw) {
    da = 0;
    E = da + align256((size_t)B * kDa * hw * sizeof(float));
    dglo = E + align256((size_t)B * kDa * sizeof(float));
    Ew = dglo + align256((size_t)B * kGruC * sizeof(float));
    part = Ew + align256((size_t)B * kGruC * sizeof(float));
    total = part + align256((size_t)wgrad_chunks(B, hw) * 256 * kGruK3 * sizeof(float));
  }
};

}  // namespace dba

using namespace dba;

static int check_gru_shape(int B, int ht, int wd) {
  DBA_CHECK_ARG(B >= 1 && ht >= 1 && wd >= 1, "conv_gru needs b, ht, wd >= 1");
  DBA_CHECK_ARG(B <= 65535, "more than 65535 edges per call");
  DBA_CHECK_ARG((long long)B * kGruIn * ht * wd <= 0x7fffffffLL, "b * 448 * ht * wd must fit in 31 bits");
  return DBA_OK;
}

static int check_gru_workspace(const char* fn, void* ws, size_t bytes, size_t need) {
  if (!ws || bytes < need) {
    set_error("invalid argument: %s needs a workspace of %zu bytes (dba_conv_gru_workspace_bytes), got %zu", fn, need, ws ? bytes : (size_t)0);
    return DBA_ERR_INVALID;
  }
  DBA_CHECK_ARG(((uintptr_t)ws & 255) == 0, "workspace must be 256-byte aligned");
  return DBA_OK;
}

extern "C" size_t dba_conv_gru_workspace_bytes(int b, int ht, int wd, int backward) {
  if (b <= 0 || ht <= 0 || wd <= 0) return 0;
  return backward ? BwdLayout(b, ht * wd).total : align256((size_t)b * kDa * sizeof(float));
}

extern "C" int dba_conv_gru_forward(const float* net, const float* inp, const float* corr, const float* flow, const float* const* params,
                                    float* out, float* zr, float* q, float* glo, int b, int ht, int wd, void* workspace,
                                    size_t workspace_bytes, dba_stream_t stream) {
  int rc = check_gru_shape(b, ht, wd);
  if (rc) return rc;
  DBA_CHECK_ARG(net && inp && corr && flow && params && out && zr && q && glo, "null pointer");
  GruParams P;
  for (int i = 0; i < kGruParams; i++) {
    DBA_CHECK_ARG(params[i], "null parameter pointer");
    P.p[i] = params[i];
  }
  rc = check_gru_workspace("conv_gru_forward", workspace, workspace_bytes, dba_conv_gru_workspace_bytes(b, ht, wd, 0));
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int hw = ht * wd;
  const GruMaps s{net, inp, corr, flow, ht, wd, hw};
  float* vec = (float*)workspace;

  GloFwd gf{};
  gf.M = kGruC; gf.N = hw; gf.K = kGruC; gf.s = s; gf.w = P.p[kWw]; gf.bias = P.p[kBw]; gf.out = q;      // q's buffer holds s until q
  if ((rc = gemm(gf, b, st, "conv_gru_forward(glo)"))) return rc;
  gru_rowsum_kernel<<<b * kGruC, 256, 0, st>>>(q, glo, kGruC, kGruC, hw, (double)hw);
  DBA_CHECK_LAUNCH("conv_gru_forward(glo mean)");
  gru_vec_kernel<<<(b * kDa + 127) / 128, 128, 0, st>>>(P, glo, vec, b);
  DBA_CHECK_LAUNCH("conv_gru_forward(vec)");

  ConvFwd<false> fzr{};
  fzr.M = 256; fzr.N = hw; fzr.K = kGruK3; fzr.s = s; fzr.wz = P.p[kWz]; fzr.wr = P.p[kWr]; fzr.vec = vec; fzr.zr = zr;
  if ((rc = gemm(fzr, b, st, "conv_gru_forward(zr)"))) return rc;
  ConvFwd<true> fq{};
  fq.M = kGruC; fq.N = hw; fq.K = kGruK3; fq.s = s; fq.wq = P.p[kWq]; fq.vec = vec; fq.zr = zr; fq.q = q; fq.out = out;
  return gemm(fq, b, st, "conv_gru_forward(q)");
}

extern "C" int dba_conv_gru_backward(const float* grad_out, const float* net, const float* inp, const float* corr, const float* flow,
                                     const float* const* params, const float* zr, const float* q, const float* glo, float* grad_net,
                                     float* grad_inp, float* grad_corr, float* grad_flow, float* const* grad_params, int b, int ht, int wd,
                                     void* workspace, size_t workspace_bytes, dba_stream_t stream) {
  int rc = check_gru_shape(b, ht, wd);
  if (rc) return rc;
  DBA_CHECK_ARG(grad_out && net && inp && corr && flow && params && zr && q && glo && grad_net && grad_inp && grad_corr && grad_flow &&
                grad_params, "null pointer");
  GruParams P;
  GruGradParams G;
  for (int i = 0; i < kGruParams; i++) {
    DBA_CHECK_ARG(params[i] && grad_params[i], "null parameter pointer");
    P.p[i] = params[i];
    G.p[i] = grad_params[i];
  }
  rc = check_gru_workspace("conv_gru_backward", workspace, workspace_bytes, dba_conv_gru_workspace_bytes(b, ht, wd, 1));
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int hw = ht * wd, total = b * hw, S = wgrad_chunks(b, hw);
  const GruMaps s{net, inp, corr, flow, ht, wd, hw};
  const BwdLayout L(b, hw);
  uint8_t* ws = (uint8_t*)workspace;
  float *da = (float*)(ws + L.da), *E = (float*)(ws + L.E), *dglo = (float*)(ws + L.dglo), *Ew = (float*)(ws + L.Ew);
  float* part = (float*)(ws + L.part);
  const GruGrads gr{grad_net, grad_inp, grad_corr, grad_flow};

  const long long n128 = (long long)b * kGruC * hw;
  gru_gate_grad_kernel<<<(unsigned)((n128 + 255) / 256), 256, 0, st>>>(grad_out, net, zr, q, grad_net, da, n128, hw);
  DBA_CHECK_LAUNCH("conv_gru_backward(gate)");
  ConvData<true> dq{};
  dq.M = kGruIn; dq.N = hw; dq.K = kGruC * 9; dq.s = s; dq.wq = P.p[kWq]; dq.zr = zr; dq.da = da; dq.gr = gr;
  if ((rc = gemm(dq, b, st, "conv_gru_backward(data q)"))) return rc;
  ConvData<false> dzr{};
  dzr.M = kGruIn; dzr.N = hw; dzr.K = 256 * 9; dzr.s = s; dzr.wz = P.p[kWz]; dzr.wr = P.p[kWr]; dzr.zr = zr; dzr.da = da; dzr.gr = gr;
  if ((rc = gemm(dzr, b, st, "conv_gru_backward(data zr)"))) return rc;

  // the 3x3 weight gradients: partials over kWgradChunk pixels, summed in chunk order
  Wgrad<1> wq{};
  wq.M = kGruC; wq.N = kGruK3; wq.total = total; wq.off = 256; wq.s = s; wq.da = da; wq.zr = zr; wq.part = part;
  if ((rc = gemm(wq, S, st, "conv_gru_backward(grad W_q)"))) return rc;
  const long long nq = (long long)kGruC * kGruK3;
  gru_sum_partials_kernel<<<(unsigned)((nq + 255) / 256), 256, 0, st>>>(part, S, nq, nq, G.p[kWq], nullptr);
  DBA_CHECK_LAUNCH("conv_gru_backward(sum W_q)");
  Wgrad<0> wzr{};
  wzr.M = 256; wzr.N = kGruK3; wzr.total = total; wzr.off = 0; wzr.s = s; wzr.da = da; wzr.part = part;
  if ((rc = gemm(wzr, S, st, "conv_gru_backward(grad W_z, W_r)"))) return rc;
  gru_sum_partials_kernel<<<(unsigned)((2 * nq + 255) / 256), 256, 0, st>>>(part, S, 2 * nq, nq, G.p[kWz], G.p[kWr]);
  DBA_CHECK_LAUNCH("conv_gru_backward(sum W_z, W_r)");

  // the biases and the glo path
  gru_rowsum_kernel<<<b * kDa, 256, 0, st>>>(da, E, kDa, kDa, hw, 1.0);
  DBA_CHECK_LAUNCH("conv_gru_backward(edge sums)");
  gru_glo_param_grad_kernel<<<(3 * kGruC * (kGruC + 1) + 127) / 128, 128, 0, st>>>(G, E, glo, b);
  DBA_CHECK_LAUNCH("conv_gru_backward(glo params)");
  gru_glo_grad_kernel<<<(b * kGruC + 127) / 128, 128, 0, st>>>(P, E, dglo, b, hw);
  DBA_CHECK_LAUNCH("conv_gru_backward(glo)");
  GloGrad gg{};
  gg.M = kGruC; gg.N = hw; gg.K = kGruC; gg.s = s; gg.w = P.p[kWw]; gg.bias = P.p[kBw]; gg.dglo = dglo; gg.da = da; gg.gnet = grad_net;
  if ((rc = gemm(gg, b, st, "conv_gru_backward(glo gate)"))) return rc;                  // a_w over a_z, which nothing reads any more
  GloData gd{};
  gd.M = kGruC; gd.N = hw; gd.K = kGruC; gd.hw = hw; gd.w = P.p[kWw]; gd.da = da; gd.gnet = grad_net;
  if ((rc = gemm(gd, b, st, "conv_gru_backward(data w)"))) return rc;
  Wgrad<2> ww{};
  ww.M = kGruC; ww.N = kGruC; ww.total = total; ww.off = 0; ww.s = s; ww.da = da; ww.part = part;
  if ((rc = gemm(ww, S, st, "conv_gru_backward(grad W_w)"))) return rc;
  const long long nw = (long long)kGruC * kGruC;
  gru_sum_partials_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, st>>>(part, S, nw, nw, G.p[kWw], nullptr);
  DBA_CHECK_LAUNCH("conv_gru_backward(sum W_w)");
  gru_rowsum_kernel<<<b * kGruC, 256, 0, st>>>(da, Ew, kGruC, kDa, hw, 1.0);
  DBA_CHECK_LAUNCH("conv_gru_backward(edge sums w)");
  gru_sum_edges_kernel<<<1, 128, 0, st>>>(Ew, G.p[kBw], b, kGruC, kGruC);
  DBA_CHECK_LAUNCH("conv_gru_backward(b_w)");
  return DBA_OK;
}
