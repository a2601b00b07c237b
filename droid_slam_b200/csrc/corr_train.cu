// CorrBlock for DroidNet's training forward (reference droid_slam/modules/corr.py:6-71 on fp32 feature maps) and its backward.
//
// Per edge e (fmap1, fmap2 [E,C,ht,wd] f32, already gathered per edge as DroidNet passes them):
//   V0[p][q]   = sum_c (f1[c][p] / 4)(f2[c][q] / 4),  V_{l+1} = avg_pool2d(V_l, 2, 2) (floor rule)     corr_volume_f32_kernel
//   lookups    = cat_l corr_index_forward(V_l, coords / 2^l, 3)                                       corr_index.cu (f32 pyramid lookup)
//   backward:  G_l[p][.] += the bilinear-weighted gradient of pixel p's 196 taps, for every call       corr_grad_accumulate_kernel
//              g_f1 = sum_l G_l P_l(f2) / 16,  g_f2 = sum_l P_l^T (G_l^T f1) / 16, once per backward     corr_adjoint_* kernels
// P_l is the 2^l x 2^l block mean over the complete blocks of the image (the rows and columns the floor rule drops get nothing).
//
// The gradient pyramid is one private buffer [E][HW][Q], Q = sum_l (ht >> l)(wd >> l), level l at column offset off_l: row p of it is
// written only by source pixel p's own lookups, so one thread per (edge, p) owns it -- no atomics, and every run gives the same bits.
// Both adjoint products are then plain GEMMs over the concatenated levels: the pooling adjoint is folded into the operands (a pooled
// copy of f2 for g_f1, a spread of the level columns of G^T f1 for g_f2), G is never expanded to level 0.
//
// The products run on the tf32 tensor cores (mma.sync m16n8k8) with 3xTF32 operand splitting (tf32x3.cuh), which keeps the error of an
// fp32 FMA chain.  The reduction order is fixed (channel order for the volume, level then pixel order for the adjoint), so every
// run gives the same bits.
#include "corr_pixel.cuh"
#include "tf32x3.cuh"

namespace dba {

// elements per gradient-pyramid row: the four level planes (ht >> l) x (wd >> l), level 0 first
struct Levels {
  long long Q;
  __host__ __device__ Levels(int ht, int wd) {
    Q = 0;
    for (int l = 0; l < 4; l++) Q += (long long)(ht >> l) * (wd >> l);
  }
};

// ---- the volume and its pooled levels ------------------------------------------------------------------------------------------------
// CTA = (64 source pixels from p0, 8x8 block (by, bx) of target pixels, edge e); the 64 x 64 product goes through shared memory to the
// epilogue, where thread (tp, tq) takes source pixels p0 + tp + 16 i (i < 4), targets = the 2x2 block at rows 8 by + 2 (tq >> 2) + {0,1}, columns 8 bx + 2 (tq & 3) + {0,1}.  Level 1 is thread-local; levels 2 and
// 3 combine lanes tq ^ 1, tq ^ 4 and tq ^ 2, tq ^ 8 (tq = lane bits 0..3) by shuffles.  Targets outside the image stage as zeros and are
// not stored; a pooled element is stored when its block lies inside the floor grid of its level, so it never sums such a zero.
__global__ void __launch_bounds__(kCtThreads) corr_volume_f32_kernel(const float* __restrict__ f1, const float* __restrict__ f2,
                                                                     float* __restrict__ out0, float* __restrict__ out1,
                                                                     float* __restrict__ out2, float* __restrict__ out3, int C, int ht,
                                                                     int wd, int nbx) {
  __shared__ __align__(16) float smem[2 * kCtK * kLd];       // the staged chunks; after the products, the 64 x 65 result tile
  float (*sA)[kLd] = reinterpret_cast<float (*)[kLd]>(smem);
  float (*sB)[kLd] = reinterpret_cast<float (*)[kLd]>(smem + kCtK * kLd);
  const int HW = ht * wd;
  const int e = blockIdx.z, p0 = blockIdx.x * kCtTile;
  const int by = blockIdx.y / nbx, bx = blockIdx.y - by * nbx;
  const int tid = threadIdx.x, tq = tid & 15, tp = tid >> 4, lane = tid & 31, warp = tid >> 5;
  const int ty = 2 * (tq >> 2), tx = 2 * (tq & 3);
  const float* A = f1 + (size_t)e * C * HW;
  const float* B = f2 + (size_t)e * C * HW;
  float acc[2][2][4] = {};

  for (int k0 = 0; k0 < C; k0 += kCtK) {
#pragma unroll 2
    for (int r = 0; r < kCtK * kCtTile / kCtThreads; r++) {
      const int idx = tid + r * kCtThreads, k = idx / kCtTile, m = idx % kCtTile;
      const int p = p0 + m, y = 8 * by + m / 8, x = 8 * bx + m % 8;
      sA[k][m] = p < HW ? A[(size_t)(k0 + k) * HW + p] : 0.f;
      sB[k][m] = (y < ht && x < wd) ? B[(size_t)(k0 + k) * HW + y * wd + x] : 0.f;
    }
    __syncthreads();
    chunk_mma_3xtf32(sA, sB, acc, warp & 1, warp >> 1, lane);
    __syncthreads();
  }
  float (*sC)[kCtTile + 1] = reinterpret_cast<float (*)[kCtTile + 1]>(smem);   // [source m][target j = 8 (y - 8 by) + (x - 8 bx)]
  {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int m = 32 * (warp & 1) + 16 * i + g, n = 16 * (warp >> 1) + 8 * j + 2 * t;
        sC[m][n] = acc[i][j][0]; sC[m][n + 1] = acc[i][j][1]; sC[m + 8][n] = acc[i][j][2]; sC[m + 8][n + 1] = acc[i][j][3];
      }
  }
  __syncthreads();

  const int h1 = ht >> 1, w1 = wd >> 1, h2 = ht >> 2, w2 = wd >> 2, h3 = ht >> 3, w3 = wd >> 3;
  const int y = 8 * by + ty, x = 8 * bx + tx;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int p = p0 + tp + 16 * i;
    const bool ok = p < HW;
    const size_t r = (size_t)e * HW + p;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; j++) v[j] = sC[tp + 16 * i][(ty + (j >> 1)) * 8 + tx + (j & 1)] * 0.0625f;   // (f1/4).(f2/4), exactly
    if (ok) {
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int yy = y + (j >> 1), xx = x + (j & 1);
        if (yy < ht && xx < wd) out0[r * HW + (size_t)yy * wd + xx] = v[j];
      }
    }
    const float v1 = ((v[0] + v[1]) + (v[2] + v[3])) * 0.25f;
    const int y1 = y >> 1, x1 = x >> 1;
    if (ok && y1 < h1 && x1 < w1) out1[r * (h1 * w1) + (size_t)y1 * w1 + x1] = v1;
    const float s1 = v1 + __shfl_xor_sync(0xffffffffu, v1, 1);
    const float v2 = (s1 + __shfl_xor_sync(0xffffffffu, s1, 4)) * 0.25f;
    const int y2 = y >> 2, x2 = x >> 2;
    if (ok && (tq & 5) == 0 && y2 < h2 && x2 < w2) out2[r * (h2 * w2) + (size_t)y2 * w2 + x2] = v2;
    const float s2 = v2 + __shfl_xor_sync(0xffffffffu, v2, 2);
    const float v3 = (s2 + __shfl_xor_sync(0xffffffffu, s2, 8)) * 0.25f;
    if (ok && tq == 0 && by < h3 && bx < w3) out3[r * (h3 * w3) + (size_t)by * w3 + bx] = v3;
  }
}

// ---- gradient accumulation -----------------------------------------------------------------------------------------------------------
// One thread per (edge, source pixel): the call's gradient [E,196,ht,wd] of this pixel is added into its own row of the gradient
// pyramid.  Per level and tap the gradient is that of corr_index_backward (the same four products in the same order), then added once.
__global__ void __launch_bounds__(128) corr_grad_accumulate_kernel(const float* __restrict__ coords, const float* __restrict__ grad,
                                                                   float* __restrict__ gpyr, long long total, int ht, int wd) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int hw1 = ht * wd;
  const int n = (int)(p / hw1);
  const int pin = (int)(p - (long long)n * hw1);
  const float x0 = coords[((size_t)n * 2 + 0) * hw1 + pin];
  const float y0 = coords[((size_t)n * 2 + 1) * hw1 + pin];
  float* plane = gpyr + (size_t)p * Levels(ht, wd).Q;   // level l's columns follow level l - 1's
#pragma unroll 1
  for (int l = 0; l < 4; l++) {
    const float s = 1.0f / (float)(1 << l);
    const float xs = x0 * s, ys = y0 * s;
    const float fxf = floorf(xs), fyf = floorf(ys);
    const float dx = xs - fxf, dy = ys - fyf;
    const int fx = floor_to_int_sat(fxf), fy = floor_to_int_sat(fyf);
    const float w11 = dx * dy, w10 = dx * (1.0f - dy), w01 = (1.0f - dx) * dy, w00 = (1.0f - dx) * (1.0f - dy);
    const int h2 = ht >> l, w2 = wd >> l;
    const float* g_in = grad + ((size_t)n * 196 + 49 * l) * hw1 + pin;
    float g[49];
#pragma unroll
    for (int c = 0; c < 49; c++) g[c] = g_in[(size_t)c * hw1];
#pragma unroll
    for (int j = 0; j < 8; j++) {             // footprint rows; along a row the 8 taps are adjacent floats (one or two sectors)
      const int y1 = fy - 3 + j;
      if ((unsigned)y1 >= (unsigned)h2) continue;
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int x1 = fx - 3 + i;
        if ((unsigned)x1 >= (unsigned)w2) continue;
        float t = 0.f;
        if (i > 0 && j > 0) t = fmaf(g[(i - 1) * 7 + (j - 1)], w11, t);
        if (i > 0 && j < 7) t = fmaf(g[(i - 1) * 7 + j], w10, t);
        if (i < 7 && j > 0) t = fmaf(g[i * 7 + (j - 1)], w01, t);
        if (i < 7 && j < 7) t = fmaf(g[i * 7 + j], w00, t);
        plane[(size_t)y1 * w2 + x1] += t;
      }
    }
    plane += (size_t)h2 * w2;
  }
}

// ---- adjoint -------------------------------------------------------------------------------------------------------------------------
// F2cat[e][c][off_l + q] = P_l(f2)[e][c][q]: the level-l block mean of f2, summed row by row in image order
__global__ void __launch_bounds__(256) corr_adjoint_pool_kernel(const float* __restrict__ f2, float* __restrict__ f2cat, long long total,
                                                                int ht, int wd) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const long long Q = Levels(ht, wd).Q;
  const long long ec = t / Q;
  int ql = (int)(t - ec * Q), l = 0;
  while (ql >= (ht >> l) * (wd >> l)) { ql -= (ht >> l) * (wd >> l); l++; }
  const int wl = wd >> l, yl = ql / wl, xl = ql - yl * wl, b = 1 << l;
  const float* src = f2 + (size_t)ec * ht * wd + (size_t)(yl * b) * wd + xl * b;
  float s = 0.f;
  for (int dy = 0; dy < b; dy++)
    for (int dx = 0; dx < b; dx++) s += src[(size_t)dy * wd + dx];
  f2cat[t] = s * (1.0f / (float)(b * b));
}

// Batched C[e][m][n] = alpha * sum_k A[e][m][k] * B(e, k, n), fixed k order.  A: [M][K] rows (lda = K).  B_T: B(k, n) = B[e][n][k] ([N][K]);
// else B(k, n) = B[e][k][n] ([K][N]).  CTA = 64 x 64 outputs; grid x over n, y over m, z over e.
template <bool B_T>
__global__ void __launch_bounds__(kCtThreads) corr_adjoint_gemm_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                                       float* __restrict__ Cout, int M, int N, long long K, float alpha) {
  __shared__ __align__(16) float sA[kCtK][kLd];
  __shared__ __align__(16) float sB[kCtK][kLd];
  const int e = blockIdx.z, n0 = blockIdx.x * kCtTile, m0 = blockIdx.y * kCtTile;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* Ae = A + (size_t)e * M * K;
  const float* Be = B + (size_t)e * N * K;
  float acc[2][2][4] = {};

  for (long long k0 = 0; k0 < K; k0 += kCtK) {
#pragma unroll
    for (int r = 0; r < kCtK * kCtTile / kCtThreads; r++) {
      const int idx = tid + r * kCtThreads;
      {   // A rows: 32 consecutive k per row
        const int k = idx % kCtK, m = idx / kCtK;
        sA[k][m] = (m0 + m < M && k0 + k < K) ? Ae[(size_t)(m0 + m) * K + k0 + k] : 0.f;
      }
      if (B_T) {
        const int k = idx % kCtK, n = idx / kCtK;
        sB[k][n] = (n0 + n < N && k0 + k < K) ? Be[(size_t)(n0 + n) * K + k0 + k] : 0.f;
      } else {
        const int n = idx % kCtTile, k = idx / kCtTile;
        sB[k][n] = (n0 + n < N && k0 + k < K) ? Be[(size_t)(k0 + k) * N + n0 + n] : 0.f;
      }
    }
    __syncthreads();
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
        if (m < M && n < N) Cout[((size_t)e * M + m) * N + n] = acc[i][j][h] * alpha;
      }
}

// g_f2[e][c][y][x] = sum over the levels whose floor grid holds (y >> l, x >> l) of H[e][c][off_l + (y >> l) w_l + (x >> l)] / 4^l
__global__ void __launch_bounds__(256) corr_adjoint_spread_kernel(const float* __restrict__ H, float* __restrict__ g2, long long total,
                                                                  int ht, int wd) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int HW = ht * wd;
  const long long ec = t / HW;
  const int pin = (int)(t - ec * HW), y = pin / wd, x = pin - y * wd;
  const float* h = H + (size_t)ec * Levels(ht, wd).Q;
  float s = h[pin];
#pragma unroll
  for (int l = 1; l < 4; l++) {
    h += (size_t)(ht >> (l - 1)) * (wd >> (l - 1));
    const int yl = y >> l, xl = x >> l;
    if (yl < (ht >> l) && xl < (wd >> l)) s += h[(size_t)yl * (wd >> l) + xl] * (1.0f / (float)(1 << (2 * l)));
  }
  g2[t] = s;
}

static size_t adjoint_buffer_bytes(int n, int C, int ht, int wd) {
  return ((size_t)n * C * Levels(ht, wd).Q * sizeof(float) + 255) & ~(size_t)255;
}

}  // namespace dba

using namespace dba;

static int check_train_shape(int n, int channels, int ht, int wd) {
  DBA_CHECK_ARG(n >= 0, "negative number of edges");
  DBA_CHECK_ARG(channels == 128, "128 feature channels expected (reference fnet)");
  DBA_CHECK_ARG(ht >= 8 && wd >= 8, "ht and wd must be at least 8 (level 3 must have at least one pixel)");
  DBA_CHECK_ARG(n <= 65535, "more than 65535 edges per call");
  DBA_CHECK_ARG((long long)((ht + 7) / 8) * ((wd + 7) / 8) <= 65535, "more than 65535 blocks of 8x8 pixels per feature map");
  return DBA_OK;
}

extern "C" int dba_corr_volume_pyramid_f32(const float* fmap1, const float* fmap2, float* out0, float* out1, float* out2, float* out3, int n,
                                           int channels, int ht, int wd, dba_stream_t stream) {
  int rc = check_train_shape(n, channels, ht, wd);
  if (rc) return rc;
  if (n == 0) return DBA_OK;
  DBA_CHECK_ARG(fmap1 && fmap2 && out0 && out1 && out2 && out3, "null pointer");
  const int nby = (ht + 7) / 8, nbx = (wd + 7) / 8;
  const dim3 grid((ht * wd + kCtTile - 1) / kCtTile, nby * nbx, n);
  corr_volume_f32_kernel<<<grid, kCtThreads, 0, (cudaStream_t)stream>>>(fmap1, fmap2, out0, out1, out2, out3, channels, ht, wd, nbx);
  DBA_CHECK_LAUNCH("corr_volume_pyramid_f32");
  return DBA_OK;
}

extern "C" int dba_corr_grad_accumulate(const float* coords, const float* grad, float* gpyr, int n, int ht, int wd, dba_stream_t stream) {
  DBA_CHECK_ARG(n >= 0, "negative number of edges");
  DBA_CHECK_ARG(ht >= 8 && wd >= 8, "ht and wd must be at least 8 (level 3 must have at least one pixel)");
  const long long total = (long long)n * ht * wd;
  if (total == 0) return DBA_OK;
  DBA_CHECK_ARG(coords && grad && gpyr, "null pointer");
  DBA_CHECK_ARG((total + 127) / 128 < 0x7fffffffLL, "too many pixels for one launch");
  corr_grad_accumulate_kernel<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)stream>>>(coords, grad, gpyr, total, ht, wd);
  DBA_CHECK_LAUNCH("corr_grad_accumulate");
  return DBA_OK;
}

extern "C" size_t dba_corr_adjoint_workspace_bytes(int n, int channels, int ht, int wd) {
  if (n <= 0 || channels <= 0 || ht <= 0 || wd <= 0) return 0;
  return 2 * adjoint_buffer_bytes(n, channels, ht, wd);
}

extern "C" int dba_corr_adjoint(const float* fmap1, const float* fmap2, const float* gpyr, float* grad1, float* grad2, int n, int channels,
                                int ht, int wd, void* workspace, size_t workspace_bytes, dba_stream_t stream) {
  int rc = check_train_shape(n, channels, ht, wd);
  if (rc) return rc;
  if (n == 0) return DBA_OK;
  DBA_CHECK_ARG(fmap1 && fmap2 && gpyr && grad1 && grad2, "null pointer");
  const size_t need = dba_corr_adjoint_workspace_bytes(n, channels, ht, wd);
  if (!workspace || workspace_bytes < need) {
    set_error("invalid argument: corr_adjoint needs a workspace of %zu bytes (dba_corr_adjoint_workspace_bytes), got %zu", need,
              workspace ? workspace_bytes : (size_t)0);
    return DBA_ERR_INVALID;
  }
  DBA_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const Levels L(ht, wd);
  const int HW = ht * wd;
  float* f2cat = (float*)workspace;
  float* H = (float*)((uint8_t*)workspace + adjoint_buffer_bytes(n, channels, ht, wd));
  const long long n_cat = (long long)n * channels * L.Q, n_map = (long long)n * channels * HW;
  corr_adjoint_pool_kernel<<<(unsigned)((n_cat + 255) / 256), 256, 0, st>>>(fmap2, f2cat, n_cat, ht, wd);
  DBA_CHECK_LAUNCH("corr_adjoint(pool)");
  // g_f1[c][p] = sum_k F2cat[c][k] G[p][k] / 16
  corr_adjoint_gemm_kernel<true><<<dim3((HW + kCtTile - 1) / kCtTile, (channels + kCtTile - 1) / kCtTile, n), kCtThreads, 0, st>>>(
      f2cat, gpyr, grad1, channels, HW, L.Q, 0.0625f);
  DBA_CHECK_LAUNCH("corr_adjoint(g1)");
  // H[c][k] = sum_p f1[c][p] G[p][k] / 16, then spread over each level's blocks
  corr_adjoint_gemm_kernel<false><<<dim3((unsigned)((L.Q + kCtTile - 1) / kCtTile), (channels + kCtTile - 1) / kCtTile, n), kCtThreads, 0, st>>>(
      fmap1, gpyr, H, channels, (int)L.Q, HW, 0.0625f);
  DBA_CHECK_LAUNCH("corr_adjoint(h)");
  corr_adjoint_spread_kernel<<<(unsigned)((n_map + 255) / 256), 256, 0, st>>>(H, grad2, n_map, ht, wd);
  DBA_CHECK_LAUNCH("corr_adjoint(g2)");
  return DBA_OK;
}
