// The feature and context encoders of DROID-SLAM as sm_90a kernels: BasicEncoder.forward (reference
// droid_slam/modules/extractor.py:118-198) for the two instances DroidNet builds (droid_net.py:149-150), fnet = BasicEncoder(128,
// 'instance') and cnet = BasicEncoder(256, 'none').  Every convolution runs on the implicit-GEMM engine of conv_engine.cuh:
//   * conv1 (7x7/2 on 3 channels): image_im2col_kernel writes, per output pixel, the 147 taps of the stride-2 window as one row
//     (pitch 152; the TMA box's out-of-bounds fill supplies zeros for K 147..191), then ONE 1x1 GEMM with N = 32;
//   * the stride-2 blocks (layer2.0, layer3.0): s2_gather_kernel writes the 9 taps of the 3x3/2 window at output resolution
//     (K = 9 C = 288 / 576), and conv1 and the 1x1/2 downsample run as ONE 1x1 GEMM with N = 2 planes: the downsample's input pixel
//     (2y, 2x) is the centre tap of that window, so its weights sit in the centre-tap K rows;
//   * 32-channel activations (stem output, layer1) are stored with a 32-channel pitch; the 64-channel TMA box reads zeros for K 32..63;
//   * instance norm (fnet): the conv epilogue EPI_STATS stores the raw f16 output plus per-16-pixel (mean, M2) slots from the fp32
//     accumulators, inorm_finalize_kernel merges the slots into mean / rstd per (image, channel), and inorm_act_kernel applies
//     relu(norm(a)) or relu(relu(norm(a)) + r), r = norm(b) (the downsample) or the block input;
//   * no norm (cnet): the epilogue EPI_RELU_RES applies the ReLU and the residual relu(x + relu(acc + bias)); no separate pass;
//   * conv2 (1x1 128 -> output_dim) writes NCHW f16 through EPI_NCHW.
#include "conv_engine.cuh"
#include <limits.h>

namespace dba {

constexpr int kStemTaps = 147;    // 7 x 7 taps x 3 channels
constexpr int kStemPitch = 152;   // im2col row pitch (16-byte rows)

// How uint8 camera frames are normalised on load (dba_encoder_forward_frames); unused for f32 / f16 images.
struct FrameNorm {
  int bgr;                  // source channel of RGB channel c: 2 - c (BGR frames) or c
  float inv255;             // 1.0f / 255.0f, rounded once in fp32 as ATen does for a division by a Python scalar
  float mean[3], stdv[3];   // per RGB channel
};

// tap (channel c, pixel off) of image e: f32 / f16 images as stored; uint8 frames normalised exactly like the reference's ATen
// sequence x / 255.0, .sub_(MEAN), .div_(STDV) on CUDA: a multiply by the fp32 reciprocal, a subtraction and an IEEE division, each
// rounded on its own (the _rn intrinsics keep the compiler from contracting the first two into an fma)
__device__ __forceinline__ float image_tap(const float* img, size_t plane, int c, size_t off, const FrameNorm&) { return img[c * plane + off]; }
__device__ __forceinline__ float image_tap(const __half* img, size_t plane, int c, size_t off, const FrameNorm&) {
  return __half2float(img[c * plane + off]);
}
__device__ __forceinline__ float image_tap(const uint8_t* img, size_t plane, int c, size_t off, const FrameNorm& f) {
  const float x = (float)img[(f.bgr ? 2 - c : c) * plane + off];
  return __fdiv_rn(__fsub_rn(__fmul_rn(x, f.inv255), f.mean[c]), f.stdv[c]);
}

// conv1's im2col: dst[(e*Ho*Wo + p) * 152 + (dy*7 + dx)*3 + c] = f16(img[e][c][2y+dy-3][2x+dx-3]) (0 outside; K 147..151 = 0).
// CTA = 64 output pixels of one output row; the 3 x 7 x 133 input halo goes through shared memory.
template <typename T>
__global__ void __launch_bounds__(256) image_im2col_kernel(const T* __restrict__ img, __half* __restrict__ dst, int H, int W, FrameNorm fn) {
  constexpr int kCols = 2 * 64 + 5;
  __shared__ float halo[3][7][kCols];
  const int e = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * 64;
  const int Ho = H >> 1, Wo = W >> 1;
  const size_t plane = (size_t)H * W;
  for (int i = threadIdx.x; i < 3 * 7 * kCols; i += 256) {
    const int c = i / (7 * kCols), r = (i - c * 7 * kCols) / kCols, col = i - c * 7 * kCols - r * kCols;
    const int yy = 2 * y + r - 3, xx = 2 * x0 + col - 3;
    float v = 0.f;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = image_tap(img + (size_t)e * 3 * plane, plane, c, (size_t)yy * W + xx, fn);
    halo[c][r][col] = v;
  }
  __syncthreads();
  const int npx = min(64, Wo - x0);
  __half* out = dst + ((size_t)e * Ho * Wo + (size_t)y * Wo + x0) * kStemPitch;
  for (int i = threadIdx.x; i < npx * (kStemPitch / 2); i += 256) {
    const int px = i / (kStemPitch / 2), k = 2 * (i - px * (kStemPitch / 2));
    float v[2];
#pragma unroll
    for (int q = 0; q < 2; q++) {
      const int kk = k + q, tap = kk / 3, c = kk - 3 * tap, dy = tap / 7, dx = tap - 7 * dy;
      v[q] = kk < kStemTaps ? halo[c][dy][2 * px + dx] : 0.f;
    }
    *reinterpret_cast<uint32_t*>(out + (size_t)i * 2) = pack_h2(v[0], v[1]);
  }
}

// 3x3 / stride 2 / pad 1 taps at output resolution: dst[((e*ho + y)*wo + x) * 9C + (dy*3 + dx)*C + c] = src[e][2y+dy-1][2x+dx-1][c]
// (0 outside); src channels-last [E][h][w][C], C % 8 == 0.  One thread = 8 channels of one tap.
__global__ void __launch_bounds__(256) s2_gather_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int C, int h, int w, long long total) {
  const long long id = (long long)blockIdx.x * 256 + threadIdx.x;
  if (id >= total) return;
  const int cg = C >> 3, ho = h >> 1, wo = w >> 1;
  const int q = (int)(id % cg);
  long long r = id / cg;
  const int t = (int)(r % 9); r /= 9;
  const int x = (int)(r % wo); r /= wo;
  const int y = (int)(r % ho);
  const long long e = r / ho;
  const int yy = 2 * y + t / 3 - 1, xx = 2 * x + t % 3 - 1;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (yy >= 0 && yy < h && xx >= 0 && xx < w) v = __ldg(reinterpret_cast<const uint4*>(src + ((e * h + yy) * w + xx) * C + q * 8));
  *reinterpret_cast<uint4*>(dst + id * 8) = v;
}

// Chan's pairwise update: (n, mean, m2) <- merge with (nb, mb, m2b)
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float mb, float m2b) {
  const float nab = n + nb, d = mb - mean, f = nb / nab;
  mean = fmaf(d, f, mean);
  m2 += m2b + d * d * n * f;
  n = nab;
}

// instance-norm statistics from the EPI_STATS slots: ms[e*N + c] = (mean, 1/sqrt(var + 1e-5)), biased variance.
// CTA = 32 channels (lanes) x 32 slot strides (warps) of one image.
__global__ void __launch_bounds__(1024) inorm_finalize_kernel(const float* __restrict__ partial, const float* __restrict__ counts, int slots, int N,
                                                               float2* __restrict__ ms) {
  __shared__ float3 red[32][32];
  const int e = blockIdx.y, lane = threadIdx.x, w = threadIdx.y, c = blockIdx.x * 32 + lane;
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (int s = w; s < slots; s += 32) {
    const float nb = __ldg(counts + (size_t)e * slots + s);
    if (nb > 0.f) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(partial + (((size_t)e * slots + s) * N + c) * 2));
      chan_merge(n, mean, m2, nb, b.x, b.y);
    }
  }
  red[w][lane] = make_float3(n, mean, m2);
  __syncthreads();
  if (w == 0) {
    for (int k = 1; k < 32; k++) {
      const float3 b = red[k][lane];
      if (b.x > 0.f) chan_merge(n, mean, m2, b.x, b.y, b.z);
    }
    ms[(size_t)e * N + c] = make_float2(mean, rsqrtf(m2 / n + 1e-5f));
  }
}

// out[pix][c] = relu(relu((a[pix][c] - mean_a[c]) * rstd_a[c]) + r), r = (b[pix][c] - mean_b[c]) * rstd_b[c] when b is set, x[pix][c]
// when x is set, else 0 (ResidualBlock: y = relu(norm2(conv2(.))), out = relu(x + y)); ms_* per image with the given strides.  All channels-last f16; one thread = 8 channels of one pixel.  out may be x.
__global__ void __launch_bounds__(256) inorm_act_kernel(const __half* __restrict__ a, int a_stride, const float2* __restrict__ ms_a, int msa_stride,
                                                        const __half* __restrict__ b, int b_stride, const float2* __restrict__ ms_b, int msb_stride,
                                                        const __half* x, int x_stride, __half* out, int out_stride, int C, int HW, long long total) {
  const long long id = (long long)blockIdx.x * 256 + threadIdx.x;
  if (id >= total) return;
  const int cg = C >> 3;
  const int c = (int)(id % cg) * 8;
  const long long pix = id / cg;
  const long long e = pix / HW;
  float v[8];
  {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(a + pix * a_stride + c));
    const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
    const float2* m = ms_a + e * msa_stride + c;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float2 f = unpack2(uw[k]), m0 = m[2 * k], m1 = m[2 * k + 1];
      v[2 * k] = relu_nan1((f.x - m0.x) * m0.y);
      v[2 * k + 1] = relu_nan1((f.y - m1.x) * m1.y);
    }
  }
  if (b) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(b + pix * b_stride + c));
    const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
    const float2* m = ms_b + e * msb_stride + c;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float2 f = unpack2(uw[k]), m0 = m[2 * k], m1 = m[2 * k + 1];
      v[2 * k] += (f.x - m0.x) * m0.y;
      v[2 * k + 1] += (f.y - m1.x) * m1.y;
    }
  } else if (x) {
    const uint4 u = *reinterpret_cast<const uint4*>(x + pix * x_stride + c);
    const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float2 f = unpack2(uw[k]);
      v[2 * k] += f.x;
      v[2 * k + 1] += f.y;
    }
  }
#pragma unroll
  for (int k = 0; k < 8; k++) v[k] = relu_nan1(v[k]);
  *reinterpret_cast<uint4*>(out + pix * out_stride + c) = make_uint4(pack_h2(v[0], v[1]), pack_h2(v[2], v[3]), pack_h2(v[4], v[5]), pack_h2(v[6], v[7]));
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
static size_t enc_al256(size_t x) { return (x + 255) & ~(size_t)255; }

// upper bound of launch_conv's EPI_STATS slot count at ht x wd (any MT: ceil(ht / (MT*RM)) * MT <= 2 ceil(ht / RM) for the MT it picks)
static size_t enc_slot_bound(int ht, int wd) {
  const int tw = (wd % 64 == 0) ? 64 : 32, rm = 128 / tw;
  return (size_t)((wd + tw - 1) / tw) * ((ht + rm - 1) / rm) * kSlotsPerMTile * 2;
}

struct EncWs { size_t big, act[4], partial, counts, ms[2], total, big_bytes, act_bytes, partial_bytes, counts_bytes, ms_bytes; };
static EncWs enc_layout(int E, int H, int W) {
  EncWs L;
  const int h1 = H / 2, w1 = W / 2, h2 = H / 4, w2 = W / 4, h3 = H / 8, w3 = W / 8;
  const size_t px1 = (size_t)E * h1 * w1, px2 = (size_t)E * h2 * w2, px3 = (size_t)E * h3 * w3;
  size_t big = px1 * kStemPitch;
  if (px2 * 288 > big) big = px2 * 288;
  if (px3 * 576 > big) big = px3 * 576;
  size_t stat_cols = enc_slot_bound(h1, w1) * 32;                 // slots x N of the widest statistics among the layers
  if (enc_slot_bound(h2, w2) * 128 > stat_cols) stat_cols = enc_slot_bound(h2, w2) * 128;
  if (enc_slot_bound(h3, w3) * 256 > stat_cols) stat_cols = enc_slot_bound(h3, w3) * 256;
  size_t o = 0;
  L.big_bytes = enc_al256(big * 2);
  L.act_bytes = enc_al256(px1 * 32 * 2);                           // the largest activation: [E][H/2][W/2][32] = [E][H/4][W/4][128]
  L.partial_bytes = enc_al256((size_t)E * stat_cols * 2 * 4);
  L.counts_bytes = enc_al256((size_t)E * enc_slot_bound(h1, w1) * 4);
  L.ms_bytes = enc_al256((size_t)E * 256 * 8);
  L.big = o; o += L.big_bytes;
  for (int k = 0; k < 4; k++) { L.act[k] = o; o += L.act_bytes; }
  L.partial = o; o += L.partial_bytes;
  L.counts = o; o += L.counts_bytes;
  for (int k = 0; k < 2; k++) { L.ms[k] = o; o += L.ms_bytes; }
  L.total = o;
  return L;
}

struct Enc {
  int E;
  cudaStream_t st;
  float* partial;
  float* counts;
  int limit;        // launches to run: the schedule stops launching after this many (dba_encoder_forward_prefix; 0 plans only)
  int launches;     // launches the schedule has reached so far
  int* plans;       // when set: [DBA_ENCODER_CONVS][5] = TW, MT, tiles_x, tiles_y, EPI_STATS slots (0 without statistics) per convolution
  int convs;        // convolutions reached so far
};

// every launch of the schedule asks this first, so a prefix and the launch count come from the one schedule
static bool enc_next(Enc& c) { return c.launches++ < c.limit; }

// one convolution of the encoder (E images of ht x wd, channels-last source)
template <int EPI>
static int enc_conv(Enc& c, int ht, int wd, int ks, ConvSrc src, const void* w, const float* b, int N, __half* out, int out_stride,
                    int relu_cols = 0, const __half* res = nullptr, int res_stride = 0, int* slots = nullptr) {
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.E = c.E; p.HT = ht; p.WD = wd; p.n_ntiles = 1; p.KS = ks; p.N = N; p.bias = b;
  p.out = out; p.out_stride = out_stride; p.relu_cols = relu_cols; p.h = res; p.h_stride = res_stride;
  p.partial = c.partial; p.counts = c.counts;
  if (EPI == EPI_NCHW) { p.nchw = out; p.nchw_C = N; }
  const int k = c.convs++;
  if (enc_next(c)) return launch_conv<EPI>(p, src, ConvSrc{nullptr, 0, 0}, w, c.st, slots);
  bool flat = false;
  int box_rows = 0;
  const int rc = conv_plan(p, src.C, 0, false, &flat, &box_rows); if (rc) return rc;      // the tiling launch_conv would take
  if (slots) *slots = p.slots;
  if (c.plans) {
    const int v[5] = {p.TW, p.MT, p.tiles_x, p.tiles_y, EPI == EPI_STATS ? p.slots : 0};
    memcpy(c.plans + 5 * k, v, sizeof(v));
  }
  return DBA_OK;
}

// convolution + instance-norm statistics: raw f16 output in out, ms[e*N + n] = (mean, rstd)
static int enc_conv_stats(Enc& c, int ht, int wd, int ks, ConvSrc src, const void* w, const float* b, int N, __half* out, float2* ms) {
  int slots = 0;
  int rc = enc_conv<EPI_STATS>(c, ht, wd, ks, src, w, b, N, out, N, 0, nullptr, 0, &slots);
  if (rc) return rc;
  if (!enc_next(c)) return DBA_OK;
  inorm_finalize_kernel<<<dim3(N / 32, c.E), dim3(32, 32), 0, c.st>>>(c.partial, c.counts, slots, N, ms);
  DBA_CHECK_LAUNCH("inorm_finalize_kernel");
  return DBA_OK;
}

static int enc_act(Enc& c, const __half* a, int a_stride, const float2* ms_a, int msa_stride, const __half* b, int b_stride, const float2* ms_b,
                   int msb_stride, const __half* x, int x_stride, __half* out, int out_stride, int C, int HW) {
  const long long total = (long long)c.E * HW * (C / 8);
  if (!enc_next(c)) return DBA_OK;
  inorm_act_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c.st>>>(a, a_stride, ms_a, msa_stride, b, b_stride, ms_b, msb_stride, x, x_stride, out,
                                                                     out_stride, C, HW, total);
  DBA_CHECK_LAUNCH("inorm_act_kernel");
  return DBA_OK;
}

// ResidualBlock(P, P, stride 1) (extractor.py:47-55) on X [E][ht][wd][P], result written back into X; T1, T2 scratch
static int enc_block_s1(Enc& c, bool inorm, int ht, int wd, int P, __half* X, __half* T1, __half* T2, float2* msA, float2* msB,
                        const void* w1, const float* b1, const void* w2, const float* b2) {
  int rc;
  if (inorm) {
    if ((rc = enc_conv_stats(c, ht, wd, 3, ConvSrc{X, P, P}, w1, b1, P, T1, msA))) return rc;
    if ((rc = enc_act(c, T1, P, msA, P, nullptr, 0, nullptr, 0, nullptr, 0, T2, P, P, ht * wd))) return rc;
    if ((rc = enc_conv_stats(c, ht, wd, 3, ConvSrc{T2, P, P}, w2, b2, P, T1, msB))) return rc;
    return enc_act(c, T1, P, msB, P, nullptr, 0, nullptr, 0, X, P, X, P, P, ht * wd);
  }
  if ((rc = enc_conv<EPI_RELU_RES>(c, ht, wd, 3, ConvSrc{X, P, P}, w1, b1, P, T1, P, P))) return rc;
  return enc_conv<EPI_RELU_RES>(c, ht, wd, 3, ConvSrc{T1, P, P}, w2, b2, P, X, P, P, X, P);
}

// ResidualBlock(Cin, P, stride 2) on X [E][ht][wd][Cin] -> X [E][ht/2][wd/2][P].  conv1 and the downsample are one GEMM on the gathered
// taps, output T1 [.][2P] = conv1 | downsample; T2 scratch
static int enc_block_s2(Enc& c, bool inorm, int ht, int wd, int Cin, int P, __half* X, __half* big, __half* T1, __half* T2, float2* msA, float2* msB,
                        const void* w1, const float* b1, const void* w2, const float* b2) {
  const int ho = ht / 2, wo = wd / 2;
  const long long total = (long long)c.E * ho * wo * 9 * (Cin / 8);
  if (enc_next(c)) {
    s2_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c.st>>>(X, big, Cin, ht, wd, total);
    DBA_CHECK_LAUNCH("s2_gather_kernel");
  }
  const ConvSrc taps{big, 9 * Cin, 9 * Cin};
  int rc;
  if (inorm) {
    if ((rc = enc_conv_stats(c, ho, wo, 1, taps, w1, b1, 2 * P, T1, msA))) return rc;
    if ((rc = enc_act(c, T1, 2 * P, msA, 2 * P, nullptr, 0, nullptr, 0, nullptr, 0, T2, P, P, ho * wo))) return rc;
    if ((rc = enc_conv_stats(c, ho, wo, 3, ConvSrc{T2, P, P}, w2, b2, P, X, msB))) return rc;
    return enc_act(c, X, P, msB, P, T1 + P, 2 * P, msA + P, 2 * P, nullptr, 0, X, P, P, ho * wo);
  }
  if ((rc = enc_conv<EPI_RELU_RES>(c, ho, wo, 1, taps, w1, b1, 2 * P, T1, 2 * P, P))) return rc;
  return enc_conv<EPI_RELU_RES>(c, ho, wo, 3, ConvSrc{T1, P, 2 * P}, w2, b2, P, X, P, P, T1 + P, 2 * P);
}

// the schedule of both encoders: launches its first `limit` kernels (limit 0: none, the tilings and the launch count only, with a
// null workspace) and reports how many it has in all and, in plans, each convolution's tiling.  frames set: a->images are uint8
// camera frames normalised on load by that format.
static int enc_forward(const dba_encoder_args* a, int limit, int* n_launches, int* plans, const dba_frame_format* frames = nullptr) {
  const int E = a->n_images, H = a->H, W = a->W;
  const dba_encoder_weights* Wt = a->weights;
  const EncWs L = enc_layout(E, H, W);
  cudaStream_t st = (cudaStream_t)a->stream;
  uint8_t* ws = (uint8_t*)a->workspace;
  __half* big = (__half*)(ws + L.big);
  __half* X = (__half*)(ws + L.act[0]);     // block input / output
  __half* T1 = (__half*)(ws + L.act[1]);
  __half* T2 = (__half*)(ws + L.act[2]);
  float2* msA = (float2*)(ws + L.ms[0]);
  float2* msB = (float2*)(ws + L.ms[1]);
  Enc c{E, st, (float*)(ws + L.partial), (float*)(ws + L.counts), limit, 0, plans, 0};
  const bool inorm = a->norm == 1;
  const int h1 = H / 2, w1 = W / 2;
  int rc;
  // conv1 7x7/2 3->32, norm1, relu1 (extractor.py:187-189)
  if (enc_next(c)) {
    const dim3 g((w1 + 63) / 64, h1, E);
    FrameNorm fn;
    memset(&fn, 0, sizeof(fn));
    if (frames) {
      fn.bgr = frames->channel_order == DBA_FRAME_BGR;
      fn.inv255 = 1.0f / 255.0f;
      for (int c = 0; c < 3; c++) { fn.mean[c] = frames->mean[c]; fn.stdv[c] = frames->std[c]; }
      image_im2col_kernel<uint8_t><<<g, 256, 0, st>>>((const uint8_t*)a->images, big, H, W, fn);
    } else if (a->images_dtype == DBA_F32) {
      image_im2col_kernel<float><<<g, 256, 0, st>>>((const float*)a->images, big, H, W, fn);
    } else {
      image_im2col_kernel<__half><<<g, 256, 0, st>>>((const __half*)a->images, big, H, W, fn);
    }
    DBA_CHECK_LAUNCH("image_im2col_kernel");
  }
  const ConvSrc stem{big, kStemTaps, kStemPitch};
  if (inorm) {
    if ((rc = enc_conv_stats(c, h1, w1, 1, stem, Wt->w[0], Wt->b[0], 32, T1, msA))) return rc;
    if ((rc = enc_act(c, T1, 32, msA, 32, nullptr, 0, nullptr, 0, nullptr, 0, X, 32, 32, h1 * w1))) return rc;
  } else if ((rc = enc_conv<EPI_RELU_RES>(c, h1, w1, 1, stem, Wt->w[0], Wt->b[0], 32, X, 32, 32))) {
    return rc;
  }
  // layer1, layer2, layer3 (:191-193)
  for (int k = 1; k <= 3; k += 2)
    if ((rc = enc_block_s1(c, inorm, h1, w1, 32, X, T1, T2, msA, msB, Wt->w[k], Wt->b[k], Wt->w[k + 1], Wt->b[k + 1]))) return rc;
  if ((rc = enc_block_s2(c, inorm, h1, w1, 32, 64, X, big, T1, T2, msA, msB, Wt->w[5], Wt->b[5], Wt->w[6], Wt->b[6]))) return rc;
  if ((rc = enc_block_s1(c, inorm, H / 4, W / 4, 64, X, T1, T2, msA, msB, Wt->w[7], Wt->b[7], Wt->w[8], Wt->b[8]))) return rc;
  if ((rc = enc_block_s2(c, inorm, H / 4, W / 4, 64, 128, X, big, T1, T2, msA, msB, Wt->w[9], Wt->b[9], Wt->w[10], Wt->b[10]))) return rc;
  if ((rc = enc_block_s1(c, inorm, H / 8, W / 8, 128, X, T1, T2, msA, msB, Wt->w[11], Wt->b[11], Wt->w[12], Wt->b[12]))) return rc;
  // conv2 1x1 128->output_dim, NCHW f16 (:195)
  rc = enc_conv<EPI_NCHW>(c, H / 8, W / 8, 1, ConvSrc{X, 128, 128}, Wt->w[13], Wt->b[13], a->output_dim, (__half*)a->out, 0);
  if (n_launches) *n_launches = c.launches;
  return rc;
}

}  // namespace dba
using namespace dba;

extern "C" size_t dba_encoder_workspace_bytes(int n_images, int H, int W, int output_dim) {
  if (n_images < 1 || H <= 0 || W <= 0 || H % 8 || W % 8 || (output_dim != 128 && output_dim != 256)) return 0;
  return enc_layout(n_images, H, W).total;
}

extern "C" int dba_encoder_workspace_layout(int n_images, int H, int W, int norm, size_t* offsets, size_t* sizes, int* n_launches, int* plans) {
  DBA_CHECK_ARG(offsets && sizes && n_launches && plans, "null pointer");
  DBA_CHECK_ARG(n_images > 0 && H > 0 && W > 0 && H % 8 == 0 && W % 8 == 0, "encoder: n_images must be positive and H, W positive multiples of 8");
  DBA_CHECK_ARG(norm == 0 || norm == 1, "encoder: norm must be 0 (none) or 1 (instance)");
  const EncWs L = enc_layout(n_images, H, W);
  const size_t off[DBA_ENCWS_COUNT] = {L.big, L.act[0], L.act[1], L.act[2], L.partial, L.counts, L.ms[0], L.ms[1]};
  const size_t sz[DBA_ENCWS_COUNT] = {L.big_bytes, L.act_bytes, L.act_bytes, L.act_bytes, L.partial_bytes, L.counts_bytes, L.ms_bytes, L.ms_bytes};
  memcpy(offsets, off, sizeof(off));
  memcpy(sizes, sz, sizeof(sz));
  dba_encoder_weights none;
  memset(&none, 0, sizeof(none));
  dba_encoder_args a;
  memset(&a, 0, sizeof(a));
  a.n_images = n_images; a.H = H; a.W = W; a.norm = norm; a.output_dim = norm ? 128 : 256; a.weights = &none;
  return enc_forward(&a, 0, n_launches, plans);
}

static int enc_checked(const dba_encoder_args* a, int n_launches, const dba_frame_format* frames) {
  DBA_CHECK_ARG(a, "null args");
  const int E = a->n_images, H = a->H, W = a->W;
  DBA_CHECK_ARG(n_launches >= 0, "encoder: negative launch count");
  DBA_CHECK_ARG(E > 0 && H > 0 && W > 0 && H % 8 == 0 && W % 8 == 0, "encoder: n_images must be positive and H, W positive multiples of 8");
  DBA_CHECK_ARG(a->norm == 0 || a->norm == 1, "encoder: norm must be 0 (none) or 1 (instance)");
  DBA_CHECK_ARG(a->output_dim == 128 || a->output_dim == 256, "encoder: output_dim must be 128 or 256");
  if (frames)
    DBA_CHECK_ARG(frames->channel_order == DBA_FRAME_RGB || frames->channel_order == DBA_FRAME_BGR, "encoder: channel_order must be DBA_FRAME_RGB or DBA_FRAME_BGR");
  else
    DBA_CHECK_ARG(a->images_dtype == DBA_F32 || a->images_dtype == DBA_F16, "encoder: images must be DBA_F32 or DBA_F16");
  DBA_CHECK_ARG(a->images && a->weights && a->out && a->workspace, "null pointer");
  const dba_encoder_weights* Wt = a->weights;
  for (int k = 0; k < DBA_ENCODER_CONVS; k++)
    DBA_CHECK_ARG(Wt->w[k] && Wt->b[k] && ((uintptr_t)Wt->w[k] & 15) == 0, "encoder: packed weights must be non-null, w[k] 16-byte aligned");
  if (a->workspace_bytes < enc_layout(E, H, W).total) { set_error("invalid argument: workspace too small (dba_encoder_workspace_bytes)"); return DBA_ERR_WORKSPACE; }
  DBA_CHECK_ARG(((uintptr_t)a->workspace & 255) == 0, "encoder: workspace must be 256-byte aligned");
  return enc_forward(a, n_launches, nullptr, nullptr, frames);
}

extern "C" int dba_encoder_forward_prefix(const dba_encoder_args* a, int n_launches) { return enc_checked(a, n_launches, nullptr); }

extern "C" int dba_encoder_forward(const dba_encoder_args* a) { return enc_checked(a, INT_MAX, nullptr); }

extern "C" int dba_encoder_forward_frames(const dba_encoder_args* a, const dba_frame_format* f) {
  DBA_CHECK_ARG(f, "encoder: null frame format");
  return enc_checked(a, INT_MAX, f);
}
