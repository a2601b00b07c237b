// The update operator of DROID-SLAM (SURVEY section 8a row A6) as hand-written sm_90a kernels:
//   UpdateModule.forward   reference droid_slam/droid_net.py:111-143  (encoders :83-93, heads :95-106)
//   ConvGRU.forward        reference droid_slam/modules/gru.py:19-32
//   GraphAgg.forward       reference droid_slam/droid_net.py:59-75
//
// Every convolution is an implicit GEMM on the Hopper tensor cores (wgmma) -- no im2col buffer, no library call:
//   * activations live channels-last ([image, y, x, C], f16), so a tile of 128 pixels x 64 channels is a K-major operand
//     with 128-byte rows; a 3x3 tap (dy,dx) is the same tile shifted by one pixel, which TMA delivers with the zero padding
//     for free (cp.async.bulk.tensor.4d with out-of-bounds fill at negative / beyond-the-edge coordinates);
//   * per (64-channel block, dx) ONE halo tile of (rows + 2) image rows is loaded and the three dy taps are the same
//     shared-memory buffer at +dy*TW*128 bytes (a multiple of the 1024-byte swizzle atom), so a 3x3 convolution reads its
//     input 3x (not 9x) from L2; widths that are not a multiple of 8 take row-flattened tiles instead (128 consecutive pixels of
//     the image on a row pitch rounded up to 8, conv_engine.cuh), so odd widths cost ~1.1x, not ~1.5x, the tensor work they need;
//   * weights are pre-packed [tap][N][K] f16 (K contiguous) and stream through a second TMA ring;
//   * wgmma.m64nNk16 (f16 operands from shared memory, fp32 accumulators in registers), N = the output channels of the tile
//     (up to 256; 384 outputs run as two 192-wide N tiles), M = 128 pixels per tile (x MT tiles sharing every weight stage);
//     persistent CTAs (one per SM) with a static tile schedule: warp 8 = TMA producer (runs ahead across tiles), warps 0..7 =
//     two consumer warpgroups, warpgroup w computing pixels 64 w .. 64 w + 63 of every M tile and running its own epilogue
//     straight from the register fragment while the producer already streams the next tile's operands;
//   * the epilogues fuse everything elementwise: bias, ReLU, the GRU gates (z, r*h, tanh, (1-z)h + zq), the gated global
//     context sum, sigmoid / softplus of the heads and the NCHW layout of the upsampling mask.
// Segment mean (GraphAgg's scatter_mean), the 7x7 flow encoder's im2col (4 input channels: 49 taps x 4 = one 196-wide K),
// the global-context mat-vec and the NCHW -> channels-last transposes are small SIMT kernels around it.
#include "conv_engine.cuh"

namespace dba {

// ---------------------------------------------------------------------------------------------------------------------------
// small SIMT kernels around the tensor-core convolutions
// ---------------------------------------------------------------------------------------------------------------------------

// [E][C][HW] (f16 or f32) -> channels-last f16 dst[(e*HW + p) * dst_stride + c] for c < cwrite (channels C..cwrite-1 are zeros).
// 64 channels x 64 pixels per CTA; a thread loads a 2 x 2 (channel pair x pixel pair) patch, transposes it in registers and parks
// the two channel-pair words in shared memory, so that both the global loads (pixel pairs of one channel row) and the global stores
// (channel pairs of one pixel) are 4-byte lanes of 128-byte rows.
template <typename T> struct Load2;
template <> struct Load2<__half> {
  static __device__ __forceinline__ float2 ld(const __half* p, bool ok0, bool ok1, bool aligned) {
    if (ok1 && aligned) return __half22float2(*reinterpret_cast<const __half2*>(p));
    return make_float2(ok0 ? __half2float(p[0]) : 0.f, ok1 ? __half2float(p[1]) : 0.f);
  }
};
template <> struct Load2<float> {
  static __device__ __forceinline__ float2 ld(const float* p, bool ok0, bool ok1, bool aligned) {
    if (ok1 && aligned) return *reinterpret_cast<const float2*>(p);
    return make_float2(ok0 ? p[0] : 0.f, ok1 ? p[1] : 0.f);
  }
};
template <typename T>
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const T* __restrict__ src, __half* __restrict__ dst, int C, int HW, int dst_stride, int cwrite) {
  __shared__ uint32_t tile[2][64][33];                      // [channel block][pixel][channel pair]
  // a CTA moves TWO 64-channel blocks of a 64-pixel tile: 16 loads per thread are in flight before the first use, and a pixel's
  // output row is one 256-byte run
  const int e = blockIdx.z, p0 = blockIdx.x * 64;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const bool even = (HW & 1) == 0;                           // pixel pairs are 4 / 8-byte aligned when HW is even
  float2 va[2][4], vb[2][4];
#pragma unroll
  for (int cbk = 0; cbk < 2; cbk++) {
    const int c0 = (blockIdx.y * 2 + cbk) * 64;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int cp = w + 8 * k;                              // channel pair 0..31
      const int c = c0 + 2 * cp, pp = p0 + 2 * lane;
      va[cbk][k] = make_float2(0.f, 0.f); vb[cbk][k] = make_float2(0.f, 0.f);
      if (c < C && pp < HW) va[cbk][k] = Load2<T>::ld(src + ((size_t)e * C + c) * HW + pp, true, pp + 1 < HW, even);
      if (c + 1 < C && pp < HW) vb[cbk][k] = Load2<T>::ld(src + ((size_t)e * C + c + 1) * HW + pp, true, pp + 1 < HW, even);
    }
  }
#pragma unroll
  for (int cbk = 0; cbk < 2; cbk++)
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int cp = w + 8 * k;
      tile[cbk][2 * lane][cp] = pack_h2(va[cbk][k].x, vb[cbk][k].x);
      tile[cbk][2 * lane + 1][cp] = pack_h2(va[cbk][k].y, vb[cbk][k].y);
    }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int px = w + 8 * k, pp = p0 + px;
#pragma unroll
    for (int cbk = 0; cbk < 2; cbk++) {
      const int c = (blockIdx.y * 2 + cbk) * 64 + 2 * lane;
      if (pp < HW && c < cwrite) *reinterpret_cast<uint32_t*>(dst + ((size_t)e * HW + pp) * dst_stride + c) = tile[cbk][px][lane];   // cwrite and strides are even
    }
  }
}

// 7x7 / 4-channel flow encoder input as one 196-wide K: dst[(e*HW + p) * 200 + (dy*7+dx)*4 + c] = flow[e][c][y+dy-3][x+dx-3] (0 outside;
// slot 49 = the 4 zero padding channels).  CTA = 64 pixels of one image row: the 4 x 7 x 70 halo goes through shared memory
// (coalesced row loads), the 64 x 400-byte output rows leave as consecutive 8-byte lanes.
__global__ void __launch_bounds__(256) flow_im2col_kernel(const float* __restrict__ flow, __half* __restrict__ dst, int HT, int WD) {
  __shared__ float halo[4][7][72];
  const int e = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * 64;
  const int HW = HT * WD;
  for (int i = threadIdx.x; i < 4 * 7 * 70; i += 256) {
    const int c = i / 490, r = (i - c * 490) / 70, col = i - c * 490 - r * 70;
    const int yy = y + r - 3, xx = x0 + col - 3;
    float v = 0.f;
    if (flow && yy >= 0 && yy < HT && xx >= 0 && xx < WD) v = __ldg(flow + ((size_t)e * 4 + c) * HW + (size_t)yy * WD + xx);
    halo[c][r][col] = v;
  }
  __syncthreads();
  const int npx = min(64, WD - x0);
  __half* out = dst + ((size_t)e * HW + (size_t)y * WD + x0) * 200;
  for (int i = threadIdx.x; i < npx * 50; i += 256) {
    const int px = i / 50, slot = i - px * 50;
    uint2 o = make_uint2(0u, 0u);
    if (slot < 49) {
      const int dy = slot / 7, dx = slot - dy * 7;
      o = make_uint2(pack_h2(halo[0][dy][px + dx], halo[1][dy][px + dx]), pack_h2(halo[2][dy][px + dx], halo[3][dy][px + dx]));
    }
    *reinterpret_cast<uint2*>(out + (size_t)i * 4) = o;
  }
}

// The 3x3 convolutions with 1-2 output channels (delta.2, weight.2, agg.eta.0) are computed as ONE 1x1 convolution that produces, per
// pixel, the 9 per-tap partial sums of every output (Y[p][t*no + o] = sum_c act[p][c] w[t][o][c]; on the tensor cores, the input is read
// once instead of three times), followed by this gather: out[p][o] = bias[o] + sum_t Y[p + shift_t][t*no + o] (zero outside the image).
// mode 0: no = 4 -> delta (o = 0,1) and sigmoid weight (o = 2,3), [img,ht,wd,2] each;  mode 1: no = 1 -> eta = 0.01 * softplus
__global__ void __launch_bounds__(256) head_gather_kernel(const float* __restrict__ Y, int ystride, int no, const float* __restrict__ bias, int mode,
                                                          float* __restrict__ out_a, float* __restrict__ out_b, int n_img, int HT, int WD) {
  const long long total = (long long)n_img * HT * WD;
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= total) return;
  const int HW = HT * WD;
  const int pin = (int)(id % HW);
  const long long img = id / HW;
  const int y = pin / WD, x = pin - y * WD;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int t = 0; t < 9; t++) {
    const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
    if (yy < 0 || yy >= HT || xx < 0 || xx >= WD) continue;
    const float* q = Y + ((size_t)img * HW + (size_t)yy * WD + xx) * ystride + t * no;
    if (no == 4) { const float4 v = __ldg(reinterpret_cast<const float4*>(q)); acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w; }
    else acc[0] += __ldg(q);
  }
  if (mode == 0) {
    *reinterpret_cast<float2*>(out_a + (size_t)id * 2) = make_float2(acc[0] + bias[0], acc[1] + bias[1]);
    *reinterpret_cast<float2*>(out_b + (size_t)id * 2) = make_float2(1.f / (1.f + __expf(-(acc[2] + bias[2]))), 1.f / (1.f + __expf(-(acc[3] + bias[3]))));
  } else {
    const float xx = acc[0] + bias[0];
    out_a[id] = 0.01f * (xx > 20.f ? xx : log1pf(__expf(xx)));     // torch Softplus(beta = 1, threshold = 20)
  }
}

// global context (gru.py:25-30): g = mean over pixels of sigmoid(w(h)) * h (from the EPI_GATE partial sums), then the three 1x1
// convolutions on g as one [384 x 128] mat-vec per edge -> glo[e][384] = z | r | q terms
__global__ void __launch_bounds__(384) glo_kernel(const float* __restrict__ partial, int slots, float inv_hw, const float* __restrict__ wg /*[384][128]*/,
                                                  const float* __restrict__ bg, float* __restrict__ glo) {
  __shared__ float g[128];
  const int e = blockIdx.x;
  if (threadIdx.x < 128) {
    float s = 0.f;
    for (int k = 0; k < slots; k++) s += partial[((size_t)e * slots + k) * 128 + threadIdx.x];
    g[threadIdx.x] = s * inv_hw;
  }
  __syncthreads();
  const float* w = wg + (size_t)threadIdx.x * 128;
  float acc = bg[threadIdx.x];
#pragma unroll 8
  for (int k = 0; k < 128; k++) acc = fmaf(__ldg(w + k), g[k], acc);
  glo[(size_t)e * 384 + threadIdx.x] = acc;
}

// CSR of the edges by aggregation segment (segment = rank of the source frame among the distinct sources, ascending), edge order kept
__global__ void seg_csr_kernel(const int64_t* __restrict__ ix, int E, int n_seg, int* __restrict__ seg_ptr, int* __restrict__ seg_edges) {
  extern __shared__ int cnt[];
  for (int s = threadIdx.x; s < n_seg; s += blockDim.x) {
    int c = 0;
    for (int e = 0; e < E; e++) c += ((int)ix[e] == s);
    cnt[s] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0;
    for (int s = 0; s < n_seg; s++) { seg_ptr[s] = a; a += cnt[s]; }
    seg_ptr[n_seg] = a;
  }
  __syncthreads();
  for (int s = threadIdx.x; s < n_seg; s += blockDim.x) {
    int o = seg_ptr[s];
    for (int e = 0; e < E; e++) if ((int)ix[e] == s) seg_edges[o++] = e;
  }
}

// scatter_mean over edges with equal source frame (droid_net.py:63-67): src channels-last with stride src_stride, dst [n_seg][HW][128]
__global__ void __launch_bounds__(256) segment_mean_kernel(const __half* __restrict__ src, int src_stride, const int* __restrict__ seg_ptr,
                                                           const int* __restrict__ seg_edges, __half* __restrict__ dst, int HW) {
  const int s = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;     // (pixel, 8-channel group)
  if (i >= HW * 16) return;
  const int pp = i >> 4, cg = (i & 15) * 8;
  const int b = seg_ptr[s], en = seg_ptr[s + 1];
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int k = b; k < en; k++) {
    const int e = seg_edges[k];
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(src + ((size_t)e * HW + pp) * src_stride + cg));
    float2 a = unpack2(u.x), bb = unpack2(u.y), c = unpack2(u.z), d = unpack2(u.w);
    acc[0] += a.x; acc[1] += a.y; acc[2] += bb.x; acc[3] += bb.y; acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
  }
  const float inv = en > b ? 1.f / (float)(en - b) : 0.f;
  *reinterpret_cast<uint4*>(dst + ((size_t)s * HW + pp) * 128 + cg) =
      make_uint4(pack_h2(acc[0] * inv, acc[1] * inv), pack_h2(acc[2] * inv, acc[3] * inv), pack_h2(acc[4] * inv, acc[5] * inv), pack_h2(acc[6] * inv, acc[7] * inv));
}


static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

// byte offsets of the intermediates in the caller's workspace; yh ([E,HW,36] f32 head partials) reuses cc and ye ([n_src,HW,12] f32
// eta partials) reuses f0, both dead by then.  The fields up to b2 are in the order of DBA_UPWS_* (droid_b200.h).
struct UpWs {
  size_t hin, x320, cc, f0, c1, f1, z, rh, s, partial, glo, am, b2, yh, ye, segptr, segedges, total;
};
static UpWs up_layout(int E, int n_src, int ht, int wd) {
  UpWs w;
  const size_t px = (size_t)E * ht * wd, spx = (size_t)(n_src > 0 ? n_src : 1) * ht * wd;
  const int tw = (wd % 64 == 0) ? 64 : 32, rm = 128 / tw;
  size_t slots = (size_t)((wd + tw - 1) / tw) * ((ht + rm - 1) / rm) * kSlotsPerMTile * 2;   // upper bound over MT
  if (wd % 8 != 0) {
    // row-flattened tiles (launch_conv): ceil(P / (128 MT)) CTA tiles of MT M tiles, P = ht * (wd rounded up to 8), so at most
    // ceil(P / 128) + MT - 1 <= ceil(P / 128) + 3 M tiles
    const size_t flat = ((size_t)ht * ((wd + 7) & ~7) + 127) / 128 + 3;
    if (flat * kSlotsPerMTile > slots) slots = flat * kSlotsPerMTile;
  }
  size_t o = 0;
  w.hin = o; o += al256(px * 128 * 2);
  w.x320 = o; o += al256(px * 320 * 2);
  w.cc = o; o += al256(px * 200 * 2);
  w.f0 = o; o += al256(px * 200 * 2);
  w.c1 = o; o += al256(px * 128 * 2);
  w.f1 = o; o += al256(px * 128 * 2);
  w.z = o; o += al256(px * 128 * 2);
  w.rh = o; o += al256(px * 128 * 2);
  w.s = o; o += al256(px * 384 * 2);
  w.partial = o; o += al256((size_t)E * slots * 128 * 4);
  w.glo = o; o += al256((size_t)E * 384 * 4);
  w.am = o; o += al256(spx * 128 * 2);
  w.b2 = o; o += al256(spx * 128 * 2);
  w.yh = w.cc;
  w.ye = w.f0;
  w.segptr = o; o += al256((size_t)(n_src + 2) * 4);
  w.segedges = o; o += al256((size_t)(E + 1) * 4);
  w.total = o;
  return w;
}

// the extents every convolution of the operator starts from, and the ConvGRU gate convolution (1x1 128 -> 128, EPI_GATE) built on
// them: dba_update_forward launches it and dba_update_workspace_layout plans it, so both count the same partial-sum slots
static ConvParams up_base(int E, int ht, int wd) {
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.E = E; p.HT = ht; p.WD = wd; p.n_ntiles = 1;
  return p;
}
static ConvParams gate_conv(const ConvParams& base) { ConvParams p = base; p.KS = 1; p.N = 128; return p; }

}  // namespace dba
using namespace dba;

extern "C" size_t dba_update_workspace_bytes(int n_edges, int n_src, int ht, int wd) {
  if (n_edges <= 0 || ht <= 0 || wd <= 0) return 0;
  return up_layout(n_edges, n_src, ht, wd).total;
}

extern "C" int dba_update_workspace_layout(int n_edges, int n_src, int ht, int wd, size_t* offsets, int* gate_slots) {
  DBA_CHECK_ARG(offsets && gate_slots, "null pointer");
  DBA_CHECK_ARG(n_edges > 0 && ht > 0 && wd > 0 && n_src >= 0, "bad extents");
  const UpWs L = up_layout(n_edges, n_src, ht, wd);
  const size_t v[DBA_UPWS_COUNT] = {L.hin, L.x320, L.cc, L.f0, L.c1, L.f1, L.z, L.rh, L.s, L.partial, L.glo, L.am, L.b2, L.yh, L.ye};
  memcpy(offsets, v, sizeof(v));
  ConvParams p = gate_conv(up_base(n_edges, ht, wd));
  bool flat = false;
  int box_rows = 0;
  int rc = conv_plan(p, 128, 0, true, &flat, &box_rows); if (rc) return rc;
  *gate_slots = p.slots;
  return DBA_OK;
}

extern "C" int dba_update_forward(const dba_update_args* a) {
  DBA_CHECK_ARG(a, "null args");
  const int E = a->n_edges, ht = a->ht, wd = a->wd, n_src = a->n_src;
  DBA_CHECK_ARG(E >= 0 && ht > 0 && wd > 0 && n_src >= 0, "bad extents");
  if (E == 0) return DBA_OK;
  DBA_CHECK_ARG(a->net && a->inp && a->corr && a->net_out && a->delta && a->weight && a->weights && a->workspace, "null pointer");
  DBA_CHECK_ARG(n_src == 0 || (a->seg && a->eta && a->upmask), "aggregation outputs / segment ids missing");
  const UpWs L = up_layout(E, n_src, ht, wd);
  DBA_CHECK_ARG(a->workspace_bytes >= L.total, "workspace too small (dba_update_workspace_bytes)");
  DBA_CHECK_ARG(((uintptr_t)a->workspace & 255) == 0 && ((uintptr_t)a->net_out & 15) == 0 && ((uintptr_t)a->net & 15) == 0, "pointers must be 16-byte aligned (workspace 256)");
  cudaStream_t st = (cudaStream_t)a->stream;
  uint8_t* ws = (uint8_t*)a->workspace;
  const dba_update_weights* W = a->weights;
  const int HW = ht * wd;
  __half* X = (__half*)(ws + L.x320);
  __half* Cc = (__half*)(ws + L.cc);
  __half* F0 = (__half*)(ws + L.f0);
  __half* C1 = (__half*)(ws + L.c1);
  __half* F1 = (__half*)(ws + L.f1);
  __half* Z = (__half*)(ws + L.z);
  __half* RH = (__half*)(ws + L.rh);
  __half* S = (__half*)(ws + L.s);
  float* partial = (float*)(ws + L.partial);
  float* glo = (float*)(ws + L.glo);
  __half* Am = (__half*)(ws + L.am);
  __half* B2 = (__half*)(ws + L.b2);
  int* seg_ptr = (int*)(ws + L.segptr);
  int* seg_edges = (int*)(ws + L.segedges);

  // ---- layout changes into channels-last f16 --------------------------------------------------------------------------
  const dim3 tgrid128((HW + 63) / 64, 1, E);
  const __half* H;      // hidden state, channels-last [E][HW][128]
  if (a->net_layout == 1) H = (const __half*)a->net;
  else {
    __half* hin = (__half*)(ws + L.hin);
    if (a->net_dtype == DBA_F16) nchw_to_nhwc_kernel<__half><<<tgrid128, 256, 0, st>>>((const __half*)a->net, hin, 128, HW, 128, 128);
    else if (a->net_dtype == DBA_F32) nchw_to_nhwc_kernel<float><<<tgrid128, 256, 0, st>>>((const float*)a->net, hin, 128, HW, 128, 128);
    else { set_error("invalid argument: net dtype must be f16 or f32"); return DBA_ERR_INVALID; }
    H = hin;
  }
  // inp -> X[:, 0:128] (X = inp | corr features | flow features, 320 channels)
  if (a->inp_dtype == DBA_F16) nchw_to_nhwc_kernel<__half><<<tgrid128, 256, 0, st>>>((const __half*)a->inp, X, 128, HW, 320, 128);
  else if (a->inp_dtype == DBA_F32) nchw_to_nhwc_kernel<float><<<tgrid128, 256, 0, st>>>((const float*)a->inp, X, 128, HW, 320, 128);
  else { set_error("invalid argument: inp dtype must be f16 or f32"); return DBA_ERR_INVALID; }
  {
    const dim3 g((HW + 63) / 64, 2, E);
    if (a->corr_dtype == DBA_F16) nchw_to_nhwc_kernel<__half><<<g, 256, 0, st>>>((const __half*)a->corr, Cc, 196, HW, 200, 200);
    else if (a->corr_dtype == DBA_F32) nchw_to_nhwc_kernel<float><<<g, 256, 0, st>>>((const float*)a->corr, Cc, 196, HW, 200, 200);
    else { set_error("invalid argument: corr dtype must be f16 or f32"); return DBA_ERR_INVALID; }
  }
  flow_im2col_kernel<<<dim3((wd + 63) / 64, ht, E), 256, 0, st>>>(a->flow, F0, ht, wd);
  DBA_CHECK_LAUNCH("update layout kernels");

  const ConvParams base = up_base(E, ht, wd);
  const ConvSrc none = {nullptr, 0, 0};
  int rc;
  // ---- corr_encoder: 1x1 196->128 + ReLU, 3x3 128->128 + ReLU -> X[:, 128:256]   (droid_net.py:83-87)
  { ConvParams p = base; p.KS = 1; p.N = 128; p.bias = W->b_corr0; p.relu = 1; p.out = C1; p.out_stride = 128;
    rc = launch_conv<EPI_STORE, true>(p, ConvSrc{Cc, 196, 200}, none, W->w_corr0, st); if (rc) return rc; }
  { ConvParams p = base; p.KS = 3; p.N = 128; p.bias = W->b_corr2; p.relu = 1; p.out = X + 128; p.out_stride = 320;
    rc = launch_conv<EPI_STORE, true>(p, ConvSrc{C1, 128, 128}, none, W->w_corr2, st); if (rc) return rc; }
  // ---- flow_encoder: 7x7 4->128 + ReLU (as a 196-wide 1x1 over the im2col rows), 3x3 128->64 + ReLU -> X[:, 256:320]   (:89-93)
  { ConvParams p = base; p.KS = 1; p.N = 128; p.bias = W->b_flow0; p.relu = 1; p.out = F1; p.out_stride = 128;
    rc = launch_conv<EPI_STORE, true>(p, ConvSrc{F0, 196, 200}, none, W->w_flow0, st); if (rc) return rc; }
  { ConvParams p = base; p.KS = 3; p.N = 64; p.bias = W->b_flow2; p.relu = 1; p.out = X + 256; p.out_stride = 320;
    rc = launch_conv<EPI_STORE, true>(p, ConvSrc{F1, 128, 128}, none, W->w_flow2, st); if (rc) return rc; }
  // ---- ConvGRU (gru.py:19-32): global context
  int slots = 0;
  { ConvParams p = gate_conv(base); p.bias = W->b_gate; p.h = H; p.h_stride = 128; p.partial = partial;
    rc = launch_conv<EPI_GATE, true>(p, ConvSrc{H, 128, 128}, none, W->w_gate, st, &slots); if (rc) return rc; }
  glo_kernel<<<E, 384, 0, st>>>(partial, slots, 1.f / (float)HW, W->w_glo, W->b_glo, glo);
  DBA_CHECK_LAUNCH("glo_kernel");
  // z, r = sigmoid(conv3x3(h | x) + glo): one 256-output convolution; epilogue writes z and r*h
  { ConvParams p = base; p.KS = 3; p.N = 256; p.bias = W->b_zr; p.h = H; p.h_stride = 128; p.glo = glo; p.z = Z; p.rh = RH;
    rc = launch_conv<EPI_ZR, true>(p, ConvSrc{H, 128, 128}, ConvSrc{X, 320, 320}, W->w_zr, st); if (rc) return rc; }
  // q = tanh(conv3x3(r*h | x) + glo); h' = (1-z) h + z q
  { ConvParams p = base; p.KS = 3; p.N = 128; p.bias = W->b_q; p.h = H; p.h_stride = 128; p.glo = glo; p.z = Z;
    p.out = (__half*)a->net_out; p.out_stride = 128;
    rc = launch_conv<EPI_Q, true>(p, ConvSrc{RH, 128, 128}, ConvSrc{X, 320, 320}, W->w_q, st); if (rc) return rc; }
  // ---- heads: stems delta.0 | weight.0 | agg.conv1 as one 384-output convolution + ReLU (droid_net.py:95-106, :60)
  const int stemN = n_src > 0 ? 384 : 256;
  { ConvParams p = base; p.KS = 3; p.N = stemN; p.w_rows = 384; p.bias = W->b_stem; p.relu = 1; p.out = S; p.out_stride = 384;
    rc = launch_conv<EPI_STORE, true>(p, ConvSrc{a->net_out, 128, 128}, none, W->w_stem, st); if (rc) return rc; }
  // delta.2 and weight.2 (3x3 128->2 each): per-tap partial sums by one 1x1 convolution 256 -> 36 (block-diagonal weights), then the
  // 9-tap gather with bias / sigmoid
  float* Yh = (float*)(ws + L.yh);                        // [E,HW,36] f32 on the (dead) corr staging buffer
  { ConvParams p = base; p.KS = 1; p.N = 64; p.bias = W->b_zero; p.f32a = Yh; p.f32_cols = 36; p.f32_stride = 36;
    rc = launch_conv<EPI_F32, true>(p, ConvSrc{S, 256, 384}, none, W->w_heads, st); if (rc) return rc; }
  head_gather_kernel<<<(unsigned)(((size_t)E * HW + 255) / 256), 256, 0, st>>>(Yh, 36, 4, W->b_heads, 0, a->delta, a->weight, E, ht, wd);
  DBA_CHECK_LAUNCH("head_gather_kernel");
  if (n_src > 0) {
    // ---- GraphAgg (droid_net.py:59-75): segment mean over edges with equal source frame, conv2, eta, upmask
    seg_csr_kernel<<<1, 256, (size_t)n_src * sizeof(int), st>>>(a->seg, E, n_src, seg_ptr, seg_edges);
    segment_mean_kernel<<<dim3((HW * 16 + 255) / 256, n_src), 256, 0, st>>>(S + 256, 384, seg_ptr, seg_edges, Am, HW);
    DBA_CHECK_LAUNCH("segment mean");
    ConvParams fb = base; fb.E = n_src;
    { ConvParams p = fb; p.KS = 3; p.N = 128; p.bias = W->b_agg2; p.relu = 1; p.out = B2; p.out_stride = 128;
      rc = launch_conv<EPI_STORE, true>(p, ConvSrc{Am, 128, 128}, none, W->w_agg2, st); if (rc) return rc; }
    float* Ye = (float*)(ws + L.ye);                      // [n_src,HW,12] f32 (9 used) on the (dead) flow im2col buffer
    { ConvParams p = fb; p.KS = 1; p.N = 32; p.bias = W->b_zero; p.f32a = Ye; p.f32_cols = 12; p.f32_stride = 12;
      rc = launch_conv<EPI_F32, true>(p, ConvSrc{B2, 128, 128}, none, W->w_eta, st); if (rc) return rc; }
    head_gather_kernel<<<(unsigned)(((size_t)n_src * HW + 255) / 256), 256, 0, st>>>(Ye, 12, 1, W->b_eta, 1, a->eta, nullptr, n_src, ht, wd);
    DBA_CHECK_LAUNCH("head_gather_kernel(eta)");
    { ConvParams p = fb; p.KS = 1; p.N = 192; p.n_ntiles = 3; p.bias = W->b_upmask; p.nchw = (__half*)a->upmask; p.nchw_C = 576;
      rc = launch_conv<EPI_NCHW, true>(p, ConvSrc{B2, 128, 128}, none, W->w_upmask, st); if (rc) return rc; }
  }
  return DBA_OK;
}

// the shape checks dba_conv_nhwc and dba_conv_nhwc_plan share (c1 = 0: no second source)
static int conv_nhwc_check_shape(int c0, int c1, int ht, int wd, int ksize, int n_out) {
  DBA_CHECK_ARG(ht > 0 && wd > 0, "bad extents");
  DBA_CHECK_ARG(ksize == 1 || ksize == 3, "kernel size must be 1 or 3");
  DBA_CHECK_ARG(n_out >= 32 && n_out <= 384 && (n_out <= 256 ? n_out % 32 == 0 : n_out == 384), "n_out must be 32..256 (multiple of 32) or 384");
  DBA_CHECK_ARG(c0 > 0 && c1 >= 0, "bad channel counts");
  DBA_CHECK_ARG(c1 == 0 || c0 % 64 == 0, "with two sources the first must hold a multiple of 64 channels");
  return DBA_OK;
}

// channels-last tensor-core convolution building block (the kernel behind every layer of dba_update_forward), exported for
// tests and for callers that keep activations channels-last: out[e,y,x,n] = act(bias[n] + sum_{tap,k} src[e,y+dy,x+dx,k] w[tap][n][k]).
// Any ht, wd > 0, tiled by the same rule as dba_update_forward.
extern "C" int dba_conv_nhwc(const void* src0, int c0, int stride0, const void* src1, int c1, int stride1, const void* wpk, const float* bias,
                             void* out, int out_stride, int n_images, int ht, int wd, int ksize, int n_out, int relu, dba_stream_t stream) {
  DBA_CHECK_ARG(src0 && wpk && bias && out, "null pointer");
  DBA_CHECK_ARG(n_images >= 0, "bad extents");
  DBA_CHECK_ARG(!src1 || c1 > 0, "bad channel counts");
  int rc = conv_nhwc_check_shape(c0, src1 ? c1 : 0, ht, wd, ksize, n_out); if (rc) return rc;
  DBA_CHECK_ARG(stride0 % 8 == 0 && stride0 >= c0 && (!src1 || (stride1 % 8 == 0 && stride1 >= c1)), "row pitches must be multiples of 8 elements and hold the channels");
  DBA_CHECK_ARG(out_stride % 8 == 0 && out_stride >= n_out, "bad output stride");
  if (n_images == 0) return DBA_OK;
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.E = n_images; p.HT = ht; p.WD = wd; p.n_ntiles = 1; p.KS = ksize; p.N = n_out; p.bias = bias; p.relu = relu;
  p.out = (__half*)out; p.out_stride = out_stride;
  return launch_conv<EPI_STORE, true>(p, ConvSrc{src0, c0, stride0}, ConvSrc{src1, c1, stride1}, wpk, (cudaStream_t)stream);
}

extern "C" int dba_conv_nhwc_plan(int ht, int wd, int c0, int c1, int ksize, int n_out, int* plan) {
  DBA_CHECK_ARG(plan, "null pointer");
  int rc = conv_nhwc_check_shape(c0, c1, ht, wd, ksize, n_out); if (rc) return rc;
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.E = 1; p.HT = ht; p.WD = wd; p.n_ntiles = 1; p.KS = ksize; p.N = n_out;
  bool flat = false;
  int box_rows = 0;
  rc = conv_plan(p, c0, c1, true, &flat, &box_rows); if (rc) return rc;
  const int v[8] = {flat ? 1 : 0, p.TW, p.MT, p.N, p.n_ntiles, p.tiles_x * p.tiles_y, p.a_stages, p.b_stages};
  memcpy(plan, v, sizeof(v));
  return DBA_OK;
}
