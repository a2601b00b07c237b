// The channels-last implicit-GEMM convolution engine (wgmma / TMA, sm_90a) shared by the update operator (update_op.cu) and
// the feature / context encoders (encoder.cu): ConvParams, the fused epilogues, conv_tc_kernel, the TMA map builders and
// launch_conv.  The design notes are at the top of update_op.cu and in DESIGN section 4.4.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"
#include <string.h>

namespace dba {

enum { EPI_STORE = 0, EPI_GATE = 1, EPI_ZR = 2, EPI_Q = 3, EPI_F32 = 4, EPI_NCHW = 5, EPI_STATS = 6, EPI_RELU_RES = 7 };

constexpr int kUpThreads = 288;   // warps 0..7 two consumer warpgroups, warp 8 TMA
constexpr int kSlotsPerMTile = 8;  // EPI_GATE / EPI_STATS partial-sum slots per 128-pixel M tile (one per consumer warp)

struct ConvParams {
  int E, HT, WD;                    // images (edges or frames), image height / width
  int TW, RM, MT;                   // tile width in pixels, image rows per 128-pixel M tile (RM * TW = 128), M tiles per CTA tile
                                    // (row-flattened tiles: TW = row pitch TWp, RM unused)
  int tiles_x, tiles_y, n_ntiles;   // CTA tiles per image (row-flattened: tiles_x linear tiles, tiles_y = 1), N tiles (output-channel blocks)
  int KS;                           // kernel size 1 or 3
  int nk0, nk1;                     // 64-channel K blocks taken from source 0 / source 1
  int N;                            // output channels per N tile (<= 256)
  int w_rows;                       // rows per tap of the packed weight tensor (0: n_ntiles * N); larger when only the first N rows are used
  int boxn;                         // weight rows per TMA box
  int a_stages, b_stages, a_bytes, b_bytes;
  const float* bias;                // [n_ntiles * N]
  int relu;
  __half* out; int out_stride;      // EPI_STORE / EPI_Q: channels-last f16, out[pix * out_stride + n]
  const __half* h; int h_stride;    // hidden state, channels-last (EPI_GATE, EPI_ZR, EPI_Q)
  const float* glo;                 // [E][384] global-context terms: z | r | q
  __half* z; __half* rh;            // EPI_ZR outputs [pix][128]; EPI_Q reads z
  float* partial; int slots;        // EPI_GATE: [E][slots][128] column sums of sigmoid(.) * h over 16-pixel groups
  float* f32a; int f32_cols, f32_stride;      // EPI_F32: f32 out[pix * f32_stride + n] for n < f32_cols (per-tap partial sums of the narrow heads)
  __half* nchw; int nchw_C;         // EPI_NCHW: out[(img * nchw_C + n) * HT*WD + pixel]
  // encoder epilogues.  EPI_STATS: out = acc + bias (f16) and, per 16-pixel slot, partial[((img * slots + slot) * N + n) * 2 + {0,1}]
  // = (mean, sum of squared deviations from that mean) of the fp32 values, counts[img * slots + slot] = valid pixels of the slot.
  // EPI_RELU_RES: v = acc + bias, ReLU on columns n < relu_cols, then v = relu(v + h[pix * h_stride + n]) when h is set.
  int relu_cols;
  float* counts;
};

__device__ __forceinline__ float tanh_fast(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sigmoid_fast(float x) { return fmaf(0.5f, tanh_fast(0.5f * x), 0.5f); }
// ReLU that keeps NaN, like torch.relu: fmaxf alone would turn a NaN input into 0 and hide it from every later stage
__device__ __forceinline__ float relu_nan(float x) { return isnan(x) ? x : fmaxf(x, 0.f); }
// the same values in one instruction (max.NaN returns NaN when an operand is NaN) for the encoder epilogues, where relu_nan's
// compare and select cost cnet 4.7 % (H100 80GB HBM3, 700 W limit); the update operator's kernels keep relu_nan and their code
__device__ __forceinline__ float relu_nan1(float x) { float y; asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float2 unpack2(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }

__device__ __forceinline__ float2 ldh2(const __half* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }

// M tiles per CTA tile a consumer warpgroup can hold in registers: MT * N / 2 <= 128 fp32 accumulators per thread
constexpr int conv_max_mt(int nw) { return 256 / nw < 4 ? 256 / nw : 4; }

// epilogue of one 64-pixel x N fragment (M tile t of the CTA tile) of consumer warpgroup wg: this thread holds pixels r, r + 8
// (r = 16 (warp % 4) + lane / 4) and columns 8 j + 2 (lane % 4) + {0, 1}.  Row-flattened tiles (FLAT): ty = 0, tx = linear tile,
// pixel m is flat index q = tx * 128 MT + 128 t + m on the padded row pitch TW, i.e. y = q / TW, x = q mod TW.
template <int EPI, int NW, bool FLAT>
__device__ __forceinline__ void conv_epilogue(const ConvParams& p, const float (&acc)[NW / 2], int t, int wg, int warp, int lane, int nt, int e, int ty,
                                              int tx) {
  const int qd = lane & 3;
  const float* bias = p.bias + nt * p.N;
  float csum[NW / 4];                                                  // EPI_GATE: per-column sums over this thread's two pixels
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
    int y, x;
    if constexpr (FLAT) {
      const int q = (tx * p.MT + t) * 128 + m;
      y = q / p.TW; x = q - y * p.TW;
    } else {
      const int my = m / p.TW, mx = m - my * p.TW;
      y = ty * (p.MT * p.RM) + t * p.RM + my; x = tx * p.TW + mx;
    }
    const bool valid = y < p.HT && x < p.WD;
    const size_t pix = ((size_t)e * p.HT + (valid ? y : 0)) * p.WD + (valid ? x : 0);
#pragma unroll
    for (int j = 0; j < NW / 8; j++) {
      const int c = 8 * j + 2 * qd;
      float v0 = acc[4 * j + 2 * i] + __ldg(bias + c), v1 = acc[4 * j + 2 * i + 1] + __ldg(bias + c + 1);
      if (EPI == EPI_STORE) {
        if (p.relu) { v0 = relu_nan(v0); v1 = relu_nan(v1); }
        if (valid) *reinterpret_cast<uint32_t*>(p.out + pix * p.out_stride + nt * p.N + c) = pack_h2(v0, v1);
      } else if (EPI == EPI_GATE) {
        float g0 = 0.f, g1 = 0.f;
        if (valid) { const float2 hh = ldh2(p.h + pix * p.h_stride + c); g0 = sigmoid_fast(v0) * hh.x; g1 = sigmoid_fast(v1) * hh.y; }
        if (i == 0) { csum[2 * j] = g0; csum[2 * j + 1] = g1; }
        else { csum[2 * j] += g0; csum[2 * j + 1] += g1; }
      } else if (EPI == EPI_ZR) {
        const float* g = p.glo + (size_t)e * 384 + c;
        v0 = sigmoid_fast(v0 + __ldg(g)); v1 = sigmoid_fast(v1 + __ldg(g + 1));
        if (valid) {
          if (c < 128) {
            *reinterpret_cast<uint32_t*>(p.z + pix * 128 + c) = pack_h2(v0, v1);
          } else {
            const float2 hh = ldh2(p.h + pix * p.h_stride + (c - 128));
            *reinterpret_cast<uint32_t*>(p.rh + pix * 128 + (c - 128)) = pack_h2(v0 * hh.x, v1 * hh.y);
          }
        }
      } else if (EPI == EPI_Q) {
        const float* g = p.glo + (size_t)e * 384 + 256 + c;
        if (valid) {
          const float2 hh = ldh2(p.h + pix * p.h_stride + c), zz = ldh2(p.z + pix * 128 + c);
          const float q0 = tanh_fast(v0 + __ldg(g)), q1 = tanh_fast(v1 + __ldg(g + 1));
          *reinterpret_cast<uint32_t*>(p.out + pix * p.out_stride + c) = pack_h2((1.f - zz.x) * hh.x + zz.x * q0, (1.f - zz.y) * hh.y + zz.y * q1);
        }
      } else if (EPI == EPI_F32) {
        if (valid && c < p.f32_cols) *reinterpret_cast<float2*>(p.f32a + pix * p.f32_stride + c) = make_float2(v0, v1);   // f32_cols even
      } else if (EPI == EPI_NCHW) {
        if (valid) {
          const size_t HW = (size_t)p.HT * p.WD;
          __half* o = p.nchw + ((size_t)e * p.nchw_C + nt * p.N + c) * HW + (size_t)y * p.WD + x;
          o[0] = __float2half_rn(v0);
          o[HW] = __float2half_rn(v1);
        }
      } else if (EPI == EPI_STATS) {
        if (valid) *reinterpret_cast<uint32_t*>(p.out + pix * p.out_stride + c) = pack_h2(v0, v1);
      } else if (EPI == EPI_RELU_RES) {
        if (c < p.relu_cols) { v0 = relu_nan1(v0); v1 = relu_nan1(v1); }
        if (valid) {
          if (p.h) { const float2 hh = ldh2(p.h + pix * p.h_stride + c); v0 = relu_nan1(v0 + hh.x); v1 = relu_nan1(v1 + hh.y); }
          *reinterpret_cast<uint32_t*>(p.out + pix * p.out_stride + c) = pack_h2(v0, v1);
        }
      }
    }
  }
  if (EPI == EPI_GATE) {
    // column sums over the warp's 16 pixels (lanes with equal lane % 4 hold the same columns), one slot per warp and M tile
#pragma unroll
    for (int k = 0; k < NW / 4; k++) {
      csum[k] += __shfl_xor_sync(0xffffffffu, csum[k], 4);
      csum[k] += __shfl_xor_sync(0xffffffffu, csum[k], 8);
      csum[k] += __shfl_xor_sync(0xffffffffu, csum[k], 16);
    }
    if (lane < 4) {
      const int slot = ((ty * p.tiles_x + tx) * p.MT + t) * kSlotsPerMTile + wg * 4 + (warp & 3);
      float* dst = p.partial + ((size_t)e * p.slots + slot) * 128;
#pragma unroll
      for (int j = 0; j < NW / 8; j++) *reinterpret_cast<float2*>(dst + 8 * j + 2 * qd) = make_float2(csum[2 * j], csum[2 * j + 1]);
    }
  }
  if (EPI == EPI_STATS) {
    // per column: mean and squared deviations about it over the warp's 16 pixels (two passes over the fp32 accumulators, so the
    // statistics stay exact when |mean| >> std); the finalize kernel merges the slots with Chan's pairwise update
    bool ok[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
      const int my = m / p.TW, mx = m - my * p.TW;
      ok[i] = ty * (p.MT * p.RM) + t * p.RM + my < p.HT && tx * p.TW + mx < p.WD;
    }
    float cnt = (float)ok[0] + (float)ok[1];
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 4);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 8);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 16);
    const float inv = cnt > 0.f ? 1.f / cnt : 0.f;
    const int slot = ((ty * p.tiles_x + tx) * p.MT + t) * kSlotsPerMTile + wg * 4 + (warp & 3);
    float* dst = p.partial + ((size_t)e * p.slots + slot) * p.N * 2;
#pragma unroll
    for (int j = 0; j < NW / 4; j++) {
      const int c = 8 * (j >> 1) + 2 * qd + (j & 1);
      const float b = __ldg(bias + c);
      const float x0 = acc[4 * (j >> 1) + (j & 1)] + b, x1 = acc[4 * (j >> 1) + 2 + (j & 1)] + b;
      float s = (ok[0] ? x0 : 0.f) + (ok[1] ? x1 : 0.f);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 8);
      s += __shfl_xor_sync(0xffffffffu, s, 16);
      const float mean = s * inv;
      float q = (ok[0] ? (x0 - mean) * (x0 - mean) : 0.f) + (ok[1] ? (x1 - mean) * (x1 - mean) : 0.f);
      q += __shfl_xor_sync(0xffffffffu, q, 4);
      q += __shfl_xor_sync(0xffffffffu, q, 8);
      q += __shfl_xor_sync(0xffffffffu, q, 16);
      if (lane < 4) *reinterpret_cast<float2*>(dst + 2 * c) = make_float2(mean, q);
    }
    if (lane == 0) p.counts[(size_t)e * p.slots + slot] = cnt;
  }
}

// Two tilings, chosen at compile time:
//  * FLAT = false: a CTA tile is MT M tiles of RM image rows x TW columns (TW = 64 or 32); per (K block, dx) one TMA box of
//    TW x (MT RM + KS - 1) pixels, the A operand of tap dy at box pixel (t RM + dy) TW + 64 wg.
//  * FLAT = true (row-flattened): pixels are numbered row-major on the row pitch TW = TWp = wd rounded up to a multiple of 8, and a
//    CTA tile is the 128 MT consecutive pixels from p0 = tx * 128 MT (it may start mid-row).  Per (K block, dx) one TMA box of TWp
//    columns x box_rows rows anchored at row y0 - pad (y0 = p0 / TWp), column dx - pad; columns >= wd and rows outside [0, ht) are
//    TMA zero fill, so no buffer needs padded columns.  The A operand of tap dy is box pixel c0 + 128 t + dy TWp + 64 wg with
//    c0 = p0 mod TWp.  TWp and c0 are multiples of 8, so every such offset is a multiple of the 1024-byte 128B-swizzle atom (8 rows
//    of 128 bytes) and the gmma_desc_sw128 descriptors hold unchanged: this is why TWp is wd rounded up to 8 and not wd itself.
template <int EPI, int NW, bool FLAT = false>
__global__ void __launch_bounds__(kUpThreads, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                                                               const __grid_constant__ CUtensorMap tmW, const ConvParams p) {
  constexpr int kMT = conv_max_mt(NW);
  extern __shared__ uint8_t up_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(up_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + p.a_stages * p.a_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + p.b_stages * p.b_bytes);
  uint64_t* a_full = bars;              // [4]
  uint64_t* a_empty = bars + 4;         // [4]
  uint64_t* b_full = bars + 8;          // [8]
  uint64_t* b_empty = bars + 16;        // [8]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int total_tiles = p.n_ntiles * p.E * tiles_per_img;
  const int nk = p.nk0 + p.nk1;
  const int pad = p.KS >> 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.a_stages; s++) { mbar_init(a_full + s, 1); mbar_init(a_empty + s, 8); }
    for (int s = 0; s < p.b_stages; s++) { mbar_init(b_full + s, 1); mbar_init(b_empty + s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ================= TMA producer (one thread) =================
    if (lane == 0) {
      uint32_t ac = 0, bc = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = tile / (p.E * tiles_per_img);
        const int r0 = tile - nt * (p.E * tiles_per_img);
        const int e = r0 / tiles_per_img;
        const int r1 = r0 - e * tiles_per_img;
        const int ty = r1 / p.tiles_x, tx = r1 - ty * p.tiles_x;
        int y0, x0;
        if constexpr (FLAT) {
          y0 = (tx * p.MT * 128) / p.TW; x0 = 0;
        } else {
          y0 = ty * (p.MT * p.RM); x0 = tx * p.TW;
        }
        for (int kb = 0; kb < nk; kb++) {
          const CUtensorMap* am = kb < p.nk0 ? &tmA0 : &tmA1;
          const int ch = (kb < p.nk0 ? kb : kb - p.nk0) * 64;
          for (int dx = 0; dx < p.KS; dx++) {
            const int as = ac % p.a_stages;
            mbar_wait(a_empty + as, ((ac / p.a_stages) & 1) ^ 1);
            mbar_expect_tx(a_full + as, p.a_bytes);
            tma_load_4d(sA + as * p.a_bytes, am, a_full + as, ch, x0 + dx - pad, y0 - pad, e);
            ac++;
            for (int dy = 0; dy < p.KS; dy++) {
              const int bs = bc % p.b_stages;
              mbar_wait(b_empty + bs, ((bc / p.b_stages) & 1) ^ 1);
              mbar_expect_tx(b_full + bs, p.b_bytes);
              for (int n = 0; n < p.N; n += p.boxn)
                tma_load_3d(sB + bs * p.b_bytes + n * 128, &tmW, b_full + bs, kb * 64, nt * p.N + n, dy * p.KS + dx);
              bc++;
            }
          }
        }
      }
    }
    return;
  }
  // ================= consumers: warpgroup wg = pixels 64 wg .. 64 wg + 63 of every M tile =================
  // A stage is released (one arrival per warp) when the wgmma batch after the last one reading it has been issued and the
  // batch reading it has completed (wgmma.wait_group 1), so one batch is always in flight.
  const int wg = warp >> 2;
  const uint32_t sA_u = smem_u32(sA), sB_u = smem_u32(sB);
  float acc[kMT][NW / 2];
  uint32_t ac = 0, bc = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int nt = tile / (p.E * tiles_per_img);
    const int r0 = tile - nt * (p.E * tiles_per_img);
    const int e = r0 / tiles_per_img;
    const int r1 = r0 - e * tiles_per_img;
    const int ty = r1 / p.tiles_x, tx = r1 - ty * p.tiles_x;
    const int c0 = FLAT ? (tx * p.MT * 128) % p.TW : 0;               // row-flattened: column of the tile's first pixel in box row 0
    bool first = true;
    int pend_a = -1, pend_b = -1;
    for (int kb = 0; kb < nk; kb++) {
      for (int dx = 0; dx < p.KS; dx++) {
        const int as = ac % p.a_stages;
        mbar_wait(a_full + as, (ac / p.a_stages) & 1);
        for (int dy = 0; dy < p.KS; dy++) {
          const int bs = bc % p.b_stages;
          mbar_wait(b_full + bs, (bc / p.b_stages) & 1);
          const uint32_t b_base = sB_u + bs * p.b_bytes;
          wgmma_fence();
#pragma unroll
          for (int t = 0; t < kMT; t++) {
            if (t < p.MT) {
              const uint32_t a_base = sA_u + as * p.a_bytes +
                                      (uint32_t)(FLAT ? c0 + t * 128 + dy * p.TW + wg * 64 : (t * p.RM + dy) * p.TW + wg * 64) * 128u;
#pragma unroll
              for (int k = 0; k < 4; k++)
                wgmma_f16<NW>(acc[t], gmma_desc_sw128(a_base + k * 32, 16, 1024), gmma_desc_sw128(b_base + k * 32, 16, 1024), (first && k == 0) ? 0 : 1, 0);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) {
            if (pend_b >= 0) mbar_arrive(b_empty + pend_b);
            if (pend_a >= 0) mbar_arrive(a_empty + pend_a);
          }
          pend_a = -1;
          pend_b = bs;
          first = false;
          bc++;
        }
        pend_a = as;
        ac++;
      }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) {
      if (pend_b >= 0) mbar_arrive(b_empty + pend_b);
      if (pend_a >= 0) mbar_arrive(a_empty + pend_a);
    }
#pragma unroll
    for (int t = 0; t < kMT; t++) {
      wgmma_fence_regs(acc[t]);
      if (t < p.MT) conv_epilogue<EPI, NW, FLAT>(p, acc[t], t, wg, warp, lane, nt, e, ty, tx);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
// activation map: channels-last f16 [E][HT][WD][stride], channels [0, C) of the slice starting at `base`
static int make_act_map(CUtensorMap* map, const void* base, int C, int stride, int WD, int HT, int E, int TW, int box_rows) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)WD, (cuuint64_t)HT, (cuuint64_t)E};
  const cuuint64_t strides[3] = {(cuuint64_t)stride * 2, (cuuint64_t)WD * stride * 2, (cuuint64_t)HT * WD * stride * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)TW, (cuuint32_t)box_rows, 1};
  return tma_encode_f16(map, base, 4, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "activation, C=%d stride=%d %dx%d E=%d box %dx%d",
                        C, stride, HT, WD, E, TW, box_rows);
}
// weight map: [taps][Ntot][Kpad] f16
static int make_weight_map(CUtensorMap* map, const void* base, int Kpad, int Ntot, int taps, int boxn) {
  const cuuint64_t dims[3] = {(cuuint64_t)Kpad, (cuuint64_t)Ntot, (cuuint64_t)taps};
  const cuuint64_t strides[2] = {(cuuint64_t)Kpad * 2, (cuuint64_t)Ntot * Kpad * 2};
  const cuuint32_t box[3] = {64, (cuuint32_t)boxn, 1};
  return tma_encode_f16(map, base, 3, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "weights K=%d N=%d taps=%d", Kpad, Ntot, taps);
}

struct ConvSrc { const void* base; int C; int stride; };

static int g_num_sms = 0;

template <int EPI>
constexpr bool conv_width_used(int nw) {
  return EPI == EPI_STORE || (EPI == EPI_GATE && nw == 128) || (EPI == EPI_ZR && nw == 256) || (EPI == EPI_Q && nw == 128) ||
         (EPI == EPI_F32 && (nw == 32 || nw == 64)) || (EPI == EPI_NCHW && (nw == 128 || nw == 192 || nw == 256)) ||
         ((EPI == EPI_STATS || EPI == EPI_RELU_RES) && (nw == 32 || nw == 64 || nw == 128 || nw == 256));
}

template <int EPI, int NW, bool FLAT>
static int launch_conv_nw(const ConvParams& p, const CUtensorMap& tA0, const CUtensorMap& tA1, const CUtensorMap& tW, int grid, int smem, cudaStream_t st) {
  if constexpr (!conv_width_used<EPI>(NW) || (FLAT && (EPI == EPI_STATS || EPI == EPI_RELU_RES))) {
    set_error("update operator: no convolution kernel for this epilogue with %d output channels", NW);
    return DBA_ERR_INVALID;
  } else {
    static bool attr_set = false;
    if (!attr_set) {
      DBA_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_kernel<EPI, NW, FLAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024), "conv_tc smem attr");
      attr_set = true;
    }
    conv_tc_kernel<EPI, NW, FLAT><<<grid, kUpThreads, smem, st>>>(tA0, tA1, tW, p);
    DBA_CHECK_LAUNCH("conv_tc_kernel");
    return DBA_OK;
  }
}

template <int EPI, bool FLAT>
static int launch_conv_n(const ConvParams& p, const CUtensorMap& tA0, const CUtensorMap& tA1, const CUtensorMap& tW, int grid, int smem, cudaStream_t st) {
  switch (p.N) {
    case 32: return launch_conv_nw<EPI, 32, FLAT>(p, tA0, tA1, tW, grid, smem, st);
    case 64: return launch_conv_nw<EPI, 64, FLAT>(p, tA0, tA1, tW, grid, smem, st);
    case 96: return launch_conv_nw<EPI, 96, FLAT>(p, tA0, tA1, tW, grid, smem, st);
    case 128: return launch_conv_nw<EPI, 128, FLAT>(p, tA0, tA1, tW, grid, smem, st);
    case 160: return launch_conv_nw<EPI, 160, FLAT>(p, tA0, tA1, tW, grid, smem, st);
    case 192: return launch_conv_nw<EPI, 192, FLAT>(p, tA0, tA1, tW, grid, smem, st);
    case 224: return launch_conv_nw<EPI, 224, FLAT>(p, tA0, tA1, tW, grid, smem, st);
    default: return launch_conv_nw<EPI, 256, FLAT>(p, tA0, tA1, tW, grid, smem, st);
  }
}

// the tiling of one convolution (host only, no device query): fills the N tiles, TW, RM, MT, tiles_x / tiles_y, nk0 / nk1, boxn,
// stage counts and sizes and slots of p from p.E, HT, WD, KS, N, n_ntiles, w_rows and the channel counts c0, c1 (0: no second source);
// *flat = row-flattened tiles, *box_rows = halo box rows.
// row_flat (the update operator): widths that are not a multiple of 8 take the row-flattened tiles of conv_tc_kernel where 2 halo
// and 2 weight stages of them fit in shared memory; the rectangular tiles, correct at every width, run everywhere else.
static int conv_plan(ConvParams& p, int c0, int c1, bool row_flat, bool* flat_out, int* box_rows_out) {
  if (p.N > 256) {                // 384 outputs: two 192-wide N tiles (the register accumulator holds at most 256 columns)
    if (p.w_rows == 0) p.w_rows = p.n_ntiles * p.N;
    p.n_ntiles *= p.N / 192;
    p.N = 192;
  }
  if (p.N % 32 != 0 || p.N < 32) { set_error("update operator: %d output channels per tile", p.N); return DBA_ERR_INVALID; }
  const int budget = 227 * 1024 - 2048;
  const int nk = (c0 + 63) / 64 + (c1 + 63) / 64;
  int box_rows = 0;
  bool flat = false;
  if (row_flat) {
    if (p.WD % 8 != 0) {
      // row-flattened tiles (conv_tc_kernel): 128 MT consecutive pixels on the row pitch twp; the halo box spans the rows those
      // pixels touch from any start column c0 <= twp - 8, plus KS - 1 halo rows.  MT as for the rectangular tiles below.
      const int twp = (p.WD + 7) & ~7, px = p.HT * twp;
      int mt = px >= 2 * 128 ? 2 : 1;
      if (p.N <= 64 && px >= 4 * 128 && nk >= 4 && p.KS == 3) mt = 4;
      if (mt > conv_max_mt(p.N)) mt = conv_max_mt(p.N);
      const int rows = (twp - 8 + 128 * mt + twp - 1) / twp + p.KS - 1;
      if (twp <= 256 && 2 * rows * twp * 128 + 2 * p.N * 128 <= budget) {   // TMA box extents <= 256; 2 halo + 2 weight stages
        flat = true;
        p.TW = twp; p.RM = 0; p.MT = mt;
        p.tiles_x = (px + 128 * mt - 1) / (128 * mt);
        p.tiles_y = 1;
        box_rows = rows;
      }
    }
  }
  if (!flat) {
    p.TW = (p.WD % 64 == 0) ? 64 : 32;
    p.RM = 128 / p.TW;
    // M tiles per CTA tile: every weight stage is shared by MT tiles (and every halo row by 3 taps), so larger is better for the
    // L2 -> SM traffic per MAC; bounded by the register accumulators (MT * N <= 256 columns) and by the image height
    p.MT = (p.HT >= 2 * p.RM) ? 2 : 1;
    if (p.N <= 64 && p.HT >= 4 * p.RM && nk >= 4 && p.KS == 3) p.MT = 4;
    if (p.MT > conv_max_mt(p.N)) p.MT = conv_max_mt(p.N);
    p.tiles_x = (p.WD + p.TW - 1) / p.TW;
    p.tiles_y = (p.HT + p.MT * p.RM - 1) / (p.MT * p.RM);
    box_rows = p.MT * p.RM + p.KS - 1;
  }
  p.nk0 = (c0 + 63) / 64;
  p.nk1 = (c1 + 63) / 64;
  p.boxn = p.N;
  p.a_bytes = box_rows * p.TW * 128;
  p.b_bytes = p.N * 128;
  // shared memory: at least 2 halo stages and 3 weight stages; what is left goes to more halo stages (up to 4: with narrow N the
  // MMAs of a stage are short and the TMA latency of the next halo tile is what the pipeline has to cover), then weight stages
  p.a_stages = 2;
  while (p.a_stages < 4 && (p.a_stages + 1) * p.a_bytes + 4 * p.b_bytes <= budget) p.a_stages++;
  p.b_stages = (budget - p.a_stages * p.a_bytes) / p.b_bytes;
  if (p.b_stages > 8) p.b_stages = 8;
  if (p.b_stages < 2) { set_error("update operator: tile does not fit shared memory"); return DBA_ERR_INVALID; }
  p.slots = p.tiles_x * p.tiles_y * p.MT * kSlotsPerMTile;
  *flat_out = flat;
  *box_rows_out = box_rows;
  return DBA_OK;
}

// one convolution launch.  src0 (+ optional src1) = channels-last sources concatenated along K; wpk = packed weights
// [KS*KS][n_ntiles*N][Kpad] with Kpad = 64 * (kblocks(src0) + kblocks(src1)); tiled by conv_plan.
template <int EPI, bool ROW_FLAT = false>
static int launch_conv(ConvParams p, ConvSrc s0, ConvSrc s1, const void* wpk, cudaStream_t st, int* slots_out = nullptr) {
  if (!g_num_sms) {
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceProp prop; DBA_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev), "cudaGetDeviceProperties");
    g_num_sms = prop.multiProcessorCount;
  }
  bool flat = false;
  int box_rows = 0;
  int rc = conv_plan(p, s0.C, s1.base ? s1.C : 0, ROW_FLAT, &flat, &box_rows); if (rc) return rc;
  if (slots_out) *slots_out = p.slots;
  const int smem = p.a_stages * p.a_bytes + p.b_stages * p.b_bytes + 1024 + 256;
  CUtensorMap tA0, tA1, tW;
  rc = make_act_map(&tA0, s0.base, s0.C, s0.stride, p.WD, p.HT, p.E, p.TW, box_rows); if (rc) return rc;
  if (s1.base) { rc = make_act_map(&tA1, s1.base, s1.C, s1.stride, p.WD, p.HT, p.E, p.TW, box_rows); if (rc) return rc; }
  else tA1 = tA0;
  rc = make_weight_map(&tW, wpk, 64 * (p.nk0 + p.nk1), p.w_rows > 0 ? p.w_rows : p.n_ntiles * p.N, p.KS * p.KS, p.boxn); if (rc) return rc;
  const long long total = (long long)p.n_ntiles * p.E * p.tiles_x * p.tiles_y;
  if (total <= 0) return DBA_OK;
  const int grid = (int)(total < g_num_sms ? total : g_num_sms);
  if constexpr (ROW_FLAT) {
    if (flat) return launch_conv_n<EPI, true>(p, tA0, tA1, tW, grid, smem, st);
  }
  return launch_conv_n<EPI, false>(p, tA0, tA1, tW, grid, smem, st);
}

}  // namespace dba
