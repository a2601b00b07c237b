// All-pairs correlation volume + 4-level pooled pyramid in ONE pass on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Replaces CorrBlock.__init__ / CorrBlock.corr (reference droid_slam/modules/corr.py:24-38, 63-71): a cuBLAS batched GEMM
// writing the [E,HW,HW] level-0 volume followed by three avg_pool2d passes that re-read it.  Here, per edge e:
//     L0[m][n]  = fp16( (1/16) * sum_c f1[ii[e]][c][m] * f2[jj[e]][c][n] )           (fp32 accumulation in registers)
//     L1..L3    = 2x2 average pooling over n = (y2,x2) (ATen rounds every level to fp16 before pooling the next; here the
//                 cascade runs in fp32 on the accumulator and each level is rounded once -- closer to exact, within fp16 ulp)
// are produced by one kernel: the GEMM is write bound (2*HW^2*128 flop vs 1.33*HW^2*2 bytes per edge, ~150 flop/B, far
// below the H100 ridge), so the pyramid is computed in the epilogue from the accumulator while it is still on chip and the
// volume is written exactly once (25.1 MB/edge at 48x64 instead of ~50 MB of traffic for GEMM + 3 pooling passes).
//
// CTA = (edge, 128 source pixels m), 288 threads.  Warp 8: TMA producer (cp.async.bulk.tensor, 128B swizzle) -- the A tile
// [128 ch x 128 px] once, then B chunks [128 ch x 4 boxes of 64 px] (4 image rows x 64 columns of frame j), double buffered.
// Warps 0-7: two consumer warpgroups, warpgroup w owns source pixels 64 w .. 64 w + 63; per chunk it runs wgmma.m64n128k16 x 8
// (K = 128) on each half of the chunk (2 image rows), both operands MN-major straight from the [C,H,W] feature layout (no
// transposes), and pools the register accumulator.  A thread holds two source pixels x (8-column groups, 2 adjacent columns each);
// 2x2 windows are thread-local, 4x4 / 8x8 windows combine lanes of a quad by shuffles, and a 4x4 word transpose inside the quad
// turns the fragment into 8-element row pieces before the stores.  A 64-column tile never splits a level-3 block.
//
// Two tilings of the target image, one kernel template (corr_volume_pyramid_kernel<P>) whose parameter type P supplies the
// tiling-specific parts -- B-box coordinates, the source pixel of a fragment row, and the four level stores:
//   CvParams      wd = 64, ht % 8 == 0 (512-wide inputs at 1/8 resolution): chunk c = pixels 256 c .. 256 c + 255, whole aligned
//                 16-byte stores, optionally in the tiled layout of levels 0-1.
//   CvRowsParams  every other ht, wd >= 8: step = (column tile t, row chunk c), bounded stores.  Measured 10-12 % slower at the
//                 wd = 64 shapes (DESIGN section 5), so those keep CvParams.
#include "common.cuh"
#include "wgmma.cuh"

namespace dba {

constexpr int kCvThreads = 288;          // warps 0..7 consumers (two warpgroups), warp 8 TMA
constexpr int kCvM = 128;                // source pixels per CTA
constexpr int kCvN = 256;                // target pixels per chunk (4 image rows at wd = 64)
constexpr int kCvK = 128;                // channels
constexpr int kBoxBytes = 64 * kCvK * 2; // one TMA box: 64 pixels x 128 channels fp16 = 16 KB
constexpr int kSmemA = 2 * kBoxBytes;    // 32 KB
constexpr int kSmemB = 4 * kBoxBytes;    // 64 KB per stage
constexpr int kCvSmem = kSmemA + 2 * kSmemB + 1024 /*alignment slack*/ + 256 /*barriers*/;

// the first n (<= 8 valid, may be <= 0) halves of v to dst: one 16-byte store when aligned and whole, else 4- or 2-byte pieces
__device__ __forceinline__ void store_h8(__half* dst, const uint4& v, int n) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  const uintptr_t a = reinterpret_cast<uintptr_t>(dst);
  if (n >= 8 && (a & 15) == 0) {
    *reinterpret_cast<uint4*>(dst) = v;
  } else if ((a & 3) == 0) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      if (2 * k + 1 < n) reinterpret_cast<uint32_t*>(dst)[k] = w[k];
      else if (2 * k < n) reinterpret_cast<unsigned short*>(dst)[2 * k] = (unsigned short)(w[k] & 0xffffu);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; k++)
      if (k < n) reinterpret_cast<unsigned short*>(dst)[k] = (unsigned short)(w[k >> 1] >> (16 * (k & 1)));
  }
}

// Fragment row i of this thread (the m64nNk16 accumulator layout), counted from `base`.
template <class T>
__device__ __forceinline__ T frag_row(T base, int wg, int warp, int lane, int i) { return base + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i; }

// What each tiling supplies to corr_volume_pyramid_kernel:
//   n_steps(), step(k, t, c)   B chunks per CTA; chunk k covers column tile t, target rows 4c .. 4c + 3
//   load_b(..., t, c, b, fj)   TMA box b (target row 4c + b, 64 columns) of chunk (t, c) of frame fj
//   source(e, m0, ..., ok)     edge e's plane index of this thread's fragment row i; ok = that source pixel exists
//   store0, store1             one 8-element piece of level 0 (row 4c + row, 8-column group gx of the 64-column tile) or level 1
//                              (row 2c + h, group qd of the 32-column tile), r = plane index from source(), skipped where the
//                              source pixel or the row is not part of the output
//   stored(ok, l, y)           for levels l = 2, 3, whose pieces only some lanes of a quad store: whether row y is part of the output
//   store2, store3             level 2 row c, columns 16 t + half .. + 7; level 3 row c / 2, columns 8 t .. 8 t + 7

// wd = 64, ht % 8 == 0: B chunk c = target pixels 256 c .. 256 c + 255 of a [frame][C][HW] map (3-D boxes of 64 pixels)
struct CvParams {
  const int64_t* ii; const int64_t* jj;
  __half* out0; __half* out1; __half* out2; __half* out3;
  int HW, wd, n_chunks;
  int tiled;     // levels 0 and 1 in 4x8-element tiles ([h/4][w/8][4][8], one 64-byte DRAM atom per tile) for corr_lookup_pyramid

  __device__ __forceinline__ int n_steps() const { return n_chunks; }
  __device__ __forceinline__ void step(int k, int& t, int& c) const { t = 0; c = k; }
  __device__ __forceinline__ void load_b(void* dst, const CUtensorMap* map, uint64_t* bar, int t, int c, int b, int fj) const {
    tma_load_3d(dst, map, bar, c * kCvN + 64 * b, 0, fj);
  }
  __device__ __forceinline__ size_t source(int e, int m0, int wg, int warp, int lane, int i, bool& ok) const {
    ok = true;
    return frag_row((size_t)e * HW + m0, wg, warp, lane, i);
  }
  __device__ __forceinline__ bool stored(bool, int, int) const { return true; }
  __device__ __forceinline__ void store0(size_t r, bool, int, int c, int row, int gx, const uint4& v) const {
    __half* dst = tiled ? out0 + r * (size_t)HW + ((size_t)c * 8 + gx) * 32 + row * 8 : out0 + r * (size_t)HW + (size_t)c * kCvN + row * 64 + gx * 8;
    *reinterpret_cast<uint4*>(dst) = v;
  }
  __device__ __forceinline__ void store1(size_t r, bool, int, int c, int h, int qd, const uint4& v) const {
    __half* dst = tiled ? out1 + r * (size_t)(HW / 4) + ((size_t)(c >> 1) * 4 + qd) * 32 + (2 * (c & 1) + h) * 8
                        : out1 + r * (size_t)(HW / 4) + (size_t)(2 * c + h) * (wd / 2) + qd * 8;
    *reinterpret_cast<uint4*>(dst) = v;
  }
  __device__ __forceinline__ void store2(size_t r, int, int c, int half, const uint4& v) const {
    *reinterpret_cast<uint4*>(out2 + r * (size_t)(HW / 16) + (size_t)c * (wd / 4) + half) = v;
  }
  __device__ __forceinline__ void store3(size_t r, int, int c, const uint4& v) const {
    *reinterpret_cast<uint4*>(out3 + r * (size_t)(HW / 64) + (size_t)(c >> 1) * (wd / 8)) = v;
  }
};

// every other size: step k = (column tile t = k / n_rchunks of 64 target columns, chunk c of 4 target rows); one B chunk = 4 TMA boxes
// of one image row x 64 columns from a row-structured map [frame][C][ht][wp], wp = row pitch (wd, or wd rounded up to 8 in the staged
// copy when wd % 8 != 0: TMA global strides must be multiples of 16 bytes).  Source pixels m run over the padded grid ht x wp.  Tails
// (source pixels past ht x wp, target rows past ht, target columns past wp) come in as zeros from TMA's out-of-bounds fill, the staged
// pad columns [wd, wp) as stored zeros; none of them is stored: a source pixel is stored when x < wd, a level-l target element when it
// lies in the floor((ht >> l) x (wd >> l)) grid of complete blocks.  Output rows are not 16-byte aligned in general, so every
// level's 8-element piece goes through store_h8.
struct CvRowsParams {
  const int64_t* ii; const int64_t* jj;
  __half* out0; __half* out1; __half* out2; __half* out3;
  size_t P0, P1, P2, P3;                 // plane sizes (ht >> l) * (wd >> l)
  int ht, wd, wp, n_ctiles, n_rchunks;
  int h1, w1, h2, w2, h3, w3;            // level extents ht >> l, wd >> l

  __device__ __forceinline__ int n_steps() const { return n_ctiles * n_rchunks; }
  __device__ __forceinline__ void step(int k, int& t, int& c) const { t = k / n_rchunks; c = k - t * n_rchunks; }
  __device__ __forceinline__ void load_b(void* dst, const CUtensorMap* map, uint64_t* bar, int t, int c, int b, int fj) const {
    tma_load_4d(dst, map, bar, 64 * t, 4 * c + b, 0, fj);
  }
  __device__ __forceinline__ size_t source(int e, int m0, int wg, int warp, int lane, int i, bool& ok) const {
    const int m = frag_row(m0, wg, warp, lane, i), ys = m / wp, xs = m - ys * wp;
    ok = ys < ht && xs < wd;
    return (size_t)e * P0 + (size_t)ys * wd + xs;
  }
  __device__ __forceinline__ bool stored(bool ok, int l, int y) const { return ok && y < (l == 2 ? h2 : h3); }
  __device__ __forceinline__ void store0(size_t r, bool ok, int t, int c, int row, int gx, const uint4& v) const {
    const int y = 4 * c + row, x = 64 * t + gx * 8;
    if (ok && y < ht) store_h8(out0 + r * P0 + (size_t)y * wd + x, v, wd - x);
  }
  __device__ __forceinline__ void store1(size_t r, bool ok, int t, int c, int h, int qd, const uint4& v) const {
    const int y = 2 * c + h, x = 32 * t + 8 * qd;
    if (ok && y < h1) store_h8(out1 + r * P1 + (size_t)y * w1 + x, v, w1 - x);
  }
  __device__ __forceinline__ void store2(size_t r, int t, int c, int half, const uint4& v) const {
    store_h8(out2 + r * P2 + (size_t)c * w2 + 16 * t + half, v, w2 - 16 * t - half);
  }
  __device__ __forceinline__ void store3(size_t r, int t, int c, const uint4& v) const {
    store_h8(out3 + r * P3 + (size_t)(c >> 1) * w3 + 8 * t, v, w3 - 8 * t);
  }
};

__device__ __forceinline__ uint32_t sel4(const uint32_t (&w)[4], int i) { return i == 0 ? w[0] : i == 1 ? w[1] : i == 2 ? w[2] : w[3]; }
// 4x4 transpose of 32-bit words inside a quad of lanes: on return lane q of the quad holds o[j] = (word q of lane j)
__device__ __forceinline__ void quad_transpose(const uint32_t (&w)[4], uint32_t (&o)[4], int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int s = 0; s < 4; s++) {
    const int src = (q + s) & 3;
    const uint32_t v = __shfl_sync(0xffffffffu, sel4(w, (q - s) & 3), (lane & ~3) | src);
#pragma unroll
    for (int j = 0; j < 4; j++) if (j == src) o[j] = v;
  }
}

template <class P>
__global__ void __launch_bounds__(kCvThreads, 1) corr_volume_pyramid_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                           const __grid_constant__ CUtensorMap tmB, P p) {
  extern __shared__ uint8_t cv_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(cv_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + kSmemA;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kSmemA + 2 * kSmemB);
  uint64_t* bar_a = bars + 0;
  uint64_t* full_b = bars + 1;       // [2]
  uint64_t* empty_b = bars + 3;      // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.y;
  const int m0 = blockIdx.x * kCvM;
  const int fi = (int)p.ii[e], fj = (int)p.jj[e];
  const int n_steps = p.n_steps();

  if (threadIdx.x == 0) {
    mbar_init(bar_a, 1);
    for (int s = 0; s < 2; s++) { mbar_init(full_b + s, 1); mbar_init(empty_b + s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ================= TMA producer =================
    if (lane == 0) {
      mbar_expect_tx(bar_a, kSmemA);
      tma_load_3d(sA, &tmA, bar_a, m0, 0, fi);
      tma_load_3d(sA + kBoxBytes, &tmA, bar_a, m0 + 64, 0, fi);
      for (int k = 0; k < n_steps; k++) {
        int t, c;
        p.step(k, t, c);
        const int s = k & 1;
        if (k >= 2) mbar_wait(empty_b + s, ((k >> 1) - 1) & 1);
        mbar_expect_tx(full_b + s, kSmemB);
        for (int b = 0; b < 4; b++) p.load_b(sB + s * kSmemB + b * kBoxBytes, &tmB, full_b + s, t, c, b, fj);
      }
    }
    return;
  }
  // ================= consumers: warpgroup wg = source pixels 64 wg .. 64 wg + 63 =================
  const int wg = warp >> 2, qd = lane & 3;
  const float sc = 0.0625f;                                            // (f1/4).(f2/4)
  const uint32_t a0 = smem_u32(sA + wg * kBoxBytes);
  size_t rowoff[2];                                                    // this thread's two source pixels (fragment rows)
  bool srcok[2];
#pragma unroll
  for (int i = 0; i < 2; i++) rowoff[i] = p.source(e, m0, wg, warp, lane, i, srcok[i]);
  float acc[64];
  float l1h0[2][8], l2prev[2][8];
  mbar_wait(bar_a, 0);
  for (int k = 0; k < n_steps; k++) {
    int t, c;
    p.step(k, t, c);
    const int s = k & 1;
    mbar_wait(full_b + s, (k >> 1) & 1);
    const uint32_t b0 = smem_u32(sB + s * kSmemB);
#pragma unroll 1
    for (int h = 0; h < 2; h++) {                                      // image rows 4c + 2h, 4c + 2h + 1 = columns 128 h .. 128 h + 127
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kCvK / 16; kk++)
        wgmma_f16<128>(acc, gmma_desc_sw128(a0 + kk * 2048, kBoxBytes, 1024), gmma_desc_sw128(b0 + 2 * h * kBoxBytes + kk * 2048, kBoxBytes, 1024),
                       kk > 0 ? 1 : 0, 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (h == 1) {                                                    // the smem stage may be refilled
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_b + s);
      }
#pragma unroll
      for (int i = 0; i < 2; i++) {
        // level 0: per image row, two blocks of four 8-column groups -> one 8-column piece per lane
#pragma unroll
        for (int ry = 0; ry < 2; ry++) {
#pragma unroll
          for (int b = 0; b < 2; b++) {
            uint32_t w[4], o[4];
#pragma unroll
            for (int g = 0; g < 4; g++) {
              const int j = ry * 8 + b * 4 + g;
              w[g] = pack_h2(acc[4 * j + 2 * i] * sc, acc[4 * j + 2 * i + 1] * sc);
            }
            quad_transpose(w, o, lane);
            p.store0(rowoff[i], srcok[i], t, c, 2 * h + ry, b * 4 + qd, make_uint4(o[0], o[1], o[2], o[3]));
          }
        }
        // level 1 row 2c + h: column 4 gx + qd of this lane's 32-column tile
        float l1[8];
#pragma unroll
        for (int gx = 0; gx < 8; gx++)
          l1[gx] = ((acc[4 * gx + 2 * i] + acc[4 * gx + 2 * i + 1]) + (acc[4 * (8 + gx) + 2 * i] + acc[4 * (8 + gx) + 2 * i + 1])) * (0.25f * sc);
        {
          uint32_t w[4], r[4];
#pragma unroll
          for (int kk = 0; kk < 4; kk++) w[kk] = pack_h2(l1[2 * kk], l1[2 * kk + 1]);
          quad_transpose(w, r, lane);                                  // lane qd: columns 8 qd + {0..3} (low halves), 8 qd + 4 + {0..3} (high)
          const uint4 v = make_uint4(__byte_perm(r[0], r[1], 0x5410), __byte_perm(r[2], r[3], 0x5410), __byte_perm(r[0], r[1], 0x7632),
                                     __byte_perm(r[2], r[3], 0x7632));
          p.store1(rowoff[i], srcok[i], t, c, h, qd, v);
        }
        if (h == 0) {
#pragma unroll
          for (int gx = 0; gx < 8; gx++) l1h0[i][gx] = l1[gx];
          continue;
        }
        // level 2 row c: column 2 gx + qd / 2 (lanes qd, qd ^ 1 hold the same value)
        float l2[8], ot[8];
#pragma unroll
        for (int gx = 0; gx < 8; gx++) {
          const float s0 = l1h0[i][gx] + __shfl_xor_sync(0xffffffffu, l1h0[i][gx], 1);
          const float s1 = l1[gx] + __shfl_xor_sync(0xffffffffu, l1[gx], 1);
          l2[gx] = (s0 + s1) * 0.25f;
        }
#pragma unroll
        for (int gx = 0; gx < 8; gx++) ot[gx] = __shfl_xor_sync(0xffffffffu, l2[gx], 2);
        const bool l2ok = p.stored(srcok[i], 2, c);
        if (qd == 0 && l2ok)
          p.store2(rowoff[i], t, c, 0, make_uint4(pack_h2(l2[0], ot[0]), pack_h2(l2[1], ot[1]), pack_h2(l2[2], ot[2]), pack_h2(l2[3], ot[3])));
        else if (qd == 2 && l2ok)
          p.store2(rowoff[i], t, c, 8, make_uint4(pack_h2(ot[4], l2[4]), pack_h2(ot[5], l2[5]), pack_h2(ot[6], l2[6]), pack_h2(ot[7], l2[7])));
        if (c & 1) {   // level 3 row c/2: column gx (lanes 0 and 2 of the quad hold the two level-2 columns 2 gx, 2 gx + 1)
          float l3[8];
#pragma unroll
          for (int gx = 0; gx < 8; gx++) {
            const float a = l2prev[i][gx] + __shfl_xor_sync(0xffffffffu, l2prev[i][gx], 2);
            const float b = l2[gx] + ot[gx];
            l3[gx] = (a + b) * 0.25f;
          }
          if (qd == 0 && p.stored(srcok[i], 3, c >> 1))
            p.store3(rowoff[i], t, c, make_uint4(pack_h2(l3[0], l3[1]), pack_h2(l3[2], l3[3]), pack_h2(l3[4], l3[5]), pack_h2(l3[6], l3[7])));
        } else {
#pragma unroll
          for (int gx = 0; gx < 8; gx++) l2prev[i][gx] = l2[gx];
        }
      }
    }
  }
}

// staged copy for wd % 8 != 0: [F][C][ht][wd] -> [F][C][ht][wp], pad columns zero.  One thread per 8 output columns (one 16-byte store).
__global__ void __launch_bounds__(256) corr_volume_stage_kernel(const __half* __restrict__ src, __half* __restrict__ dst, long long n_rows,
                                                                int wd, int wp) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int gpr = wp >> 3;
  if (q >= n_rows * gpr) return;
  const long long row = q / gpr;
  const int x0 = (int)(q - row * gpr) * 8;
  const unsigned short* s = reinterpret_cast<const unsigned short*>(src) + row * wd;
  uint32_t w[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint32_t lo = x0 + 2 * k < wd ? s[x0 + 2 * k] : 0u, hi = x0 + 2 * k + 1 < wd ? s[x0 + 2 * k + 1] : 0u;
    w[k] = lo | (hi << 16);
  }
  *reinterpret_cast<uint4*>(dst + row * wp + x0) = make_uint4(w[0], w[1], w[2], w[3]);
}

// ---- host ------------------------------------------------------------------------------------------------------------------
// [frame][C][HW] -> boxes of 64 consecutive pixels x C channels
static int make_fmap_tensor_map(CUtensorMap* map, const void* base, int n_frames, int C, int HW) {
  const cuuint64_t dims[3] = {(cuuint64_t)HW, (cuuint64_t)C, (cuuint64_t)n_frames};
  const cuuint64_t strides[2] = {(cuuint64_t)HW * 2, (cuuint64_t)HW * C * 2};
  const cuuint32_t box[3] = {64, (cuuint32_t)C, 1};
  return tma_encode_f16(map, base, 3, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "features, %d frames x %d ch x %d px", n_frames, C, HW);
}

// [frame][C][ht][wp] -> boxes of 64 columns of one image row x C channels (same shared-memory image as a box of the map above)
static int make_fmap_rows_tensor_map(CUtensorMap* map, const void* base, int n_frames, int C, int ht, int wp) {
  const cuuint64_t dims[4] = {(cuuint64_t)wp, (cuuint64_t)ht, (cuuint64_t)C, (cuuint64_t)n_frames};
  const cuuint64_t strides[3] = {(cuuint64_t)wp * 2, (cuuint64_t)ht * wp * 2, (cuuint64_t)C * ht * wp * 2};
  const cuuint32_t box[4] = {64, 1, (cuuint32_t)C, 1};
  return tma_encode_f16(map, base, 4, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "feature rows, %d frames x %d ch x %d x %d",
                        n_frames, C, ht, wp);
}

// bytes of one staged copy [n_frames][C][ht][wp], rounded to 256 so the second copy stays aligned
static size_t staged_bytes(int n_frames, int C, int ht, int wd) {
  const size_t wp = (size_t)((wd + 7) & ~7);
  return ((size_t)n_frames * C * ht * wp * 2 + 255) & ~(size_t)255;
}

template <class P>
static int corr_volume_kernel_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const P& p, dim3 grid, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    DBA_CHECK_CUDA(cudaFuncSetAttribute(corr_volume_pyramid_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, kCvSmem), "corr_volume smem attr");
    attr = true;
  }
  corr_volume_pyramid_kernel<P><<<grid, kCvThreads, kCvSmem, st>>>(tmA, tmB, p);
  DBA_CHECK_LAUNCH("corr_volume_pyramid");
  return DBA_OK;
}

}  // namespace dba
using namespace dba;

// the shapes of the CvParams tiling (512-wide inputs at 1/8 resolution); it alone writes the tiled layout
static bool is_wd64_shape(int ht, int wd) { return wd == 64 && ht % 8 == 0; }

extern "C" int dba_corr_volume_supported(int channels, int ht, int wd, int dtype, int tiled) {
  return (dtype == DBA_F16 && channels == 128 && ht >= 8 && wd >= 8 && (!tiled || is_wd64_shape(ht, wd))) ? 1 : 0;
}

extern "C" size_t dba_corr_volume_workspace_bytes(int n_frames1, int n_frames2, int channels, int ht, int wd) {
  if (n_frames1 <= 0 || n_frames2 <= 0 || channels <= 0 || ht <= 0 || wd <= 0 || wd % 8 == 0) return 0;
  return staged_bytes(n_frames1, channels, ht, wd) + staged_bytes(n_frames2, channels, ht, wd);
}

extern "C" int dba_corr_volume_pyramid(const void* fmap1, const void* fmap2, const int64_t* ii, const int64_t* jj, void* out0, void* out1,
                                       void* out2, void* out3, int n_edges, int n_frames1, int n_frames2, int channels, int ht, int wd,
                                       int dtype, int tiled, void* workspace, size_t workspace_bytes, dba_stream_t stream) {
  DBA_CHECK_ARG(n_edges >= 0 && n_frames1 > 0 && n_frames2 > 0, "bad extents");
  DBA_CHECK_ARG(dtype == DBA_F16, "corr_volume_pyramid: only f16 features (the live system's autocast dtype) are implemented");
  DBA_CHECK_ARG(channels == 128, "corr_volume_pyramid: 128 feature channels expected (reference fnet)");
  DBA_CHECK_ARG(ht >= 8 && wd >= 8, "corr_volume_pyramid: ht and wd must be at least 8 (level 3 must have at least one pixel)");
  DBA_CHECK_ARG(!tiled || is_wd64_shape(ht, wd), "corr_volume_pyramid: the tiled layout is implemented for wd = 64, ht % 8 == 0 (512-wide inputs at 1/8 resolution)");
  const size_t ws_need = dba_corr_volume_workspace_bytes(n_frames1, n_frames2, channels, ht, wd);
  if (n_edges == 0) return DBA_OK;
  DBA_CHECK_ARG(fmap1 && fmap2 && ii && jj && out0 && out1 && out2 && out3, "null pointer");
  DBA_CHECK_ARG((((uintptr_t)fmap1 | (uintptr_t)fmap2 | (uintptr_t)out0 | (uintptr_t)out1 | (uintptr_t)out2 | (uintptr_t)out3) & 15) == 0, "pointers must be 16-byte aligned");
  DBA_CHECK_ARG(n_edges <= 65535, "more than 65535 edges per call");
  if (ws_need > 0) {
    if (!workspace || workspace_bytes < ws_need) {
      set_error("invalid argument: corr_volume_pyramid: wd %% 8 != 0 needs a workspace of %zu bytes (dba_corr_volume_workspace_bytes), got %zu",
                ws_need, workspace ? workspace_bytes : (size_t)0);
      return DBA_ERR_INVALID;
    }
    DBA_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "workspace must be 16-byte aligned");
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int wp = (wd + 7) & ~7;
  const void* f1 = fmap1;
  const void* f2 = fmap2;
  if (wp != wd) {   // TMA strides must be multiples of 16 bytes: copy the frames into rows padded to 8 pixels
    __half* s1 = (__half*)workspace;
    __half* s2 = (__half*)((uint8_t*)workspace + staged_bytes(n_frames1, channels, ht, wd));
    const long long r1 = (long long)n_frames1 * channels * ht, r2 = (long long)n_frames2 * channels * ht;
    corr_volume_stage_kernel<<<(unsigned)((r1 * (wp / 8) + 255) / 256), 256, 0, st>>>((const __half*)fmap1, s1, r1, wd, wp);
    DBA_CHECK_LAUNCH("corr_volume_pyramid(stage fmap1)");
    corr_volume_stage_kernel<<<(unsigned)((r2 * (wp / 8) + 255) / 256), 256, 0, st>>>((const __half*)fmap2, s2, r2, wd, wp);
    DBA_CHECK_LAUNCH("corr_volume_pyramid(stage fmap2)");
    f1 = s1; f2 = s2;
  }
  const dim3 grid((ht * wp + kCvM - 1) / kCvM, n_edges);
  CUtensorMap tmA, tmB;
  int rc = make_fmap_tensor_map(&tmA, f1, n_frames1, channels, ht * wp); if (rc) return rc;
  if (is_wd64_shape(ht, wd)) {
    rc = make_fmap_tensor_map(&tmB, f2, n_frames2, channels, ht * wd); if (rc) return rc;
    CvParams p;
    p.ii = ii; p.jj = jj; p.out0 = (__half*)out0; p.out1 = (__half*)out1; p.out2 = (__half*)out2; p.out3 = (__half*)out3;
    p.HW = ht * wd; p.wd = wd; p.n_chunks = ht * wd / kCvN; p.tiled = tiled;
    return corr_volume_kernel_launch(tmA, tmB, p, grid, st);
  }
  rc = make_fmap_rows_tensor_map(&tmB, f2, n_frames2, channels, ht, wp); if (rc) return rc;
  CvRowsParams p;
  p.ii = ii; p.jj = jj; p.out0 = (__half*)out0; p.out1 = (__half*)out1; p.out2 = (__half*)out2; p.out3 = (__half*)out3;
  p.ht = ht; p.wd = wd; p.wp = wp; p.n_ctiles = (wd + 63) / 64; p.n_rchunks = (ht + 3) / 4;
  p.h1 = ht >> 1; p.w1 = wd >> 1; p.h2 = ht >> 2; p.w2 = wd >> 2; p.h3 = ht >> 3; p.w3 = wd >> 3;
  p.P0 = (size_t)ht * wd; p.P1 = (size_t)p.h1 * p.w1; p.P2 = (size_t)p.h2 * p.w2; p.P3 = (size_t)p.h3 * p.w3;
  return corr_volume_kernel_launch(tmA, tmB, p, grid, st);
}
