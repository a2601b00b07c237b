// 3xTF32 products on the tf32 tensor cores (mma.sync m16n8k8), shared by the training kernels (corr_train.cu, gru_train.cu).
//
// x = hi + lo, both rounded to tf32, and a.b = a_lo.b_hi + a_hi.b_lo + a_hi.b_hi accumulated in fp32, which keeps the error of an fp32
// FMA chain.  The unit of work is a 64 x 64 output tile computed by 256 threads from reduction chunks of kCtK staged in shared memory.
#pragma once
#include <stdint.h>

namespace dba {

constexpr int kCtThreads = 256;
constexpr int kCtTile = 64;    // output tile 64 x 64: warp w computes rows 32 (w & 1) .. + 31, columns 16 (w >> 1) .. + 15
constexpr int kCtK = 32;       // reduction chunk staged in shared memory
constexpr int kLd = kCtTile + 8;   // row pitch of a staged chunk: the fragment loads (8 t + g) hit 32 distinct banks

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(x - __uint_as_float(hi)));
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// acc += the 64 x 64 product of one staged chunk, sa[k][m] x sb[k][n] (k < kCtK), for this warp's 32 x 16 part.  acc[i][j] is the
// m16n8 accumulator of rows 32 wm + 16 i + {g, g + 8}, columns 16 wn + 8 j + {2 t, 2 t + 1} (g = lane / 4, t = lane % 4).  The chunk's
// products accumulate on the tensor cores from zero and are added to acc with fp32 adds: accumulating thousands of terms inside the
// MMA loses low bits of a large running sum (at the training shape, grad fmap2's K = 3072 sums came out 7.5x less accurate than fp32's).
__device__ __forceinline__ void chunk_mma_3xtf32(const float (*sa)[kLd], const float (*sb)[kLd], float (&acc)[2][2][4], int wm, int wn,
                                                 int lane) {
  const int g = lane >> 2, t = lane & 3;
  float part[2][2][4] = {};
#pragma unroll
  for (int k0 = 0; k0 < kCtK; k0 += 8) {
    uint32_t ah[2][4], al[2][4], bh[2][2], bl[2][2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const int m = 32 * wm + 16 * i + g;
      split_tf32(sa[k0 + t][m], ah[i][0], al[i][0]);
      split_tf32(sa[k0 + t][m + 8], ah[i][1], al[i][1]);
      split_tf32(sa[k0 + t + 4][m], ah[i][2], al[i][2]);
      split_tf32(sa[k0 + t + 4][m + 8], ah[i][3], al[i][3]);
    }
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int n = 16 * wn + 8 * j + g;
      split_tf32(sb[k0 + t][n], bh[j][0], bl[j][0]);
      split_tf32(sb[k0 + t + 4][n], bh[j][1], bl[j][1]);
    }
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
      for (int j = 0; j < 2; j++) {
        mma_tf32(part[i][j], al[i], bh[j]);
        mma_tf32(part[i][j], ah[i], bl[j]);
        mma_tf32(part[i][j], ah[i], bh[j]);
      }
  }
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int h = 0; h < 4; h++) acc[i][j][h] += part[i][j][h];
}

}  // namespace dba
