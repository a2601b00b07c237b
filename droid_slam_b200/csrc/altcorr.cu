// altcorr_forward / altcorr_backward for sm_90a (on-the-fly correlation, no stored volume).
//
// Replaces reference src/altcorr_kernel.cu:24-225.  Forward semantics (oracle/corr.py::altcorr_forward):
//   raw[b,m,a,c,y,x] = sum_ch T(f1[b,ii[m],ch,y,x]/4) * T(f2[b,jj[m],ch,floor(y0)+a-r,floor(x0)+c-r]/4)   (fp32 accumulation,
//   product rounded in the feature dtype T), zero outside fmap2;  then the bilinear blend of the four shifted
//   (2r+1)^2 sub-windows, every elementwise step rounded in T exactly like the eight ATen ops of the reference
//   (:160-169).  The reference returns a permuted view; this kernel writes the contiguous [B,M,y-off,x-off,H,W]
//   tensor and the binding returns the same permuted view.
//
// Mapping: CTA = 32 consecutive pixels x (2r+2) window rows.  A warp is one window row of 32 neighbouring pixels, so
// for smooth flow its 2r+2 taps per channel are contiguous runs of fmap2 (coalesced through L1) and the fmap1 value
// is a coalesced load shared by the rows through L1.  Raw windows go through shared memory; the blend and the
// [.., y-off, x-off, H, W] stores are coalesced over the 32 pixels.  One launch replaces kernel + 8 ATen passes.
#include "common.cuh"

namespace dba {

template <typename T> struct AltMath;
template <> struct AltMath<float> {
  static __device__ __forceinline__ float quarter(float v) { return (float)((double)v / 4.0); }
  static __device__ __forceinline__ float mac(float s, float a, float b) { return fmaf(a, b, s); }   // nvcc contracts `s += f1*f2`
  static __device__ __forceinline__ float from_f32(float v) { return v; }
  static __device__ __forceinline__ float to_f32(float v) { return v; }
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
};
template <> struct AltMath<double> {
  static __device__ __forceinline__ double quarter(double v) { return v / 4.0; }
  static __device__ __forceinline__ float mac(float s, double a, double b) { return s + (float)(a * b); }
  static __device__ __forceinline__ double from_f32(float v) { return (double)v; }
  static __device__ __forceinline__ float to_f32(double v) { return (float)v; }
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
};
template <> struct AltMath<__half> {
  static __device__ __forceinline__ __half quarter(__half v) { return __float2half_rn((float)((double)__half2float(v) / 4.0)); }
  static __device__ __forceinline__ float mac(float s, __half a, __half b) { return s + __half2float(__hmul_rn(a, b)); }
  static __device__ __forceinline__ __half from_f32(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half mul(__half a, __half b) { return __hmul_rn(a, b); }
  static __device__ __forceinline__ __half add(__half a, __half b) { return __hadd_rn(a, b); }
  static __device__ __forceinline__ __half sub(__half a, __half b) { return __hsub_rn(a, b); }
};
template <> struct AltMath<__nv_bfloat16> {   // extension (not dispatched by the reference): same scheme with bf16 rounding
  static __device__ __forceinline__ __nv_bfloat16 quarter(__nv_bfloat16 v) { return __float2bfloat16_rn(__bfloat162float(v) * 0.25f); }
  static __device__ __forceinline__ float mac(float s, __nv_bfloat16 a, __nv_bfloat16 b) {
    return s + __bfloat162float(__float2bfloat16_rn(__bfloat162float(a) * __bfloat162float(b)));
  }
  static __device__ __forceinline__ __nv_bfloat16 from_f32(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 mul(__nv_bfloat16 a, __nv_bfloat16 b) { return __float2bfloat16_rn(__bfloat162float(a) * __bfloat162float(b)); }
  static __device__ __forceinline__ __nv_bfloat16 add(__nv_bfloat16 a, __nv_bfloat16 b) { return __float2bfloat16_rn(__bfloat162float(a) + __bfloat162float(b)); }
  static __device__ __forceinline__ __nv_bfloat16 sub(__nv_bfloat16 a, __nv_bfloat16 b) { return __float2bfloat16_rn(__bfloat162float(a) - __bfloat162float(b)); }
};

constexpr int kAltMaxD = 16;   // 2r+2 <= 16  (r <= 7)

template <typename T, int D>
__global__ void __launch_bounds__(32 * D) altcorr_fwd_kernel(const T* __restrict__ fmap1, const T* __restrict__ fmap2,
                                                              const float* __restrict__ coords, const int64_t* __restrict__ us,
                                                              const int64_t* __restrict__ vs, T* __restrict__ out,
                                                              int N1, int N2, int C, int HW, int W, int H2, int W2, int M) {
  typedef AltMath<T> A;
  constexpr int R = (D - 2) / 2;
  __shared__ float s_raw[D][D][33];
  const int lane = threadIdx.x;       // pixel within the group of 32
  const int a = threadIdx.y;          // window row (y offset)
  const int m = blockIdx.y, b = blockIdx.z;
  const int p = blockIdx.x * 32 + lane;
  const bool pok = p < HW;
  const int pc = pok ? p : HW - 1;
  const int ix = (int)us[m], jx = (int)vs[m];
  const float x = coords[(((size_t)b * M + m) * 2 + 0) * HW + pc];
  const float y = coords[(((size_t)b * M + m) * 2 + 1) * HW + pc];
  const int i1 = floor_to_int_sat(floorf(y)) + (a - R);
  const int j1 = floor_to_int_sat(floorf(x)) - R;
  const bool rowok = (unsigned)i1 < (unsigned)H2;
  const T* f1 = fmap1 + (((size_t)b * N1 + ix) * C) * HW + pc;
  const T* f2 = fmap2 + (((size_t)b * N2 + jx) * C) * (size_t)H2 * W2 + (size_t)(rowok ? i1 : 0) * W2;
  float acc[D];
  bool inb[D];
#pragma unroll
  for (int c = 0; c < D; c++) { acc[c] = 0.f; inb[c] = rowok && (unsigned)(j1 + c) < (unsigned)W2; }
  for (int ch = 0; ch < C; ch++) {
    const T v1 = A::quarter(f1[(size_t)ch * HW]);
    const T* row = f2 + (size_t)ch * H2 * W2;
#pragma unroll
    for (int c = 0; c < D; c++) {
      if (inb[c]) acc[c] = A::mac(acc[c], v1, A::quarter(row[j1 + c]));
    }
  }
#pragma unroll
  for (int c = 0; c < D; c++) s_raw[a][c][lane] = A::to_f32(A::from_f32(acc[c]));   // raw window is stored in T (:74)
  __syncthreads();
  // ---- bilinear blend, all steps rounded in T (reference :158-169)
  const T dx = A::from_f32(x - floorf(x));
  const T dy = A::from_f32(y - floorf(y));
  const T one = A::from_f32(1.0f);
  const T w00 = A::mul(A::sub(one, dx), A::sub(one, dy));
  const T w01 = A::mul(dx, A::sub(one, dy));       // pairs with raw[a][c+1]
  const T w10 = A::mul(A::sub(one, dx), dy);       // pairs with raw[a+1][c]
  const T w11 = A::mul(dx, dy);
  constexpr int RD = D - 1;
  if (pok) {
    for (int o = a; o < RD * RD; o += D) {
      const int oa = o / RD, oc = o - oa * RD;
      T v = A::mul(w00, A::from_f32(s_raw[oa][oc][lane]));
      v = A::add(v, A::mul(w01, A::from_f32(s_raw[oa][oc + 1][lane])));
      v = A::add(v, A::mul(w10, A::from_f32(s_raw[oa + 1][oc][lane])));
      v = A::add(v, A::mul(w11, A::from_f32(s_raw[oa + 1][oc + 1][lane])));
      out[((((size_t)b * M + m) * RD + oa) * RD + oc) * HW + p] = v;
    }
  }
}

// backward (training only; kept for API parity): thread per (pixel, tap), loop over channels, atomics in T.
// Takes the gradient of the BLENDED output like the reference host function (src/altcorr_kernel.cu:175-225).
template <typename T> __device__ __forceinline__ void atomic_add_t(T* p, T v) { atomicAdd(p, v); }

template <typename T>
__global__ void __launch_bounds__(256) altcorr_bwd_kernel(int R, const T* __restrict__ fmap1, const T* __restrict__ fmap2,
                                                          const float* __restrict__ coords, const int64_t* __restrict__ us,
                                                          const int64_t* __restrict__ vs, const float* __restrict__ corr_grad,
                                                          T* __restrict__ g1, T* __restrict__ g2, int B, int N1, int N2, int C, int H,
                                                          int W, int H2, int W2, int M) {
  typedef AltMath<T> A;
  const int D = 2 * R + 2;
  long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)B * M * H * W * D * D;
  if (n >= total) return;
  const int jj = (int)(n % D); n /= D;
  const int ii = (int)(n % D); n /= D;
  const int j0 = (int)(n % W); n /= W;
  const int i0 = (int)(n % H); n /= H;
  const int m = (int)(n % M); n /= M;
  const int b = (int)n;
  const int ix = (int)us[m], jx = (int)vs[m];
  const size_t HW = (size_t)H * W;
  const float x = coords[(((size_t)b * M + m) * 2 + 0) * HW + (size_t)i0 * W + j0];
  const float y = coords[(((size_t)b * M + m) * 2 + 1) * HW + (size_t)i0 * W + j0];
  const int i1 = floor_to_int_sat(floorf(y)) + (ii - R);
  const int j1 = floor_to_int_sat(floorf(x)) + (jj - R);
  if (!((unsigned)i1 < (unsigned)H2 && (unsigned)j1 < (unsigned)W2)) return;
  // raw-window gradient from the gradient of the blended output (reference altcorr_cuda_backward, :190-207):
  // corr_grad is [B,M,x-off,y-off,H,W] (what autograd hands back for the permuted view), RD = 2r+1
  const int RD = D - 1;
  const float dx = x - floorf(x), dy = y - floorf(y);
  const size_t gbase = ((size_t)b * M + m) * RD * RD;
  const size_t pix = (size_t)i0 * W + j0;
  auto G = [&](int a, int c) -> float { return corr_grad[(gbase + (size_t)c * RD + a) * HW + pix]; };
  float gsum = 0.f;
  bool first = true;
  auto acc_term = [&](float w, float gv) { const float t = __fmul_rn(w, gv); gsum = first ? t : __fadd_rn(gsum, t); first = false; };
  // g1 + g2 + g3 + g4 with zeros where the slice does not cover (ii,jj)
  acc_term(__fmul_rn(1.f - dx, 1.f - dy), (ii < RD && jj < RD) ? G(ii, jj) : 0.f);
  acc_term(__fmul_rn(dx, 1.f - dy), (ii < RD && jj >= 1) ? G(ii, jj - 1) : 0.f);
  acc_term(__fmul_rn(1.f - dx, dy), (ii >= 1 && jj < RD) ? G(ii - 1, jj) : 0.f);
  acc_term(__fmul_rn(dx, dy), (ii >= 1 && jj >= 1) ? G(ii - 1, jj - 1) : 0.f);
  const T g = A::from_f32(gsum);
  const size_t o1 = (((size_t)b * N1 + ix) * C) * HW + (size_t)i0 * W + j0;
  const size_t o2 = (((size_t)b * N2 + jx) * C) * (size_t)H2 * W2 + (size_t)i1 * W2 + j1;
  for (int ch = 0; ch < C; ch++) {
    atomic_add_t<T>(g1 + o1 + (size_t)ch * HW, A::mul(g, fmap2[o2 + (size_t)ch * H2 * W2]));
    atomic_add_t<T>(g2 + o2 + (size_t)ch * H2 * W2, A::mul(g, fmap1[o1 + (size_t)ch * HW]));
  }
}

template <typename T>
static int launch_alt_fwd(const void* f1, const void* f2, const float* coords, const int64_t* ii, const int64_t* jj, void* out, int B,
                          int N1, int N2, int C, int H, int W, int H2, int W2, int M, int radius, cudaStream_t st) {
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, M, B);
#define ALT_CASE(Dv)                                                                                                        \
  case Dv:                                                                                                                  \
    altcorr_fwd_kernel<T, Dv><<<grid, dim3(32, Dv), 0, st>>>((const T*)f1, (const T*)f2, coords, ii, jj, (T*)out, N1, N2, C, HW, W, \
                                                              H2, W2, M);                                                   \
    break;
  switch (2 * radius + 2) {
    ALT_CASE(2) ALT_CASE(4) ALT_CASE(6) ALT_CASE(8) ALT_CASE(10) ALT_CASE(12) ALT_CASE(14) ALT_CASE(16)
    default: dba::set_error("altcorr radius %d unsupported (0..7)", radius); return DBA_ERR_INVALID;
  }
#undef ALT_CASE
  DBA_CHECK_LAUNCH("altcorr_forward");
  return DBA_OK;
}

template <typename T>
static int launch_alt_bwd(const void* f1, const void* f2, const float* coords, const float* cg, const int64_t* ii, const int64_t* jj,
                          void* g1, void* g2, int B, int N1, int N2, int C, int H, int W, int H2, int W2, int M, int radius,
                          cudaStream_t st) {
  DBA_CHECK_CUDA(cudaMemsetAsync(g1, 0, (size_t)B * N1 * C * H * W * sizeof(T), st), "altcorr_backward memset");
  DBA_CHECK_CUDA(cudaMemsetAsync(g2, 0, (size_t)B * N2 * C * H2 * W2 * sizeof(T), st), "altcorr_backward memset");
  const int D = 2 * radius + 2;
  const long long total = (long long)B * M * H * W * D * D;
  if (total == 0) return DBA_OK;
  const long long blocks = (total + 255) / 256;
  DBA_CHECK_ARG(blocks < 0x7fffffffLL, "altcorr_backward problem too large");
  altcorr_bwd_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(radius, (const T*)f1, (const T*)f2, coords, ii, jj, cg, (T*)g1, (T*)g2, B, N1,
                                                          N2, C, H, W, H2, W2, M);
  DBA_CHECK_LAUNCH("altcorr_backward");
  return DBA_OK;
}

// ---- AltCorrBlock (reference modules/corr.py:89-117) on a private channels-last pyramid -------------------------------------
//
// altcorr_pyramid_kernel: level l of the reference is F.avg_pool2d applied l times to the feature maps (each pass: fp32 sum of the
// 2x2 window in the order (0,0),(0,1),(1,0),(1,1) starting from 0, / 4, rounded to T; floor sizes).  Every level is stored as
// AltMath::quarter(level value) in [BN, H>>l, W>>l, C], so the /4 of the correlation (reference altcorr_kernel.cu:67-68) is paid once per
// element.  CTA = one channel chunk of kPyrCC channels x kPyrTX column tiles of S x S level-0 pixels (S = 2^(L-1)); a thread walks the
// whole pooling chain of one tile and one channel in registers (reads: a warp covers 4 channel rows of 8S contiguous pixels), the
// quartered levels are transposed through shared memory and written as 16-byte channel vectors.  In shared memory every tile row
// of a level is followed by one padding pixel, so the 8 tiles of a warp write to different banks.
constexpr int kPyrTX = 8;
constexpr int kPyrCC = 8;

constexpr int pyr_smem_elems(int L) {   // the L quartered levels of one CTA, level l having s = S >> l rows of kPyrTX padded tile rows
  int n = 0;
  for (int l = 0; l < L; l++) n += kPyrCC * ((1 << (L - 1)) >> l) * kPyrTX * (((1 << (L - 1)) >> l) + 1);
  return n;
}
__device__ __forceinline__ int pyr_slot(int r, int col, int s) { return r * kPyrTX * (s + 1) + col + col / s; }   // s = tile width

template <typename T>
__device__ __forceinline__ T pool4(T a, T b, T c, T d) {   // ATen avg_pool2d (CUDA, NCHW): float aveval = 0; aveval += x ...; / 4
  float s = __fadd_rn(0.f, AltMath<T>::to_f32(a));
  s = __fadd_rn(s, AltMath<T>::to_f32(b));
  s = __fadd_rn(s, AltMath<T>::to_f32(c));
  s = __fadd_rn(s, AltMath<T>::to_f32(d));
  return AltMath<T>::from_f32(__fdiv_rn(s, 4.f));
}

template <typename T, int L>
__global__ void __launch_bounds__(kPyrTX * kPyrCC) altcorr_pyramid_kernel(const T* __restrict__ fmaps, T* __restrict__ o0, T* __restrict__ o1,
                                                                          T* __restrict__ o2, T* __restrict__ o3, int C, int H, int W, int TY, int TXB) {
  typedef AltMath<T> A;
  constexpr int S = 1 << (L - 1);
  constexpr int SW = kPyrTX * S;
  __shared__ __align__(16) T sm[pyr_smem_elems(L)];
  const int NC = C / kPyrCC;
  long long blk = blockIdx.x;
  const int chunk = (int)(blk % NC); blk /= NC;
  const int txb = (int)(blk % TXB); blk /= TXB;
  const int ty = (int)(blk % TY);
  const long long bn = blk / TY;
  const int tx = threadIdx.x, cc = threadIdx.y;
  const T* src = fmaps + ((size_t)bn * C + chunk * kPyrCC + cc) * H * W;
  const int y0 = ty * S, x0 = (txb * kPyrTX + tx) * S;
  T v[S][S];
#pragma unroll
  for (int r = 0; r < S; r++)
#pragma unroll
    for (int q = 0; q < S; q++) {
      const int y = y0 + r, x = x0 + q;
      v[r][q] = (y < H && x < W) ? src[(size_t)y * W + x] : A::from_f32(0.f);
      sm[pyr_slot(r, tx * S + q, S) * kPyrCC + cc] = A::quarter(v[r][q]);
    }
  int off = S * kPyrTX * (S + 1) * kPyrCC;
#pragma unroll
  for (int l = 1; l < L; l++) {
    const int s = S >> l;
#pragma unroll
    for (int r = 0; r < (S >> l); r++)
#pragma unroll
      for (int q = 0; q < (S >> l); q++) {   // in place: (r,q) is written after its 2x2 source block was read, and no later block reads it
        v[r][q] = pool4<T>(v[2 * r][2 * q], v[2 * r][2 * q + 1], v[2 * r + 1][2 * q], v[2 * r + 1][2 * q + 1]);
        sm[off + pyr_slot(r, tx * s + q, s) * kPyrCC + cc] = A::quarter(v[r][q]);
      }
    off += s * kPyrTX * (s + 1) * kPyrCC;
  }
  __syncthreads();
  constexpr int VPP = kPyrCC * sizeof(T) / 16;   // 16-byte vectors per pixel and chunk
  T* outs[4] = {o0, o1, o2, o3};
  off = 0;
  const int tid = cc * kPyrTX + tx;
#pragma unroll
  for (int l = 0; l < L; l++) {
    const int s = S >> l, sw = SW >> l, Hl = H >> l, Wl = W >> l;
    for (int t = tid; t < s * sw * VPP; t += kPyrTX * kPyrCC) {
      const int pix = t / VPP, k = t - pix * VPP;
      const int r = pix / sw, col = pix - r * sw;
      const int y = ty * s + r, x = txb * sw + col;
      if (y < Hl && x < Wl)
        reinterpret_cast<uint4*>(outs[l] + (((size_t)bn * Hl + y) * Wl + x) * C + chunk * kPyrCC)[k] =
            reinterpret_cast<const uint4*>(sm + off + pyr_slot(r, col, s) * kPyrCC)[k];
    }
    off += s * kPyrTX * (s + 1) * kPyrCC;
  }
}

// altcorr_lookup_pyramid_kernel: AltCorrBlock.__call__ = for every level l, altcorr_forward(level 0, level l, coords / 2^l) flattened
// and stacked, i.e. out[b,m,l*49 + xo*7 + yo,y,x].  Same arithmetic as altcorr_fwd_kernel (R = 3): per raw tap one fp32 sum in
// ascending channel order of T-rounded products, raw window rounded to T, bilinear blend in T.  Same mapping too (CTA = 32 pixels x 8
// window rows, a warp = one window row), but the operands come as 16-byte channel vectors: the 32 source-pixel vectors are staged in
// shared memory once for all levels (row padded by 16 bytes: conflict-free), each tap reads 8 (f16) or 4 (f32) channels per load.
constexpr int kLkMaxDynSmem = 200 * 1024;

template <typename T> struct AltVec;
template <> struct AltVec<__half> {
  static __device__ __forceinline__ float mac(float s, const uint4& u1, const uint4& u2) {
    const __half2* a = reinterpret_cast<const __half2*>(&u1);
    const __half2* b = reinterpret_cast<const __half2*>(&u2);
#pragma unroll
    for (int i = 0; i < 4; i++) {   // each lane of __hmul2_rn rounds like __hmul_rn (AltMath<__half>::mac)
      const __half2 p = __hmul2_rn(a[i], b[i]);
      s = s + __low2float(p);
      s = s + __high2float(p);
    }
    return s;
  }
};
template <> struct AltVec<float> {
  static __device__ __forceinline__ float mac(float s, const uint4& u1, const uint4& u2) {
    const float4 a = *reinterpret_cast<const float4*>(&u1), b = *reinterpret_cast<const float4*>(&u2);
    s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); s = fmaf(a.w, b.w, s);
    return s;
  }
};

template <typename T, int L>
__global__ void __launch_bounds__(256) altcorr_lookup_pyramid_kernel(const T* __restrict__ p0, const T* __restrict__ p1, const T* __restrict__ p2,
                                                                     const T* __restrict__ p3, const float* __restrict__ coords,
                                                                     const int64_t* __restrict__ us, const int64_t* __restrict__ vs,
                                                                     T* __restrict__ out, int N, int C, int H, int W, int M) {
  typedef AltMath<T> A;
  constexpr int R = 3, D = 2 * R + 2, RD = D - 1;
  constexpr int VE = 16 / sizeof(T);   // channels per 16-byte vector
  extern __shared__ uint4 s_f1[];      // [32][C/VE + 1]
  __shared__ float s_raw[D][D][33];
  const int lane = threadIdx.x, a = threadIdx.y;
  const int m = blockIdx.y, b = blockIdx.z;
  const int HW = H * W;
  const int p = blockIdx.x * 32 + lane;
  const bool pok = p < HW;
  const int pc = pok ? p : HW - 1;
  const int ix = (int)us[m], jx = (int)vs[m];
  const int CV = C / VE, CVP = CV + 1;
  {
    const uint4* f1 = reinterpret_cast<const uint4*>(p0 + ((size_t)b * N + ix) * HW * C);
    for (int t = a * 32 + lane; t < 32 * CV; t += 32 * D) {
      const int q = t / CV, k = t - q * CV;
      s_f1[q * CVP + k] = f1[(size_t)min(blockIdx.x * 32 + q, HW - 1) * CV + k];
    }
  }
  const float x = coords[(((size_t)b * M + m) * 2 + 0) * HW + pc];
  const float y = coords[(((size_t)b * M + m) * 2 + 1) * HW + pc];
  const uint4* f1s = s_f1 + lane * CVP;
  T* o = out + ((size_t)b * M + m) * (L * RD * RD) * HW + p;
  __syncthreads();
#pragma unroll 1
  for (int l = 0; l < L; l++) {
    const int Hl = H >> l, Wl = W >> l;
    const float sc = 1.f / (float)(1 << l);   // exact: x * 2^-l == x / 2^l (reference: coords / 2**i)
    const float xl = __fmul_rn(x, sc), yl = __fmul_rn(y, sc);
    const int i1 = floor_to_int_sat(floorf(yl)) + (a - R);
    const int j1 = floor_to_int_sat(floorf(xl)) - R;
    const bool rowok = (unsigned)i1 < (unsigned)Hl;
    const T* level = l == 0 ? p0 : l == 1 ? p1 : l == 2 ? p2 : p3;   // a select, not an indexed array: no local-memory stack frame
    const uint4* f2 = reinterpret_cast<const uint4*>(level + (((size_t)b * N + jx) * Hl + (rowok ? i1 : 0)) * Wl * C);
    float acc[D];
    bool inb[D];
#pragma unroll
    for (int c = 0; c < D; c++) { acc[c] = 0.f; inb[c] = rowok && (unsigned)(j1 + c) < (unsigned)Wl; }
    for (int k = 0; k < CV; k++) {
      const uint4 u1 = f1s[k];
#pragma unroll
      for (int c = 0; c < D; c++) {
        if (inb[c]) acc[c] = AltVec<T>::mac(acc[c], u1, __ldg(f2 + (size_t)(j1 + c) * CV + k));
      }
    }
#pragma unroll
    for (int c = 0; c < D; c++) s_raw[a][c][lane] = A::to_f32(A::from_f32(acc[c]));
    __syncthreads();
    const T dx = A::from_f32(xl - floorf(xl));
    const T dy = A::from_f32(yl - floorf(yl));
    const T one = A::from_f32(1.0f);
    const T w00 = A::mul(A::sub(one, dx), A::sub(one, dy));
    const T w01 = A::mul(dx, A::sub(one, dy));
    const T w10 = A::mul(A::sub(one, dx), dy);
    const T w11 = A::mul(dx, dy);
    if (pok) {
      for (int t = a; t < RD * RD; t += D) {
        const int oa = t / RD, oc = t - oa * RD;   // oa: y offset (window row), oc: x offset
        T v = A::mul(w00, A::from_f32(s_raw[oa][oc][lane]));
        v = A::add(v, A::mul(w01, A::from_f32(s_raw[oa][oc + 1][lane])));
        v = A::add(v, A::mul(w10, A::from_f32(s_raw[oa + 1][oc][lane])));
        v = A::add(v, A::mul(w11, A::from_f32(s_raw[oa + 1][oc + 1][lane])));
        o[(size_t)(l * RD * RD + oc * RD + oa) * HW] = v;   // channel l*49 + xo*7 + yo
      }
    }
    __syncthreads();
  }
}

template <typename T, int L>
static int launch_alt_pyramid_l(const void* fmaps, void* const* outs, int BN, int C, int H, int W, cudaStream_t st) {
  constexpr int S = 1 << (L - 1);
  const int TY = (H + S - 1) / S, TXB = (W + kPyrTX * S - 1) / (kPyrTX * S);
  const long long blocks = (long long)BN * TY * TXB * (C / kPyrCC);
  DBA_CHECK_ARG(blocks < 0x7fffffffLL, "altcorr_pyramid problem too large");
  altcorr_pyramid_kernel<T, L><<<(unsigned)blocks, dim3(kPyrTX, kPyrCC), 0, st>>>((const T*)fmaps, (T*)outs[0], (T*)outs[1], (T*)outs[2],
                                                                                 (T*)outs[3], C, H, W, TY, TXB);
  DBA_CHECK_LAUNCH("altcorr_pyramid");
  return DBA_OK;
}

template <typename T>
static int launch_alt_pyramid(const void* fmaps, void* const* outs, int BN, int C, int H, int W, int levels, cudaStream_t st) {
  switch (levels) {
    case 1: return launch_alt_pyramid_l<T, 1>(fmaps, outs, BN, C, H, W, st);
    case 2: return launch_alt_pyramid_l<T, 2>(fmaps, outs, BN, C, H, W, st);
    case 3: return launch_alt_pyramid_l<T, 3>(fmaps, outs, BN, C, H, W, st);
    default: return launch_alt_pyramid_l<T, 4>(fmaps, outs, BN, C, H, W, st);
  }
}

template <typename T, int L>
static int launch_alt_lookup_l(const void* const* pyr, const float* coords, const int64_t* ii, const int64_t* jj, void* out, int B, int N,
                               int C, int H, int W, int M, cudaStream_t st) {
  const size_t smem = (size_t)32 * (C / (16 / sizeof(T)) + 1) * 16;
  DBA_CHECK_ARG(smem <= (size_t)kLkMaxDynSmem, "altcorr_lookup_pyramid: too many channels");
  auto kern = altcorr_lookup_pyramid_kernel<T, L>;
  if (smem > 32 * 1024)
    DBA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "altcorr_lookup_pyramid smem");
  dim3 grid((H * W + 31) / 32, M, B);
  kern<<<grid, dim3(32, 8), smem, st>>>((const T*)pyr[0], (const T*)pyr[1], (const T*)pyr[2], (const T*)pyr[3], coords, ii, jj, (T*)out, N,
                                        C, H, W, M);
  DBA_CHECK_LAUNCH("altcorr_lookup_pyramid");
  return DBA_OK;
}

template <typename T>
static int launch_alt_lookup(const void* const* pyr, const float* coords, const int64_t* ii, const int64_t* jj, void* out, int B, int N,
                             int C, int H, int W, int M, int levels, cudaStream_t st) {
  switch (levels) {
    case 1: return launch_alt_lookup_l<T, 1>(pyr, coords, ii, jj, out, B, N, C, H, W, M, st);
    case 2: return launch_alt_lookup_l<T, 2>(pyr, coords, ii, jj, out, B, N, C, H, W, M, st);
    case 3: return launch_alt_lookup_l<T, 3>(pyr, coords, ii, jj, out, B, N, C, H, W, M, st);
    default: return launch_alt_lookup_l<T, 4>(pyr, coords, ii, jj, out, B, N, C, H, W, M, st);
  }
}

}  // namespace dba
using namespace dba;

static int check_alt(int B, int N1, int N2, int C, int H, int W, int H2, int W2, int M, int radius, int dtype) {
  DBA_CHECK_ARG(B >= 0 && N1 >= 0 && N2 >= 0 && C >= 0 && H >= 0 && W >= 0 && H2 >= 0 && W2 >= 0 && M >= 0, "negative extent");
  DBA_CHECK_ARG(radius >= 0 && radius <= 7, "radius out of range (0..7)");
  DBA_CHECK_ARG(dtype == DBA_F32 || dtype == DBA_F16 || dtype == DBA_F64 || dtype == DBA_BF16, "unsupported dtype");
  DBA_CHECK_ARG(M <= 65535 && B <= 65535, "more than 65535 edges per altcorr call");
  return DBA_OK;
}

extern "C" int dba_altcorr_forward(const void* fmap1, const void* fmap2, const float* coords, const int64_t* ii, const int64_t* jj,
                                   void* out, int B, int N1, int N2, int C, int H, int W, int H2, int W2, int M, int radius, int dtype,
                                   dba_stream_t stream) {
  int rc = check_alt(B, N1, N2, C, H, W, H2, W2, M, radius, dtype);
  if (rc) return rc;
  if ((long long)B * M * H * W == 0) return DBA_OK;
  DBA_CHECK_ARG(fmap1 && fmap2 && coords && ii && jj && out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case DBA_F32: return launch_alt_fwd<float>(fmap1, fmap2, coords, ii, jj, out, B, N1, N2, C, H, W, H2, W2, M, radius, st);
    case DBA_F16: return launch_alt_fwd<__half>(fmap1, fmap2, coords, ii, jj, out, B, N1, N2, C, H, W, H2, W2, M, radius, st);
    case DBA_F64: return launch_alt_fwd<double>(fmap1, fmap2, coords, ii, jj, out, B, N1, N2, C, H, W, H2, W2, M, radius, st);
    default: return launch_alt_fwd<__nv_bfloat16>(fmap1, fmap2, coords, ii, jj, out, B, N1, N2, C, H, W, H2, W2, M, radius, st);
  }
}

extern "C" int dba_altcorr_backward(const void* fmap1, const void* fmap2, const float* coords, const float* corr_grad,
                                    const int64_t* ii, const int64_t* jj, void* fmap1_grad, void* fmap2_grad, int B, int N1, int N2, int C,
                                    int H, int W, int H2, int W2, int M, int radius, int dtype, dba_stream_t stream) {
  int rc = check_alt(B, N1, N2, C, H, W, H2, W2, M, radius, dtype);
  if (rc) return rc;
  DBA_CHECK_ARG(fmap1_grad && fmap2_grad, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case DBA_F32: return launch_alt_bwd<float>(fmap1, fmap2, coords, corr_grad, ii, jj, fmap1_grad, fmap2_grad, B, N1, N2, C, H, W, H2, W2, M, radius, st);
    case DBA_F16: return launch_alt_bwd<__half>(fmap1, fmap2, coords, corr_grad, ii, jj, fmap1_grad, fmap2_grad, B, N1, N2, C, H, W, H2, W2, M, radius, st);
    case DBA_F64: return launch_alt_bwd<double>(fmap1, fmap2, coords, corr_grad, ii, jj, fmap1_grad, fmap2_grad, B, N1, N2, C, H, W, H2, W2, M, radius, st);
    default: return launch_alt_bwd<__nv_bfloat16>(fmap1, fmap2, coords, corr_grad, ii, jj, fmap1_grad, fmap2_grad, B, N1, N2, C, H, W, H2, W2, M, radius, st);
  }
}

// shapes the channels-last pyramid kernels are built for (include/droid_b200.h); extents as in check_alt
static int check_alt_pyramid(int B, int N, int C, int H, int W, int M, int levels, int radius, int dtype) {
  int rc = check_alt(B, N, N, C, H, W, H >> 1, W >> 1, M, radius, dtype);
  if (rc) return rc;
  DBA_CHECK_ARG(dtype == DBA_F32 || dtype == DBA_F16, "altcorr pyramid: float16 or float32 feature maps expected");
  DBA_CHECK_ARG(radius == 3, "altcorr pyramid: radius 3 expected");
  DBA_CHECK_ARG(levels >= 1 && levels <= 4, "altcorr pyramid: 1..4 levels expected");
  DBA_CHECK_ARG(C % 8 == 0, "altcorr pyramid: the channel count must be a multiple of 8");
  DBA_CHECK_ARG(H >= (1 << (levels - 1)) && W >= (1 << (levels - 1)), "altcorr pyramid: H and W must be at least 2^(levels-1)");
  DBA_CHECK_ARG((long long)H * W < 0x7fffffffLL, "altcorr pyramid: image too large");
  return DBA_OK;
}

extern "C" int dba_altcorr_pyramid(const void* fmaps, void* out0, void* out1, void* out2, void* out3, int B, int N, int C, int H, int W,
                                   int levels, int dtype, dba_stream_t stream) {
  int rc = check_alt_pyramid(B, N, C, H, W, 0, levels, 3, dtype);
  if (rc) return rc;
  if ((long long)B * N * C == 0) return DBA_OK;
  void* outs[4] = {out0, out1, out2, out3};
  DBA_CHECK_ARG(fmaps, "null pointer");
  for (int l = 0; l < levels; l++) DBA_CHECK_ARG(outs[l], "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DBA_F16) return launch_alt_pyramid<__half>(fmaps, outs, B * N, C, H, W, levels, st);
  return launch_alt_pyramid<float>(fmaps, outs, B * N, C, H, W, levels, st);
}

extern "C" int dba_altcorr_lookup_pyramid(const void* p0, const void* p1, const void* p2, const void* p3, const float* coords,
                                          const int64_t* ii, const int64_t* jj, void* out, int B, int N, int C, int H, int W, int M,
                                          int levels, int radius, int dtype, dba_stream_t stream) {
  int rc = check_alt_pyramid(B, N, C, H, W, M, levels, radius, dtype);
  if (rc) return rc;
  if ((long long)B * M == 0) return DBA_OK;
  const void* pyr[4] = {p0, p1, p2, p3};
  DBA_CHECK_ARG(coords && ii && jj && out, "null pointer");
  for (int l = 0; l < levels; l++) DBA_CHECK_ARG(pyr[l], "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DBA_F16) return launch_alt_lookup<__half>(pyr, coords, ii, jj, out, B, N, C, H, W, M, levels, st);
  return launch_alt_lookup<float>(pyr, coords, ii, jj, out, B, N, C, H, W, M, levels, st);
}
