// `droid_backends` -- drop-in Python extension.  It exports the reference's nine callables (reference src/droid.cpp:93-259: ba,
// frame_distance, projmap, depth_filter, iproj, altcorr_forward, altcorr_backward, corr_index_forward, corr_index_backward) with identical
// positional signatures and return shapes, plus the native extensions below them (correlation pyramids, reprojection, factor-graph
// step, update operator, encoders, edge selection, trajectory filler).  Everything runs on the C ABI of include/droid_b200.h
// (libdroid_b200.so, hand-written sm_90a kernels).
//
// torch is used here for what the reference binding uses it for: tensor handles, the caching allocator, the current stream.
// Differences from the reference binding, all strictly safer: a CUDAGuard on the tensors' device, launches on torch's CURRENT stream
// (the reference uses the legacy default stream), and every tensor argument's device, dtype, layout and shape checked before any launch
// (Expect below), with messages that name the entry point and the argument.  There is no CPU fallback: every call needs CUDA tensors and
// fails loudly otherwise.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <algorithm>
#include <string>
#include <vector>
#include <cuda_runtime_api.h>
#include <cstring>
#include "../../../include/droid_b200.h"
#include "../../../include/droid_b200_training.h"

static inline void check_status(int rc, const char* op) {
  TORCH_CHECK(rc == DBA_OK, "droid_backends.", op, " failed (status ", rc, "): ", dba_last_error());
}
static inline dba_stream_t cur_stream() { return (dba_stream_t)at::cuda::getCurrentCUDAStream().stream(); }

// no host synchronisation is possible while the current stream is being captured into a CUDA graph
static bool stream_capturing() {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(at::cuda::getCurrentCUDAStream().stream(), &cap);
  return cap != cudaStreamCaptureStatusNone;
}

// A device workspace of `bytes` from the caching allocator, 256-byte aligned; `keep` owns the allocation until the call returns.
static void* workspace(size_t bytes, const torch::Device& dev, torch::Tensor& keep) {
  keep = torch::empty({(int64_t)bytes + 256}, torch::TensorOptions().dtype(torch::kUInt8).device(dev));
  return (void*)(((uintptr_t)keep.data_ptr() + 255) & ~(uintptr_t)255);
}

static int dtype_code(const torch::Tensor& t, const char* what) {
  switch (t.scalar_type()) {
    case torch::kFloat32: return DBA_F32;
    case torch::kFloat16: return DBA_F16;
    case torch::kFloat64: return DBA_F64;
    case torch::kBFloat16: return DBA_BF16;
    default: TORCH_CHECK(false, what, ": unsupported dtype ", t.scalar_type());
  }
  return -1;
}

// ---- argument checks --------------------------------------------------------------------------------------------------------------

constexpr torch::ScalarType F16 = torch::kFloat16, F32 = torch::kFloat32, I64 = torch::kInt64;
using Dtypes = c10::ArrayRef<torch::ScalarType>;   // the dtypes an argument may have; empty: any (dtype_code or a conversion decides)
constexpr int64_t kAny = -1;                        // an extent that may take any value

// The extents an argument must have.  kDims: this rank and these extents.  kRows: a flat array of rows of per_row elements (numel a
// multiple of per_row) with n rows.  first_at_least: dims[0] / n is a lower bound -- the kernels read a prefix of the leading dimension.
struct Shape {
  enum Kind { kAnyShape, kDims, kRows } kind = kAnyShape;
  c10::IntArrayRef dims;
  int64_t per_row = 0, n = kAny;
  bool first_at_least = false;
};
static Shape dims(c10::IntArrayRef d) { return {Shape::kDims, d}; }
static Shape dims_min(c10::IntArrayRef d) { return {Shape::kDims, d, 0, kAny, true}; }
static Shape rows(int64_t per_row, int64_t n = kAny) { return {Shape::kRows, {}, per_row, n}; }
static Shape rows_min(int64_t per_row, int64_t n) { return {Shape::kRows, {}, per_row, n, true}; }
static Shape at_least(int64_t n) { return rows_min(1, n); }

enum Layout { kContiguous, kAnyLayout };   // kAnyLayout: the binding makes its own contiguous copy

static std::string describe(const Shape& s) {
  std::string r;
  if (s.kind == Shape::kDims) {
    for (size_t d = 0; d < s.dims.size(); d++)
      r += (d ? "," : "") + std::string(d == 0 && s.first_at_least ? ">=" : "") + (s.dims[d] == kAny ? "*" : std::to_string(s.dims[d]));
    return "[" + r + "]";
  }
  r = s.n == kAny ? std::string("any number of") : (s.first_at_least ? "at least " : "") + std::to_string(s.n);
  return s.per_row == 1 ? r + " elements" : r + " rows of " + std::to_string(s.per_row) + " elements";
}

static std::string item(const char* list, size_t k) { return std::string(list) + "[" + std::to_string(k) + "]"; }

// The argument checks of one entry point, run before anything is launched.  The device is that of the entry point's first tensor
// argument; every tensor argument must be a CUDA tensor on it, have an accepted dtype, be contiguous where the kernel reads its raw
// layout, and have the extents the kernel reads.  Each error names the entry point and the argument, what was expected and what arrived.
struct Expect {
  const char* fn;
  torch::Device dev;
  Expect(const char* fn, const torch::Tensor& first, const char* first_name) : fn(fn), dev(first.device()) {
    cuda(first, first_name);
  }
  void cuda(const torch::Tensor& t, const char* name) const {
    TORCH_CHECK(t.is_cuda(), "droid_backends.", fn, ": ", name, " must be a CUDA tensor (droid_backends has no CPU path), got a ", t.device(),
                " tensor");
  }
  void operator()(const torch::Tensor& t, const char* name, Dtypes dtypes, const Shape& shape = {}, Layout layout = kContiguous) const {
    cuda(t, name);
    TORCH_CHECK(t.device() == dev, "droid_backends.", fn, ": ", name, " must be on ", dev, " (the device of the first tensor argument), got ",
                t.device());
    TORCH_CHECK(dtypes.empty() || std::find(dtypes.begin(), dtypes.end(), t.scalar_type()) != dtypes.end(), "droid_backends.", fn, ": ", name,
                " must be ", (dtypes.size() == 1 ? c10::toString(dtypes[0]) : "one of"), (dtypes.size() == 1 ? "" : c10::str(" ", dtypes)),
                ", got ", t.scalar_type());
    TORCH_CHECK(layout == kAnyLayout || t.is_contiguous(), "droid_backends.", fn, ": ", name, " must be contiguous, got strides ", t.strides());
    bool ok = true;
    if (shape.kind == Shape::kDims) {
      ok = t.dim() == (int64_t)shape.dims.size();
      for (int64_t d = 0; ok && d < t.dim(); d++) {
        const int64_t want = shape.dims[d], got = t.size(d);
        ok = want == kAny || got == want || (d == 0 && shape.first_at_least && got > want);
      }
    } else if (shape.kind == Shape::kRows) {
      const int64_t n = shape.per_row > 0 ? t.numel() / shape.per_row : 0;
      ok = t.dim() >= 1 && n * shape.per_row == t.numel() && (shape.n == kAny || n == shape.n || (shape.first_at_least && n > shape.n));
    }
    TORCH_CHECK(ok, "droid_backends.", fn, ": ", name, " must be ", describe(shape), ", got shape ", t.sizes());
  }
  // an optional argument: checked as above when given; returns it, or an undefined tensor for None
  torch::Tensor opt(const c10::optional<torch::Tensor>& t, const char* name, Dtypes dtypes, const Shape& shape = {},
                    Layout layout = kContiguous) const {
    if (!t.has_value() || !t->defined()) return {};
    (*this)(*t, name, dtypes, shape, layout);
    return *t;
  }
};

// ---- the reference's nine callables -----------------------------------------------------------------------------------------------

// sticky device status word of a ba call (include/droid_b200.h: dba_ba_read_info)
static void check_ba_status(int st, bool after_solve) {
  TORCH_CHECK(!(st & 1), "droid_backends.ba: ii/jj hold frame indices outside [0, n_frames) (the reference reads out of bounds here)");
  TORCH_CHECK(!(st & 8), "droid_backends.ba: a source frame has more than 254 out-edges; the Schur complement kernels hold at most 255 rows per depth frame");
  TORCH_CHECK(!(st & 2), "droid_backends.ba: eta row count does not match the number of depth frames");
  if (after_solve && (st & 4))
    TORCH_WARN("droid_backends.ba: the damped pose system was not positive definite in at least one Gauss-Newton iteration; that iteration's "
               "update is zero (the reference does the same silently, src/droid_kernels.cu:1216-1219)");
}

std::vector<torch::Tensor> ba(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor disps_sens,
                              torch::Tensor targets, torch::Tensor weights, torch::Tensor eta, torch::Tensor ii, torch::Tensor jj,
                              const int t0, const int t1, const int iterations, const float lm, const float ep,
                              const bool motion_only) {
  const Expect expect("ba", poses, "poses");
  expect(poses, "poses", F32, dims({kAny, 7}));
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  const int N = (int)disps.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  const int HW = ht * wd;
  expect(intrinsics, "intrinsics", F32, at_least(4));
  expect(disps_sens, "disps_sens", F32, dims({N, ht, wd}));
  expect(ii, "ii", I64);
  const int E = (int)ii.size(0);
  expect(jj, "jj", I64, rows(1, E));
  expect(targets, "targets", F32, rows(2 * HW, E));
  expect(weights, "weights", F32, rows(2 * HW, E));
  TORCH_CHECK(poses.size(0) >= N || poses.size(0) >= t1, "poses has fewer rows than the optimisation window");
  TORCH_CHECK(t0 >= 0 && t1 >= t0 && t1 <= N, "invalid window [t0,t1)");
  if (iterations <= 0) return {torch::Tensor(), torch::Tensor()};   // reference returns two undefined tensors
  if (!motion_only) expect(eta, "eta", F32, rows_min(HW, 1), kAnyLayout);   // [M,ht,wd]; the reference only needs it .view()-able (SURVEY Q12)
  c10::cuda::CUDAGuard guard(expect.dev);

  const torch::Tensor eta_c = motion_only ? eta : eta.contiguous();
  const int eta_rows = motion_only ? 1 : (int)(eta_c.numel() / HW);
  const int n_frames = std::min<int>(N, (int)poses.size(0));
  const size_t ws_bytes = dba_ba_workspace_bytes(n_frames, E, ht, wd, t0, t1);
  torch::Tensor ws;
  const int P = t1 - t0;
  auto dx = torch::empty({P, 6}, poses.options());

  dba_ba_args a;
  memset(&a, 0, sizeof(a));
  a.poses = poses.data_ptr<float>(); a.disps = disps.data_ptr<float>(); a.intrinsics = intrinsics.data_ptr<float>();
  a.disps_sens = disps_sens.data_ptr<float>(); a.targets = targets.data_ptr<float>(); a.weights = weights.data_ptr<float>();
  a.eta = motion_only ? nullptr : eta_c.data_ptr<float>(); a.eta_rows = eta_rows;
  a.ii = ii.data_ptr<int64_t>(); a.jj = jj.data_ptr<int64_t>();
  a.n_frames = n_frames; a.n_edges = E; a.ht = ht; a.wd = wd; a.t0 = t0; a.t1 = t1;
  a.lm = lm; a.ep = ep; a.motion_only = motion_only ? 1 : 0;
  a.dx_out = dx.data_ptr<float>(); a.dz_out = nullptr;
  a.workspace = workspace(ws_bytes, expect.dev, ws); a.workspace_bytes = ws_bytes; a.stream = cur_stream();
  a.own_lo = 0; a.own_hi = n_frames; a.eta_by_frame = 0;

  // The graph bookkeeping runs first and its result is read back (one stream synchronisation; the reference's ba synchronises a
  // dozen times per call): the number of depth frames M sizes dz, eta must have 1 or M rows (the reference raises a broadcast
  // error otherwise, src/droid_kernels.cu:1407), and out-of-range indices are reported instead of being dropped.  While the stream
  // is being captured into a CUDA graph no synchronisation is possible: dz is sized from eta and the checks are skipped (the
  // caller validated the same tensors eagerly).
  const bool capturing = stream_capturing();
  torch::Tensor dz;
  int M = eta_rows;
  if (!capturing) {
    check_status(dba_ba_prepare(&a), "ba");
    int st = 0;
    check_status(dba_ba_read_info(&a, &M, &st), "ba");
    check_ba_status(st, /*after_solve=*/false);
    TORCH_CHECK(motion_only || eta_rows == 1 || eta_rows == M, "ba: eta has ", eta_rows, " rows but the graph has ", M,
                " depth frames (unique(ii U [t0,t1)))");
  } else {
    TORCH_CHECK(motion_only || eta_rows > 1, "ba: a broadcast (1-row) eta needs the depth-frame count from the device and cannot be used during CUDA graph capture");
  }
  if (!motion_only) {
    dz = torch::empty({M, HW}, poses.options());
    a.dz_out = dz.data_ptr<float>();
  }
  check_status(dba_ba(&a, iterations), "ba");
  if (!capturing) {
    int st = 0, m2 = 0;
    check_status(dba_ba_read_info(&a, &m2, &st), "ba");
    check_ba_status(st, /*after_solve=*/true);
  }
  return {dx, dz};
}

torch::Tensor frame_distance(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj,
                             const float beta) {
  const Expect expect("frame_distance", poses, "poses");
  expect(poses, "poses", F32, dims({kAny, 7}));
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  expect(intrinsics, "intrinsics", F32, at_least(4));
  expect(ii, "ii", I64);
  const int num = (int)ii.size(0);
  expect(jj, "jj", I64, rows_min(1, num));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto dist = torch::empty({num}, poses.options());
  check_status(dba_frame_distance(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                                  jj.data_ptr<int64_t>(), dist.data_ptr<float>(), num, (int)disps.size(1), (int)disps.size(2), beta,
                                  cur_stream()), "frame_distance");
  return dist;
}

std::vector<torch::Tensor> projmap(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj) {
  const Expect expect("projmap", poses, "poses");
  expect(poses, "poses", F32, dims({kAny, 7}));
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  expect(intrinsics, "intrinsics", F32, at_least(4));
  expect(ii, "ii", I64);
  const int num = (int)ii.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  expect(jj, "jj", I64, rows_min(1, num));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto coords = torch::empty({num, ht, wd, 3}, poses.options());
  auto valid = torch::empty({num, ht, wd, 1}, poses.options());
  check_status(dba_projmap(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                           jj.data_ptr<int64_t>(), coords.data_ptr<float>(), valid.data_ptr<float>(), num, ht, wd, cur_stream()), "projmap");
  return {coords, valid};
}

torch::Tensor iproj(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics) {
  const Expect expect("iproj", poses, "poses");
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  const int nm = (int)disps.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  expect(poses, "poses", F32, dims_min({nm, 7}));   // one pose per disparity map
  expect(intrinsics, "intrinsics", F32, at_least(4));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto points = torch::empty({nm, ht, wd, 3}, disps.options());
  check_status(dba_iproj(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), points.data_ptr<float>(), nm, ht,
                         wd, cur_stream()), "iproj");
  return points;
}

torch::Tensor depth_filter(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ix, torch::Tensor thresh) {
  const Expect expect("depth_filter", poses, "poses");
  expect(poses, "poses", F32, dims({kAny, 7}));
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  expect(intrinsics, "intrinsics", F32, at_least(4));
  expect(ix, "ix", I64);
  const int num = (int)ix.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  expect(thresh, "thresh", F32, at_least(num));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto counter = torch::empty({num, ht, wd}, disps.options());
  check_status(dba_depth_filter(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ix.data_ptr<int64_t>(),
                                thresh.data_ptr<float>(), counter.data_ptr<float>(), num, (int)disps.size(0), ht, wd, cur_stream()),
               "depth_filter");
  return counter;
}

std::vector<torch::Tensor> corr_index_forward(torch::Tensor volume, torch::Tensor coords, int radius) {
  const Expect expect("corr_index_forward", volume, "volume");
  expect(volume, "volume", {}, dims({kAny, kAny, kAny, kAny, kAny}));
  const int n = (int)volume.size(0), h1 = (int)volume.size(1), w1 = (int)volume.size(2), h2 = (int)volume.size(3), w2 = (int)volume.size(4);
  expect(coords, "coords", F32, dims({n, 2, h1, w1}));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto corr = torch::empty({n, 2 * radius + 1, 2 * radius + 1, h1, w1}, volume.options());
  check_status(dba_corr_index_forward(volume.data_ptr(), coords.data_ptr<float>(), corr.data_ptr(), n, h1, w1, h2, w2, radius,
                                      dtype_code(volume, "corr_index_forward"), cur_stream()), "corr_index_forward");
  return {corr};
}

std::vector<torch::Tensor> corr_index_backward(torch::Tensor volume, torch::Tensor coords, torch::Tensor corr_grad, int radius) {
  const Expect expect("corr_index_backward", volume, "volume");
  expect(volume, "volume", {}, dims({kAny, kAny, kAny, kAny, kAny}));
  const int n = (int)volume.size(0), h1 = (int)volume.size(1), w1 = (int)volume.size(2), h2 = (int)volume.size(3), w2 = (int)volume.size(4);
  const int D = 2 * radius + 1;
  expect(coords, "coords", F32, dims_min({n, 2, h1, w1}));
  expect(corr_grad, "corr_grad", volume.scalar_type(), dims_min({n, D, D, h1, w1}));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto volume_grad = torch::empty_like(volume);
  check_status(dba_corr_index_backward(coords.data_ptr<float>(), corr_grad.data_ptr(), volume_grad.data_ptr(), n, h1, w1, h2, w2, radius,
                                       dtype_code(volume, "corr_index_backward"), cur_stream()), "corr_index_backward");
  return {volume_grad};
}

std::vector<torch::Tensor> altcorr_forward(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor coords, torch::Tensor ii,
                                           torch::Tensor jj, int radius) {
  const Expect expect("altcorr_forward", fmap1, "fmap1");
  expect(coords, "coords", F32, dims({kAny, kAny, 2, kAny, kAny}));
  const int B = (int)coords.size(0), M = (int)coords.size(1), H = (int)coords.size(3), W = (int)coords.size(4);
  expect(fmap1, "fmap1", {}, dims_min({B, kAny, kAny, H, W}));
  const int C = (int)fmap1.size(2);
  expect(fmap2, "fmap2", fmap1.scalar_type(), dims_min({B, kAny, C, kAny, kAny}));
  expect(ii, "ii", I64, rows(1, M), kAnyLayout);
  expect(jj, "jj", I64, rows(1, M), kAnyLayout);
  c10::cuda::CUDAGuard guard(expect.dev);
  auto iic = ii.contiguous(), jjc = jj.contiguous();
  const int D = 2 * radius + 1;
  auto out = torch::empty({B, M, D, D, H, W}, fmap1.options());
  check_status(dba_altcorr_forward(fmap1.data_ptr(), fmap2.data_ptr(), coords.data_ptr<float>(), iic.data_ptr<int64_t>(),
                                   jjc.data_ptr<int64_t>(), out.data_ptr(), B, (int)fmap1.size(1), (int)fmap2.size(1), C, H, W,
                                   (int)fmap2.size(3), (int)fmap2.size(4), M, radius, dtype_code(fmap1, "altcorr_forward"), cur_stream()),
               "altcorr_forward");
  return {out.permute({0, 1, 3, 2, 4, 5})};   // reference src/altcorr_kernel.cu:171
}

std::vector<torch::Tensor> altcorr_backward(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor coords, torch::Tensor corr_grad,
                                            torch::Tensor ii, torch::Tensor jj, int radius) {
  // corr_grad is the gradient of the tensor altcorr_forward returned ([B,M,x-off,y-off,H,W]); the reference
  // (src/droid.cpp:212-226 -> src/altcorr_kernel.cu:175-225) un-permutes it and spreads it over the raw window.
  const Expect expect("altcorr_backward", fmap1, "fmap1");
  expect(coords, "coords", F32, dims({kAny, kAny, 2, kAny, kAny}));
  const int B = (int)coords.size(0), M = (int)coords.size(1), H = (int)coords.size(3), W = (int)coords.size(4);
  const int D = 2 * radius + 1;
  expect(fmap1, "fmap1", {}, dims_min({B, kAny, kAny, H, W}));
  const int C = (int)fmap1.size(2);
  expect(fmap2, "fmap2", fmap1.scalar_type(), dims_min({B, kAny, C, kAny, kAny}));
  expect(corr_grad, "corr_grad", {}, rows(1, (int64_t)B * M * D * D * H * W));   // [B,M,2r+1,2r+1,H,W], any dtype (read as f32)
  expect(ii, "ii", I64, rows_min(1, M), kAnyLayout);
  expect(jj, "jj", I64, rows_min(1, M), kAnyLayout);
  c10::cuda::CUDAGuard guard(expect.dev);
  auto iic = ii.contiguous(), jjc = jj.contiguous();
  auto cg = corr_grad.to(torch::kFloat32).contiguous();   // kernel reads a float accessor (src/altcorr_kernel.cu:84)
  auto g1 = torch::empty_like(fmap1), g2 = torch::empty_like(fmap2);
  check_status(dba_altcorr_backward(fmap1.data_ptr(), fmap2.data_ptr(), coords.data_ptr<float>(), cg.data_ptr<float>(), iic.data_ptr<int64_t>(),
                                    jjc.data_ptr<int64_t>(), g1.data_ptr(), g2.data_ptr(), B, (int)fmap1.size(1), (int)fmap2.size(1), C, H, W,
                                    (int)fmap2.size(3), (int)fmap2.size(4), M, radius, dtype_code(fmap1, "altcorr_backward"), cur_stream()),
               "altcorr_backward");
  return {g1, g2};
}

// ---- extensions -------------------------------------------------------------------------------------------------------------------

// CorrBlock.__init__ in one tensor-core kernel (reference droid_slam/modules/corr.py:24-38,63-71).  fmap1/fmap2 [N,128,ht,wd] f16
// (ht, wd >= 8), ii/jj [E] -> 4 pyramid levels.  tiled (levels 0-1 in the private tiled layout) only where
// dba_corr_volume_supported(..., tiled = 1); wd % 8 != 0 takes a staging workspace from the caching allocator.
std::vector<torch::Tensor> corr_volume_pyramid(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor ii, torch::Tensor jj, bool tiled) {
  const Expect expect("corr_volume_pyramid", fmap1, "fmap1");
  expect(fmap1, "fmap1", F16, dims({kAny, kAny, kAny, kAny}));
  const int C = (int)fmap1.size(1), ht = (int)fmap1.size(2), wd = (int)fmap1.size(3);
  expect(fmap2, "fmap2", F16, dims({kAny, C, ht, wd}));
  expect(ii, "ii", I64);
  const int E = (int)ii.size(0);
  expect(jj, "jj", I64, rows(1, E));
  c10::cuda::CUDAGuard guard(expect.dev);
  std::vector<torch::Tensor> out;
  for (int l = 0; l < 4; l++) out.push_back(torch::empty({E, ht, wd, ht >> l, wd >> l}, fmap1.options()));
  const int n1 = (int)fmap1.size(0), n2 = (int)fmap2.size(0);
  const size_t ws_bytes = dba_corr_volume_workspace_bytes(n1, n2, C, ht, wd);
  torch::Tensor ws;
  void* ws_p = (ws_bytes > 0 && E > 0) ? workspace(ws_bytes, expect.dev, ws) : nullptr;
  check_status(dba_corr_volume_pyramid(fmap1.data_ptr(), fmap2.data_ptr(), ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), out[0].data_ptr(),
                                       out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), E, n1, n2, C, ht, wd, DBA_F16, tiled ? 1 : 0,
                                       ws_p, ws_p ? ws_bytes : 0, cur_stream()),
               "corr_volume_pyramid");
  return out;
}

// CorrBlock.__call__ (reference modules/corr.py:40-50) in one launch.  pyramid = 4 f16 tensors [E,h1,w1,h1/2^l,w1/2^l] (reference
// layout, or levels 0-1 tiled when `tiled`) or 4 f32 tensors in the reference layout, coords [E,2,h1,w1] f32 at level-0 scale -> [E,196,h1,w1] = cat over levels of corr_index_forward
torch::Tensor corr_lookup_pyramid(std::vector<torch::Tensor> pyramid, torch::Tensor coords, bool tiled) {
  TORCH_CHECK(pyramid.size() == 4, "droid_backends.corr_lookup_pyramid: 4 pyramid levels expected, got ", pyramid.size());
  const Expect expect("corr_lookup_pyramid", pyramid[0], "pyramid[0]");
  expect(pyramid[0], "pyramid[0]", {F16, F32}, dims({kAny, kAny, kAny, kAny, kAny}));
  const torch::ScalarType vt = pyramid[0].scalar_type();
  const int n = (int)pyramid[0].size(0), h1 = (int)pyramid[0].size(1), w1 = (int)pyramid[0].size(2);
  for (int l = 0; l < 4; l++) expect(pyramid[l], item("pyramid", l).c_str(), vt, dims({n, h1, w1, h1 >> l, w1 >> l}));
  expect(coords, "coords", F32, dims({n, 2, h1, w1}));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto out = torch::empty({n, 196, h1, w1}, pyramid[0].options());
  check_status(dba_corr_lookup_pyramid(pyramid[0].data_ptr(), pyramid[1].data_ptr(), pyramid[2].data_ptr(), pyramid[3].data_ptr(), coords.data_ptr<float>(), out.data_ptr(),
                                       n, h1, w1, tiled ? 3 : 0, dtype_code(pyramid[0], "corr_lookup_pyramid"), cur_stream()), "corr_lookup_pyramid");
  return out;
}

// The training CorrBlock (include/droid_b200.h): fmap1, fmap2 [E,128,ht,wd] f32 -> 4 f32 pyramid levels [E,ht,wd,ht>>l,wd>>l]
std::vector<torch::Tensor> corr_volume_pyramid_f32(torch::Tensor fmap1, torch::Tensor fmap2) {
  const Expect expect("corr_volume_pyramid_f32", fmap1, "fmap1");
  expect(fmap1, "fmap1", F32, dims({kAny, kAny, kAny, kAny}));
  const int E = (int)fmap1.size(0), C = (int)fmap1.size(1), ht = (int)fmap1.size(2), wd = (int)fmap1.size(3);
  expect(fmap2, "fmap2", F32, dims({E, C, ht, wd}));
  c10::cuda::CUDAGuard guard(expect.dev);
  std::vector<torch::Tensor> out;
  for (int l = 0; l < 4; l++) out.push_back(torch::empty({E, ht, wd, ht >> l, wd >> l}, fmap1.options()));
  check_status(dba_corr_volume_pyramid_f32(fmap1.data_ptr<float>(), fmap2.data_ptr<float>(), out[0].data_ptr<float>(), out[1].data_ptr<float>(),
                                           out[2].data_ptr<float>(), out[3].data_ptr<float>(), E, C, ht, wd, cur_stream()),
               "corr_volume_pyramid_f32");
  return out;
}

static int64_t grad_pyramid_row(int64_t ht, int64_t wd) {
  int64_t q = 0;
  for (int l = 0; l < 4; l++) q += (ht >> l) * (wd >> l);
  return q;
}

// gpyr [E,ht*wd,Q] f32 += the gradient of one corr_lookup_pyramid call: grad [E,196,ht,wd] f32 at coords [E,2,ht,wd]
void corr_grad_accumulate(torch::Tensor coords, torch::Tensor grad, torch::Tensor gpyr) {
  const Expect expect("corr_grad_accumulate", coords, "coords");
  expect(coords, "coords", F32, dims({kAny, 2, kAny, kAny}));
  const int E = (int)coords.size(0), ht = (int)coords.size(2), wd = (int)coords.size(3);
  expect(grad, "grad", F32, dims({E, 196, ht, wd}));
  expect(gpyr, "gpyr", F32, dims({E, (int64_t)ht * wd, grad_pyramid_row(ht, wd)}));
  c10::cuda::CUDAGuard guard(expect.dev);
  check_status(dba_corr_grad_accumulate(coords.data_ptr<float>(), grad.data_ptr<float>(), gpyr.data_ptr<float>(), E, ht, wd, cur_stream()),
               "corr_grad_accumulate");
}

// (grad_fmap1, grad_fmap2) [E,128,ht,wd] of the training CorrBlock from its accumulated gradient pyramid gpyr [E,ht*wd,Q]
std::vector<torch::Tensor> corr_adjoint(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor gpyr) {
  const Expect expect("corr_adjoint", fmap1, "fmap1");
  expect(fmap1, "fmap1", F32, dims({kAny, kAny, kAny, kAny}));
  const int E = (int)fmap1.size(0), C = (int)fmap1.size(1), ht = (int)fmap1.size(2), wd = (int)fmap1.size(3);
  expect(fmap2, "fmap2", F32, dims({E, C, ht, wd}));
  expect(gpyr, "gpyr", F32, dims({E, (int64_t)ht * wd, grad_pyramid_row(ht, wd)}));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto g1 = torch::empty_like(fmap1), g2 = torch::empty_like(fmap2);
  const size_t ws_bytes = dba_corr_adjoint_workspace_bytes(E, C, ht, wd);
  torch::Tensor ws;
  void* ws_p = ws_bytes > 0 ? workspace(ws_bytes, expect.dev, ws) : nullptr;
  check_status(dba_corr_adjoint(fmap1.data_ptr<float>(), fmap2.data_ptr<float>(), gpyr.data_ptr<float>(), g1.data_ptr<float>(), g2.data_ptr<float>(),
                                E, C, ht, wd, ws_p, ws_bytes, cur_stream()),
               "corr_adjoint");
  return {g1, g2};
}

// AltCorrBlock.__init__ (reference modules/corr.py:90-101) as one launch.  fmaps [B,N,C,H,W] f16/f32 -> num_levels tensors
// [B,N,H>>l,W>>l,C] in the private channels-last, pre-quartered layout of include/droid_b200.h (dba_altcorr_pyramid).
std::vector<torch::Tensor> altcorr_pyramid(torch::Tensor fmaps, int num_levels) {
  const Expect expect("altcorr_pyramid", fmaps, "fmaps");
  expect(fmaps, "fmaps", {F16, F32}, dims({kAny, kAny, kAny, kAny, kAny}));
  TORCH_CHECK(num_levels >= 1 && num_levels <= 4, "altcorr_pyramid: 1..4 levels expected");
  c10::cuda::CUDAGuard guard(expect.dev);
  const int B = (int)fmaps.size(0), N = (int)fmaps.size(1), C = (int)fmaps.size(2), H = (int)fmaps.size(3), W = (int)fmaps.size(4);
  std::vector<torch::Tensor> out;
  void* p[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int l = 0; l < num_levels; l++) {
    out.push_back(torch::empty({B, N, H >> l, W >> l, C}, fmaps.options()));
    p[l] = out.back().data_ptr();
  }
  check_status(dba_altcorr_pyramid(fmaps.data_ptr(), p[0], p[1], p[2], p[3], B, N, C, H, W, num_levels, dtype_code(fmaps, "altcorr_pyramid"), cur_stream()),
               "altcorr_pyramid");
  return out;
}

// AltCorrBlock.__call__ (reference modules/corr.py:104-117) in one launch.  pyramid from altcorr_pyramid, coords [B,M,2,H,W] f32
// at level-0 scale, ii/jj [M] -> [B,M,L*49,H,W] = stack over levels of altcorr_forward(level 0, level l, coords / 2^l, ii, jj, radius)
torch::Tensor altcorr_lookup_pyramid(std::vector<torch::Tensor> pyramid, torch::Tensor coords, torch::Tensor ii, torch::Tensor jj, int radius) {
  const int L = (int)pyramid.size();
  TORCH_CHECK(L >= 1 && L <= 4, "droid_backends.altcorr_lookup_pyramid: 1..4 pyramid levels expected, got ", L);
  const Expect expect("altcorr_lookup_pyramid", pyramid[0], "pyramid[0]");
  const auto& p0 = pyramid[0];
  expect(p0, "pyramid[0]", {}, dims({kAny, kAny, kAny, kAny, kAny}));
  const int B = (int)p0.size(0), N = (int)p0.size(1), H = (int)p0.size(2), W = (int)p0.size(3), C = (int)p0.size(4);
  for (int l = 1; l < L; l++) expect(pyramid[l], item("pyramid", l).c_str(), p0.scalar_type(), dims({B, N, H >> l, W >> l, C}));
  expect(coords, "coords", F32, dims({B, kAny, 2, H, W}));
  const int M = (int)coords.size(1);
  expect(ii, "ii", I64, dims({M}), kAnyLayout);
  expect(jj, "jj", I64, dims({M}), kAnyLayout);
  c10::cuda::CUDAGuard guard(expect.dev);
  auto iic = ii.contiguous(), jjc = jj.contiguous();
  auto out = torch::empty({B, M, L * (2 * radius + 1) * (2 * radius + 1), H, W}, p0.options());
  const void* p[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int l = 0; l < L; l++) p[l] = pyramid[l].data_ptr();
  check_status(dba_altcorr_lookup_pyramid(p[0], p[1], p[2], p[3], coords.data_ptr<float>(), iic.data_ptr<int64_t>(), jjc.data_ptr<int64_t>(),
                                          out.data_ptr(), B, N, C, H, W, M, L, radius, dtype_code(p0, "altcorr_lookup_pyramid"), cur_stream()),
               "altcorr_lookup_pyramid");
  return out;
}

// fused DepthVideo.reproject (reference depth_video.py:171-179 -> geom/projective_ops.py:165-198, jacobian=False)
std::vector<torch::Tensor> reproject(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj) {
  const Expect expect("reproject", poses, "poses");
  expect(poses, "poses", F32);
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  expect(intrinsics, "intrinsics", F32, dims({kAny, 4}));
  expect(ii, "ii", I64);
  const int num = (int)ii.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  expect(jj, "jj", I64, rows_min(1, num));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto coords = torch::empty({num, ht, wd, 2}, poses.options());
  auto valid = torch::empty({num, ht, wd, 1}, poses.options());
  check_status(dba_reproject(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                             jj.data_ptr<int64_t>(), coords.data_ptr<float>(), valid.data_ptr<float>(), num, ht, wd, cur_stream()), "reproject");
  return {coords, valid};
}

// FactorGraph.update / update_lowmem motion features (reference factor_graph.py:220-222, :280-282) fused with the reprojection.
// poses [N,7], disps [N,ht,wd], intrinsics [N,4], ii / jj [E] int64, target [(1,)E,ht,wd,2] f32; call row r reads edge edge_index[r]
// (all E edges in order when edge_index is None).  Returns [coords [n,ht,wd,2], coords_t [n,2,ht,wd], motn [n,4,ht,wd]].
std::vector<torch::Tensor> motion_features(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj,
                                           torch::Tensor target, c10::optional<torch::Tensor> edge_index) {
  const Expect expect("motion_features", poses, "poses");
  expect(poses, "poses", F32);
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  expect(intrinsics, "intrinsics", F32, dims({kAny, 4}));
  expect(ii, "ii", I64);
  const int E = (int)ii.numel(), ht = (int)disps.size(1), wd = (int)disps.size(2);
  expect(jj, "jj", I64, rows(1, E));
  expect(target, "target", F32, rows((int64_t)ht * wd * 2, E));
  const torch::Tensor ei = expect.opt(edge_index, "edge_index", I64);
  const int n = ei.defined() ? (int)ei.numel() : E;
  c10::cuda::CUDAGuard guard(expect.dev);
  auto coords = torch::empty({n, ht, wd, 2}, poses.options());
  auto coords_t = torch::empty({n, 2, ht, wd}, poses.options());
  auto motn = torch::empty({n, 4, ht, wd}, poses.options());
  check_status(dba_motion_features(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                                   jj.data_ptr<int64_t>(), ei.defined() ? ei.data_ptr<int64_t>() : nullptr, target.data_ptr<float>(),
                                   coords.data_ptr<float>(), coords_t.data_ptr<float>(), motn.data_ptr<float>(), n, ht, wd, cur_stream()),
               "motion_features");
  return {coords, coords_t, motn};
}

// write-back of one update-operator call into the factor graph and BA's inputs (reference factor_graph.py:234-251, :304-320).
// delta / weight / coords [n,ht,wd,2] f32 (call rows), edge_index [n] int64 or None (row r = edge r); target / weight_out [(1,)E,ht,wd,2] and
// ba_target / ba_weight [E_ba,2,ht,wd] written in place (row n_inactive + e); eta [n_src,ht,wd] scattered to damping[src_frames];
// then, when ba_frames is given, ba_damping[r] = .2 * damping[ba_frames[r]] + ep.
void graph_writeback(torch::Tensor delta, torch::Tensor weight, torch::Tensor coords, c10::optional<torch::Tensor> edge_index,
                     torch::Tensor target, torch::Tensor weight_out, torch::Tensor ba_target, torch::Tensor ba_weight, int64_t n_inactive,
                     c10::optional<torch::Tensor> eta, c10::optional<torch::Tensor> src_frames, torch::Tensor damping,
                     c10::optional<torch::Tensor> ba_frames, c10::optional<torch::Tensor> ba_damping, double ep) {
  const Expect expect("graph_writeback", delta, "delta");
  expect(damping, "damping", F32, dims({kAny, kAny, kAny}));   // [n_frames,ht,wd]
  const int ht = (int)damping.size(1), wd = (int)damping.size(2);
  const int64_t hw = (int64_t)ht * wd, px2 = hw * 2;
  expect(delta, "delta", F32, rows(px2));
  const int n = (int)(delta.numel() / px2);
  expect(weight, "weight", F32, rows(px2, n));
  expect(coords, "coords", F32, rows(px2, n));
  expect(target, "target", F32, rows(px2));
  const int64_t E = target.numel() / px2;
  expect(weight_out, "weight_out", F32, rows(px2, E));
  expect(ba_target, "ba_target", F32, rows(px2));
  const int64_t E_ba = ba_target.numel() / px2;
  expect(ba_weight, "ba_weight", F32, rows(px2, E_ba));
  TORCH_CHECK(n_inactive >= 0 && n_inactive + E <= E_ba, "ba_target must hold n_inactive + E rows");
  const torch::Tensor ei = expect.opt(edge_index, "edge_index", I64, rows(1, n));
  TORCH_CHECK(ei.defined() || n <= E, "more call rows than graph edges");
  int n_src = 0;
  torch::Tensor eta_t, src_t;
  if ((eta_t = expect.opt(eta, "eta", F32, rows(hw))).defined()) {
    n_src = (int)(eta_t.numel() / hw);
    src_t = expect.opt(src_frames, "src_frames", I64, rows(1, n_src));
    TORCH_CHECK(src_t.defined(), "src_frames is required with eta");
  }
  const torch::Tensor baf = expect.opt(ba_frames, "ba_frames", I64);
  const int n_ba = baf.defined() ? (int)baf.numel() : 0;
  torch::Tensor bad;
  if (baf.defined()) {
    bad = expect.opt(ba_damping, "ba_damping", F32, rows(hw, n_ba));   // [len(ba_frames),ht,wd]
    TORCH_CHECK(bad.defined(), "ba_damping is required with ba_frames");
  }
  c10::cuda::CUDAGuard guard(expect.dev);
  check_status(dba_graph_writeback(delta.data_ptr<float>(), weight.data_ptr<float>(), coords.data_ptr<float>(),
                                   ei.defined() ? ei.data_ptr<int64_t>() : nullptr, n, target.data_ptr<float>(), weight_out.data_ptr<float>(),
                                   ba_target.data_ptr<float>(), ba_weight.data_ptr<float>(), (int)n_inactive,
                                   eta_t.defined() ? eta_t.data_ptr<float>() : nullptr, src_t.defined() ? src_t.data_ptr<int64_t>() : nullptr,
                                   n_src, damping.data_ptr<float>(), baf.defined() ? baf.data_ptr<int64_t>() : nullptr, n_ba,
                                   bad.defined() ? bad.data_ptr<float>() : nullptr, (float)ep, ht, wd, cur_stream()), "graph_writeback");
}

// the pose interpolation of PoseTrajectoryFiller.__fill (reference trajectory_filler.py:51-65).  poses [N,7] and tstamps [N] of
// the keyframes, t [F] f32 -> [t0 [F] int64, t1 [F] int64, poses [F,7]].
std::vector<torch::Tensor> fill_interpolate(torch::Tensor poses, torch::Tensor tstamps, torch::Tensor t) {
  const Expect expect("fill_interpolate", poses, "poses");
  expect(poses, "poses", F32, dims({kAny, 7}));
  TORCH_CHECK(poses.size(0) >= 1, "fill_interpolate: no keyframe to interpolate from (the reference indexes an empty tensor here)");
  expect(tstamps, "tstamps", F32, dims({poses.size(0)}));
  expect(t, "t", F32, dims({kAny}));
  c10::cuda::CUDAGuard guard(expect.dev);
  const int F = (int)t.size(0);
  auto t0 = torch::empty({F}, poses.options().dtype(torch::kInt64));
  auto t1 = torch::empty({F}, poses.options().dtype(torch::kInt64));
  auto out = torch::empty({F, 7}, poses.options());
  check_status(dba_fill_interpolate(poses.data_ptr<float>(), tstamps.data_ptr<float>(), (int)poses.size(0), t.data_ptr<float>(), F,
                                    t0.data_ptr<int64_t>(), t1.data_ptr<int64_t>(), out.data_ptr<float>(), cur_stream()), "fill_interpolate");
  return {t0, t1, out};
}

// motion-only BA of the trajectory filler's graph (every edge from a fixed frame ii < t0 to one frame t0 <= jj < t1), all
// iterations in one launch.  Arguments as ba (intrinsics: the single camera; disps: only the rows of the fixed frames are read).  Returns
// [status (int32 [1] on the device)], with diagnostics also dx [t1-t0,6] and the undamped blocks sys [t1-t0,42] f64 (H row-major, then b)
// of the last iteration.  check: read the status back (one stream synchronisation) and raise when an edge breaks the structure (no pose has then
// changed) / warn when a block was not positive definite; skipped while the stream is being captured.
std::vector<torch::Tensor> pose_only_ba(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor targets,
                                        torch::Tensor weights, torch::Tensor ii, torch::Tensor jj, const int t0, const int t1, const int iterations,
                                        const float lm, const float ep, const bool check, const bool diagnostics) {
  const Expect expect("pose_only_ba", poses, "poses");
  expect(poses, "poses", F32, dims({kAny, 7}));
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  expect(intrinsics, "intrinsics", F32, at_least(4));
  expect(ii, "ii", I64);
  const int N = (int)poses.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  const int E = (int)ii.numel();
  expect(jj, "jj", I64, rows(1, E));
  expect(targets, "targets", F32, rows((int64_t)2 * ht * wd, E));
  expect(weights, "weights", F32, rows((int64_t)2 * ht * wd, E));
  TORCH_CHECK(t0 >= 0 && t1 >= t0 && t1 <= N, "invalid window [t0,t1)");
  TORCH_CHECK(iterations >= 0, "iterations must be >= 0");
  c10::cuda::CUDAGuard guard(expect.dev);
  auto status = torch::empty({1}, poses.options().dtype(torch::kInt32));
  torch::Tensor dx, sys;
  if (diagnostics) {
    dx = torch::zeros({t1 - t0, 6}, poses.options());
    sys = torch::zeros({t1 - t0, 42}, poses.options().dtype(torch::kFloat64));
  }
  check_status(dba_pose_only_ba(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), targets.data_ptr<float>(),
                                weights.data_ptr<float>(), ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), N, (int)disps.size(0), E, ht, wd, t0, t1,
                                iterations, lm, ep, status.data_ptr<int>(), diagnostics ? sys.data_ptr<double>() : nullptr,
                                diagnostics ? dx.data_ptr<float>() : nullptr, cur_stream()),
               "pose_only_ba");
  if (check && !stream_capturing()) {
    const int st = status.cpu().data_ptr<int>()[0];
    TORCH_CHECK(!(st & 1), "droid_backends.pose_only_ba: an edge is not (0 <= ii < min(t0, len(disps)), t0 <= jj < t1); no pose was changed");
    if (st & 2)
      TORCH_WARN("droid_backends.pose_only_ba: a damped pose block was not positive definite in at least one iteration; that frame's update "
                 "is zero in that iteration (the reference zeroes the whole window's update)");
  }
  if (!diagnostics) return {status};
  return {status, dx, sys};
}

// extents of the 27 packed update-operator weights in dba_update_weights order (include/droid_b200.h), as
// droid_slam_b200.update.pack_update_weights makes them: w_* f16 [taps][N][Kpad], then b_* f32 [N], then w_glo, b_glo, b_zero f32
static const std::vector<int64_t> kUpdateWeightShapes[27] = {
    {1, 128, 256}, {9, 128, 128}, {1, 128, 256}, {9, 64, 128}, {1, 128, 128}, {9, 256, 448}, {9, 128, 448}, {9, 384, 128}, {1, 64, 256},
    {9, 128, 128}, {1, 32, 128},  {1, 576, 128}, {128},        {128},         {128},         {64},          {128},         {256},
    {128},         {384},         {4},           {128},        {1},           {576},         {384, 128},    {384},         {64}};

// the update operator (reference droid_slam/droid_net.py:111-143, modules/gru.py:19-32, droid_net.py:59-75) on the tensor
// cores.  net [E,128,ht,wd] f16/f32 (or channels-last f16 [E,ht,wd,128] when net_channels_last), inp [E,128,ht,wd], corr [E,196,ht,wd],
// flow [E,4,ht,wd] f32 or None, seg [E] int64 (torch.unique inverse of the source frames) or None, n_src distinct sources,
// packed = the 27 tensors of droid_slam_b200.update.pack_update_weights in dba_update_weights order.
// Returns [net' (channels-last f16 [E,ht,wd,128]), delta [E,ht,wd,2] f32, weight [E,ht,wd,2] f32 (, eta [n_src,ht,wd] f32, upmask [n_src,576,ht,wd] f16)].
std::vector<torch::Tensor> update_forward(torch::Tensor net, torch::Tensor inp, torch::Tensor corr, c10::optional<torch::Tensor> flow,
                                          c10::optional<torch::Tensor> seg, int64_t n_src, std::vector<torch::Tensor> packed, bool net_channels_last) {
  const Expect expect("update_forward", net, "net");
  if (net_channels_last) expect(net, "net", F16, dims({kAny, kAny, kAny, 128}));
  else expect(net, "net", {}, dims({kAny, 128, kAny, kAny}));
  const int E = (int)net.size(0), ht = (int)net.size(net_channels_last ? 1 : 2), wd = (int)net.size(net_channels_last ? 2 : 3);
  expect(inp, "inp", {}, dims({E, 128, ht, wd}));
  expect(corr, "corr", {}, dims({E, 196, ht, wd}));
  // flow [E,4,ht,wd] of any dtype and layout is converted to a contiguous f32 copy
  const torch::Tensor flow_t = expect.opt(flow, "flow", {}, rows((int64_t)4 * ht * wd, E), kAnyLayout);
  const torch::Tensor flow_c = flow_t.defined() ? flow_t.to(torch::kFloat32).contiguous() : flow_t;
  const bool agg = seg.has_value() && seg->defined() && n_src > 0;
  torch::Tensor seg_c;
  if (agg) seg_c = expect.opt(seg, "seg", I64, rows(1, E), kAnyLayout).contiguous();
  TORCH_CHECK(packed.size() == 27, "droid_backends.update_forward: 27 packed weights expected, got ", packed.size());
  dba_update_weights W;
  const void** wp = reinterpret_cast<const void**>(&W);
  for (int k = 0; k < 27; k++) {
    expect(packed[k], item("packed", k).c_str(), k < 12 ? F16 : F32, dims(kUpdateWeightShapes[k]));
    wp[k] = packed[k].data_ptr();
  }
  c10::cuda::CUDAGuard guard(expect.dev);
  auto o16 = torch::TensorOptions().dtype(torch::kFloat16).device(expect.dev);
  auto o32 = torch::TensorOptions().dtype(torch::kFloat32).device(expect.dev);
  auto net_out = torch::empty({E, ht, wd, 128}, o16);
  auto delta = torch::empty({E, ht, wd, 2}, o32);
  auto weight = torch::empty({E, ht, wd, 2}, o32);
  torch::Tensor eta, upmask;
  if (agg) { eta = torch::empty({n_src, ht, wd}, o32); upmask = torch::empty({n_src, 576, ht, wd}, o16); }
  const size_t ws_bytes = dba_update_workspace_bytes(E, agg ? (int)n_src : 0, ht, wd);
  torch::Tensor ws;
  dba_update_args a;
  memset(&a, 0, sizeof(a));
  a.n_edges = E; a.ht = ht; a.wd = wd;
  a.net = net.data_ptr(); a.net_dtype = dtype_code(net, "update_forward"); a.net_layout = net_channels_last ? 1 : 0;
  a.inp = inp.data_ptr(); a.inp_dtype = dtype_code(inp, "update_forward");
  a.corr = corr.data_ptr(); a.corr_dtype = dtype_code(corr, "update_forward");
  a.flow = flow_c.defined() ? flow_c.data_ptr<float>() : nullptr;
  a.seg = agg ? seg_c.data_ptr<int64_t>() : nullptr; a.n_src = agg ? (int)n_src : 0;
  a.weights = &W;
  a.net_out = net_out.data_ptr(); a.delta = delta.data_ptr<float>(); a.weight = weight.data_ptr<float>();
  a.eta = agg ? eta.data_ptr<float>() : nullptr; a.upmask = agg ? upmask.data_ptr() : nullptr;
  a.workspace = workspace(ws_bytes, expect.dev, ws); a.workspace_bytes = ws_bytes; a.stream = cur_stream();
  check_status(dba_update_forward(&a), "update_forward");
  if (agg) return {net_out, delta, weight, eta, upmask};
  return {net_out, delta, weight};
}

// BasicEncoder.forward (reference droid_slam/modules/extractor.py:183-198) for DroidNet's fnet (norm 1 = instance, output_dim
// 128) and cnet (norm 0 = none, output_dim 256).  images [n,3,H,W] f32/f16, H and W multiples of 8; packed = the 28 tensors of
// droid_slam_b200.encoder.pack_encoder_weights (w[0..13] f16, then b[0..13] f32, include/droid_b200.h).  Returns [n,output_dim,H/8,W/8] f16.
// frames: null for f32 / f16 images (dba_encoder_forward), else uint8 camera frames in that format (dba_encoder_forward_frames)
static torch::Tensor run_encoder(const char* fn, torch::Tensor images, const std::vector<torch::Tensor>& packed, int64_t norm, int64_t output_dim,
                                 const dba_frame_format* frames) {
  const Expect expect(fn, images, frames ? "frames" : "images");
  if (frames) expect(images, "frames", torch::kUInt8, dims({kAny, 3, kAny, kAny}));
  else expect(images, "images", {F32, F16}, dims({kAny, 3, kAny, kAny}));
  TORCH_CHECK(norm == 0 || norm == 1, fn, ": norm must be 0 (none) or 1 (instance)");
  TORCH_CHECK(output_dim == 128 || output_dim == 256, fn, ": output_dim must be 128 or 256");
  TORCH_CHECK(packed.size() == 2 * DBA_ENCODER_CONVS, fn, ": 28 packed tensors expected");
  const int n = (int)images.size(0), H = (int)images.size(2), W = (int)images.size(3);
  TORCH_CHECK(n > 0 && H > 0 && W > 0 && H % 8 == 0 && W % 8 == 0, fn, ": H and W must be positive multiples of 8, got ", H, "x", W);
  // [taps, N, Kpad] of each packed weight
  const int64_t shapes[DBA_ENCODER_CONVS][3] = {{1, 32, 192}, {9, 32, 64}, {9, 32, 64}, {9, 32, 64}, {9, 32, 64}, {1, 128, 320}, {9, 64, 64},
                                                {9, 64, 64}, {9, 64, 64}, {1, 256, 576}, {9, 128, 128}, {9, 128, 128}, {9, 128, 128}, {1, output_dim, 128}};
  dba_encoder_weights Wt;
  for (int k = 0; k < DBA_ENCODER_CONVS; k++) {
    expect(packed[k], item("packed_weights", k).c_str(), F16, dims(shapes[k]));
    expect(packed[DBA_ENCODER_CONVS + k], item("packed_weights", DBA_ENCODER_CONVS + k).c_str(), F32, rows(1, shapes[k][1]));
    Wt.w[k] = packed[k].data_ptr();
    Wt.b[k] = packed[DBA_ENCODER_CONVS + k].data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(expect.dev);
  auto out = torch::empty({n, output_dim, H / 8, W / 8}, images.options().dtype(torch::kFloat16));
  const size_t ws_bytes = dba_encoder_workspace_bytes(n, H, W, (int)output_dim);
  torch::Tensor ws;
  dba_encoder_args a;
  memset(&a, 0, sizeof(a));
  a.images = images.data_ptr(); a.images_dtype = frames ? DBA_F32 : dtype_code(images, fn);
  a.n_images = n; a.H = H; a.W = W;
  a.weights = &Wt; a.norm = (int)norm; a.output_dim = (int)output_dim;
  a.out = out.data_ptr();
  a.workspace = workspace(ws_bytes, expect.dev, ws); a.workspace_bytes = ws_bytes; a.stream = cur_stream();
  check_status(frames ? dba_encoder_forward_frames(&a, frames) : dba_encoder_forward(&a), fn);
  return out;
}

torch::Tensor encoder_forward(torch::Tensor images, std::vector<torch::Tensor> packed, int64_t norm, int64_t output_dim) {
  return run_encoder("encoder_forward", images, packed, norm, output_dim, nullptr);
}

// encoder_forward on uint8 camera frames [n,3,H,W] (BGR when bgr, else RGB), normalised on load as the reference does in fp32:
// x / 255 - mean[c], / std[c] per RGB channel (dba_encoder_forward_frames).  The same bits as encoder_forward on the normalised frames.
torch::Tensor encoder_forward_frames(torch::Tensor frames, std::vector<torch::Tensor> packed, int64_t norm, int64_t output_dim, bool bgr,
                                     std::vector<double> mean, std::vector<double> std) {
  TORCH_CHECK(mean.size() == 3 && std.size() == 3, "droid_backends.encoder_forward_frames: mean and std must hold 3 values (one per RGB channel), got ",
              mean.size(), " and ", std.size());
  dba_frame_format f;
  memset(&f, 0, sizeof(f));
  f.channel_order = bgr ? DBA_FRAME_BGR : DBA_FRAME_RGB;
  for (int c = 0; c < 3; c++) { f.mean[c] = (float)mean[c]; f.std[c] = (float)std[c]; }
  return run_encoder("encoder_forward_frames", frames, packed, norm, output_dim, &f);
}

// channels-last tensor-core convolution (building block of update_forward).  src0 [E,ht,wd,C0] f16 (+ src1 [E,ht,wd,C1]),
// wpk f16 [k*k][N][Kpad], bias f32 [N] -> [E,ht,wd,N] f16
torch::Tensor conv_nhwc(torch::Tensor src0, c10::optional<torch::Tensor> src1, torch::Tensor wpk, torch::Tensor bias, int64_t ksize, bool relu) {
  const Expect expect("conv_nhwc", src0, "src0");
  expect(src0, "src0", F16, dims({kAny, kAny, kAny, kAny}));
  const int E = (int)src0.size(0), ht = (int)src0.size(1), wd = (int)src0.size(2), C0 = (int)src0.size(3);
  const torch::Tensor s1 = expect.opt(src1, "src1", F16, dims_min({E, ht, wd, kAny}));
  const int C1 = s1.defined() ? (int)s1.size(3) : 0;
  expect(wpk, "wpk", F16, dims({ksize * ksize, kAny, 64 * ((C0 + 63) / 64) + 64 * ((C1 + 63) / 64)}));
  const int N = (int)wpk.size(1);
  expect(bias, "bias", F32, rows(1, N));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto out = torch::empty({E, ht, wd, N}, src0.options());
  check_status(dba_conv_nhwc(src0.data_ptr(), C0, C0, s1.defined() ? s1.data_ptr() : nullptr, C1, C1, wpk.data_ptr(), bias.data_ptr<float>(),
                             out.data_ptr(), N, E, ht, wd, (int)ksize, N, relu ? 1 : 0, cur_stream()), "conv_nhwc");
  return out;
}

// cvx_upsample of inverse depths (reference droid_net.py:21-42 via DepthVideo.upsample, depth_video.py:155-159).
// disps [n,ht,wd] f32, mask [n,576,ht,wd] f16/f32 -> [n,8ht,8wd] f32
torch::Tensor cvx_upsample(torch::Tensor disps, torch::Tensor mask) {
  const Expect expect("cvx_upsample", disps, "disps");
  expect(disps, "disps", F32, dims({kAny, kAny, kAny}));
  const int n = (int)disps.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  expect(mask, "mask", {F16, F32}, dims({n, 576, ht, wd}));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto out = torch::empty({n, 8 * ht, 8 * wd}, disps.options());
  check_status(dba_cvx_upsample(disps.data_ptr<float>(), mask.data_ptr(), out.data_ptr<float>(), n, ht, wd, dtype_code(mask, "cvx_upsample"), cur_stream()), "cvx_upsample");
  return out;
}

// (row F1) the edge selection of FactorGraph.add_proximity_factors (reference factor_graph.py:357-411) on the device.
// d [(t-t0)*(t-t1)] f32 as returned by frame_distance over the meshgrid of :351-356, ii_known / jj_known int64 = the graph's active, bad
// and inactive edges.  Returns es [n,2] int64 in the reference's emission order (one host read of the row count).
torch::Tensor proximity_edges(torch::Tensor d, int64_t t0, int64_t t1, int64_t t, torch::Tensor ii_known, torch::Tensor jj_known, int64_t rad, int64_t nms,
                              double thresh, int64_t max_factors, bool stereo) {
  const Expect expect("proximity_edges", d, "d");
  TORCH_CHECK(t0 >= 0 && t1 >= 0, "t0, t1 >= 0");
  const int64_t n_i = std::max<int64_t>(t - t0, 0), n_j = std::max<int64_t>(t - t1, 0), n = n_i * n_j;
  expect(d, "d", F32, rows(1, n));   // the (t - t0) * (t - t1) distances
  expect(ii_known, "ii_known", I64);
  expect(jj_known, "jj_known", I64, rows(1, ii_known.numel()));
  c10::cuda::CUDAGuard guard(expect.dev);
  const int64_t cap = 2 * n + (3 + 2 * rad) * n_i + 2;
  auto es = torch::empty({cap, 2}, ii_known.options());
  auto hdr = torch::zeros({2}, torch::dtype(torch::kInt32).device(expect.dev));
  const size_t wsb = dba_proximity_workspace_bytes((int)t0, (int)t1, (int)t);
  torch::Tensor ws;
  void* ws_p = workspace(wsb, expect.dev, ws);
  check_status(dba_proximity_edges(d.data_ptr<float>(), (int)t0, (int)t1, (int)t, ii_known.data_ptr<int64_t>(), jj_known.data_ptr<int64_t>(), (int)ii_known.numel(), (int)rad,
                                   (int)nms, (float)thresh, (int)max_factors, stereo ? 1 : 0, es.data_ptr<int64_t>(), (int)cap, hdr.data_ptr<int>(), ws_p, wsb,
                                   cur_stream()), "proximity_edges");
  auto h = hdr.cpu();
  const int rows = h.data_ptr<int>()[0], status = h.data_ptr<int>()[1];
  TORCH_CHECK((status & 2) == 0, "proximity_edges: index (i - t0) * (t - t1) + (j - t1) out of range (the reference raises IndexError here)");
  TORCH_CHECK((status & 1) == 0, "proximity_edges: internal capacity exceeded");
  return es.narrow(0, 0, rows);
}

// DroidAsync's hand-over of the frontend's keyframes [t0,t1) to the backend (reference droid_slam/droid_async.py:54-119).  front / back:
// the two DepthVideo's buffers in the order poses, disps, disps_sens, images, tstamp, intrinsics, fmaps, nets, inps; front on one
// device, back on another or the same one.  On the back device's current stream: the slices [t0,t1) of every buffer go to the back
// buffers (a peer copy across devices, a device copy otherwise; torch's cross-device copy orders both devices' current streams), the
// front's poses[t0-10:t0-1] to a staging tensor, then dba_fragment_handover aligns and re-anchors in place.  The front's disps_sens is
// read where it is on one device and copied whole across devices (the reference's torch.any spans the whole buffer).  No host
// synchronisation.  Returns [diagnostics [9] f64: s, dG, align_scale] with diagnostics, else [].
std::vector<torch::Tensor> fragment_handover(std::vector<torch::Tensor> front, std::vector<torch::Tensor> back, int64_t t0, int64_t t1, bool stereo,
                                             bool diagnostics) {
  static const char* names[9] = {"poses", "disps", "disps_sens", "images", "tstamp", "intrinsics", "fmaps", "nets", "inps"};
  TORCH_CHECK(front.size() == 9 && back.size() == 9, "droid_backends.fragment_handover: front and back must each hold the 9 buffers ",
              "(poses, disps, disps_sens, images, tstamp, intrinsics, fmaps, nets, inps), got ", front.size(), " and ", back.size());
  const Expect fx("fragment_handover", front[0], "front poses");
  const Expect bx("fragment_handover", back[0], "back poses");
  fx(front[0], "front poses", F32, dims({kAny, 7}));
  const int64_t N = front[0].size(0);
  fx(front[1], "front disps", F32, dims({N, kAny, kAny}), kAnyLayout);
  const int64_t ht = front[1].size(1), wd = front[1].size(2);
  fx(front[2], "front disps_sens", F32, dims({N, ht, wd}));
  for (int k = 3; k < 9; k++) {
    const std::string name = std::string("front ") + names[k];
    fx(front[k], name.c_str(), {}, {}, kAnyLayout);
    TORCH_CHECK(front[k].dim() >= 1 && front[k].size(0) == N, "droid_backends.fragment_handover: ", name, " must have ", N,
                " frames (as poses), got shape ", front[k].sizes());
  }
  bx(back[0], "back poses", F32, dims({N, 7}));
  bx(back[1], "back disps", F32, dims({N, ht, wd}));
  for (int k = 2; k < 9; k++) {
    const std::string name = std::string("back ") + names[k];
    bx(back[k], name.c_str(), front[k].scalar_type(), dims(front[k].sizes()), kAnyLayout);
  }
  TORCH_CHECK(t0 == 0 || t0 >= 10, "droid_backends.fragment_handover: t0 must be 0 or at least 10 (the frames [t0-10, t0-1) are aligned), got ", t0);
  TORCH_CHECK(t0 <= N && t1 >= 0 && t1 <= N, "droid_backends.fragment_handover: t0 = ", t0, ", t1 = ", t1, " outside the ", N, "-frame buffers");
  c10::cuda::CUDAGuard guard(bx.dev);
  const int64_t n = std::max<int64_t>(t1 - t0, 0);
  if (n > 0)
    for (int k = 0; k < 9; k++) back[k].narrow(0, t0, n).copy_(front[k].narrow(0, t0, n), true);
  torch::Tensor align, sens = front[2];
  const auto on_back = torch::TensorOptions().device(bx.dev);
  if (t0 > 0) align = front[0].narrow(0, t0 - 10, 9).to(on_back, true, true);     // a snapshot: the front may move on
  if (fx.dev != bx.dev) sens = sens.to(on_back, true);
  torch::Tensor ws, diag;
  void* ws_p = workspace(DBA_HANDOVER_WORKSPACE_BYTES, bx.dev, ws);
  if (diagnostics) diag = torch::empty({9}, back[0].options().dtype(torch::kFloat64));
  check_status(dba_fragment_handover(t0 > 0 ? align.data_ptr<float>() : nullptr, back[0].data_ptr<float>(), back[1].data_ptr<float>(),
                                     sens.data_ptr<float>(), sens.numel(), (int)t0, (int)t1, (int)(ht * wd), stereo ? 1 : 0, ws_p,
                                     diagnostics ? diag.data_ptr<double>() : nullptr, cur_stream()), "fragment_handover");
  if (!diagnostics) return {};
  return {diag};
}

// ---- Lie groups SO3 / SE3 (droid_slam_b200/lietorch) -------------------------------------------------------------------------------
constexpr torch::ScalarType F64 = torch::kFloat64;

// The checks of one lie_forward / lie_backward call: the operands' device and dtype (float32 / float64, one for all), the last dimension
// of each (the operation's record sizes), the rank and broadcast compatibility (each batch size equal or 1, at most DBA_LIE_MAX_DIMS batch
// dimensions).  Makes the operands contiguous (never expanded) and gives the output batch shape and each operand's batch strides in
// records, 0 where it broadcasts.
struct LieCall {
  int da = 0, db = 0, dout = 0;
  torch::Tensor a, b;
  std::vector<int64_t> shape, sa, sb;
  LieCall(const char* fn, int op, int group, const torch::Tensor& a_in, const c10::optional<torch::Tensor>& b_in, const Expect& expect) {
    TORCH_CHECK(dba_lie_record_sizes(op, group, &da, &db, &dout) == DBA_OK, "droid_backends.", fn, ": no operation ", op, " for group ", group);
    expect(a_in, "a", {F32, F64}, {}, kAnyLayout);
    TORCH_CHECK(a_in.dim() >= 1 && a_in.size(-1) == da, "droid_backends.", fn, ": a must be [...,", da, "], got shape ", a_in.sizes());
    const int64_t nd = a_in.dim() - 1;
    TORCH_CHECK(nd <= DBA_LIE_MAX_DIMS, "droid_backends.", fn, ": at most ", DBA_LIE_MAX_DIMS, " batch dimensions, got ", nd);
    a = a_in.contiguous();
    if (db > 0) {
      TORCH_CHECK(b_in.has_value() && b_in->defined(), "droid_backends.", fn, ": operation ", op, " takes a second operand");
      expect(*b_in, "b", {a_in.scalar_type()}, {}, kAnyLayout);
      TORCH_CHECK(b_in->dim() == a_in.dim() && b_in->size(-1) == db, "droid_backends.", fn, ": b must be [...,", db, "] of a's rank ",
                  a_in.dim(), ", got shape ", b_in->sizes());
      b = b_in->contiguous();
    } else {
      TORCH_CHECK(!b_in.has_value() || !b_in->defined(), "droid_backends.", fn, ": operation ", op, " takes one operand");
    }
    shape.resize(nd); sa.resize(nd); sb.resize(nd, 0);
    int64_t ra = 1, rb = 1;
    for (int64_t d = nd - 1; d >= 0; d--) {
      const int64_t n = a.size(d), m = db > 0 ? b.size(d) : n;
      TORCH_CHECK(n == m || n == 1 || m == 1, "droid_backends.", fn, ": a ", a.sizes(), " and b ", b.sizes(), " do not broadcast in dimension ", d,
                  " (sizes must be equal or 1)");
      shape[d] = n == 1 ? m : n;
      sa[d] = n == 1 ? 0 : ra;
      ra *= n;
      if (db > 0) { sb[d] = m == 1 ? 0 : rb; rb *= m; }
    }
  }
  std::vector<int64_t> out_sizes(int64_t last) const { auto s = shape; s.push_back(last); return s; }
};

torch::Tensor lie_forward(int op, int group, torch::Tensor a, c10::optional<torch::Tensor> b) {
  const Expect expect("lie_forward", a, "a");
  const LieCall c("lie_forward", op, group, a, b, expect);
  c10::cuda::CUDAGuard guard(expect.dev);
  auto out = torch::empty(c.out_sizes(c.dout), c.a.options());
  check_status(dba_lie_forward(op, group, c.a.scalar_type() == F64 ? DBA_F64 : DBA_F32, c.a.data_ptr(), c.sa.data(),
                               c.db > 0 ? c.b.data_ptr() : nullptr, c.db > 0 ? c.sb.data() : nullptr, out.data_ptr(), (int)c.shape.size(),
                               c.shape.data(), cur_stream()), "lie_forward");
  return out;
}

// need_a / need_b: which gradients to compute; one not asked for is returned as None and never computed (at least one must be asked for)
std::vector<c10::optional<torch::Tensor>> lie_backward(int op, int group, torch::Tensor grad, torch::Tensor a, c10::optional<torch::Tensor> b,
                                                       bool need_a, bool need_b) {
  const Expect expect("lie_backward", a, "a");
  const LieCall c("lie_backward", op, group, a, b, expect);
  const auto grad_sizes = c.out_sizes(c.dout);
  expect(grad, "grad", {a.scalar_type()}, dims(grad_sizes), kAnyLayout);
  c10::cuda::CUDAGuard guard(expect.dev);
  need_b = need_b && c.db > 0;
  TORCH_CHECK(need_a || need_b, "droid_backends.lie_backward: no gradient asked for");
  auto g = grad.contiguous();
  const bool empty = g.numel() == 0;
  torch::Tensor ga, gb;
  if (need_a) ga = empty ? torch::zeros_like(c.a) : torch::empty_like(c.a);
  if (need_b) gb = empty ? torch::zeros_like(c.b) : torch::empty_like(c.b);
  check_status(dba_lie_backward(op, group, c.a.scalar_type() == F64 ? DBA_F64 : DBA_F32, g.data_ptr(), c.a.data_ptr(), c.sa.data(),
                                c.db > 0 ? c.b.data_ptr() : nullptr, c.db > 0 ? c.sb.data() : nullptr, need_a ? ga.data_ptr() : nullptr,
                                need_b ? gb.data_ptr() : nullptr, (int)c.shape.size(), c.shape.data(), cur_stream()), "lie_backward");
  std::vector<c10::optional<torch::Tensor>> out;
  out.push_back(need_a ? c10::optional<torch::Tensor>(ga) : c10::nullopt);
  if (c.db > 0) out.push_back(need_b ? c10::optional<torch::Tensor>(gb) : c10::nullopt);
  return out;
}

// ---- the differentiable dense BA layer (droid_slam_b200.modules.ba_layer) ---------------------------------------------------------
// The checks of one ba_layer_forward / ba_layer_backward call: every tensor fp32 (ii / jj int64), contiguous, on one device, with the
// extents of include/droid_b200.h; fixedp in [0, N) and at most DBA_BA_LAYER_MAX_POSES pose unknowns.  Fills the args struct and the
// workspace.
static dba_ba_layer_args ba_layer_args(const char* fn, const Expect& expect, const torch::Tensor& target, const torch::Tensor& weight,
                                       const torch::Tensor& eta, const torch::Tensor& poses, const torch::Tensor& disps,
                                       const torch::Tensor& intrinsics, const torch::Tensor& ii, const torch::Tensor& jj, int64_t fixedp,
                                       double ep, double lm, torch::Tensor& ws) {
  expect(disps, "disps", {F32}, dims({kAny, kAny, kAny, kAny}));
  const int64_t B = disps.size(0), N = disps.size(1), ht = disps.size(2), wd = disps.size(3);
  expect(ii, "ii", {I64}, dims({kAny}));
  const int64_t E = ii.size(0);
  expect(jj, "jj", {I64}, dims({E}));
  expect(target, "target", {F32}, dims({B, E, ht, wd, 2}));
  expect(weight, "weight", {F32}, dims({B, E, ht, wd, 2}));
  expect(eta, "eta", {F32}, dims({B, kAny, ht, wd}));
  expect(poses, "poses", {F32}, dims({B, N, 7}));
  expect(intrinsics, "intrinsics", {F32}, dims({B, N, 4}));
  TORCH_CHECK(B >= 1 && N >= 1 && E >= 1 && ht >= 1 && wd >= 1 && eta.size(1) >= 1, "droid_backends.", fn,
              ": empty batch, frames, edges, depth frames or image");
  TORCH_CHECK(fixedp >= 0 && fixedp < N, "droid_backends.", fn, ": fixedp must be in [0, N) = [0, ", N, "), got ", fixedp);
  TORCH_CHECK(N - fixedp <= DBA_BA_LAYER_MAX_POSES, "droid_backends.", fn, ": at most ", DBA_BA_LAYER_MAX_POSES,
              " pose unknowns (N - fixedp) are factored in one launch, got ", N - fixedp);
  dba_ba_layer_args a{};
  a.target = target.data_ptr<float>(); a.weight = weight.data_ptr<float>(); a.eta = eta.data_ptr<float>();
  a.poses = poses.data_ptr<float>(); a.disps = disps.data_ptr<float>(); a.intrinsics = intrinsics.data_ptr<float>();
  a.ii = ii.data_ptr<int64_t>(); a.jj = jj.data_ptr<int64_t>();
  a.B = (int)B; a.N = (int)N; a.E = (int)E; a.M = (int)eta.size(1); a.ht = (int)ht; a.wd = (int)wd; a.fixedp = (int)fixedp;
  a.ep = (float)ep; a.lm = (float)lm;
  const size_t bytes = dba_ba_layer_workspace_bytes(a.B, a.N, a.E, a.M, a.ht, a.wd, a.fixedp);
  ws = torch::empty({(int64_t)bytes}, disps.options().dtype(torch::kUInt8));
  a.workspace = ws.data_ptr(); a.workspace_bytes = bytes;
  a.stream = cur_stream();
  return a;
}

// -> [poses', disps', factor, dx, dz, flags]; check=True reads the status word (one host sync) and raises on an out-of-range ii / jj or
// a source-frame count other than eta's M
std::vector<torch::Tensor> ba_layer_forward(torch::Tensor target, torch::Tensor weight, torch::Tensor eta, torch::Tensor poses, torch::Tensor disps,
                                            torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj, int64_t fixedp, double ep, double lm,
                                            bool check) {
  const Expect expect("ba_layer_forward", disps, "disps");
  c10::cuda::CUDAGuard guard(expect.dev);
  torch::Tensor ws;
  dba_ba_layer_args a = ba_layer_args("ba_layer_forward", expect, target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp, ep, lm, ws);
  const int64_t n = 6 * (a.N - a.fixedp);
  auto f64 = disps.options().dtype(F64);
  auto poses_out = torch::empty_like(poses), disps_out = torch::empty_like(disps);
  auto factor = torch::empty({a.B, n, n}, f64), dx = torch::empty({a.B, n}, f64), dz = torch::zeros({a.B, a.M, a.ht * a.wd}, f64);
  auto flags = torch::empty({1 + a.B}, disps.options().dtype(torch::kInt32));
  a.poses_out = poses_out.data_ptr<float>(); a.disps_out = disps_out.data_ptr<float>();
  a.factor = factor.data_ptr<double>(); a.dx = dx.data_ptr<double>(); a.dz = dz.data_ptr<double>(); a.flags = flags.data_ptr<int>();
  check_status(dba_ba_layer_forward(&a), "ba_layer_forward");
  if (check) {
    const int st = flags[0].item<int>();
    TORCH_CHECK_INDEX(!(st & DBA_BA_LAYER_BAD_INDEX), "droid_backends.ba_layer_forward: ii / jj index a frame outside [0, ", a.N, ")");
    TORCH_CHECK(!(st & DBA_BA_LAYER_BAD_M), "droid_backends.ba_layer_forward: eta has ", a.M, " depth frames, not the number of distinct ii");
  }
  return {poses_out, disps_out, factor, dx, dz, flags};
}

// -> [grad_target, grad_weight, grad_eta, grad_poses, grad_disps]
std::vector<torch::Tensor> ba_layer_backward(torch::Tensor grad_poses, torch::Tensor grad_disps, torch::Tensor target, torch::Tensor weight,
                                             torch::Tensor eta, torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii,
                                             torch::Tensor jj, int64_t fixedp, double ep, double lm, torch::Tensor factor, torch::Tensor dx,
                                             torch::Tensor dz, torch::Tensor flags) {
  const Expect expect("ba_layer_backward", disps, "disps");
  c10::cuda::CUDAGuard guard(expect.dev);
  torch::Tensor ws;
  dba_ba_layer_args a = ba_layer_args("ba_layer_backward", expect, target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp, ep, lm, ws);
  const int64_t n = 6 * (a.N - a.fixedp);
  expect(grad_poses, "grad_poses", {F32}, dims({a.B, a.N, 7}));
  expect(grad_disps, "grad_disps", {F32}, dims({a.B, a.N, a.ht, a.wd}));
  expect(factor, "factor", {F64}, dims({a.B, n, n}));
  expect(dx, "dx", {F64}, dims({a.B, n}));
  expect(dz, "dz", {F64}, dims({a.B, a.M, a.ht * a.wd}));
  expect(flags, "flags", {torch::kInt32}, dims({1 + a.B}));
  auto g_target = torch::empty_like(target), g_weight = torch::empty_like(weight), g_eta = torch::empty_like(eta);
  auto g_poses = torch::empty_like(poses), g_disps = torch::empty_like(disps);
  a.factor = factor.data_ptr<double>(); a.dx = dx.data_ptr<double>(); a.dz = dz.data_ptr<double>(); a.flags = flags.data_ptr<int>();
  a.grad_poses_out = grad_poses.data_ptr<float>(); a.grad_disps_out = grad_disps.data_ptr<float>();
  a.grad_target = g_target.data_ptr<float>(); a.grad_weight = g_weight.data_ptr<float>(); a.grad_eta = g_eta.data_ptr<float>();
  a.grad_poses = g_poses.data_ptr<float>(); a.grad_disps = g_disps.data_ptr<float>();
  check_status(dba_ba_layer_backward(&a), "ba_layer_backward");
  return {g_target, g_weight, g_eta, g_poses, g_disps};
}

// ---- training's tail: the flow loss and upsample_disp's backward (droid_slam_b200.modules.flow_loss / upsample_disp) ----------------

// a device array of the tensors' data pointers, staged in pinned memory and copied on the current stream (no host synchronisation;
// the caching host allocator keeps the staging buffer until the copy has run)
static torch::Tensor device_pointers(const std::vector<torch::Tensor>& ts, const torch::Device& dev) {
  auto host = torch::empty({(int64_t)ts.size()}, torch::TensorOptions().dtype(I64).pinned_memory(true));
  int64_t* p = host.data_ptr<int64_t>();
  for (size_t k = 0; k < ts.size(); k++) p[k] = (int64_t)(uintptr_t)ts[k].data_ptr();
  return host.to(dev, /*non_blocking=*/true);
}

// The checks of one flow_loss_forward / flow_loss_backward call: every tensor fp32, contiguous, on one device; Ps [B,N,7], disps
// [B,N,ht,wd], intrinsics [B,N,4], and every element of poses_est / disps_est (as many of each, at least one) [B,N,7] / [B,N,ht,wd];
// N >= 2 (the chain graph has an edge), a non-empty batch and image.
struct FlowArgs {
  int B, N, ht, wd, n;
};
static FlowArgs flow_loss_args(const char* fn, const Expect& expect, const torch::Tensor& Ps, const torch::Tensor& disps,
                               const std::vector<torch::Tensor>& poses_est, const std::vector<torch::Tensor>& disps_est,
                               const torch::Tensor& intrinsics) {
  expect(disps, "disps", {F32}, dims({kAny, kAny, kAny, kAny}));
  const int64_t B = disps.size(0), N = disps.size(1), ht = disps.size(2), wd = disps.size(3);
  expect(Ps, "Ps", {F32}, dims({B, N, 7}));
  expect(intrinsics, "intrinsics", {F32}, dims({B, N, 4}));
  TORCH_CHECK(!poses_est.empty() && poses_est.size() == disps_est.size(), "droid_backends.", fn, ": poses_est and disps_est must hold "
              "the same number (at least one) of iterates, got ", poses_est.size(), " and ", disps_est.size());
  for (size_t k = 0; k < poses_est.size(); k++) {
    expect(poses_est[k], item("poses_est", k).c_str(), {F32}, dims({B, N, 7}));
    expect(disps_est[k], item("disps_est", k).c_str(), {F32}, dims({B, N, ht, wd}));
  }
  TORCH_CHECK(B >= 1 && ht >= 1 && wd >= 1, "droid_backends.", fn, ": empty batch or image");
  TORCH_CHECK(N >= 2, "droid_backends.", fn, ": N must be at least 2 (the chain graph of one frame has no edge), got ", N);
  TORCH_CHECK(B <= 65535 && N <= 32768, "droid_backends.", fn, ": at most 65535 batch elements and 32768 frames, got ", B, " and ", N);
  return {(int)B, (int)N, (int)ht, (int)wd, (int)poses_est.size()};
}

// -> [loss (0-dim f32), metrics (f64 [3]: sum of epe where v > 0.5, that count, the count with epe < 1, for the last iterate)]
std::vector<torch::Tensor> flow_loss_forward(torch::Tensor Ps, torch::Tensor disps, std::vector<torch::Tensor> poses_est,
                                             std::vector<torch::Tensor> disps_est, torch::Tensor intrinsics, double gamma) {
  const Expect expect("flow_loss_forward", disps, "disps");
  const FlowArgs a = flow_loss_args("flow_loss_forward", expect, Ps, disps, poses_est, disps_est, intrinsics);
  c10::cuda::CUDAGuard guard(expect.dev);
  torch::Tensor keep;
  const size_t bytes = dba_flow_loss_workspace_bytes(a.B, a.N, a.ht, a.wd, a.n);
  void* ws = workspace(bytes, expect.dev, keep);
  auto pp = device_pointers(poses_est, expect.dev), dp = device_pointers(disps_est, expect.dev);
  auto loss = torch::empty({}, disps.options()), metrics = torch::empty({3}, disps.options().dtype(torch::kFloat64));
  check_status(dba_flow_loss_forward(Ps.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(),
                                     (const float* const*)pp.data_ptr(), (const float* const*)dp.data_ptr(), a.n, loss.data_ptr<float>(),
                                     metrics.data_ptr<double>(), a.B, a.N, a.ht, a.wd, gamma, ws, bytes, cur_stream()), "flow_loss_forward");
  return {loss, metrics};
}

// -> [grad_poses_est[0..n), grad_disps_est[0..n)]; grad: the loss's upstream gradient (0-dim f32 on the device)
std::vector<torch::Tensor> flow_loss_backward(torch::Tensor grad, torch::Tensor Ps, torch::Tensor disps, std::vector<torch::Tensor> poses_est,
                                              std::vector<torch::Tensor> disps_est, torch::Tensor intrinsics, double gamma) {
  const Expect expect("flow_loss_backward", disps, "disps");
  const FlowArgs a = flow_loss_args("flow_loss_backward", expect, Ps, disps, poses_est, disps_est, intrinsics);
  expect(grad, "grad", {F32}, Shape{Shape::kDims, c10::IntArrayRef()});
  c10::cuda::CUDAGuard guard(expect.dev);
  torch::Tensor keep;
  const size_t bytes = dba_flow_loss_workspace_bytes(a.B, a.N, a.ht, a.wd, a.n);
  void* ws = workspace(bytes, expect.dev, keep);
  std::vector<torch::Tensor> gp, gd;
  for (int k = 0; k < a.n; k++) { gp.push_back(torch::empty_like(poses_est[k])); gd.push_back(torch::empty_like(disps_est[k])); }
  auto pp = device_pointers(poses_est, expect.dev), dp = device_pointers(disps_est, expect.dev);
  auto gpp = device_pointers(gp, expect.dev), gdp = device_pointers(gd, expect.dev);
  check_status(dba_flow_loss_backward(grad.data_ptr<float>(), Ps.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(),
                                      (const float* const*)pp.data_ptr(), (const float* const*)dp.data_ptr(), a.n, (float* const*)gpp.data_ptr(),
                                      (float* const*)gdp.data_ptr(), a.B, a.N, a.ht, a.wd, gamma, ws, bytes, cur_stream()), "flow_loss_backward");
  gp.insert(gp.end(), gd.begin(), gd.end());
  return gp;
}

// the backward of cvx_upsample for fp32 masks: disps [n,ht,wd], mask [n,576,ht,wd], grad_out [n,8ht,8wd] -> [grad_disps, grad_mask]
std::vector<torch::Tensor> cvx_upsample_backward(torch::Tensor disps, torch::Tensor mask, torch::Tensor grad_out) {
  const Expect expect("cvx_upsample_backward", disps, "disps");
  expect(disps, "disps", {F32}, dims({kAny, kAny, kAny}));
  const int64_t n = disps.size(0), ht = disps.size(1), wd = disps.size(2);
  expect(mask, "mask", {F32}, dims({n, 576, ht, wd}));
  expect(grad_out, "grad_out", {F32}, dims({n, 8 * ht, 8 * wd}));
  c10::cuda::CUDAGuard guard(expect.dev);
  auto g = ((uintptr_t)grad_out.data_ptr() & 15) ? grad_out.clone() : grad_out;     // the kernel reads 16-byte vectors
  auto grad_disps = torch::empty_like(disps), grad_mask = torch::empty_like(mask);
  auto taps = torch::empty({n, 9, 8, ht, wd}, disps.options());
  check_status(dba_cvx_upsample_backward(disps.data_ptr<float>(), mask.data_ptr<float>(), g.data_ptr<float>(), grad_disps.data_ptr<float>(),
                                         grad_mask.data_ptr<float>(), taps.data_ptr<float>(), (int)n, (int)ht, (int)wd, cur_stream()),
               "cvx_upsample_backward");
  return {grad_disps, grad_mask};
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "H100-native droid_backends (drop-in for princeton-vl/DROID-SLAM src/droid.cpp)";
  // bundle adjustment kernels
  m.def("ba", &ba, "bundle adjustment");
  m.def("frame_distance", &frame_distance, "frame_distance");
  m.def("projmap", &projmap, "projmap");
  m.def("depth_filter", &depth_filter, "depth_filter");
  m.def("iproj", &iproj, "back projection");
  // correlation volume kernels
  m.def("altcorr_forward", &altcorr_forward, "ALTCORR forward");
  m.def("altcorr_backward", &altcorr_backward, "ALTCORR backward");
  m.def("corr_index_forward", &corr_index_forward, "INDEX forward");
  m.def("corr_index_backward", &corr_index_backward, "INDEX backward");
  m.def("corr_volume_pyramid", &corr_volume_pyramid, "all-pairs correlation + 4-level pyramid (wgmma), native extension", pybind11::arg("fmap1"), pybind11::arg("fmap2"),
        pybind11::arg("ii"), pybind11::arg("jj"), pybind11::arg("tiled") = false);
  m.def("corr_volume_pyramid_f32", &corr_volume_pyramid_f32, "training CorrBlock: fp32 correlation volume + 4-level pyramid, native extension",
        pybind11::arg("fmap1"), pybind11::arg("fmap2"));
  m.def("corr_grad_accumulate", &corr_grad_accumulate, "training CorrBlock: add one lookup's gradient into the gradient pyramid, native extension",
        pybind11::arg("coords"), pybind11::arg("grad"), pybind11::arg("gpyr"));
  m.def("corr_adjoint", &corr_adjoint, "training CorrBlock: feature-map gradients from the gradient pyramid, native extension",
        pybind11::arg("fmap1"), pybind11::arg("fmap2"), pybind11::arg("gpyr"));
  m.def("corr_lookup_pyramid", &corr_lookup_pyramid, "4-level radius-3 lookup in one launch -> [E,196,H,W], native extension", pybind11::arg("pyramid"), pybind11::arg("coords"),
        pybind11::arg("tiled") = false);
  m.def("altcorr_pyramid", &altcorr_pyramid, "AltCorrBlock pyramid in one launch -> levels [B,N,H>>l,W>>l,C] (private channels-last layout), native extension",
        pybind11::arg("fmaps"), pybind11::arg("num_levels") = 4);
  m.def("altcorr_lookup_pyramid", &altcorr_lookup_pyramid, "AltCorrBlock lookup over all levels in one launch -> [B,M,L*49,H,W], native extension",
        pybind11::arg("pyramid"), pybind11::arg("coords"), pybind11::arg("ii"), pybind11::arg("jj"), pybind11::arg("radius") = 3);
  m.def("corr_volume_supported", [](int dim, int ht, int wd, bool tiled) { return dba_corr_volume_supported(dim, ht, wd, DBA_F16, tiled ? 1 : 0) != 0; },
        "does corr_volume_pyramid (tiled: with tiled=True) have a kernel for f16 [.,dim,ht,wd] feature maps", pybind11::arg("dim"), pybind11::arg("ht"),
        pybind11::arg("wd"), pybind11::arg("tiled") = false);
  m.def("reproject", &reproject, "fused pops.projective_transform(jacobian=False), native extension");
  m.def("motion_features", &motion_features, "reprojection + FactorGraph motion features in one launch -> [coords, coords_t, motn], native extension",
        pybind11::arg("poses"), pybind11::arg("disps"), pybind11::arg("intrinsics"), pybind11::arg("ii"), pybind11::arg("jj"), pybind11::arg("target"),
        pybind11::arg("edge_index") = pybind11::none());
  m.def("graph_writeback", &graph_writeback, "update-operator outputs -> factor graph target / weight / damping and BA inputs (in place), native extension",
        pybind11::arg("delta"), pybind11::arg("weight"), pybind11::arg("coords"), pybind11::arg("edge_index"), pybind11::arg("target"),
        pybind11::arg("weight_out"), pybind11::arg("ba_target"), pybind11::arg("ba_weight"), pybind11::arg("n_inactive"), pybind11::arg("eta"),
        pybind11::arg("src_frames"), pybind11::arg("damping"), pybind11::arg("ba_frames") = pybind11::none(),
        pybind11::arg("ba_damping") = pybind11::none(), pybind11::arg("ep") = 1e-7);
  m.def("update_workspace_bytes", [](int n_edges, int n_src, int ht, int wd) { return dba_update_workspace_bytes(n_edges, n_src, ht, wd); },
        "device workspace of one update_forward call (dba_update_workspace_bytes)");
  m.def("update_forward", &update_forward, "update operator (ConvGRU + heads + GraphAgg) on wgmma, native extension");
  m.def("encoder_forward", &encoder_forward, "feature / context encoder (BasicEncoder: fnet norm=1, cnet norm=0) on wgmma -> [n,output_dim,H/8,W/8] f16, native extension",
        pybind11::arg("images"), pybind11::arg("packed_weights"), pybind11::arg("norm"), pybind11::arg("output_dim"));
  m.def("encoder_forward_frames", &encoder_forward_frames,
        "encoder_forward on uint8 camera frames [n,3,H,W], channel reorder and normalisation on load -> [n,output_dim,H/8,W/8] f16, native extension",
        pybind11::arg("frames"), pybind11::arg("packed_weights"), pybind11::arg("norm"), pybind11::arg("output_dim"), pybind11::arg("bgr"),
        pybind11::arg("mean"), pybind11::arg("std"));
  m.def("conv_nhwc", &conv_nhwc,"channels-last 1x1/3x3 convolution on wgmma, native extension");
  m.def("cvx_upsample", &cvx_upsample, "convex upsampling of inverse depth maps (droid_net.cvx_upsample, dim = 1), native extension");
  m.def("proximity_edges", &proximity_edges, "edge selection of FactorGraph.add_proximity_factors (factor_graph.py:357-411), native extension");
  m.def("fill_interpolate", &fill_interpolate, "pose interpolation of PoseTrajectoryFiller.__fill -> [t0, t1, poses], native extension",
        pybind11::arg("poses"), pybind11::arg("tstamps"), pybind11::arg("t"));
  m.def("pose_only_ba", &pose_only_ba, "motion-only BA of the trajectory filler's graph, all iterations in one launch -> [status(, dx, sys)], native extension",
        pybind11::arg("poses"), pybind11::arg("disps"), pybind11::arg("intrinsics"), pybind11::arg("targets"), pybind11::arg("weights"),
        pybind11::arg("ii"), pybind11::arg("jj"), pybind11::arg("t0"), pybind11::arg("t1"), pybind11::arg("iterations") = 2,
        pybind11::arg("lm") = 1e-4f, pybind11::arg("ep") = 0.1f, pybind11::arg("check") = true,
        pybind11::arg("diagnostics") = false);
  m.def("fragment_handover", &fragment_handover,
        "DroidAsync's frontend -> backend hand-over of frames [t0,t1): slice copies, fragment alignment and re-anchoring on the back device "
        "-> [diagnostics (s, dG, align_scale)] or [], native extension",
        pybind11::arg("front"), pybind11::arg("back"), pybind11::arg("t0"), pybind11::arg("t1"), pybind11::arg("stereo"),
        pybind11::arg("diagnostics") = false);
  m.def("lie_forward", &lie_forward, "SO3 / SE3 group operation (group 1: SO3, 3: SE3; op: include/droid_b200.h DBA_LIE_*) with broadcasting in "
        "the kernel -> out, native extension", pybind11::arg("op"), pybind11::arg("group"), pybind11::arg("a"), pybind11::arg("b") = pybind11::none());
  m.def("lie_backward", &lie_backward, "gradients of lie_forward (lietorch's convention; broadcast operands reduced in the kernel) -> [grad_a(, "
        "grad_b)], None for a gradient not asked for, native extension", pybind11::arg("op"), pybind11::arg("group"), pybind11::arg("grad"),
        pybind11::arg("a"), pybind11::arg("b") = pybind11::none(), pybind11::arg("need_a") = true, pybind11::arg("need_b") = true);
  m.def("ba_layer_forward", &ba_layer_forward, "the dense BA layer of DroidNet (reference geom/ba.py BA), forward -> [poses', disps', factor, "
        "dx, dz, flags], native extension", pybind11::arg("target"), pybind11::arg("weight"), pybind11::arg("eta"), pybind11::arg("poses"),
        pybind11::arg("disps"), pybind11::arg("intrinsics"), pybind11::arg("ii"), pybind11::arg("jj"), pybind11::arg("fixedp") = 1,
        pybind11::arg("ep") = 0.1, pybind11::arg("lm") = 1e-4, pybind11::arg("check") = true);
  m.def("ba_layer_backward", &ba_layer_backward, "gradients of ba_layer_forward -> [grad_target, grad_weight, grad_eta, grad_poses, grad_disps], "
        "native extension", pybind11::arg("grad_poses"), pybind11::arg("grad_disps"), pybind11::arg("target"), pybind11::arg("weight"),
        pybind11::arg("eta"), pybind11::arg("poses"), pybind11::arg("disps"), pybind11::arg("intrinsics"), pybind11::arg("ii"),
        pybind11::arg("jj"), pybind11::arg("fixedp"), pybind11::arg("ep"), pybind11::arg("lm"), pybind11::arg("factor"), pybind11::arg("dx"),
        pybind11::arg("dz"), pybind11::arg("flags"));
  m.def("flow_loss_forward", &flow_loss_forward, "training's flow loss (reference geom/losses.py flow_loss) on the chain graph, every "
        "iterate in one pass -> [loss, metrics (sum of epe where v > 0.5, that count, the count with epe < 1)], native extension",
        pybind11::arg("Ps"), pybind11::arg("disps"), pybind11::arg("poses_est"), pybind11::arg("disps_est"), pybind11::arg("intrinsics"),
        pybind11::arg("gamma") = 0.9);
  m.def("flow_loss_backward", &flow_loss_backward, "gradients of flow_loss_forward -> [grad_poses_est..., grad_disps_est...], native extension",
        pybind11::arg("grad"), pybind11::arg("Ps"), pybind11::arg("disps"), pybind11::arg("poses_est"), pybind11::arg("disps_est"),
        pybind11::arg("intrinsics"), pybind11::arg("gamma") = 0.9);
  m.def("cvx_upsample_backward", &cvx_upsample_backward, "gradients of cvx_upsample for fp32 masks -> [grad_disps, grad_mask], native extension",
        pybind11::arg("disps"), pybind11::arg("mask"), pybind11::arg("grad_out"));
  m.def("_b200_native", []() { return true; });
}
