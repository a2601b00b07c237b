// `droid_backends` -- drop-in Python extension exporting the reference's nine callables
// (reference src/droid.cpp:93-259: ba, frame_distance, projmap, depth_filter, iproj, altcorr_forward,
// altcorr_backward, corr_index_forward, corr_index_backward) with identical positional signatures and return
// shapes, implemented on the C ABI of include/droid_b200.h (libdroid_b200.so, hand-written sm_90a kernels).
//
// torch is used here for what the reference binding uses it for: tensor handles, the caching allocator, the current
// stream.  Differences from the reference binding, all strictly safer: a CUDAGuard on the tensors' device, launches on
// torch's CURRENT stream (the reference uses the legacy default stream), dtype/device checks with readable messages.
// There is no CPU fallback: every call needs CUDA tensors and fails loudly otherwise.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <vector>
#include <cuda_runtime_api.h>
#include <cstring>
#include "../../../include/droid_b200.h"

#define CHECK_CONTIGUOUS(x) TORCH_CHECK(x.is_contiguous(), #x " must be contiguous")   // reference src/droid.cpp:89
#define CHECK_CUDA(x) TORCH_CHECK(x.is_cuda(), #x " must be a CUDA tensor (droid_backends has no CPU path)")
#define CHECK_F32(x) TORCH_CHECK(x.scalar_type() == torch::kFloat32, #x " must be float32")
#define CHECK_I64(x) TORCH_CHECK(x.scalar_type() == torch::kInt64, #x " must be int64")
#define CHECK_INPUT(x) do { CHECK_CONTIGUOUS(x); CHECK_CUDA(x); } while (0)

static inline void check_status(int rc, const char* op) {
  TORCH_CHECK(rc == DBA_OK, "droid_backends.", op, " failed (status ", rc, "): ", dba_last_error());
}
static inline dba_stream_t cur_stream() { return (dba_stream_t)at::cuda::getCurrentCUDAStream().stream(); }

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
  CHECK_INPUT(targets); CHECK_INPUT(weights); CHECK_INPUT(poses); CHECK_INPUT(disps);
  CHECK_INPUT(intrinsics); CHECK_INPUT(disps_sens); CHECK_INPUT(ii); CHECK_INPUT(jj);
  CHECK_F32(targets); CHECK_F32(weights); CHECK_F32(poses); CHECK_F32(disps); CHECK_F32(intrinsics); CHECK_F32(disps_sens);
  CHECK_I64(ii); CHECK_I64(jj);
  TORCH_CHECK(poses.dim() == 2 && poses.size(1) == 7, "poses must be [N,7]");
  TORCH_CHECK(disps.dim() == 3, "disps must be [N,ht,wd]");
  TORCH_CHECK(disps_sens.sizes() == disps.sizes(), "disps_sens must have the shape of disps");
  TORCH_CHECK(intrinsics.numel() >= 4, "intrinsics must hold fx,fy,cx,cy");
  const int N = (int)disps.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  const int HW = ht * wd;
  const int E = (int)ii.size(0);
  TORCH_CHECK(jj.size(0) == E, "ii and jj must have the same length");
  TORCH_CHECK(targets.numel() == (int64_t)E * 2 * HW && weights.numel() == (int64_t)E * 2 * HW, "targets/weights must be [E,2,ht,wd]");
  TORCH_CHECK(poses.size(0) >= N || poses.size(0) >= t1, "poses has fewer rows than the optimisation window");
  TORCH_CHECK(t0 >= 0 && t1 >= t0 && t1 <= N, "invalid window [t0,t1)");
  if (iterations <= 0) return {torch::Tensor(), torch::Tensor()};   // reference returns two undefined tensors
  c10::cuda::CUDAGuard guard(poses.device());

  int eta_rows = 1;
  torch::Tensor eta_c = eta;
  if (!motion_only) {
    CHECK_CUDA(eta); CHECK_F32(eta);
    eta_c = eta.contiguous();   // the reference only needs it .view()-able (SURVEY Q12)
    TORCH_CHECK(eta_c.numel() % HW == 0 && eta_c.numel() > 0, "eta must be [M,ht,wd]");
    eta_rows = (int)(eta_c.numel() / HW);
  }
  const int n_frames = std::min<int>(N, (int)poses.size(0));
  const size_t ws_bytes = dba_ba_workspace_bytes(n_frames, E, ht, wd, t0, t1);
  auto ws = torch::empty({(int64_t)ws_bytes}, torch::TensorOptions().dtype(torch::kUInt8).device(poses.device()));
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
  a.workspace = ws.data_ptr(); a.workspace_bytes = ws_bytes; a.stream = cur_stream();
  a.own_lo = 0; a.own_hi = n_frames; a.eta_by_frame = 0;

  // The graph bookkeeping runs first and its result is read back (one stream synchronisation; the reference's ba synchronises a
  // dozen times per call): the number of depth frames M sizes dz, eta must have 1 or M rows (the reference raises a broadcast
  // error otherwise, src/droid_kernels.cu:1407), and out-of-range indices are reported instead of being dropped.  While the stream
  // is being captured into a CUDA graph no synchronisation is possible: dz is sized from eta and the checks are skipped (the
  // caller validated the same tensors eagerly).
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing((cudaStream_t)a.stream, &cap);
  const bool capturing = cap != cudaStreamCaptureStatusNone;
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
  CHECK_INPUT(poses); CHECK_INPUT(disps); CHECK_INPUT(intrinsics); CHECK_INPUT(ii); CHECK_INPUT(jj);
  CHECK_F32(poses); CHECK_F32(disps); CHECK_F32(intrinsics); CHECK_I64(ii); CHECK_I64(jj);
  TORCH_CHECK(disps.dim() == 3, "disps must be [N,ht,wd]");
  c10::cuda::CUDAGuard guard(poses.device());
  const int num = (int)ii.size(0);
  auto dist = torch::empty({num}, poses.options());
  check_status(dba_frame_distance(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                                  jj.data_ptr<int64_t>(), dist.data_ptr<float>(), num, (int)disps.size(1), (int)disps.size(2), beta,
                                  cur_stream()), "frame_distance");
  return dist;
}

std::vector<torch::Tensor> projmap(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj) {
  CHECK_INPUT(poses); CHECK_INPUT(disps); CHECK_INPUT(intrinsics); CHECK_INPUT(ii); CHECK_INPUT(jj);
  CHECK_F32(poses); CHECK_F32(disps); CHECK_F32(intrinsics); CHECK_I64(ii); CHECK_I64(jj);
  TORCH_CHECK(disps.dim() == 3, "disps must be [N,ht,wd]");
  c10::cuda::CUDAGuard guard(poses.device());
  const int num = (int)ii.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  auto coords = torch::empty({num, ht, wd, 3}, poses.options());
  auto valid = torch::empty({num, ht, wd, 1}, poses.options());
  check_status(dba_projmap(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                           jj.data_ptr<int64_t>(), coords.data_ptr<float>(), valid.data_ptr<float>(), num, ht, wd, cur_stream()), "projmap");
  return {coords, valid};
}

torch::Tensor iproj(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics) {
  CHECK_INPUT(poses); CHECK_INPUT(disps); CHECK_INPUT(intrinsics);
  CHECK_F32(poses); CHECK_F32(disps); CHECK_F32(intrinsics);
  TORCH_CHECK(disps.dim() == 3, "disps must be [N,ht,wd]");
  TORCH_CHECK(poses.size(0) >= disps.size(0), "need one pose per disparity map");
  c10::cuda::CUDAGuard guard(poses.device());
  const int nm = (int)disps.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  auto points = torch::empty({nm, ht, wd, 3}, disps.options());
  check_status(dba_iproj(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), points.data_ptr<float>(), nm, ht,
                         wd, cur_stream()), "iproj");
  return points;
}

torch::Tensor depth_filter(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ix, torch::Tensor thresh) {
  CHECK_INPUT(poses); CHECK_INPUT(disps); CHECK_INPUT(intrinsics); CHECK_INPUT(ix); CHECK_INPUT(thresh);
  CHECK_F32(poses); CHECK_F32(disps); CHECK_F32(intrinsics); CHECK_I64(ix); CHECK_F32(thresh);
  TORCH_CHECK(disps.dim() == 3, "disps must be [N,ht,wd]");
  c10::cuda::CUDAGuard guard(poses.device());
  const int num = (int)ix.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  auto counter = torch::empty({num, ht, wd}, disps.options());
  check_status(dba_depth_filter(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ix.data_ptr<int64_t>(),
                                thresh.data_ptr<float>(), counter.data_ptr<float>(), num, (int)disps.size(0), ht, wd, cur_stream()),
               "depth_filter");
  return counter;
}

std::vector<torch::Tensor> corr_index_forward(torch::Tensor volume, torch::Tensor coords, int radius) {
  CHECK_INPUT(volume); CHECK_INPUT(coords); CHECK_F32(coords);
  TORCH_CHECK(volume.dim() == 5 && coords.dim() == 4 && coords.size(1) == 2, "volume [N,h1,w1,h2,w2], coords [N,2,h1,w1]");
  TORCH_CHECK(coords.size(0) == volume.size(0) && coords.size(2) == volume.size(1) && coords.size(3) == volume.size(2), "coords/volume mismatch");
  c10::cuda::CUDAGuard guard(volume.device());
  const int n = (int)volume.size(0), h1 = (int)volume.size(1), w1 = (int)volume.size(2), h2 = (int)volume.size(3), w2 = (int)volume.size(4);
  auto corr = torch::empty({n, 2 * radius + 1, 2 * radius + 1, h1, w1}, volume.options());
  check_status(dba_corr_index_forward(volume.data_ptr(), coords.data_ptr<float>(), corr.data_ptr(), n, h1, w1, h2, w2, radius,
                                      dtype_code(volume, "corr_index_forward"), cur_stream()), "corr_index_forward");
  return {corr};
}

std::vector<torch::Tensor> corr_index_backward(torch::Tensor volume, torch::Tensor coords, torch::Tensor corr_grad, int radius) {
  CHECK_INPUT(volume); CHECK_INPUT(coords); CHECK_INPUT(corr_grad); CHECK_F32(coords);
  TORCH_CHECK(volume.dim() == 5 && coords.dim() == 4, "volume [N,h1,w1,h2,w2], coords [N,2,h1,w1]");
  TORCH_CHECK(corr_grad.scalar_type() == volume.scalar_type(), "corr_grad must have the dtype of volume");
  c10::cuda::CUDAGuard guard(volume.device());
  const int n = (int)volume.size(0), h1 = (int)volume.size(1), w1 = (int)volume.size(2), h2 = (int)volume.size(3), w2 = (int)volume.size(4);
  auto volume_grad = torch::empty_like(volume);
  check_status(dba_corr_index_backward(coords.data_ptr<float>(), corr_grad.data_ptr(), volume_grad.data_ptr(), n, h1, w1, h2, w2, radius,
                                       dtype_code(volume, "corr_index_backward"), cur_stream()), "corr_index_backward");
  return {volume_grad};
}

std::vector<torch::Tensor> altcorr_forward(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor coords, torch::Tensor ii,
                                           torch::Tensor jj, int radius) {
  CHECK_INPUT(fmap1); CHECK_INPUT(fmap2); CHECK_INPUT(coords); CHECK_F32(coords);
  CHECK_CUDA(ii); CHECK_CUDA(jj); CHECK_I64(ii); CHECK_I64(jj);
  TORCH_CHECK(fmap1.dim() == 5 && fmap2.dim() == 5 && coords.dim() == 5 && coords.size(2) == 2, "fmaps [B,N,C,H,W], coords [B,M,2,H,W]");
  TORCH_CHECK(fmap1.scalar_type() == fmap2.scalar_type(), "fmap1/fmap2 dtype mismatch");
  c10::cuda::CUDAGuard guard(fmap1.device());
  auto iic = ii.contiguous(), jjc = jj.contiguous();
  const int B = (int)coords.size(0), M = (int)coords.size(1), H = (int)coords.size(3), W = (int)coords.size(4);
  TORCH_CHECK(iic.size(0) == M && jjc.size(0) == M, "ii/jj must have one entry per edge");
  TORCH_CHECK(fmap1.size(3) == H && fmap1.size(4) == W, "fmap1 spatial size must match coords");
  const int D = 2 * radius + 1;
  auto out = torch::empty({B, M, D, D, H, W}, fmap1.options());
  check_status(dba_altcorr_forward(fmap1.data_ptr(), fmap2.data_ptr(), coords.data_ptr<float>(), iic.data_ptr<int64_t>(),
                                   jjc.data_ptr<int64_t>(), out.data_ptr(), B, (int)fmap1.size(1), (int)fmap2.size(1), (int)fmap1.size(2), H, W,
                                   (int)fmap2.size(3), (int)fmap2.size(4), M, radius, dtype_code(fmap1, "altcorr_forward"), cur_stream()),
               "altcorr_forward");
  return {out.permute({0, 1, 3, 2, 4, 5})};   // reference src/altcorr_kernel.cu:171
}

std::vector<torch::Tensor> altcorr_backward(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor coords, torch::Tensor corr_grad,
                                            torch::Tensor ii, torch::Tensor jj, int radius) {
  // corr_grad is the gradient of the tensor altcorr_forward returned ([B,M,x-off,y-off,H,W]); the reference
  // (src/droid.cpp:212-226 -> src/altcorr_kernel.cu:175-225) un-permutes it and spreads it over the raw window.
  CHECK_INPUT(fmap1); CHECK_INPUT(fmap2); CHECK_INPUT(coords); CHECK_INPUT(corr_grad); CHECK_F32(coords);
  CHECK_CUDA(ii); CHECK_CUDA(jj); CHECK_I64(ii); CHECK_I64(jj);
  c10::cuda::CUDAGuard guard(fmap1.device());
  auto iic = ii.contiguous(), jjc = jj.contiguous();
  auto cg = corr_grad.to(torch::kFloat32).contiguous();   // kernel reads a float accessor (src/altcorr_kernel.cu:84)
  const int B = (int)coords.size(0), M = (int)coords.size(1), H = (int)coords.size(3), W = (int)coords.size(4);
  const int D = 2 * radius + 1;
  TORCH_CHECK(cg.numel() == (int64_t)B * M * D * D * H * W, "corr_grad must be [B,M,2r+1,2r+1,H,W]");
  auto g1 = torch::empty_like(fmap1), g2 = torch::empty_like(fmap2);
  check_status(dba_altcorr_backward(fmap1.data_ptr(), fmap2.data_ptr(), coords.data_ptr<float>(), cg.data_ptr<float>(), iic.data_ptr<int64_t>(),
                                    jjc.data_ptr<int64_t>(), g1.data_ptr(), g2.data_ptr(), B, (int)fmap1.size(1), (int)fmap2.size(1),
                                    (int)fmap1.size(2), H, W, (int)fmap2.size(3), (int)fmap2.size(4), M, radius,
                                    dtype_code(fmap1, "altcorr_backward"), cur_stream()), "altcorr_backward");
  return {g1, g2};
}

// extension beyond the reference's nine callables: CorrBlock.__init__ in one tensor-core kernel
// (reference droid_slam/modules/corr.py:24-38,63-71).  fmap1/fmap2 [N,128,ht,wd] f16 (ht, wd >= 8), ii/jj [E] -> 4 pyramid levels.
// tiled (levels 0-1 in the private tiled layout) only where dba_corr_volume_tiled_supported; wd % 8 != 0 takes a staging workspace
// from the caching allocator.
std::vector<torch::Tensor> corr_volume_pyramid(torch::Tensor fmap1, torch::Tensor fmap2, torch::Tensor ii, torch::Tensor jj, bool tiled) {
  CHECK_INPUT(fmap1); CHECK_INPUT(fmap2); CHECK_INPUT(ii); CHECK_INPUT(jj); CHECK_I64(ii); CHECK_I64(jj);
  TORCH_CHECK(fmap1.dim() == 4 && fmap2.dim() == 4, "fmaps must be [N,C,ht,wd]");
  TORCH_CHECK(fmap1.scalar_type() == torch::kFloat16 && fmap2.scalar_type() == torch::kFloat16, "corr_volume_pyramid: float16 feature maps expected");
  TORCH_CHECK(fmap1.size(1) == fmap2.size(1) && fmap1.size(2) == fmap2.size(2) && fmap1.size(3) == fmap2.size(3), "fmap shapes differ");
  c10::cuda::CUDAGuard guard(fmap1.device());
  const int E = (int)ii.size(0), C = (int)fmap1.size(1), ht = (int)fmap1.size(2), wd = (int)fmap1.size(3);
  TORCH_CHECK(jj.size(0) == E, "ii and jj must have the same length");
  std::vector<torch::Tensor> out;
  for (int l = 0; l < 4; l++) out.push_back(torch::empty({E, ht, wd, ht >> l, wd >> l}, fmap1.options()));
  const int n1 = (int)fmap1.size(0), n2 = (int)fmap2.size(0);
  if (tiled) {
    check_status(dba_corr_volume_pyramid_tiled(fmap1.data_ptr(), fmap2.data_ptr(), ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), out[0].data_ptr(),
                                               out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), E, n1, n2, C, ht, wd, DBA_F16, cur_stream()),
                 "corr_volume_pyramid");
    return out;
  }
  const size_t ws_bytes = dba_corr_volume_workspace_bytes(n1, n2, C, ht, wd);
  torch::Tensor ws;
  if (ws_bytes > 0 && E > 0) ws = torch::empty({(int64_t)ws_bytes}, fmap1.options().dtype(torch::kUInt8));
  check_status(dba_corr_volume_pyramid_ws(fmap1.data_ptr(), fmap2.data_ptr(), ii.data_ptr<int64_t>(), jj.data_ptr<int64_t>(), out[0].data_ptr(),
                                          out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), E, n1, n2, C, ht, wd, DBA_F16,
                                          ws.defined() ? ws.data_ptr() : nullptr, ws.defined() ? ws_bytes : 0, cur_stream()),
               "corr_volume_pyramid");
  return out;
}

// extension: CorrBlock.__call__ (reference modules/corr.py:40-50) in one launch.  pyramid = 4 f16 tensors [E,h1,w1,h1/2^l,w1/2^l] (reference
// layout, or levels 0-1 tiled when `tiled`), coords [E,2,h1,w1] f32 at level-0 scale -> [E,196,h1,w1] = cat over levels of corr_index_forward
torch::Tensor corr_lookup_pyramid(std::vector<torch::Tensor> pyramid, torch::Tensor coords, bool tiled) {
  TORCH_CHECK(pyramid.size() == 4, "corr_lookup_pyramid: 4 pyramid levels expected");
  CHECK_INPUT(coords); CHECK_F32(coords);
  for (auto& v : pyramid) { CHECK_INPUT(v); TORCH_CHECK(v.scalar_type() == torch::kFloat16 && v.dim() == 5, "pyramid levels must be f16 [E,h1,w1,h2,w2]"); }
  const int n = (int)pyramid[0].size(0), h1 = (int)pyramid[0].size(1), w1 = (int)pyramid[0].size(2);
  TORCH_CHECK(coords.dim() == 4 && coords.size(0) == n && coords.size(1) == 2 && coords.size(2) == h1 && coords.size(3) == w1, "coords must be [E,2,h1,w1]");
  for (int l = 0; l < 4; l++)
    TORCH_CHECK(pyramid[l].size(0) == n && pyramid[l].size(1) == h1 && pyramid[l].size(2) == w1 && pyramid[l].size(3) == (h1 >> l) && pyramid[l].size(4) == (w1 >> l), "pyramid level ", l, " has the wrong shape");
  c10::cuda::CUDAGuard guard(coords.device());
  auto out = torch::empty({n, 196, h1, w1}, pyramid[0].options());
  check_status(dba_corr_lookup_pyramid(pyramid[0].data_ptr(), pyramid[1].data_ptr(), pyramid[2].data_ptr(), pyramid[3].data_ptr(), coords.data_ptr<float>(), out.data_ptr(),
                                       n, h1, w1, tiled ? 3 : 0, DBA_F16, cur_stream()), "corr_lookup_pyramid");
  return out;
}

// extension: AltCorrBlock.__init__ (reference modules/corr.py:90-101) as one launch.  fmaps [B,N,C,H,W] f16/f32 -> num_levels tensors
// [B,N,H>>l,W>>l,C] in the private channels-last, pre-quartered layout of include/droid_b200.h (dba_altcorr_pyramid).
std::vector<torch::Tensor> altcorr_pyramid(torch::Tensor fmaps, int num_levels) {
  CHECK_INPUT(fmaps);
  TORCH_CHECK(fmaps.dim() == 5, "altcorr_pyramid: fmaps must be [B,N,C,H,W]");
  TORCH_CHECK(fmaps.scalar_type() == torch::kFloat16 || fmaps.scalar_type() == torch::kFloat32, "altcorr_pyramid: float16 or float32 feature maps expected, got ",
              fmaps.scalar_type());
  TORCH_CHECK(num_levels >= 1 && num_levels <= 4, "altcorr_pyramid: 1..4 levels expected");
  c10::cuda::CUDAGuard guard(fmaps.device());
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

// extension: AltCorrBlock.__call__ (reference modules/corr.py:104-117) in one launch.  pyramid from altcorr_pyramid, coords [B,M,2,H,W] f32
// at level-0 scale, ii/jj [M] -> [B,M,L*49,H,W] = stack over levels of altcorr_forward(level 0, level l, coords / 2^l, ii, jj, radius)
torch::Tensor altcorr_lookup_pyramid(std::vector<torch::Tensor> pyramid, torch::Tensor coords, torch::Tensor ii, torch::Tensor jj, int radius) {
  const int L = (int)pyramid.size();
  TORCH_CHECK(L >= 1 && L <= 4, "altcorr_lookup_pyramid: 1..4 pyramid levels expected");
  CHECK_INPUT(coords); CHECK_F32(coords);
  CHECK_CUDA(ii); CHECK_CUDA(jj); CHECK_I64(ii); CHECK_I64(jj);
  for (auto& v : pyramid) {
    CHECK_INPUT(v);
    TORCH_CHECK(v.dim() == 5 && v.scalar_type() == pyramid[0].scalar_type() && v.device() == coords.device(),
                "altcorr_lookup_pyramid: pyramid levels must be [B,N,H>>l,W>>l,C] tensors of one dtype on the device of coords");
  }
  const auto& p0 = pyramid[0];
  const int B = (int)p0.size(0), N = (int)p0.size(1), H = (int)p0.size(2), W = (int)p0.size(3), C = (int)p0.size(4);
  TORCH_CHECK(coords.dim() == 5 && coords.size(0) == B && coords.size(2) == 2 && coords.size(3) == H && coords.size(4) == W,
              "altcorr_lookup_pyramid: coords must be [B,M,2,H,W] with B, H, W of pyramid level 0");
  for (int l = 1; l < L; l++)
    TORCH_CHECK(pyramid[l].size(0) == B && pyramid[l].size(1) == N && pyramid[l].size(2) == (H >> l) && pyramid[l].size(3) == (W >> l) &&
                    pyramid[l].size(4) == C, "altcorr_lookup_pyramid: pyramid level ", l, " has the wrong shape");
  const int M = (int)coords.size(1);
  auto iic = ii.contiguous(), jjc = jj.contiguous();
  TORCH_CHECK(iic.dim() == 1 && jjc.dim() == 1 && iic.size(0) == M && jjc.size(0) == M, "altcorr_lookup_pyramid: ii/jj must have one entry per edge");
  c10::cuda::CUDAGuard guard(coords.device());
  auto out = torch::empty({B, M, L * (2 * radius + 1) * (2 * radius + 1), H, W}, p0.options());
  const void* p[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int l = 0; l < L; l++) p[l] = pyramid[l].data_ptr();
  check_status(dba_altcorr_lookup_pyramid(p[0], p[1], p[2], p[3], coords.data_ptr<float>(), iic.data_ptr<int64_t>(), jjc.data_ptr<int64_t>(),
                                          out.data_ptr(), B, N, C, H, W, M, L, radius, dtype_code(p0, "altcorr_lookup_pyramid"), cur_stream()),
               "altcorr_lookup_pyramid");
  return out;
}

// extension: fused DepthVideo.reproject (reference depth_video.py:171-179 -> geom/projective_ops.py:165-198, jacobian=False)
std::vector<torch::Tensor> reproject(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj) {
  CHECK_INPUT(poses); CHECK_INPUT(disps); CHECK_INPUT(intrinsics); CHECK_INPUT(ii); CHECK_INPUT(jj);
  CHECK_F32(poses); CHECK_F32(disps); CHECK_F32(intrinsics); CHECK_I64(ii); CHECK_I64(jj);
  TORCH_CHECK(disps.dim() == 3 && intrinsics.dim() == 2 && intrinsics.size(1) == 4, "disps [N,ht,wd], intrinsics [N,4]");
  c10::cuda::CUDAGuard guard(poses.device());
  const int num = (int)ii.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  auto coords = torch::empty({num, ht, wd, 2}, poses.options());
  auto valid = torch::empty({num, ht, wd, 1}, poses.options());
  check_status(dba_reproject(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                             jj.data_ptr<int64_t>(), coords.data_ptr<float>(), valid.data_ptr<float>(), num, ht, wd, cur_stream()), "reproject");
  return {coords, valid};
}

static void check_rows(const torch::Tensor& t, const char* name, const torch::Device& dev, int64_t per_row, const char* shape) {
  CHECK_CONTIGUOUS(t); CHECK_F32(t);
  TORCH_CHECK(t.device() == dev, name, " must be on ", dev);
  TORCH_CHECK(t.dim() >= 1 && t.numel() % per_row == 0, name, " must be ", shape);
}

static const int64_t* opt_index(const c10::optional<torch::Tensor>& t, const torch::Device& dev, int64_t n, const char* name) {
  if (!t.has_value() || !t->defined()) return nullptr;
  CHECK_CONTIGUOUS((*t)); CHECK_I64((*t));
  TORCH_CHECK(t->device() == dev && t->numel() == n, name, " must be an int64 tensor of ", n, " entries on ", dev);
  return t->data_ptr<int64_t>();
}

// extension: FactorGraph.update / update_lowmem motion features (reference factor_graph.py:220-222, :280-282) fused with the reprojection.
// poses [N,7], disps [N,ht,wd], intrinsics [N,4], ii / jj [E] int64, target [(1,)E,ht,wd,2] f32; call row r reads edge edge_index[r]
// (all E edges in order when edge_index is None).  Returns [coords [n,ht,wd,2], coords_t [n,2,ht,wd], motn [n,4,ht,wd]].
std::vector<torch::Tensor> motion_features(torch::Tensor poses, torch::Tensor disps, torch::Tensor intrinsics, torch::Tensor ii, torch::Tensor jj,
                                           torch::Tensor target, c10::optional<torch::Tensor> edge_index) {
  CHECK_INPUT(poses); CHECK_INPUT(disps); CHECK_INPUT(intrinsics); CHECK_INPUT(ii); CHECK_INPUT(jj);
  CHECK_F32(poses); CHECK_F32(disps); CHECK_F32(intrinsics); CHECK_I64(ii); CHECK_I64(jj);
  TORCH_CHECK(disps.dim() == 3 && intrinsics.dim() == 2 && intrinsics.size(1) == 4, "disps [N,ht,wd], intrinsics [N,4]");
  const auto dev = poses.device();
  TORCH_CHECK(disps.device() == dev && intrinsics.device() == dev && ii.device() == dev && jj.device() == dev, "motion_features: all tensors on one device");
  c10::cuda::CUDAGuard guard(dev);
  const int E = (int)ii.numel(), ht = (int)disps.size(1), wd = (int)disps.size(2);
  TORCH_CHECK(jj.numel() == E, "ii and jj must have the same length");
  check_rows(target, "target", dev, (int64_t)ht * wd * 2, "[E,ht,wd,2]");
  TORCH_CHECK(target.numel() == (int64_t)E * ht * wd * 2, "target must be [E,ht,wd,2] with E = len(ii)");
  const int n = (edge_index.has_value() && edge_index->defined()) ? (int)edge_index->numel() : E;
  const int64_t* ei = opt_index(edge_index, dev, n, "edge_index");
  auto coords = torch::empty({n, ht, wd, 2}, poses.options());
  auto coords_t = torch::empty({n, 2, ht, wd}, poses.options());
  auto motn = torch::empty({n, 4, ht, wd}, poses.options());
  check_status(dba_motion_features(poses.data_ptr<float>(), disps.data_ptr<float>(), intrinsics.data_ptr<float>(), ii.data_ptr<int64_t>(),
                                   jj.data_ptr<int64_t>(), ei, target.data_ptr<float>(), coords.data_ptr<float>(), coords_t.data_ptr<float>(),
                                   motn.data_ptr<float>(), n, ht, wd, cur_stream()), "motion_features");
  return {coords, coords_t, motn};
}

// extension: write-back of one update-operator call into the factor graph and BA's inputs (reference factor_graph.py:234-251, :304-320).
// delta / weight / coords [n,ht,wd,2] f32 (call rows), edge_index [n] int64 or None (row r = edge r); target / weight_out [(1,)E,ht,wd,2] and
// ba_target / ba_weight [E_ba,2,ht,wd] written in place (row n_inactive + e); eta [n_src,ht,wd] scattered to damping[src_frames];
// then, when ba_frames is given, ba_damping[r] = .2 * damping[ba_frames[r]] + ep.
void graph_writeback(torch::Tensor delta, torch::Tensor weight, torch::Tensor coords, c10::optional<torch::Tensor> edge_index,
                     torch::Tensor target, torch::Tensor weight_out, torch::Tensor ba_target, torch::Tensor ba_weight, int64_t n_inactive,
                     c10::optional<torch::Tensor> eta, c10::optional<torch::Tensor> src_frames, torch::Tensor damping,
                     c10::optional<torch::Tensor> ba_frames, c10::optional<torch::Tensor> ba_damping, double ep) {
  const auto dev = damping.device();
  CHECK_CUDA(damping);
  check_rows(damping, "damping", dev, 1, "[n_frames,ht,wd]");
  TORCH_CHECK(damping.dim() == 3, "damping must be [n_frames,ht,wd]");
  const int ht = (int)damping.size(1), wd = (int)damping.size(2);
  const int64_t px2 = (int64_t)ht * wd * 2;
  for (auto* t : {&delta, &weight, &coords, &target, &weight_out, &ba_target, &ba_weight}) check_rows(*t, "graph_writeback tensor", dev, px2, "[rows,ht,wd,2]");
  const int n = (int)(delta.numel() / px2);
  TORCH_CHECK(weight.numel() == delta.numel() && coords.numel() == delta.numel(), "delta, weight and coords must have the same shape");
  const int64_t E = target.numel() / px2, E_ba = ba_target.numel() / px2;
  TORCH_CHECK(weight_out.numel() == target.numel() && ba_weight.numel() == ba_target.numel(), "target / weight_out and ba_target / ba_weight shapes differ");
  TORCH_CHECK(n_inactive >= 0 && n_inactive + E <= E_ba, "ba_target must hold n_inactive + E rows");
  TORCH_CHECK(edge_index.has_value() && edge_index->defined() ? true : n <= E, "more call rows than graph edges");
  c10::cuda::CUDAGuard guard(dev);
  const int64_t* ei = opt_index(edge_index, dev, n, "edge_index");
  int n_src = 0;
  const float* eta_p = nullptr;
  const int64_t* src_p = nullptr;
  if (eta.has_value() && eta->defined()) {
    check_rows(*eta, "eta", dev, (int64_t)ht * wd, "[n_src,ht,wd]");
    n_src = (int)(eta->numel() / ((int64_t)ht * wd));
    eta_p = eta->data_ptr<float>();
    src_p = opt_index(src_frames, dev, n_src, "src_frames");
    TORCH_CHECK(src_p, "src_frames is required with eta");
  }
  int n_ba = 0;
  const int64_t* baf = nullptr;
  float* bad = nullptr;
  if (ba_frames.has_value() && ba_frames->defined()) {
    n_ba = (int)ba_frames->numel();
    baf = opt_index(ba_frames, dev, n_ba, "ba_frames");
    TORCH_CHECK(ba_damping.has_value() && ba_damping->defined(), "ba_damping is required with ba_frames");
    check_rows(*ba_damping, "ba_damping", dev, (int64_t)ht * wd, "[M,ht,wd]");
    TORCH_CHECK(ba_damping->numel() == (int64_t)n_ba * ht * wd, "ba_damping must be [len(ba_frames),ht,wd]");
    bad = ba_damping->data_ptr<float>();
  }
  check_status(dba_graph_writeback(delta.data_ptr<float>(), weight.data_ptr<float>(), coords.data_ptr<float>(), ei, n, target.data_ptr<float>(),
                                   weight_out.data_ptr<float>(), ba_target.data_ptr<float>(), ba_weight.data_ptr<float>(), (int)n_inactive, eta_p, src_p,
                                   n_src, damping.data_ptr<float>(), baf, n_ba, bad, (float)ep, ht, wd, cur_stream()), "graph_writeback");
}

// extension: the update operator (reference droid_slam/droid_net.py:111-143, modules/gru.py:19-32, droid_net.py:59-75) on the tensor
// cores.  net [E,128,ht,wd] f16/f32 (or channels-last f16 [E,ht,wd,128] when net_channels_last), inp [E,128,ht,wd], corr [E,196,ht,wd],
// flow [E,4,ht,wd] f32 or None, seg [E] int64 (torch.unique inverse of the source frames) or None, n_src distinct sources,
// packed = the 27 tensors of droid_slam_b200.update.pack_update_weights in dba_update_weights order.
// Returns [net' (channels-last f16 [E,ht,wd,128]), delta [E,ht,wd,2] f32, weight [E,ht,wd,2] f32 (, eta [n_src,ht,wd] f32, upmask [n_src,576,ht,wd] f16)].
std::vector<torch::Tensor> update_forward(torch::Tensor net, torch::Tensor inp, torch::Tensor corr, c10::optional<torch::Tensor> flow,
                                          c10::optional<torch::Tensor> seg, int64_t n_src, std::vector<torch::Tensor> packed, bool net_channels_last) {
  CHECK_INPUT(net); CHECK_INPUT(inp); CHECK_INPUT(corr);
  TORCH_CHECK(net.dim() == 4 && inp.dim() == 4 && corr.dim() == 4, "net/inp/corr must be 4-D");
  TORCH_CHECK(packed.size() == 27, "packed weights: 27 tensors expected");
  c10::cuda::CUDAGuard guard(net.device());
  int E, ht, wd;
  if (net_channels_last) {
    TORCH_CHECK(net.scalar_type() == torch::kFloat16 && net.size(3) == 128, "channels-last net must be f16 [E,ht,wd,128]");
    E = (int)net.size(0); ht = (int)net.size(1); wd = (int)net.size(2);
  } else {
    TORCH_CHECK(net.size(1) == 128, "net must be [E,128,ht,wd]");
    E = (int)net.size(0); ht = (int)net.size(2); wd = (int)net.size(3);
  }
  TORCH_CHECK(inp.size(0) == E && inp.size(1) == 128 && inp.size(2) == ht && inp.size(3) == wd, "inp must be [E,128,ht,wd]");
  TORCH_CHECK(corr.size(0) == E && corr.size(1) == 196 && corr.size(2) == ht && corr.size(3) == wd, "corr must be [E,196,ht,wd]");
  torch::Tensor flow_c, seg_c;
  if (flow.has_value() && flow->defined()) {
    flow_c = flow->to(torch::kFloat32).contiguous();
    CHECK_CUDA(flow_c);
    TORCH_CHECK(flow_c.numel() == (int64_t)E * 4 * ht * wd, "flow must be [E,4,ht,wd]");
  }
  const bool agg = seg.has_value() && seg->defined() && n_src > 0;
  if (agg) { seg_c = seg->contiguous(); CHECK_CUDA(seg_c); CHECK_I64(seg_c); TORCH_CHECK(seg_c.numel() == E, "seg must have one entry per edge"); }
  dba_update_weights W;
  const void** wp = reinterpret_cast<const void**>(&W);
  for (int k = 0; k < 27; k++) {
    CHECK_INPUT(packed[k]);
    TORCH_CHECK(packed[k].scalar_type() == (k < 12 ? torch::kFloat16 : torch::kFloat32), "packed weight ", k, " has the wrong dtype");
    wp[k] = packed[k].data_ptr();
  }
  auto o16 = torch::TensorOptions().dtype(torch::kFloat16).device(net.device());
  auto o32 = torch::TensorOptions().dtype(torch::kFloat32).device(net.device());
  auto net_out = torch::empty({E, ht, wd, 128}, o16);
  auto delta = torch::empty({E, ht, wd, 2}, o32);
  auto weight = torch::empty({E, ht, wd, 2}, o32);
  torch::Tensor eta, upmask;
  if (agg) { eta = torch::empty({n_src, ht, wd}, o32); upmask = torch::empty({n_src, 576, ht, wd}, o16); }
  const size_t ws_bytes = dba_update_workspace_bytes(E, agg ? (int)n_src : 0, ht, wd);
  auto ws = torch::empty({(int64_t)ws_bytes + 256}, torch::TensorOptions().dtype(torch::kUInt8).device(net.device()));
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
  a.workspace = (void*)(((uintptr_t)ws.data_ptr() + 255) & ~(uintptr_t)255); a.workspace_bytes = ws_bytes; a.stream = cur_stream();
  check_status(dba_update_forward(&a), "update_forward");
  if (agg) return {net_out, delta, weight, eta, upmask};
  return {net_out, delta, weight};
}

// extension: BasicEncoder.forward (reference droid_slam/modules/extractor.py:183-198) for DroidNet's fnet (norm 1 = instance, output_dim
// 128) and cnet (norm 0 = none, output_dim 256).  images [n,3,H,W] f32/f16, H and W multiples of 8; packed = the 28 tensors of
// droid_slam_b200.encoder.pack_encoder_weights (w[0..13] f16, then b[0..13] f32, include/droid_b200.h).  Returns [n,output_dim,H/8,W/8] f16.
torch::Tensor encoder_forward(torch::Tensor images, std::vector<torch::Tensor> packed, int64_t norm, int64_t output_dim) {
  CHECK_INPUT(images);
  TORCH_CHECK(images.dim() == 4 && images.size(1) == 3, "encoder_forward: images must be [n,3,H,W]");
  TORCH_CHECK(images.scalar_type() == torch::kFloat32 || images.scalar_type() == torch::kFloat16, "encoder_forward: float32 or float16 images expected");
  TORCH_CHECK(norm == 0 || norm == 1, "encoder_forward: norm must be 0 (none) or 1 (instance)");
  TORCH_CHECK(output_dim == 128 || output_dim == 256, "encoder_forward: output_dim must be 128 or 256");
  TORCH_CHECK(packed.size() == 2 * DBA_ENCODER_CONVS, "encoder_forward: 28 packed tensors expected");
  const int n = (int)images.size(0), H = (int)images.size(2), W = (int)images.size(3);
  TORCH_CHECK(n > 0 && H > 0 && W > 0 && H % 8 == 0 && W % 8 == 0, "encoder_forward: H and W must be positive multiples of 8, got ", H, "x", W);
  c10::cuda::CUDAGuard guard(images.device());
  // [taps, N, Kpad] of each packed weight
  const int64_t shapes[DBA_ENCODER_CONVS][3] = {{1, 32, 192}, {9, 32, 64}, {9, 32, 64}, {9, 32, 64}, {9, 32, 64}, {1, 128, 320}, {9, 64, 64},
                                                {9, 64, 64}, {9, 64, 64}, {1, 256, 576}, {9, 128, 128}, {9, 128, 128}, {9, 128, 128}, {1, output_dim, 128}};
  dba_encoder_weights Wt;
  for (int k = 0; k < DBA_ENCODER_CONVS; k++) {
    const torch::Tensor& w = packed[k];
    const torch::Tensor& b = packed[DBA_ENCODER_CONVS + k];
    CHECK_INPUT(w); CHECK_INPUT(b);
    TORCH_CHECK(w.device() == images.device() && b.device() == images.device(), "encoder_forward: packed weights must be on the images' device");
    TORCH_CHECK(w.scalar_type() == torch::kFloat16 && w.dim() == 3 && w.size(0) == shapes[k][0] && w.size(1) == shapes[k][1] && w.size(2) == shapes[k][2],
                "encoder_forward: packed weight ", k, " must be f16 [", shapes[k][0], ",", shapes[k][1], ",", shapes[k][2], "], got ", w.sizes());
    TORCH_CHECK(b.scalar_type() == torch::kFloat32 && b.numel() == shapes[k][1], "encoder_forward: packed bias ", k, " must be f32 [", shapes[k][1], "]");
    Wt.w[k] = w.data_ptr();
    Wt.b[k] = b.data_ptr<float>();
  }
  auto out = torch::empty({n, output_dim, H / 8, W / 8}, images.options().dtype(torch::kFloat16));
  const size_t ws_bytes = dba_encoder_workspace_bytes(n, H, W, (int)output_dim);
  auto ws = torch::empty({(int64_t)ws_bytes + 256}, images.options().dtype(torch::kUInt8));
  dba_encoder_args a;
  memset(&a, 0, sizeof(a));
  a.images = images.data_ptr(); a.images_dtype = dtype_code(images, "encoder_forward");
  a.n_images = n; a.H = H; a.W = W;
  a.weights = &Wt; a.norm = (int)norm; a.output_dim = (int)output_dim;
  a.out = out.data_ptr();
  a.workspace = (void*)(((uintptr_t)ws.data_ptr() + 255) & ~(uintptr_t)255); a.workspace_bytes = ws_bytes; a.stream = cur_stream();
  check_status(dba_encoder_forward(&a), "encoder_forward");
  return out;
}

// extension: channels-last tensor-core convolution (building block of update_forward).  src0 [E,ht,wd,C0] f16 (+ src1 [E,ht,wd,C1]),
// wpk f16 [k*k][N][Kpad], bias f32 [N] -> [E,ht,wd,N] f16
torch::Tensor conv_nhwc(torch::Tensor src0, c10::optional<torch::Tensor> src1, torch::Tensor wpk, torch::Tensor bias, int64_t ksize, bool relu) {
  CHECK_INPUT(src0); CHECK_INPUT(wpk); CHECK_INPUT(bias); CHECK_F32(bias);
  TORCH_CHECK(src0.dim() == 4 && src0.scalar_type() == torch::kFloat16 && wpk.dim() == 3 && wpk.scalar_type() == torch::kFloat16, "src0 [E,ht,wd,C] f16, wpk [taps,N,K] f16");
  c10::cuda::CUDAGuard guard(src0.device());
  const int E = (int)src0.size(0), ht = (int)src0.size(1), wd = (int)src0.size(2), C0 = (int)src0.size(3), N = (int)wpk.size(1);
  const void* s1 = nullptr; int C1 = 0;
  torch::Tensor s1t;
  if (src1.has_value() && src1->defined()) { s1t = *src1; CHECK_INPUT(s1t); TORCH_CHECK(s1t.scalar_type() == torch::kFloat16 && s1t.dim() == 4, "src1 [E,ht,wd,C] f16"); s1 = s1t.data_ptr(); C1 = (int)s1t.size(3); }
  TORCH_CHECK(wpk.size(0) == ksize * ksize && wpk.size(2) == 64 * ((C0 + 63) / 64) + 64 * ((C1 + 63) / 64) && bias.numel() == N, "packed weight shape mismatch");
  auto out = torch::empty({E, ht, wd, N}, src0.options());
  check_status(dba_conv_nhwc(src0.data_ptr(), C0, C0, s1, C1, C1, wpk.data_ptr(), bias.data_ptr<float>(), out.data_ptr(), N, E, ht, wd, (int)ksize, N,
                             relu ? 1 : 0, cur_stream()), "conv_nhwc");
  return out;
}

// extension: cvx_upsample of inverse depths (reference droid_net.py:21-42 via DepthVideo.upsample, depth_video.py:155-159).
// disps [n,ht,wd] f32, mask [n,576,ht,wd] f16/f32 -> [n,8ht,8wd] f32
torch::Tensor cvx_upsample(torch::Tensor disps, torch::Tensor mask) {
  CHECK_INPUT(disps); CHECK_INPUT(mask); CHECK_F32(disps);
  TORCH_CHECK(disps.dim() == 3 && mask.dim() == 4 && mask.size(0) == disps.size(0) && mask.size(1) == 576 && mask.size(2) == disps.size(1) && mask.size(3) == disps.size(2),
              "disps [n,ht,wd], mask [n,576,ht,wd]");
  c10::cuda::CUDAGuard guard(disps.device());
  const int n = (int)disps.size(0), ht = (int)disps.size(1), wd = (int)disps.size(2);
  auto out = torch::empty({n, 8 * ht, 8 * wd}, disps.options());
  check_status(dba_cvx_upsample(disps.data_ptr<float>(), mask.data_ptr(), out.data_ptr<float>(), n, ht, wd, dtype_code(mask, "cvx_upsample"), cur_stream()), "cvx_upsample");
  return out;
}

// extension (row F1): the edge selection of FactorGraph.add_proximity_factors (reference factor_graph.py:357-411) on the device.
// d [(t-t0)*(t-t1)] f32 as returned by frame_distance over the meshgrid of :351-356, ii_known / jj_known int64 = the graph's active, bad
// and inactive edges.  Returns es [n,2] int64 in the reference's emission order (one host read of the row count).
torch::Tensor proximity_edges(torch::Tensor d, int64_t t0, int64_t t1, int64_t t, torch::Tensor ii_known, torch::Tensor jj_known, int64_t rad, int64_t nms,
                              double thresh, int64_t max_factors, bool stereo) {
  CHECK_INPUT(d); CHECK_F32(d); CHECK_INPUT(ii_known); CHECK_INPUT(jj_known);
  TORCH_CHECK(ii_known.scalar_type() == torch::kInt64 && jj_known.scalar_type() == torch::kInt64 && ii_known.numel() == jj_known.numel(), "ii_known / jj_known: int64, same length");
  TORCH_CHECK(t0 >= 0 && t1 >= 0, "t0, t1 >= 0");
  c10::cuda::CUDAGuard guard(d.device());
  const int64_t n_i = std::max<int64_t>(t - t0, 0), n_j = std::max<int64_t>(t - t1, 0), n = n_i * n_j;
  TORCH_CHECK(d.numel() == n, "d must hold (t - t0) * (t - t1) distances");
  const int64_t cap = 2 * n + (3 + 2 * rad) * n_i + 2;
  auto es = torch::empty({cap, 2}, ii_known.options());
  auto hdr = torch::zeros({2}, torch::dtype(torch::kInt32).device(d.device()));
  const size_t wsb = dba_proximity_workspace_bytes((int)t0, (int)t1, (int)t);
  auto ws = torch::empty({(int64_t)wsb}, torch::dtype(torch::kUInt8).device(d.device()));
  check_status(dba_proximity_edges(d.data_ptr<float>(), (int)t0, (int)t1, (int)t, ii_known.data_ptr<int64_t>(), jj_known.data_ptr<int64_t>(), (int)ii_known.numel(), (int)rad,
                                   (int)nms, (float)thresh, (int)max_factors, stereo ? 1 : 0, es.data_ptr<int64_t>(), (int)cap, hdr.data_ptr<int>(), ws.data_ptr(), wsb,
                                   cur_stream()), "proximity_edges");
  auto h = hdr.cpu();
  const int rows = h.data_ptr<int>()[0], status = h.data_ptr<int>()[1];
  TORCH_CHECK((status & 2) == 0, "proximity_edges: index (i - t0) * (t - t1) + (j - t1) out of range (the reference raises IndexError here)");
  TORCH_CHECK((status & 1) == 0, "proximity_edges: internal capacity exceeded");
  return es.narrow(0, 0, rows);
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
  m.def("corr_lookup_pyramid", &corr_lookup_pyramid, "4-level radius-3 lookup in one launch -> [E,196,H,W], native extension", pybind11::arg("pyramid"), pybind11::arg("coords"),
        pybind11::arg("tiled") = false);
  m.def("altcorr_pyramid", &altcorr_pyramid, "AltCorrBlock pyramid in one launch -> levels [B,N,H>>l,W>>l,C] (private channels-last layout), native extension",
        pybind11::arg("fmaps"), pybind11::arg("num_levels") = 4);
  m.def("altcorr_lookup_pyramid", &altcorr_lookup_pyramid, "AltCorrBlock lookup over all levels in one launch -> [B,M,L*49,H,W], native extension",
        pybind11::arg("pyramid"), pybind11::arg("coords"), pybind11::arg("ii"), pybind11::arg("jj"), pybind11::arg("radius") = 3);
  m.def("corr_volume_supported", [](int dim, int ht, int wd, bool tiled) { return (tiled ? dba_corr_volume_tiled_supported : dba_corr_volume_supported)(dim, ht, wd, DBA_F16) != 0; },
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
  m.def("conv_nhwc", &conv_nhwc,"channels-last 1x1/3x3 convolution on wgmma, native extension");
  m.def("cvx_upsample", &cvx_upsample, "convex upsampling of inverse depth maps (droid_net.cvx_upsample, dim = 1), native extension");
  m.def("proximity_edges", &proximity_edges, "edge selection of FactorGraph.add_proximity_factors (factor_graph.py:357-411), native extension");
  m.def("_b200_native", []() { return true; });
}
