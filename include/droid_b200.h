/*
 * droid_b200.h -- C ABI of the H100-native (sm_90a) dense-BA update hot path of DROID-SLAM.
 *
 * This is the drop-in boundary: every entry point takes plain device pointers, extents, a dtype code and a
 * CUDA stream, and returns an int status (0 = ok).  No torch types cross it.  The Python extension
 * `droid_backends` (droid_slam_b200/csrc/binding/droid_backends.cpp) is a thin pybind11 layer that forwards the
 * reference's nine callables (reference src/droid.cpp:246-259) to these functions.
 *
 * All pointers are DEVICE pointers on the current CUDA device unless stated otherwise.  All tensors are dense
 * row-major ("contiguous") exactly as the reference requires (src/droid.cpp:89-90).
 * Index tensors are int64 (reference `LongType`, src/droid_kernels.cu:19-24).
 */
#ifndef DROID_B200_H
#define DROID_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* dba_stream_t; /* a cudaStream_t */

/* dtype codes for the correlation ops (reference dispatch: AT_DISPATCH_FLOATING_TYPES_AND_HALF,
 * src/correlation_kernels.cu:146, src/altcorr_kernel.cu:150; bf16 is an extension) */
enum { DBA_F32 = 0, DBA_F16 = 1, DBA_F64 = 2, DBA_BF16 = 3 };

/* status codes */
enum {
  DBA_OK = 0,
  DBA_ERR_INVALID = 1,   /* bad argument (null pointer, negative extent, unsupported dtype/radius) */
  DBA_ERR_CUDA = 2,      /* a CUDA runtime call or launch failed; see dba_last_error() */
  DBA_ERR_WORKSPACE = 3  /* workspace too small */
};

const char* dba_last_error(void);   /* thread-local, human readable */
int dba_version(void);              /* 100 * major + minor */

/* ---- correlation volume lookup ------------------------------------------------------------------
 * replaces corr_index_cuda_forward / corr_index_cuda_backward (reference src/correlation_kernels.cu:127-185,
 * bound at src/droid.cpp:175-196).
 * volume [n,h1,w1,h2,w2], coords [n,2,h1,w1] f32, corr [n,2r+1,2r+1,h1,w1] (x-offset major), dtype of volume.
 * forward fully overwrites `corr`; backward fully overwrites `volume_grad`. */
int dba_corr_index_forward(const void* volume, const float* coords, void* corr,
                           int n, int h1, int w1, int h2, int w2, int radius, int dtype, dba_stream_t stream);
int dba_corr_index_backward(const float* coords, const void* corr_grad, void* volume_grad,
                            int n, int h1, int w1, int h2, int w2, int radius, int dtype, dba_stream_t stream);

/* ---- correlation volume + pooled pyramid (tensor cores) -----------------------------------------------
 * replaces CorrBlock.__init__ / CorrBlock.corr (reference droid_slam/modules/corr.py:24-38,63-71: torch.matmul of the
 * /4-scaled feature maps + 3x avg_pool2d).  fmap1 [n_frames1,C,ht,wd], fmap2 [n_frames2,C,ht,wd] (f16, C = 128),
 * ii,jj [E] int64 frame indices into fmap1 / fmap2;  out_l [E,ht,wd,ht/2^l,wd/2^l] f16 for l = 0..3, fully overwritten.
 * One wgmma/TMA kernel writes all four levels in a single pass over the accumulator.
 * Any ht, wd >= 8 (DBA_ERR_INVALID below: the reference's avg_pool2d fails on a 1-pixel level).  Level l keeps only the complete
 * 2^l x 2^l blocks (avg_pool2d's floor rule): a trailing odd row or column is dropped at every level.  Level 0 is
 * fp16(sum_c f1 f2 / 16) from fp32 accumulators; levels 1-3 are the fp32 cascade of 2x2 means, each rounded once.
 * Checked before any launch: more than 65535 edges, null pointers, pointers not 16-byte aligned, a missing or small workspace.
 * tiled = 1: private layout, levels 0 and 1 of every plane stored as 4x8-element tiles ([h2/4][w2/8][4][8] f16 = one 64-byte DRAM atom
 * per tile) for dba_corr_lookup_pyramid(tiled_mask = 3); levels 2, 3 and all tensor shapes are unchanged.  NOT readable by
 * dba_corr_index_forward / the reference's CorrBlock.__call__.  Only for wd = 64, ht % 8 == 0 (DBA_ERR_INVALID elsewhere).
 * workspace: 16-byte aligned, at least dba_corr_volume_workspace_bytes; may be NULL when that is 0. */
/* 1 when dba_corr_volume_pyramid has a kernel for this shape / dtype / layout (f16, 128 channels, ht >= 8, wd >= 8; tiled: wd = 64,
 * ht % 8 == 0), else 0 */
int dba_corr_volume_supported(int channels, int ht, int wd, int dtype, int tiled);
/* device workspace of dba_corr_volume_pyramid: 0 when wd % 8 == 0, else a copy of both feature-map tensors with rows padded to a
 * multiple of 8 pixels (TMA global strides are multiples of 16 bytes), about 2 * 2 * C * ht * wd bytes per frame.  Read and written once
 * per call: with one frame pair per edge about 1024 * ht * wd bytes per edge, against 2.66 * (ht * wd)^2 bytes of volume written. */
size_t dba_corr_volume_workspace_bytes(int n_frames1, int n_frames2, int channels, int ht, int wd);
int dba_corr_volume_pyramid(const void* fmap1, const void* fmap2, const int64_t* ii, const int64_t* jj,
                            void* out0, void* out1, void* out2, void* out3,
                            int n_edges, int n_frames1, int n_frames2, int channels, int ht, int wd, int dtype, int tiled,
                            void* workspace, size_t workspace_bytes, dba_stream_t stream);

/* CorrBlock.__call__ (reference droid_slam/modules/corr.py:40-50) in one launch: out [n,196,h1,w1] = concatenation over the four levels
 * of corr_index_forward(volume_l, coords / 2^l, 3) -- bit-identical values; coords [n,2,h1,w1] f32 at level-0 scale are read once.
 * f16 or f32 volumes, h1, w1 >= 8, planes of level l [h1 >> l, w1 >> l], each level tensor 16-byte aligned; no load leaves a level tensor.
 * tiled_mask: 0 = reference layout, 3 = levels 0 and 1 in the tiled layout above (f16, h1 % 8 == 0 and w1 % 64 == 0 only). */
int dba_corr_lookup_pyramid(const void* v0, const void* v1, const void* v2, const void* v3, const float* coords, void* out,
                            int n, int h1, int w1, int tiled_mask, int dtype, dba_stream_t stream);

/* ---- CorrBlock for training (fp32 feature maps, forward and backward) ------------------------------------------------------------
 * DroidNet.forward's CorrBlock(fmaps[:,ii], fmaps[:,jj]) (reference droid_slam/modules/corr.py:6-71) with train.py's fp32 maps.
 * fmap1, fmap2 [n,128,ht,wd] f32, one map pair per edge; ht, wd >= 8; n <= 65535.  Products on the tf32 tensor cores with 3xTF32 splitting
 * (fp32-level accuracy), fixed summation order, no host synchronisation.
 * dba_corr_volume_pyramid_f32: out_l [n,ht,wd,ht>>l,wd>>l] (reference layout), out_0 = (f1/4)^T (f2/4), out_{l+1} = 2x2 mean of out_l over
 *   complete blocks.  Readable by dba_corr_lookup_pyramid(dtype DBA_F32) and dba_corr_index_forward.
 * The gradient pyramid: gpyr [n][ht*wd][Q] f32, Q = sum_l (ht>>l)(wd>>l); row p holds the gradient of source pixel p's plane of each level,
 *   level 0 first.  The caller zeroes it once per backward pass.
 * dba_corr_grad_accumulate: adds the gradient of one lookup -- grad [n,196,ht,wd] of dba_corr_lookup_pyramid's output at coords [n,2,ht,wd]
 *   -- into gpyr.  One thread owns each row: no atomics, the same bits every run.
 * dba_corr_adjoint: grad1 = sum_l G_l P_l(f2) / 16, grad2 = sum_l P_l^T (G_l^T f1) / 16 into [n,128,ht,wd] (fully overwritten), P_l the
 *   2^l block mean (floor rule).  workspace: 16-byte aligned, at least dba_corr_adjoint_workspace_bytes. */
int dba_corr_volume_pyramid_f32(const float* fmap1, const float* fmap2, float* out0, float* out1, float* out2, float* out3, int n,
                                int channels, int ht, int wd, dba_stream_t stream);
int dba_corr_grad_accumulate(const float* coords, const float* grad, float* gpyr, int n, int ht, int wd, dba_stream_t stream);
size_t dba_corr_adjoint_workspace_bytes(int n, int channels, int ht, int wd);
int dba_corr_adjoint(const float* fmap1, const float* fmap2, const float* gpyr, float* grad1, float* grad2, int n, int channels, int ht,
                     int wd, void* workspace, size_t workspace_bytes, dba_stream_t stream);

/* ---- on-the-fly correlation ---------------------------------------------------------------------
 * replaces altcorr_cuda_forward / altcorr_cuda_backward (reference src/altcorr_kernel.cu:132-225, bound at
 * src/droid.cpp:198-226).
 * fmap1 [B,N1,C,H,W], fmap2 [B,N2,C,H2,W2], coords [B,M,2,H,W] f32, ii,jj [M] int64 (frame indices into
 * fmap1 / fmap2).  forward writes `out` as a CONTIGUOUS [B,M,2r+1(y-off),2r+1(x-off),H,W] tensor; the binding
 * returns its permute(0,1,3,2,4,5) view like the reference (:171).
 * backward consumes corr_grad [B,M,2r+1(x-off),2r+1(y-off),H,W] f32 -- the gradient of the returned (permuted)
 * tensor, as the reference host function does (:175-207) -- and fully overwrites fmap1_grad / fmap2_grad. */
int dba_altcorr_forward(const void* fmap1, const void* fmap2, const float* coords,
                        const int64_t* ii, const int64_t* jj, void* out,
                        int B, int N1, int N2, int C, int H, int W, int H2, int W2, int M,
                        int radius, int dtype, dba_stream_t stream);
int dba_altcorr_backward(const void* fmap1, const void* fmap2, const float* coords, const float* corr_grad,
                         const int64_t* ii, const int64_t* jj, void* fmap1_grad, void* fmap2_grad,
                         int B, int N1, int N2, int C, int H, int W, int H2, int W2, int M,
                         int radius, int dtype, dba_stream_t stream);

/* ---- AltCorrBlock on a private channels-last pyramid ----------------------------------------------------------
 * replaces AltCorrBlock.__init__ / __call__ (reference droid_slam/modules/corr.py:89-117: 3x avg_pool2d, then per level
 * altcorr_forward + flatten + stack).  Shapes: f16 or f32, C % 8 == 0, 1 <= levels <= 4, H, W >= 2^(levels-1), radius 3;
 * extents as for dba_altcorr_forward.  An empty batch (B, N or M zero) returns 0 without a launch; no host synchronisation.
 *
 * dba_altcorr_pyramid: fmaps [B,N,C,H,W] -> out_l [B,N,H>>l,W>>l,C] (channels last) for l < levels; out_l for l >= levels may be NULL.
 *   PRIVATE LAYOUT: element (b,n,y,x,c) of out_l holds (reference level l)[b,n,c,y,x] / 4 rounded to the dtype, reference level l+1
 *   being F.avg_pool2d(level l, 2, stride=2) of the rounded level l (fp32 sum of the 2x2 window, / 4, rounded; floor sizes).  The /4
 *   is the scaling the reference applies to both operands of every product (src/altcorr_kernel.cu:67-68).  NOT readable by
 *   dba_altcorr_forward / the reference's CorrLayer; level 0 is a copy, so the pyramid takes about 1.33x the feature maps.
 * dba_altcorr_lookup_pyramid: p_l = the pyramid above; coords [B,M,2,H,W] f32 at level-0 scale; ii,jj [M] int64 frame indices
 *   (source, target); out [B,M,levels*49,H,W], channel l*49 + xo*7 + yo = the reference's
 *   stack([altcorr_forward(level 0, level l, coords / 2^l, ii, jj, 3).flatten(2,3) for l], 2).flatten(2,3), bit for bit. */
int dba_altcorr_pyramid(const void* fmaps, void* out0, void* out1, void* out2, void* out3,
                        int B, int N, int C, int H, int W, int levels, int dtype, dba_stream_t stream);
int dba_altcorr_lookup_pyramid(const void* p0, const void* p1, const void* p2, const void* p3, const float* coords,
                               const int64_t* ii, const int64_t* jj, void* out,
                               int B, int N, int C, int H, int W, int M, int levels, int radius, int dtype, dba_stream_t stream);

/* ---- streaming geometry -------------------------------------------------------------------------
 * poses [n_poses,7] (tx,ty,tz,qx,qy,qz,qw) f32, disps [n_disps,ht,wd] f32, intrinsics [4] f32 (fx,fy,cx,cy).
 * replace projmap_cuda / frame_distance_cuda / depth_filter_cuda / iproj_cuda
 * (reference src/droid_kernels.cu:1447-1550, bound at src/droid.cpp:125-171,228-242). */
int dba_projmap(const float* poses, const float* disps, const float* intrinsics,
                const int64_t* ii, const int64_t* jj, float* coords /*[E,ht,wd,3]*/, float* valid /*[E,ht,wd,1]*/,
                int n_edges, int ht, int wd, dba_stream_t stream);
/* fused reprojection feeding the update operator: replaces pops.projective_transform(jacobian=False)
 * (reference droid_slam/geom/projective_ops.py:165-198 via DepthVideo.reproject, depth_video.py:171-179).
 * intrinsics_per_frame [n_frames,4]; coords [E,ht,wd,2], valid [E,ht,wd,1]; MIN_DEPTH 0.2, stereo baseline for ii == jj. */
int dba_reproject(const float* poses, const float* disps, const float* intrinsics_per_frame,
                  const int64_t* ii, const int64_t* jj, float* coords, float* valid, int n_edges, int ht, int wd, dba_stream_t stream);

/* ---- factor-graph step (FactorGraph.update / update_lowmem, reference droid_slam/factor_graph.py:214-330) -----------------
 * Call row r stands for graph edge e = edge_index[r] (edge_index null: e = r); indices are not range-checked.
 * dba_motion_features: the reprojection of dba_reproject (same device code, bit-identical coords) of edge (ii[e], jj[e]) fused with the
 * motion features (:220-222, :280-282).  target [E,ht,wd,2] (the graph's); outputs per call row: coords [n,ht,wd,2],
 * coords_t [n,2,ht,wd] (the layout dba_corr_lookup_pyramid / dba_altcorr_lookup_pyramid take), motn [n,4,ht,wd] =
 * clamp(coords - (x,y), +-64), clamp(target - coords, +-64) in fp32; NaN stays NaN like torch.clamp. */
int dba_motion_features(const float* poses, const float* disps, const float* intrinsics_per_frame, const int64_t* ii, const int64_t* jj,
                        const int64_t* edge_index, const float* target, float* coords, float* coords_t, float* motn,
                        int n_rows, int ht, int wd, dba_stream_t stream);
/* dba_graph_writeback: the update operator's delta / weight [n,ht,wd,2] for call rows whose coordinates are coords [n,ht,wd,2] go back
 * to the graph: target[e] = coords + delta and weight_out[e] = weight ([E,ht,wd,2]), and the same values to BA's channel-major inputs
 * ba_target / ba_weight [E_ba,2,ht,wd] at row n_inactive + e (inactive edges first, then graph order, as the reference concatenates).
 * damping [n_frames,ht,wd]: damping[src_frames[m]] = eta[m] for m < n_src (eta [n_src,ht,wd]).  Then, if n_ba_frames > 0 (after that
 * scatter, stream-ordered): ba_damping[r] = .2f * damping[ba_frames[r]] + ep, two roundings (:251, :320). */
int dba_graph_writeback(const float* delta, const float* weight, const float* coords, const int64_t* edge_index, int n_rows,
                        float* target, float* weight_out, float* ba_target, float* ba_weight, int n_inactive,
                        const float* eta, const int64_t* src_frames, int n_src, float* damping,
                        const int64_t* ba_frames, int n_ba_frames, float* ba_damping, float ep, int ht, int wd, dba_stream_t stream);

int dba_frame_distance(const float* poses, const float* disps, const float* intrinsics,
                       const int64_t* ii, const int64_t* jj, float* dist /*[K]*/,
                       int n_pairs, int ht, int wd, float beta, dba_stream_t stream);
int dba_depth_filter(const float* poses, const float* disps, const float* intrinsics,
                     const int64_t* ix, const float* thresh, float* counter /*[num,ht,wd]*/,
                     int num, int n_disps, int ht, int wd, dba_stream_t stream);
int dba_iproj(const float* poses, const float* disps, const float* intrinsics, float* points /*[n,ht,wd,3]*/,
              int n, int ht, int wd, dba_stream_t stream);

/* convex upsampling of inverse depth maps: replaces cvx_upsample / upsample_disp (reference droid_slam/droid_net.py:21-42) as called by
 * DepthVideo.upsample (depth_video.py:155-159).  disps [n,ht,wd] f32, mask [n,576,ht,wd] (f16 or f32; 9 taps x 8 x 8 sub-pixels, the
 * update operator's `upmask`), out [n,8*ht,8*wd] f32 = softmax-over-taps weighted sum of the 3x3 neighbourhood (zero padded). */
int dba_cvx_upsample(const float* disps, const void* mask, float* out, int n, int ht, int wd, int mask_dtype, dba_stream_t stream);

/* ---- factor-graph edge selection (row F1) --------------------------------------------------------
 * replaces the body of FactorGraph.add_proximity_factors between `video.distance(...)` and `add_factors(...)` (reference
 * droid_slam/factor_graph.py:357-411: masking, suppression around the edges the graph already has, temporal-neighbour edges, then the
 * greedy selection by increasing distance with non-maximum suppression -- a Python / NumPy triple loop on a CPU copy of d).
 * d [(t-t0)*(t-t1)] f32: frame distances over the grid i in [t0,t), j in [t1,t), row-major (what dba_frame_distance returns for the
 * meshgrid of factor_graph.py:351-356), read only.  ii_known / jj_known [n_known] int64: cat(ii, ii_bad, ii_inac) / cat(jj, ...).
 * es [cap][2] int64 receives the (i, j) rows in the reference's emission order; n_out_status [2] int32 on the device: [0] rows written,
 * [1] status (bit 0: cap too small, bit 1: the reference's unchecked index d[(i-t0)*(t-t1) + (j-t1)] left the array, where it raises
 * IndexError).  cap >= 2*n + (1+2*(rad+1))*(t-t0) always suffices.  Equal finite distances are visited in index order (torch.argsort
 * gives no order for ties).  No host synchronisation. */
size_t dba_proximity_workspace_bytes(int t0, int t1, int t);
int dba_proximity_edges(const float* d, int t0, int t1, int t, const int64_t* ii_known, const int64_t* jj_known, int n_known, int rad, int nms,
                        float thresh, int max_factors, int stereo, int64_t* es, int cap, int* n_out_status, void* workspace, size_t workspace_bytes,
                        dba_stream_t stream);

/* ---- dense bundle adjustment --------------------------------------------------------------------
 * replaces ba_cuda (reference src/droid_kernels.cu:1323-1443, bound at src/droid.cpp:93-122).
 * In place on poses [n_frames,7] and disps [n_frames,ht,wd]; disps_sens like disps; targets, weights
 * [E,2,ht,wd]; eta [M,ht,wd] with M = |unique(ii U [t0,t1))| rows in ascending frame order (or 1 row,
 * broadcast); ii,jj [E] int64.  Outputs of the LAST Gauss-Newton iteration: dx_out [t1-t0,6], dz_out [M,ht*wd]
 * (dz_out untouched when motion_only).  Everything runs on `stream` with no host synchronisation.
 * An empty window (t0 == t1) has no pose system; unless motion_only, the inverse depths still take dz = Q w (dx = 0).
 *
 * The call is split at the one point where a multi-GPU run exchanges data:
 *   dba_ba_prepare   graph bookkeeping (unique / CSR by source frame), once per call
 *   dba_ba_build     per-edge blocks + depth elimination -> reduced pose system  Hsys [6P,6P] f64 (LOWER triangle valid),
 *                    bsys [6P] f64 (edge-sharded runs all-reduce exactly this buffer, 8*(36P^2+6P) bytes)
 *   dba_ba_solve     damping + Cholesky (fp64) -> dx, back-substitution -> dz, retraction of poses and disps
 * dba_ba runs prepare + iterations x (build, solve).
 * workspace: dba_ba_workspace_bytes(); layout is private, the reduced system sits at dba_ba_system_offset(). */
size_t dba_ba_workspace_bytes(int n_frames, int n_edges, int ht, int wd, int t0, int t1);
size_t dba_ba_system_offset(int n_frames, int n_edges, int ht, int wd, int t0, int t1);  /* bytes from workspace start */
size_t dba_ba_system_bytes(int t0, int t1);                                              /* 8*(36P^2+6P) */

typedef struct {
  float* poses; float* disps; const float* intrinsics; const float* disps_sens;
  const float* targets; const float* weights; const float* eta; int eta_rows;
  const int64_t* ii; const int64_t* jj;
  int n_frames, n_edges, ht, wd, t0, t1;
  float lm, ep; int motion_only;
  float* dx_out; float* dz_out;
  void* workspace; size_t workspace_bytes;
  dba_stream_t stream;
  /* edge-sharded multi-GPU runs (one rank = the out-edges of a contiguous range of source frames):
   * only depth frames in [own_lo, own_hi) get their inverse depth updated by dba_ba_solve (the other ranks own the
   * rest); single-GPU callers pass own_lo = 0, own_hi = n_frames.  eta_by_frame != 0: eta has n_frames rows indexed by
   * FRAME id instead of M rows in depth-frame order (a rank's local depth-frame set differs from the global one). */
  int own_lo, own_hi, eta_by_frame;
  /* optional fused peer-to-peer reduction of the pose system over NVLink peer memory (p2p_world > 1), replacing the separate
   * all-reduce: the rank accumulates its partial system in p2p_system[p2p_rank] (slot p2p_epoch & 1 of two, each 36P^2+6P
   * doubles; 8 uint64 flags follow the two slots), dba_ba_p2p_signal() publishes it with release stores into every peer's
   * flags[p2p_rank], and the Cholesky kernel of dba_ba_solve waits for the W flags and sums the W peer copies in rank order
   * (bit-identical on every rank) straight out of peer memory.  p2p_system[] are peer-mapped device pointers (e.g. from
   * torch.distributed._symmetric_memory); p2p_epoch must increase by one per Gauss-Newton iteration on every rank.
   * p2p_epoch_dev (optional, rank-local device memory, zero-initialised once): when set, the published / awaited epoch VALUE is
   * this device counter (dba_ba_p2p_signal increments it on the stream), so the whole iteration can be captured in a CUDA graph
   * and replayed; p2p_epoch then only selects the slot, and a captured graph must hold an even number of iterations. */
  int p2p_world, p2p_rank;
  unsigned long long p2p_epoch;
  void* p2p_system[8];
  unsigned long long* p2p_epoch_dev;
} dba_ba_args;

int dba_ba_prepare(const dba_ba_args* a);
int dba_ba_build(const dba_ba_args* a);
int dba_ba_solve(const dba_ba_args* a);
int dba_ba(const dba_ba_args* a, int iterations);
int dba_ba_p2p_signal(const dba_ba_args* a);   /* after dba_ba_build, before dba_ba_solve, when p2p_world > 1 */
/* synchronises `stream` and reads back M = number of depth frames found by the last dba_ba_prepare on this
 * workspace and the sticky device status word (0 = ok, bit0 = index out of range, bit1 = eta rows != M,
 * bit2 = Cholesky hit a non-positive pivot in some iteration -> that iteration's dx = 0 like the reference,
 * bit3 = a source frame has more than 254 out-edges and motion_only == 0: its Schur complement would be truncated, the result is
 * not usable; dba_ba_prepare already sets it, so a caller can check before the first dba_ba_build changes any state). */
int dba_ba_read_info(const dba_ba_args* a, int* n_depth_frames, int* device_status);

/* ---- non-keyframe pose filling (PoseTrajectoryFiller, reference droid_slam/trajectory_filler.py) -----------------------
 * dba_fill_interpolate: the linear pose interpolation of `__fill` (:51-65), one thread per frame.  poses [n_keyframes,7], tstamps
 * [n_keyframes] f32 (any order), t [n] f32 -> t0_out / t1_out [n] int64, poses_out [n,7]:  t0 = #{k : tstamps[k] <= t} - 1,
 * t1 = t0 + 1 if t0 < n_keyframes - 1 else t0, dt = tstamps[t1] - tstamps[t0] + 1e-3,
 * G = Exp(Log(P[t1] P[t0]^-1) / dt * (t - tstamps[t0])) P[t0] with lietorch's SE3 formulas in fp32.  t0 = -1 (t before every keyframe) is
 * written as is; index -1 then reads keyframe n_keyframes - 1, like Python's negative indexing in the reference.  n_keyframes >= 1.
 * dba_pose_only_ba: `iterations` Gauss-Newton iterations of motion-only BA (dba_ba with motion_only = 1) in one launch, for graphs whose
 * every edge goes from a fixed frame to one optimised frame: 0 <= ii < min(t0, n_disps), t0 <= jj < t1.  The pose system is then block
 * diagonal: per optimised frame the Hjj / vj sums of its edges (ascending edge order, fp64 across warps and edges, no atomics: bit-
 * reproducible whatever other frames share the call), damping diag += ep + lm * diag, a 6x6 fp64 Cholesky, poses <- Exp(dx) poses.
 * poses [n_frames,7] (rows [t0,t1) updated in place), disps [n_disps,ht,wd], intrinsics [4] (the single camera of dba_ba), targets /
 * weights [E,2,ht,wd], ii / jj [E] int64.  status: device int32 [1], overwritten: bit 0 = an edge breaks the structure above (checked by
 * a first launch; no pose changes), bit 1 = some frame's damped block was not positive definite (its dx = 0 in that iteration; dba_ba
 * zeroes the whole window's update instead).  Optional outputs of the last iteration (may be NULL): sys_out [t1-t0][42] f64 = the
 * undamped block H (6x6 row-major) and b (6), dx_out [t1-t0][6].  No host synchronisation. */
int dba_fill_interpolate(const float* poses, const float* tstamps, int n_keyframes, const float* t, int n, int64_t* t0_out,
                         int64_t* t1_out, float* poses_out, dba_stream_t stream);
int dba_pose_only_ba(float* poses, const float* disps, const float* intrinsics, const float* targets, const float* weights,
                     const int64_t* ii, const int64_t* jj, int n_frames, int n_disps, int n_edges, int ht, int wd, int t0, int t1,
                     int iterations, float lm, float ep, int* status, double* sys_out, float* dx_out, dba_stream_t stream);

/* ---- DroidAsync fragment hand-over (reference droid_slam/droid_async.py:54-119, droid_slam/align.py) -----------------------
 * One backend round's hand-over of the frontend's keyframes [t0,t1) to the backend's video, on the backend's device, in two launches and
 * without a host synchronisation.  The caller first copies the frontend's poses[t0:t1] and disps[t0:t1] into poses2 / disps2 rows [t0,t1)
 * and, when t0 > 0, the frontend's poses[t0-10:t0-1] into poses1_align [9,7].  Then:
 *   launch 1 (one CTA per slice of disps_sens1; the first one also aligns): any = any(disps_sens1 != 0) per slice, and when t0 > 0
 *     (dG, s) = align_pose_fragements(poses1_align, poses2[t0-10:t0-1]) in fp64 from the fp32 poses: the 81 relative translations,
 *     s = sum(dt1 . dt2) / sum(dt1 . dt1), dG from the s-scaled frontend poses with 3 log-mean-exp refinements; t0 == 0: dG = identity,
 *     s = 1.
 *   launch 2 (one CTA per frame and 1024-pixel chunk): align_scale = !stereo && !any; s_eff = align_scale ? s : 1 -- dG stays the one
 *     computed from the s-scaled poses even when s is discarded, as the reference does; with s_f = (float)s_eff,
 *     poses2[f] = dG * (poses2[f] with its translation * s_f in fp32), composed in fp64 and rounded once, and disps2[f] /= s_f (fp32
 *     division), for t0 <= f < t1.
 * poses2 [>= t1, 7] f32, disps2 [>= t1, hw] f32, disps_sens1: the frontend's whole disps_sens buffer (n_sens floats) readable from this
 * device (the reference's torch.any spans the whole buffer).  Contract: t0 == 0 or t0 >= 10 -- what the reference's backend_process
 * produces (t0 = counter2 - 2, counter2 being 0 in the first round and at least 28 after it); other t0 are rejected (the reference's
 * Python slices would wrap at negative starts; that is not reproduced).  t1 <= t0 re-anchors nothing (an empty slice in the reference).
 * workspace: DBA_HANDOVER_WORKSPACE_BYTES bytes of device memory, 8-byte aligned, no initialisation needed.  diagnostics (may be NULL):
 * double [9] = s_eff, dG (tx,ty,tz,qx,qy,qz,qw), align_scale (0 / 1). */
#define DBA_HANDOVER_WORKSPACE_BYTES 4096
int dba_fragment_handover(const float* poses1_align, float* poses2, float* disps2, const float* disps_sens1, long long n_sens, int t0, int t1,
                          int hw, int stereo, void* workspace, double* diagnostics, dba_stream_t stream);

/* ---- update operator (ConvGRU + heads + GraphAgg) on the tensor cores -----------------------------------
 * replaces UpdateModule.forward (reference droid_slam/droid_net.py:111-143), ConvGRU.forward (droid_slam/modules/gru.py:19-32) and
 * GraphAgg.forward (droid_net.py:59-75) -- in the reference a chain of 19 cuDNN convolutions + ~25 elementwise launches.
 * Every convolution runs as an implicit GEMM (wgmma / TMA, f16 operands, fp32 accumulation) on channels-last
 * activations; gates, activations, the global-context sum and output layouts are fused into the epilogues.  Any ht, wd > 0: widths
 * that are not a multiple of 8 (e.g. 69, 70, 73 at 1/8 of the reference's demo / ETH3D image sizes) run row-flattened tiles.
 *
 * Packed weights (device memory, made once per checkpoint by the host side, droid_slam_b200/update.py:pack_update_weights):
 *   w_* : f16 [taps][N][Kpad]  (tap = dy*k + dx, K = input channels in the reference's concatenation order, zero padded to a
 *         multiple of 64), b_* : f32 [N]
 *   w_corr0 [1][128][256]  corr_encoder.0 (196 in)        w_corr2 [9][128][128] corr_encoder.2
 *   w_flow0 [1][128][256]  flow_encoder.0, K = (dy*7+dx)*4 + c (7x7 taps folded into K)     w_flow2 [9][64][128] flow_encoder.2
 *   w_gate  [1][128][128]  gru.w          w_glo f32 [384][128] = gru.convz_glo | convr_glo | convq_glo, b_glo [384]
 *   w_zr    [9][256][448]  gru.convz | gru.convr         w_q [9][128][448] gru.convq
 *   w_stem  [9][384][128]  delta.0 | weight.0 | agg.conv1
 *   w_heads [1][64][256]   per-tap rows: row 4t+o (t = 3 dy + dx) = tap t of delta.2 (o = 0,1; K 0..127) / weight.2 (o = 2,3; K 128..255),
 *                          rows 36..63 zero -- the 3x3 / 2-channel heads run as one 1x1 convolution + a 9-tap gather;  b_heads [4]
 *   w_agg2  [9][128][128]  agg.conv2      w_eta [1][32][128] row t = tap t of agg.eta.0, b_eta [1]      w_upmask [1][576][128] agg.upmask.0
 *   b_zero  f32 [64] zeros (bias of the per-tap partial-sum convolutions) */
typedef struct {
  const void *w_corr0, *w_corr2, *w_flow0, *w_flow2, *w_gate, *w_zr, *w_q, *w_stem, *w_heads, *w_agg2, *w_eta, *w_upmask;
  const float *b_corr0, *b_corr2, *b_flow0, *b_flow2, *b_gate, *b_zr, *b_q, *b_stem, *b_heads, *b_agg2, *b_eta, *b_upmask;
  const float *w_glo, *b_glo, *b_zero;
} dba_update_weights;

typedef struct {
  int n_edges, ht, wd;
  const void* net;  int net_dtype;  int net_layout;   /* hidden state [E,128,ht,wd] (layout 0, DBA_F16 / DBA_F32) or channels-last f16 [E,ht,wd,128] (layout 1) */
  const void* inp;  int inp_dtype;                     /* context features [E,128,ht,wd] */
  const void* corr; int corr_dtype;                    /* correlation features [E,196,ht,wd] */
  const float* flow;                                   /* motion features [E,4,ht,wd] f32, or NULL (= zeros, MotionFilter's call) */
  const int64_t* seg; int n_src;                       /* seg[e] = rank of edge e's source frame among the distinct sources (torch.unique
                                                          inverse); n_src = number of distinct sources; n_src = 0: no aggregation outputs */
  const dba_update_weights* weights;                   /* HOST struct of DEVICE pointers */
  void* net_out;                                       /* new hidden state, channels-last f16 [E,ht,wd,128] */
  float* delta;  float* weight;                        /* [E,ht,wd,2] f32: flow revision, confidence (sigmoid) */
  float* eta;    void* upmask;                         /* [n_src,ht,wd] f32 (0.01 * softplus), [n_src,576,ht,wd] f16 */
  void* workspace; size_t workspace_bytes;             /* dba_update_workspace_bytes(), 256-byte aligned */
  dba_stream_t stream;
} dba_update_args;

size_t dba_update_workspace_bytes(int n_edges, int n_src, int ht, int wd);
int dba_update_forward(const dba_update_args* a);

/* host only: where dba_update_forward leaves its intermediates in the workspace, from the layout it uses itself (for tests that
 * check each stage on the inputs the previous one wrote).  offsets[DBA_UPWS_COUNT] = byte offsets from the workspace start of:
 *   HIN  f16 [E,HW,128]  hidden state, channels-last (written for net_layout 0 only)
 *   X320 f16 [E,HW,320]  inp | corr encoder | flow encoder          CC   f16 [E,HW,200]  corr, channels-last (196 used)
 *   F0   f16 [E,HW,200]  7x7 im2col of flow (196 used)               C1, F1 f16 [E,HW,128]  first corr / flow encoder layers
 *   Z, RH f16 [E,HW,128] GRU z and r*h                               S    f16 [E,HW,384]  stems delta.0 | weight.0 | agg.conv1
 *   PARTIAL f32 [E,gate_slots,128]  sums of sigmoid(gru.w(h)) * h over 16-pixel slots            GLO f32 [E,384]  z | r | q terms
 *   AM, B2 f16 [n_src,HW,128]  segment mean of agg.conv1, agg.conv2
 *   YH f32 [E,HW,36]   per-tap partials of delta.2 / weight.2 (reuses CC)    YE f32 [n_src,HW,12]  of agg.eta.0, 9 used (reuses F0)
 * *gate_slots = the partial-sum slots glo_kernel adds per edge.  DBA_ERR_INVALID for extents dba_update_forward rejects. */
enum { DBA_UPWS_HIN, DBA_UPWS_X320, DBA_UPWS_CC, DBA_UPWS_F0, DBA_UPWS_C1, DBA_UPWS_F1, DBA_UPWS_Z, DBA_UPWS_RH, DBA_UPWS_S,
       DBA_UPWS_PARTIAL, DBA_UPWS_GLO, DBA_UPWS_AM, DBA_UPWS_B2, DBA_UPWS_YH, DBA_UPWS_YE, DBA_UPWS_COUNT };
int dba_update_workspace_layout(int n_edges, int n_src, int ht, int wd, size_t* offsets, int* gate_slots);

/* the building block of dba_update_forward, exported: 1x1 / 3x3 'same' convolution of channels-last f16 activations on the tensor
 * cores.  src0 (+ optional src1, concatenated along channels after src0) [n_images,ht,wd,stride] using channels [0,c); wpk f16
 * [ksize*ksize][n_out][Kpad] with Kpad = 64*ceil(c0/64) + 64*ceil(c1/64), K contiguous; bias f32 [n_out]; out f16
 * [n_images,ht,wd,out_stride] channels [0,n_out) written.  n_out in {32,64,...,256,384}; any ht, wd > 0, tiled as in
 * dba_update_forward. */
int dba_conv_nhwc(const void* src0, int c0, int stride0, const void* src1, int c1, int stride1, const void* wpk, const float* bias,
                  void* out, int out_stride, int n_images, int ht, int wd, int ksize, int n_out, int relu, dba_stream_t stream);
/* host only: the tiling dba_conv_nhwc launches for these extents (c1 = 0: no second source), computed by the same code.
 * plan [8] = {row-flattened tiles (0 / 1), TW (tile width, or the row pitch of row-flattened tiles), MT (128-pixel M tiles per CTA
 * tile), N tile width, number of N tiles, CTA tiles per image, halo stages, weight stages}.  DBA_ERR_INVALID for extents
 * dba_conv_nhwc rejects. */
int dba_conv_nhwc_plan(int ht, int wd, int c0, int c1, int ksize, int n_out, int* plan);

/* ---- feature / context encoders (BasicEncoder) on the tensor cores ---------------------------------------------------
 * replaces BasicEncoder.forward (reference droid_slam/modules/extractor.py:183-198) for the two encoders DroidNet builds
 * (droid_net.py:149-150): fnet = BasicEncoder(output_dim=128, norm_fn='instance') and cnet = BasicEncoder(output_dim=256,
 * norm_fn='none'), dropout 0, multidim False.  images [n_images,3,H,W] DBA_F32 or DBA_F16 (rounded to f16 on load, the cast autocast
 * applies), H and W positive multiples of 8; out [n_images,output_dim,H/8,W/8] f16, fully overwritten.  Instance norm: per image and
 * channel, biased variance, eps 1e-5, no affine parameters.  Never synchronises the host; can be captured in a CUDA graph.
 *
 * Packed weights (device memory, made once per checkpoint by droid_slam_b200/encoder.py:pack_encoder_weights), w[k] f16 [taps][N][Kpad]
 * (tap = dy*k + dx, K contiguous and zero padded to a multiple of 64), b[k] f32 [N]:
 *   k = 0       conv1 7x7/2 3->32           [1][32][192]    K = (dy*7 + dx)*3 + c (the 147 taps of the stride-2 window)
 *   k = 1..4    layer1.{0,1}.{conv1,conv2}  [9][32][64]
 *   k = 5       layer2.0.conv1 | downsample [1][128][320]   K = (dy*3 + dx)*32 + c (the 3x3/2 taps gathered at output resolution);
 *                                                           rows 0..63 conv1, rows 64..127 downsample.0 in the centre-tap rows K 128..159
 *   k = 6..8    layer2.0.conv2, layer2.1.{conv1,conv2}       [9][64][64]
 *   k = 9       layer3.0.conv1 | downsample [1][256][576]   K = (dy*3 + dx)*64 + c; rows 128..255 downsample.0 in K 256..319
 *   k = 10..12  layer3.0.conv2, layer3.1.{conv1,conv2}       [9][128][128]
 *   k = 13      conv2 1x1 128->output_dim   [1][output_dim][128] */
#define DBA_ENCODER_CONVS 14
typedef struct {
  const void* w[DBA_ENCODER_CONVS];
  const float* b[DBA_ENCODER_CONVS];
} dba_encoder_weights;

typedef struct {
  const void* images; int images_dtype;                /* [n_images,3,H,W], DBA_F32 or DBA_F16 */
  int n_images, H, W;
  const dba_encoder_weights* weights;                  /* HOST struct of DEVICE pointers */
  int norm;                                            /* 0 = none (cnet), 1 = instance (fnet) */
  int output_dim;                                      /* 128 or 256 */
  void* out;                                           /* [n_images,output_dim,H/8,W/8] f16 */
  void* workspace; size_t workspace_bytes;             /* dba_encoder_workspace_bytes(), 256-byte aligned */
  dba_stream_t stream;
} dba_encoder_args;

/* 0 for extents without a kernel (n_images < 1, H or W not a positive multiple of 8, output_dim not 128 or 256) */
size_t dba_encoder_workspace_bytes(int n_images, int H, int W, int output_dim);
int dba_encoder_forward(const dba_encoder_args* a);

/* camera frames straight into the encoders: dba_encoder_forward on a->images = uint8 frames [n_images,3,H,W] in the format's channel
 * order (a->images_dtype is ignored).  Each tap is reordered to RGB and normalised in fp32 as the reference's ATen sequence on CUDA does
 * it (motion_filter.py:62-63: x / 255.0, .sub_(MEAN), .div_(STDV)): x * (1.0f / 255.0f), then - mean[c], then an IEEE division by
 * std[c], each step rounded to fp32, c the RGB channel; then rounded to f16 like the DBA_F32 path.  The output equals
 * dba_encoder_forward on the normalised fp32 frames bit for bit; the fp32 frames are never stored.  Same workspace. */
enum { DBA_FRAME_RGB = 0, DBA_FRAME_BGR = 1 };
typedef struct {
  int channel_order;                                   /* DBA_FRAME_RGB, or DBA_FRAME_BGR (reversed to RGB on load) */
  float mean[3], std[3];                               /* per RGB channel */
} dba_frame_format;
int dba_encoder_forward_frames(const dba_encoder_args* a, const dba_frame_format* f);

/* host only: where dba_encoder_forward keeps its intermediates, from the layout and the schedule it uses itself (for tests that check
 * each launch on what the previous one wrote).  offsets / sizes [DBA_ENCWS_COUNT]: byte offset from the workspace start and size of
 *   BIG  f16  the im2col rows [n,H/2,W/2,152] (147 used), then the gathered 3x3/2 taps [n,h/2,w/2,9C] of layer2.0 and layer3.0
 *   X, T1, T2 f16 channels-last activations [n,h,w,C]: X a block's input and output, T1 / T2 its scratch (T1 [.,2P] = conv1 |
 *        downsample in the stride-2 blocks)
 *   PARTIAL f32 [n,slots,N,2] (mean, M2) per 16-pixel slot of the last statistics convolution, COUNTS f32 [n,slots] its valid pixels
 *   MSA, MSB f32 [n,N,2] (mean, rstd) per image and channel
 * *n_launches = kernels dba_encoder_forward launches; plans [DBA_ENCODER_CONVS][5] = per convolution k the tile width TW, the M tiles
 * per CTA tile MT, CTA tiles per image along x and y, and the slots its statistics use per image (0 where it takes none: every
 * convolution of norm 0, conv2 of norm 1).  DBA_ERR_INVALID for extents dba_encoder_forward rejects. */
enum { DBA_ENCWS_BIG, DBA_ENCWS_X, DBA_ENCWS_T1, DBA_ENCWS_T2, DBA_ENCWS_PARTIAL, DBA_ENCWS_COUNTS, DBA_ENCWS_MSA, DBA_ENCWS_MSB, DBA_ENCWS_COUNT };
int dba_encoder_workspace_layout(int n_images, int H, int W, int norm, size_t* offsets, size_t* sizes, int* n_launches, int* plans);
/* dba_encoder_forward stopped after its first n_launches kernels (the same schedule; out is written by the last one only) */
int dba_encoder_forward_prefix(const dba_encoder_args* a, int n_launches);

/* ---- standalone damped SPD solve (the solver inside dba_ba_solve) ---------------------------------------
 * (H + diag(ep + lm*diag(H))) x = b with H [n,n] fp64 (symmetric; only its lower triangle is read), b [n] fp64 -> x [n] fp32,
 * on the device in fp64; replaces SparseBlock::solve (reference src/droid_kernels.cu:1201-1222).  *fail_flag_device is set to 1
 * and x to 0 when a pivot is not positive and finite (reference: solver.info() != Eigen::Success).
 * On return the workspace starts with the Cholesky factor L of the damped system: row-major, leading dimension 32*ceil(n/32),
 * lower triangle valid (the entries above the diagonal are unspecified). */
size_t dba_solve_workspace_bytes(int n);
int dba_solve_spd(const double* H, const double* b, int n, float lm, float ep, float* x, int* fail_flag_device,
                  void* workspace, size_t workspace_bytes, dba_stream_t stream);
/* host only: where the resident-tile Cholesky (n <= 448) places its tiles -- map_i / map_j [128]: tile (i, j) of warp slot 8*cta + warp
 * (i == number of tile rows: a right-hand-side piece; 0xFF: none).  Returns the cluster size, 0 when n is served by the barrier kernel. */
int dba_solve_tile_placement(int n, unsigned char* map_i, unsigned char* map_j);

/* ---- Lie groups SO3 / SE3 (the `lietorch` package, droid_slam_b200/lietorch) ---------------------------------------------------------
 * replaces lietorch_backends.* (reference thirdparty/lietorch/lietorch/src/lietorch_gpu.cu).  group: DBA_LIE_SO3 (data qx,qy,qz,qw;
 * tangent 3) or DBA_LIE_SE3 (data tx,ty,tz,qx,qy,qz,qw; tangent tau,phi); dtype DBA_F32 or DBA_F64 for every operand.  The quaternion is
 * normalised on load; exp / log / the left Jacobian and its inverse take their small-angle branches below lietorch's EPS = 1e-6.
 * Operands a (and b for the binary ops), records of dba_lie_record_sizes' sizes, the last dimension contiguous.  Broadcasting: the
 * output batch is shape[ndim] (0 <= ndim <= DBA_LIE_MAX_DIMS); a_strides / b_strides [ndim] are each operand's batch strides in records,
 * 0 where it broadcasts (its size 1).  out and grad are contiguous over shape.  No operand is copied to the output's batch.
 *   op          a            b              out
 *   EXP         tangent      -              group            LOG        group   -        tangent
 *   INV         group        -              group            MUL        group   group    group
 *   ADJ / ADJT  group        tangent        tangent          JINV       group   tangent  tangent = Jl(log a)^-1 b
 *   ACT         group        point [3]      point [3]        ACT4       group   [4]      [4] (homogeneous)
 *   PROJECTOR   group        -              [N*N] row-major (the orthogonal projector vec() / InitFromVec's gradients use)
 *   VEC / FROMVEC: backward only (their forward is the identity): grad_a = grad P(a) / grad pinv(P(a)), N entries each.
 * dba_lie_backward: grad [shape, out record] -> grad_a laid out like a, grad_b like b, fully overwritten (nothing is written when the
 * output batch is empty).  grad_a or grad_b may be NULL (not both, for a binary op): that gradient is neither computed nor written, so
 * no reduction runs for a broadcast operand whose gradient is not asked for.  The gradient of a group operand is lietorch's left-tangent gradient d/de L(Exp(e) X) at e = 0 in the first K
 * entries of its N-entry record, the rest 0; a group output's upstream gradient is read from the same K entries.  A broadcast operand's
 * gradient is summed over its broadcast dimensions inside the launch, in a fixed order (bit-reproducible).  Jinv and PROJECTOR have no
 * backward.  Neither entry point synchronises the host. */
#define DBA_LIE_MAX_DIMS 8
enum { DBA_LIE_SO3 = 1, DBA_LIE_SE3 = 3 };          /* lietorch's group ids */
enum { DBA_LIE_EXP = 0, DBA_LIE_LOG, DBA_LIE_INV, DBA_LIE_MUL, DBA_LIE_ADJ, DBA_LIE_ADJT, DBA_LIE_JINV, DBA_LIE_ACT, DBA_LIE_ACT4,
       DBA_LIE_PROJECTOR, DBA_LIE_VEC, DBA_LIE_FROMVEC, DBA_LIE_OPS };
/* host only: the record sizes of operation op on group: *a, *b (0: unary), *out; DBA_ERR_INVALID for an unknown op or group */
int dba_lie_record_sizes(int op, int group, int* a, int* b, int* out);
int dba_lie_forward(int op, int group, int dtype, const void* a, const int64_t* a_strides, const void* b, const int64_t* b_strides,
                    void* out, int ndim, const int64_t* shape, dba_stream_t stream);
int dba_lie_backward(int op, int group, int dtype, const void* grad, const void* a, const int64_t* a_strides, const void* b,
                     const int64_t* b_strides, void* grad_a, void* grad_b, int ndim, const int64_t* shape, dba_stream_t stream);

/* ---- the differentiable dense BA layer (DroidNet's BA, reference geom/ba.py:31-106), forward and backward -------------------------
 * fp32, contiguous: target / weight [B,E,ht,wd,2], eta [B,M,ht,wd] (M = the number of distinct source frames), poses [B,N,7] (SE3),
 * disps [B,N,ht,wd], intrinsics [B,N,4] (per frame); ii / jj [E] int64.  Pose unknowns are frames fixedp .. N-1 (fixedp in [0, N),
 * N - fixedp <= DBA_BA_LAYER_MAX_POSES: the reduced pose system is factored by one CTA in shared memory).  Damping ep, lm as in
 * schur_solve (0.1, 1e-4).
 * dba_ba_layer_forward writes poses_out / disps_out and keeps, for the backward, the fp64 Cholesky factor [B, n, n] (n = 6 (N - fixedp),
 * lower triangle), dx [B, n] and dz [B, M, ht*wd] (zero-filled by the caller), and flags [1 + B] (device ints): flags[0] the status word
 * (DBA_BA_LAYER_BAD_*: edges with an out-of-range ii / jj are skipped instead of read), flags[1 + b] batch element b's factor failed
 * (any failure: dx = 0 for the whole batch).  dba_ba_layer_backward takes the upstream gradients grad_poses_out [B,N,7] (lietorch's
 * left-tangent convention) and grad_disps_out [B,N,ht,wd] with the same inputs and kept tensors, and writes grad_target, grad_weight,
 * grad_eta, grad_poses (all frames; 7th entry 0) and grad_disps, each shaped like its input.  The workspace is scratch for either call.
 * Neither entry point synchronises the host; no floating-point atomics (bit-reproducible, batch elements independent). */
#define DBA_BA_LAYER_MAX_POSES 20
enum { DBA_BA_LAYER_BAD_INDEX = 1, DBA_BA_LAYER_BAD_M = 2 };
typedef struct {
  const float *target, *weight, *eta, *poses, *disps, *intrinsics;
  const int64_t *ii, *jj;
  int B, N, E, M, ht, wd, fixedp;
  float ep, lm;
  float *poses_out, *disps_out;                       /* forward outputs */
  double *factor, *dx, *dz;                           /* written by the forward, read by the backward */
  int* flags;                                         /* [1 + B] */
  const float *grad_poses_out, *grad_disps_out;       /* backward inputs */
  float *grad_target, *grad_weight, *grad_eta, *grad_poses, *grad_disps;
  void* workspace;
  size_t workspace_bytes;
  dba_stream_t stream;
} dba_ba_layer_args;
size_t dba_ba_layer_workspace_bytes(int B, int N, int E, int M, int ht, int wd, int fixedp);
int dba_ba_layer_forward(const dba_ba_layer_args* args);
int dba_ba_layer_backward(const dba_ba_layer_args* args);

#ifdef __cplusplus
}
#endif
#endif /* DROID_B200_H */
