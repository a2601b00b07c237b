/* droid_b200_training.h -- the C ABI of training's tail: DroidNet's flow loss and the backward of its disparity upsampling.
 * Declared apart from droid_b200.h, whose function set (57 entry points) the project's ABI checks pin; c_api.TRAINING_PROTOTYPES
 * mirrors this file and tests/test_flow_loss_cpu.py checks the two against each other. */
#ifndef DROID_B200_TRAINING_H
#define DROID_B200_TRAINING_H
#include "droid_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---- training's flow loss (reference geom/losses.py:89-118 flow_loss), forward and backward -----------------------------------------
 * fp32, contiguous: Ps [B,N,7] (SE3, the ground truth), disps [B,N,ht,wd], intrinsics [B,N,4] (per frame, full resolution); poses_est /
 * disps_est: device arrays of n pointers to the iterates' [B,N,7] poses and [B,N,ht,wd] disparities.  N >= 2, n >= 1.  The edges are
 * the chain graph the reference builds (i -> i-1, i -> i+1 for every i, in that order).
 * dba_flow_loss_forward writes loss (device float) = sum_s gamma^(n-1-s) mean(v |c1 - c0|) over B E ht wd, and metrics (device double
 * [3]) for the last iterate: the sum of epe where v > 0.5, that pixel count, and the count with epe < 1.
 * dba_flow_loss_backward reads the upstream gradient grad_loss (device float) and writes, through device arrays of n pointers,
 * grad_poses_est[s] [B,N,7] (lietorch's left-tangent convention, 7th entry 0) and grad_disps_est[s] [B,N,ht,wd].  The workspace
 * (dba_flow_loss_workspace_bytes) is scratch for either call.  Neither synchronises the host; no floating-point atomics. */
size_t dba_flow_loss_workspace_bytes(int B, int N, int ht, int wd, int n);
int dba_flow_loss_forward(const float* Ps, const float* disps, const float* intrinsics, const float* const* poses_est,
                          const float* const* disps_est, int n, float* loss, double* metrics, int B, int N, int ht, int wd, double gamma,
                          void* workspace, size_t workspace_bytes, dba_stream_t stream);
int dba_flow_loss_backward(const float* grad_loss, const float* Ps, const float* disps, const float* intrinsics, const float* const* poses_est,
                           const float* const* disps_est, int n, float* const* grad_poses_est, float* const* grad_disps_est, int B, int N,
                           int ht, int wd, double gamma, void* workspace, size_t workspace_bytes, dba_stream_t stream);

/* the backward of dba_cvx_upsample for fp32 masks: disps [n,ht,wd], mask [n,576,ht,wd], grad_out [n,8*ht,8*wd] (16-byte aligned) ->
 * grad_disps [n,ht,wd], grad_mask [n,576,ht,wd].  The softmax is recomputed from the mask; tap_partials [n,9,8,ht,wd] floats is scratch
 * (per-tap sums, gathered in a fixed order: no atomics). */
int dba_cvx_upsample_backward(const float* disps, const float* mask, const float* grad_out, float* grad_disps, float* grad_mask,
                              float* tap_partials, int n, int ht, int wd, dba_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DROID_B200_TRAINING_H */
