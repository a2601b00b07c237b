"""ctypes view of the C ABI declared in include/droid_b200.h and include/droid_b200_training.h (used by the parity tests, the tools and
bench.py's e2e leg).

Every function of droid_b200.h has one prototype in PROTOTYPES, and every header struct that Python fills has one mirror here;
tests/test_oracle_cpu.py checks both against the header.  droid_b200_training.h's functions are in TRAINING_PROTOTYPES, checked by
tests/test_flow_loss_cpu.py.  Pointers are passed as c_void_p, except pointers to a mirrored struct."""
import ctypes
import os

_LIB = None

DBA_F32, DBA_F16, DBA_F64, DBA_BF16 = 0, 1, 2, 3
DBA_ENCODER_CONVS = 14

vp, ci, cf, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t


class BAArgs(ctypes.Structure):
    """dba_ba_args"""
    _fields_ = [
        ("poses", vp), ("disps", vp), ("intrinsics", vp), ("disps_sens", vp),
        ("targets", vp), ("weights", vp), ("eta", vp), ("eta_rows", ci),
        ("ii", vp), ("jj", vp),
        ("n_frames", ci), ("n_edges", ci), ("ht", ci), ("wd", ci),
        ("t0", ci), ("t1", ci),
        ("lm", cf), ("ep", cf), ("motion_only", ci),
        ("dx_out", vp), ("dz_out", vp),
        ("workspace", vp), ("workspace_bytes", sz),
        ("stream", vp),
        ("own_lo", ci), ("own_hi", ci), ("eta_by_frame", ci),
        ("p2p_world", ci), ("p2p_rank", ci), ("p2p_epoch", ctypes.c_ulonglong), ("p2p_system", vp * 8), ("p2p_epoch_dev", vp),
    ]


class UpdateWeights(ctypes.Structure):
    """dba_update_weights: device pointers in the order of update.PACKED_ORDER"""
    _fields_ = [(k, vp) for k in (
        "w_corr0", "w_corr2", "w_flow0", "w_flow2", "w_gate", "w_zr", "w_q", "w_stem", "w_heads", "w_agg2", "w_eta", "w_upmask",
        "b_corr0", "b_corr2", "b_flow0", "b_flow2", "b_gate", "b_zr", "b_q", "b_stem", "b_heads", "b_agg2", "b_eta", "b_upmask",
        "w_glo", "b_glo", "b_zero")]


class UpdateArgs(ctypes.Structure):
    """dba_update_args"""
    _fields_ = [("n_edges", ci), ("ht", ci), ("wd", ci),
                ("net", vp), ("net_dtype", ci), ("net_layout", ci),
                ("inp", vp), ("inp_dtype", ci), ("corr", vp), ("corr_dtype", ci),
                ("flow", vp), ("seg", vp), ("n_src", ci), ("weights", ctypes.POINTER(UpdateWeights)),
                ("net_out", vp), ("delta", vp), ("weight", vp), ("eta", vp), ("upmask", vp),
                ("workspace", vp), ("workspace_bytes", sz), ("stream", vp)]


class EncoderWeights(ctypes.Structure):
    """dba_encoder_weights: w[k] f16 and b[k] f32 device pointers of convolution k"""
    _fields_ = [("w", vp * DBA_ENCODER_CONVS), ("b", vp * DBA_ENCODER_CONVS)]


class EncoderArgs(ctypes.Structure):
    """dba_encoder_args"""
    _fields_ = [("images", vp), ("images_dtype", ci), ("n_images", ci), ("H", ci), ("W", ci),
                ("weights", ctypes.POINTER(EncoderWeights)), ("norm", ci), ("output_dim", ci), ("out", vp),
                ("workspace", vp), ("workspace_bytes", sz), ("stream", vp)]


class FrameFormat(ctypes.Structure):
    """dba_frame_format"""
    _fields_ = [("channel_order", ci), ("mean", cf * 3), ("std", cf * 3)]


_BA, _UPD, _ENC = ctypes.POINTER(BAArgs), ctypes.POINTER(UpdateArgs), ctypes.POINTER(EncoderArgs)

# name -> (restype, argtypes), in the header's order
PROTOTYPES = {
    "dba_last_error": (ctypes.c_char_p, []),
    "dba_version": (ci, []),
    "dba_corr_index_forward": (ci, [vp] * 3 + [ci] * 7 + [vp]),
    "dba_corr_index_backward": (ci, [vp] * 3 + [ci] * 7 + [vp]),
    "dba_corr_volume_supported": (ci, [ci] * 5),
    "dba_corr_volume_workspace_bytes": (sz, [ci] * 5),
    "dba_corr_volume_pyramid": (ci, [vp] * 8 + [ci] * 8 + [vp, sz, vp]),
    "dba_corr_lookup_pyramid": (ci, [vp] * 6 + [ci] * 5 + [vp]),
    "dba_corr_volume_pyramid_f32": (ci, [vp] * 6 + [ci] * 4 + [vp]),
    "dba_corr_grad_accumulate": (ci, [vp] * 3 + [ci] * 3 + [vp]),
    "dba_corr_adjoint_workspace_bytes": (sz, [ci] * 4),
    "dba_corr_adjoint": (ci, [vp] * 5 + [ci] * 4 + [vp, sz, vp]),
    "dba_altcorr_forward": (ci, [vp] * 6 + [ci] * 11 + [vp]),
    "dba_altcorr_backward": (ci, [vp] * 8 + [ci] * 11 + [vp]),
    "dba_altcorr_pyramid": (ci, [vp] * 5 + [ci] * 7 + [vp]),
    "dba_altcorr_lookup_pyramid": (ci, [vp] * 8 + [ci] * 9 + [vp]),
    "dba_projmap": (ci, [vp] * 7 + [ci] * 3 + [vp]),
    "dba_reproject": (ci, [vp] * 7 + [ci] * 3 + [vp]),
    "dba_motion_features": (ci, [vp] * 10 + [ci] * 3 + [vp]),
    "dba_graph_writeback": (ci, [vp] * 4 + [ci] + [vp] * 4 + [ci] + [vp, vp, ci, vp, vp, ci, vp, cf, ci, ci, vp]),
    "dba_frame_distance": (ci, [vp] * 6 + [ci] * 3 + [cf, vp]),
    "dba_depth_filter": (ci, [vp] * 6 + [ci] * 4 + [vp]),
    "dba_iproj": (ci, [vp] * 4 + [ci] * 3 + [vp]),
    "dba_cvx_upsample": (ci, [vp] * 3 + [ci] * 4 + [vp]),
    "dba_proximity_workspace_bytes": (sz, [ci] * 3),
    "dba_proximity_edges": (ci, [vp, ci, ci, ci, vp, vp, ci, ci, ci, cf, ci, ci, vp, ci, vp, vp, sz, vp]),
    "dba_ba_workspace_bytes": (sz, [ci] * 6),
    "dba_ba_system_offset": (sz, [ci] * 6),
    "dba_ba_system_bytes": (sz, [ci] * 2),
    "dba_ba_prepare": (ci, [_BA]),
    "dba_ba_build": (ci, [_BA]),
    "dba_ba_solve": (ci, [_BA]),
    "dba_ba": (ci, [_BA, ci]),
    "dba_ba_p2p_signal": (ci, [_BA]),
    "dba_ba_read_info": (ci, [_BA, vp, vp]),
    "dba_fill_interpolate": (ci, [vp, vp, ci, vp, ci, vp, vp, vp, vp]),
    "dba_pose_only_ba": (ci, [vp] * 7 + [ci] * 8 + [cf, cf] + [vp] * 4),
    "dba_fragment_handover": (ci, [vp] * 4 + [ctypes.c_longlong] + [ci] * 4 + [vp] * 3),
    "dba_update_workspace_bytes": (sz, [ci] * 4),
    "dba_update_forward": (ci, [_UPD]),
    "dba_update_workspace_layout": (ci, [ci] * 4 + [vp] * 2),
    "dba_conv_nhwc": (ci, [vp, ci, ci, vp, ci, ci, vp, vp, vp] + [ci] * 7 + [vp]),
    "dba_conv_nhwc_plan": (ci, [ci] * 6 + [vp]),
    "dba_encoder_workspace_bytes": (sz, [ci] * 4),
    "dba_encoder_forward": (ci, [_ENC]),
    "dba_encoder_forward_frames": (ci, [_ENC, ctypes.POINTER(FrameFormat)]),
    "dba_encoder_workspace_layout": (ci, [ci] * 4 + [vp] * 4),
    "dba_encoder_forward_prefix": (ci, [_ENC, ci]),
    "dba_solve_workspace_bytes": (sz, [ci]),
    "dba_solve_spd": (ci, [vp, vp, ci, cf, cf, vp, vp, vp, sz, vp]),
    "dba_solve_tile_placement": (ci, [ci, vp, vp]),
    "dba_lie_record_sizes": (ci, [ci] * 2 + [vp] * 3),
    "dba_lie_forward": (ci, [ci] * 3 + [vp] * 5 + [ci, vp, vp]),
    "dba_lie_backward": (ci, [ci] * 3 + [vp] * 7 + [ci, vp, vp]),
    "dba_ba_layer_workspace_bytes": (sz, [ci] * 7),
    "dba_ba_layer_forward": (ci, [vp]),                 # dba_ba_layer_args has no Python caller, so no mirror
    "dba_ba_layer_backward": (ci, [vp]),
}

SYMBOLS = list(PROTOTYPES)

# include/droid_b200_training.h (training's flow loss, upsample_disp's backward and the ConvGRU), in that header's order
TRAINING_PROTOTYPES = {
    "dba_flow_loss_workspace_bytes": (sz, [ci] * 5),
    "dba_flow_loss_forward": (ci, [vp] * 5 + [ci, vp, vp] + [ci] * 4 + [ctypes.c_double, vp, sz, vp]),
    "dba_flow_loss_backward": (ci, [vp] * 6 + [ci, vp, vp] + [ci] * 4 + [ctypes.c_double, vp, sz, vp]),
    "dba_cvx_upsample_backward": (ci, [vp] * 6 + [ci] * 3 + [vp]),
    "dba_conv_gru_workspace_bytes": (sz, [ci] * 4),
    "dba_conv_gru_forward": (ci, [vp] * 9 + [ci] * 3 + [vp, sz, vp]),
    "dba_conv_gru_backward": (ci, [vp] * 14 + [ci] * 3 + [vp, sz, vp]),
}


def ba_args(poses, disps, intrinsics, disps_sens, targets, weights, eta, ii, jj, t0, t1, lm, ep, dx_out, dz_out, workspace, stream,
            motion_only=False, own=None, eta_by_frame=False):
    """a dba_ba_args over torch tensors, which the caller keeps alive.  N, ht, wd come from disps and E from ii; eta None passes a null
    eta of one row; workspace is a byte tensor, stream a cudaStream_t as an int; own = (own_lo, own_hi), every frame by default.  The
    peer-to-peer fields stay zero."""
    N, ht, wd = disps.shape
    a = BAArgs()
    a.poses, a.disps, a.intrinsics, a.disps_sens = poses.data_ptr(), disps.data_ptr(), intrinsics.data_ptr(), disps_sens.data_ptr()
    a.targets, a.weights = targets.data_ptr(), weights.data_ptr()
    a.eta, a.eta_rows = (eta.data_ptr(), eta.shape[0]) if eta is not None else (None, 1)
    a.ii, a.jj = ii.data_ptr(), jj.data_ptr()
    a.n_frames, a.n_edges, a.ht, a.wd, a.t0, a.t1 = N, ii.shape[0], ht, wd, t0, t1
    a.lm, a.ep, a.motion_only = lm, ep, int(motion_only)
    a.dx_out, a.dz_out = dx_out.data_ptr(), dz_out.data_ptr()
    a.workspace, a.workspace_bytes = workspace.data_ptr(), workspace.nbytes
    a.stream = stream
    a.own_lo, a.own_hi = own if own is not None else (0, N)
    a.eta_by_frame = int(eta_by_frame)
    return a


def lib_path():
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libdroid_b200.so")


def load():
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not os.path.exists(p):
        raise ImportError("libdroid_b200.so not built; run `python -m droid_slam_b200.build`")
    L = ctypes.CDLL(p)
    for name, (restype, argtypes) in {**PROTOTYPES, **TRAINING_PROTOTYPES}.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _LIB = L
    return L


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError("%s failed (status %d): %s" % (what, rc, load().dba_last_error().decode()))
