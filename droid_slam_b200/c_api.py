"""ctypes view of the C ABI declared in include/droid_b200.h (used by the parity tests and by bench.py's e2e leg)."""
import ctypes
import os

_LIB = None

SYMBOLS = [
    "dba_last_error", "dba_version",
    "dba_corr_index_forward", "dba_corr_index_backward", "dba_corr_volume_pyramid", "dba_corr_lookup_pyramid", "dba_corr_volume_supported",
    "dba_corr_volume_workspace_bytes", "dba_altcorr_forward", "dba_altcorr_backward",
    "dba_altcorr_pyramid", "dba_altcorr_lookup_pyramid",
    "dba_projmap", "dba_reproject", "dba_motion_features", "dba_graph_writeback", "dba_cvx_upsample", "dba_frame_distance", "dba_depth_filter", "dba_iproj",
    "dba_ba_workspace_bytes", "dba_ba_system_offset", "dba_ba_system_bytes",
    "dba_ba_prepare", "dba_ba_build", "dba_ba_solve", "dba_ba", "dba_ba_read_info", "dba_ba_p2p_signal",
    "dba_solve_workspace_bytes", "dba_solve_spd", "dba_solve_tile_placement",
    "dba_update_workspace_bytes", "dba_update_workspace_layout", "dba_update_forward", "dba_conv_nhwc", "dba_conv_nhwc_plan", "dba_encoder_workspace_bytes", "dba_encoder_forward",
    "dba_encoder_forward_frames", "dba_encoder_workspace_layout", "dba_encoder_forward_prefix", "dba_proximity_workspace_bytes", "dba_proximity_edges",
    "dba_fill_interpolate", "dba_pose_only_ba", "dba_fragment_handover", "dba_lie_record_sizes", "dba_lie_forward", "dba_lie_backward",
    "dba_ba_layer_workspace_bytes", "dba_ba_layer_forward", "dba_ba_layer_backward",
    "dba_corr_volume_pyramid_f32", "dba_corr_grad_accumulate", "dba_corr_adjoint_workspace_bytes", "dba_corr_adjoint",
]

DBA_F32, DBA_F16, DBA_F64, DBA_BF16 = 0, 1, 2, 3


class BAArgs(ctypes.Structure):
    _fields_ = [
        ("poses", ctypes.c_void_p), ("disps", ctypes.c_void_p), ("intrinsics", ctypes.c_void_p), ("disps_sens", ctypes.c_void_p),
        ("targets", ctypes.c_void_p), ("weights", ctypes.c_void_p), ("eta", ctypes.c_void_p), ("eta_rows", ctypes.c_int),
        ("ii", ctypes.c_void_p), ("jj", ctypes.c_void_p),
        ("n_frames", ctypes.c_int), ("n_edges", ctypes.c_int), ("ht", ctypes.c_int), ("wd", ctypes.c_int),
        ("t0", ctypes.c_int), ("t1", ctypes.c_int),
        ("lm", ctypes.c_float), ("ep", ctypes.c_float), ("motion_only", ctypes.c_int),
        ("dx_out", ctypes.c_void_p), ("dz_out", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
        ("stream", ctypes.c_void_p),
        ("own_lo", ctypes.c_int), ("own_hi", ctypes.c_int), ("eta_by_frame", ctypes.c_int),
        ("p2p_world", ctypes.c_int), ("p2p_rank", ctypes.c_int), ("p2p_epoch", ctypes.c_ulonglong), ("p2p_system", ctypes.c_void_p * 8), ("p2p_epoch_dev", ctypes.c_void_p),
    ]


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
    L.dba_last_error.restype = ctypes.c_char_p
    L.dba_version.restype = ctypes.c_int
    for n in ("dba_ba_workspace_bytes", "dba_ba_system_offset"):
        getattr(L, n).restype = ctypes.c_size_t
        getattr(L, n).argtypes = [ctypes.c_int] * 6
    L.dba_ba_system_bytes.restype = ctypes.c_size_t
    L.dba_ba_system_bytes.argtypes = [ctypes.c_int] * 2
    vp, ci, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.dba_corr_index_forward.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp]
    L.dba_corr_index_backward.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp]
    L.dba_corr_volume_pyramid.argtypes = [vp] * 8 + [ci] * 8 + [vp, ctypes.c_size_t, vp]
    L.dba_corr_lookup_pyramid.argtypes = [vp] * 6 + [ci] * 5 + [vp]
    L.dba_corr_volume_supported.argtypes = [ci] * 5
    L.dba_corr_volume_workspace_bytes.restype = ctypes.c_size_t
    L.dba_corr_volume_workspace_bytes.argtypes = [ci] * 5
    L.dba_corr_volume_pyramid_f32.argtypes = [vp] * 6 + [ci] * 4 + [vp]
    L.dba_corr_grad_accumulate.argtypes = [vp] * 3 + [ci] * 3 + [vp]
    L.dba_corr_adjoint_workspace_bytes.restype = ctypes.c_size_t
    L.dba_corr_adjoint_workspace_bytes.argtypes = [ci] * 4
    L.dba_corr_adjoint.argtypes = [vp] * 5 + [ci] * 4 + [vp, ctypes.c_size_t, vp]
    L.dba_altcorr_forward.argtypes = [vp, vp, vp, vp, vp, vp] + [ci] * 11 + [vp]
    L.dba_altcorr_backward.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp] + [ci] * 11 + [vp]
    L.dba_altcorr_pyramid.argtypes = [vp] * 5 + [ci] * 7 + [vp]
    L.dba_altcorr_lookup_pyramid.argtypes = [vp] * 8 + [ci] * 9 + [vp]
    L.dba_projmap.argtypes = [vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, vp]
    L.dba_reproject.argtypes = [vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, vp]
    L.dba_motion_features.argtypes = [vp] * 10 + [ci] * 3 + [vp]
    L.dba_graph_writeback.argtypes = [vp] * 4 + [ci] + [vp] * 4 + [ci] + [vp, vp, ci, vp, vp, ci, vp, cf, ci, ci, vp]
    L.dba_update_workspace_bytes.restype = ctypes.c_size_t
    L.dba_update_workspace_bytes.argtypes = [ci] * 4
    L.dba_update_workspace_layout.argtypes = [ci] * 4 + [vp, vp]
    L.dba_frame_distance.argtypes = [vp, vp, vp, vp, vp, vp, ci, ci, ci, cf, vp]
    L.dba_depth_filter.argtypes = [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, vp]
    L.dba_iproj.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp]
    for n in ("dba_ba_prepare", "dba_ba_build", "dba_ba_solve", "dba_ba_p2p_signal"):
        getattr(L, n).argtypes = [ctypes.POINTER(BAArgs)]
    L.dba_ba.argtypes = [ctypes.POINTER(BAArgs), ci]
    L.dba_ba_read_info.argtypes = [ctypes.POINTER(BAArgs), ctypes.POINTER(ci), ctypes.POINTER(ci)]
    L.dba_solve_workspace_bytes.restype = ctypes.c_size_t
    L.dba_solve_workspace_bytes.argtypes = [ci]
    L.dba_solve_spd.argtypes = [vp, vp, ci, cf, cf, vp, vp, vp, ctypes.c_size_t, vp]
    L.dba_solve_tile_placement.argtypes = [ci, vp, vp]
    L.dba_conv_nhwc_plan.argtypes = [ci] * 6 + [vp]
    L.dba_encoder_workspace_bytes.restype = ctypes.c_size_t
    L.dba_encoder_workspace_bytes.argtypes = [ci] * 4
    L.dba_encoder_workspace_layout.argtypes = [ci] * 4 + [vp] * 4
    L.dba_encoder_forward_prefix.argtypes = [vp, ci]
    L.dba_encoder_forward_frames.argtypes = [vp, vp]
    L.dba_proximity_workspace_bytes.restype = ctypes.c_size_t
    L.dba_proximity_workspace_bytes.argtypes = [ci, ci, ci]
    L.dba_proximity_edges.argtypes = [vp, ci, ci, ci, vp, vp, ci, ci, ci, cf, ci, ci, vp, ci, vp, vp, ctypes.c_size_t, vp]
    L.dba_fill_interpolate.argtypes = [vp, vp, ci, vp, ci, vp, vp, vp, vp]
    L.dba_pose_only_ba.argtypes = [vp] * 7 + [ci] * 8 + [cf, cf] + [vp] * 4
    _LIB = L
    return L


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError("%s failed (status %d): %s" % (what, rc, load().dba_last_error().decode()))
