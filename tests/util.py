"""helpers shared by the parity tests: calling the C ABI with torch CUDA tensors, comparison metrics"""
import ctypes

import torch

from droid_slam_b200 import c_api

DT = {torch.float32: c_api.DBA_F32, torch.float16: c_api.DBA_F16, torch.float64: c_api.DBA_F64, torch.bfloat16: c_api.DBA_BF16}


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def c_corr_index_forward(L, volume, coords, r):
    n, h1, w1, h2, w2 = volume.shape
    out = torch.full((n, 2 * r + 1, 2 * r + 1, h1, w1), float("nan"), dtype=volume.dtype, device=volume.device)
    c_api.check(L.dba_corr_index_forward(ptr(volume), ptr(coords), ptr(out), n, h1, w1, h2, w2, r, DT[volume.dtype], stream()), "corr_index_forward")
    return out


def c_corr_index_backward(L, volume, coords, grad, r):
    n, h1, w1, h2, w2 = volume.shape
    out = torch.full_like(volume, float("nan"))
    c_api.check(L.dba_corr_index_backward(ptr(coords), ptr(grad), ptr(out), n, h1, w1, h2, w2, r, DT[volume.dtype], stream()), "corr_index_backward")
    return out


def c_ba(L, poses, disps, intr, disps_sens, targets, weights, eta, ii, jj, t0, t1, itrs, lm, ep, motion_only, M, ws_fill=None):
    """dba_ba through ctypes; ws_fill: byte value the workspace starts with (255 makes every float in it NaN) instead of torch.empty's"""
    N, ht, wd = disps.shape
    E = ii.shape[0]
    ws_bytes = L.dba_ba_workspace_bytes(N, E, ht, wd, t0, t1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=poses.device)
    if ws_fill is not None:
        ws.fill_(ws_fill)
    dx = torch.full((t1 - t0, 6), float("nan"), device=poses.device)
    dz = torch.full((M, ht * wd), float("nan"), device=poses.device)
    a = c_api.BAArgs()
    a.poses, a.disps, a.intrinsics, a.disps_sens = poses.data_ptr(), disps.data_ptr(), intr.data_ptr(), disps_sens.data_ptr()
    a.targets, a.weights = targets.data_ptr(), weights.data_ptr()
    a.eta = eta.data_ptr() if eta is not None else None
    a.eta_rows = eta.shape[0] if eta is not None else 1
    a.ii, a.jj = ii.data_ptr(), jj.data_ptr()
    a.n_frames, a.n_edges, a.ht, a.wd, a.t0, a.t1 = N, E, ht, wd, t0, t1
    a.lm, a.ep, a.motion_only = lm, ep, int(motion_only)
    a.dx_out, a.dz_out = dx.data_ptr(), dz.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws_bytes
    a.stream = torch.cuda.current_stream().cuda_stream
    a.own_lo, a.own_hi, a.eta_by_frame = 0, N, 0
    c_api.check(L.dba_ba(ctypes.byref(a), itrs) if itrs > 0 else L.dba_ba_prepare(ctypes.byref(a)), "ba")
    m = ctypes.c_int(0); st = ctypes.c_int(0)
    c_api.check(L.dba_ba_read_info(ctypes.byref(a), ctypes.byref(m), ctypes.byref(st)), "ba_read_info")
    return dx, dz, m.value, st.value, (a, ws)


def rel_err(a, b, floor=1.0):
    """max |a-b| / max(|b|, floor): the '1e-4 rel' of BASELINE.json with an absolute floor for values near zero"""
    a = a.double().cpu(); b = b.double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=floor)).max())


def frac_equal(a, b):
    a = a.cpu(); b = b.cpu()
    return float((a == b).float().mean())


def assert_bit_identical(a, b, what=""):
    """torch.equal with a useful message (how many elements differ and by how much)"""
    a = a.cpu(); b = b.cpu()
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    if not torch.equal(a, b):
        neq = (a != b) & ~(torch.isnan(a) & torch.isnan(b))          # NaN in the same place on both sides (NaN coordinates) counts as identical
        if bool(neq.any()):
            d = (a.double() - b.double()).abs()
            raise AssertionError("%s: %d of %d elements differ, max |diff| %.3e" % (what, int(neq.sum()), a.numel(), float(d[neq].max())))
