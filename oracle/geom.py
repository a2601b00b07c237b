"""Streaming geometry ops restated from src/droid_kernels.cu (projmap, frame_distance, depth_filter, iproj).
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import torch
from .se3 import act_se3, rel_se3

__all__ = ["projmap", "frame_distance", "depth_filter", "iproj", "MIN_DEPTH", "pixel_grid", "edge_transform", "reproject"]

MIN_DEPTH = 0.25  # src/droid_kernels.cu:35


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def pixel_grid(ht, wd, dtype):
    v, u = torch.meshgrid(torch.arange(ht, dtype=dtype), torch.arange(wd, dtype=dtype), indexing="ij")
    return u.reshape(-1), v.reshape(-1)


def edge_transform(poses, ii, jj, stereo_quirk):
    """relative transform per edge (src/droid_kernels.cu:228-258); stereo edges ii==jj get the fixed
    baseline (-0.1,0,0 | identity) only where the kernel has that branch (projective_transform_kernel)."""
    ti, qi = poses[ii, :3], poses[ii, 3:]
    tj, qj = poses[jj, :3], poses[jj, 3:]
    tij, qij = rel_se3(ti, qi, tj, qj)
    if stereo_quirk:
        s = (ii == jj)
        if bool(s.any()):
            tij = tij.clone(); qij = qij.clone()
            tij[s] = torch.tensor([-0.1, 0.0, 0.0], dtype=torch.float32).to(poses.dtype)   # an fp32 constant in the reference
            qij[s] = torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=poses.dtype)
    return tij, qij


def _backproject(disps_i, intr, ht, wd):
    fx, fy, cx, cy = [intr[k] for k in range(4)]
    u, v = pixel_grid(ht, wd, disps_i.dtype)
    X = torch.stack([((u - cx) / fx).expand_as(disps_i), ((v - cy) / fy).expand_as(disps_i),
                     torch.ones_like(disps_i), disps_i], dim=-1)
    return X, u, v


def projmap(poses, disps, intrinsics, ii, jj):
    """src/droid_kernels.cu:436-525, 1472-1497.  coords [E,ht,wd,3] (channel 2 stays 0), valid [E,ht,wd,1].
    No stereo branch in this kernel."""
    N, ht, wd = disps.shape
    E = ii.shape[0]
    fx, fy, cx, cy = [intrinsics[k] for k in range(4)]
    tij, qij = edge_transform(poses, ii, jj, stereo_quirk=False)
    Xi, u, v = _backproject(disps[ii].reshape(E, -1), intrinsics, ht, wd)
    Xj = act_se3(tij[:, None], qij[:, None], Xi)
    z = Xj[..., 2]
    ok = z > 0.01
    zz = torch.where(ok, z, torch.ones_like(z))
    cu = torch.where(ok, fx * (Xj[..., 0] / zz) + cx, u.expand_as(z))
    cv = torch.where(ok, fy * (Xj[..., 1] / zz) + cy, v.expand_as(z))
    coords = torch.stack([cu, cv, torch.zeros_like(cu)], dim=-1).reshape(E, ht, wd, 3)
    valid = (z > MIN_DEPTH).to(disps.dtype).reshape(E, ht, wd, 1)
    return coords, valid


def frame_distance(poses, disps, intrinsics, ii, jj, beta):
    """src/droid_kernels.cu:527-666, 1447-1469.  One direction only (loop `n<1`)."""
    N, ht, wd = disps.shape
    K = ii.shape[0]
    dt = disps.dtype
    fx, fy, cx, cy = [intrinsics[k] for k in range(4)]
    tij, qij = edge_transform(poses, ii, jj, stereo_quirk=False)
    Xi, u, v = _backproject(disps[ii].reshape(K, -1), intrinsics, ht, wd)
    HW = ht * wd
    beta = torch.tensor(beta, dtype=torch.float32).to(dt)  # kernel argument is `const float beta`
    # full motion
    Xj = act_se3(tij[:, None], qij[:, None], Xi)
    du = fx * (Xj[..., 0] / Xj[..., 2]) + cx - u
    dv = fy * (Xj[..., 1] / Xj[..., 2]) + cy - v
    d1 = torch.sqrt(du * du + dv * dv)
    ok1 = Xj[..., 2] > MIN_DEPTH
    # translation only
    Yj = Xi[..., :3] + Xi[..., 3:4] * tij[:, None]
    du = fx * (Yj[..., 0] / Yj[..., 2]) + cx - u
    dv = fy * (Yj[..., 1] / Yj[..., 2]) + cy - v
    d2 = torch.sqrt(du * du + dv * dv)
    ok2 = Yj[..., 2] > MIN_DEPTH
    zero = torch.zeros((), dtype=dt)
    accum = torch.where(ok1, beta * d1, zero).sum(-1) + torch.where(ok2, (1 - beta) * d2, zero).sum(-1)
    valid = torch.where(ok1, beta, zero).sum(-1) + torch.where(ok2, 1 - beta, zero).sum(-1)
    total = (beta * HW + (1 - beta) * HW).expand(K)
    frac = valid.double() / (total.double() + 1e-8)   # (:664) `total[0] + 1e-8` is fp64: in fp32 the 1e-8 would vanish
    return torch.where(frac < 0.75, torch.full_like(accum, 1000.0), accum / valid)


def _device_floor_int(x):
    """static_cast<int>(floor(x)) as the device computes it for fp32 x: cvt.rzi.s32.f32 saturates at the int range and maps NaN to 0"""
    f = torch.floor(x.double())
    return torch.where(torch.isnan(f), torch.zeros_like(f), f).clamp(-2.0 ** 31, 2.0 ** 31 - 1)


def depth_filter(poses, disps, intrinsics, ix, thresh):
    """src/droid_kernels.cu:670-784, 1500-1524.  Neighbour set ix-1,-2,-3, ix+3,+4,+5 (line 704, kept).  The cell is
    static_cast<int>(floor(uj)) with the device's conversion: a NaN projection (Z == 0 with X == Y == 0) lands in cell 0 and is
    compared with the four disparities there, and projections beyond the int range saturate."""
    num, ht, wd = disps.shape
    dt = disps.dtype
    fx, fy, cx, cy = [intrinsics[k] for k in range(4)]
    n = ix.shape[0]
    counter = torch.zeros(n, ht * wd, dtype=dt)
    for b in range(n):
        i = int(ix[b])
        t = thresh[b]
        for neigh in range(6):
            j = i - neigh - 1 if neigh < 3 else i + neigh
            if j < 0 or j >= num:
                continue
            ii = torch.tensor([i]); jj = torch.tensor([j])
            tij, qij = edge_transform(poses, ii, jj, stereo_quirk=False)
            Xi, u, v = _backproject(disps[i].reshape(1, -1), intrinsics, ht, wd)
            Xj = act_se3(tij[:, None], qij[:, None], Xi)[0]
            uj = fx * (Xj[:, 0] / Xj[:, 2]) + cx
            vj = fy * (Xj[:, 1] / Xj[:, 2]) + cy
            dj = Xj[:, 3] / Xj[:, 2]
            fu, fv = _device_floor_int(uj), _device_floor_int(vj)
            inb = (fu >= 0) & (fv >= 0) & (fu < wd - 1) & (fv < ht - 1)
            u0 = torch.where(inb, fu, torch.zeros_like(fu)).long()
            v0 = torch.where(inb, fv, torch.zeros_like(fv)).long()
            dsj = disps[j]
            d00 = dsj[v0, u0]; d01 = dsj[v0, (u0 + 1).clamp(max=wd - 1)]
            d10 = dsj[(v0 + 1).clamp(max=ht - 1), u0]; d11 = dsj[(v0 + 1).clamp(max=ht - 1), (u0 + 1).clamp(max=wd - 1)]
            # comparisons are done in double in the kernel (1.0/dj with a double literal), line 777-781
            idj = 1.0 / dj.double()
            t64 = t.double()
            hit = ((idj - 1.0 / d00.double()).abs() < t64) | ((idj - 1.0 / d01.double()).abs() < t64) | \
                  ((idj - 1.0 / d10.double()).abs() < t64) | ((idj - 1.0 / d11.double()).abs() < t64)
            counter[b] += (inb & hit).to(dt)
    return counter.reshape(n, ht, wd)


def iproj(poses, disps, intrinsics):
    """src/droid_kernels.cu:788-859, 1527-1550.  points = (T * [X,Y,1,d])[:3] / d."""
    n, ht, wd = disps.shape
    Xi, u, v = _backproject(disps.reshape(n, -1), intrinsics, ht, wd)
    Xj = act_se3(poses[:n, None, :3], poses[:n, None, 3:], Xi)
    pts = Xj[..., :3] / Xj[..., 3:4]
    return pts.reshape(n, ht, wd, 3)


def reproject(poses, disps, intrinsics, ii, jj):
    """pops.projective_transform(poses, depths, intrinsics, ii, jj, jacobian=False) as called by DepthVideo.reproject
    (droid_slam/geom/projective_ops.py:165-198, depth_video.py:171-179), restated without lietorch:
    X0 = iproj(d_i; K_i) (:16-35), Gij = G_j G_i^-1 with the stereo constant for ii == jj (:174-178), X1 = Gij X0,
    proj with Z < 0.1 -> 1 and K_j (:46-58), valid = (X1.Z > 0.2) & (X0.Z > 0.2) (:185).  intrinsics [N,4]."""
    N, ht, wd = disps.shape
    E = ii.shape[0]
    dt = disps.dtype
    tij, qij = edge_transform(poses, ii, jj, stereo_quirk=True)
    u, v = pixel_grid(ht, wd, dt)
    Ki, Kj = intrinsics[ii], intrinsics[jj]
    d_i = disps[ii].reshape(E, -1)
    X0 = torch.stack([(u[None] - Ki[:, 2:3]) / Ki[:, 0:1], (v[None] - Ki[:, 3:4]) / Ki[:, 1:2], torch.ones_like(d_i), d_i], dim=-1)
    X1 = act_se3(tij[:, None], qij[:, None], X0)
    small, min_depth = _f32(0.5 * 0.2), _f32(0.2)       # fp32 literals, as the reference's fp32 tensors compare with them
    Z = torch.where(X1[..., 2] < small, torch.ones_like(X1[..., 2]), X1[..., 2])
    d = 1.0 / Z
    x = Kj[:, 0:1] * (X1[..., 0] * d) + Kj[:, 2:3]
    y = Kj[:, 1:2] * (X1[..., 1] * d) + Kj[:, 3:4]
    coords = torch.stack([x, y], dim=-1).reshape(E, ht, wd, 2)
    valid = ((X1[..., 2] > min_depth) & (X0[..., 2] > min_depth)).to(dt).reshape(E, ht, wd, 1)
    return coords, valid
