"""Training's flow loss -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

geom/losses.py flow_loss (:89-118) restated on any device and dtype, on the lietorch stand-in (oracle/shims): the chain graph the
reference builds (graph ignored), coords / valid of projective_transform from oracle/ba_layer.py's restatement of
projective_ops.py (`_jacobians`: iproj, Gij = Pj Pi^-1, actp, proj with Z < 0.1 -> 1, valid = (X1.z > 0.2) & (X0.z > 0.2)), val0 masked
by disps > 0, loss = sum_i gamma^(n-1-i) mean(v |c1 - c0|).  Autograd through it is the yardstick for droid_slam_b200.modules.flow_loss.
That restatement also forms the reprojection's Jacobians, which the loss does not use: its time and memory overstate the reference's.
"""
import torch

from .ba_layer import SE3, _jacobians


def chain_edges(N, device=None):
    """losses.py:93-97: for i in 0..N-1 the j with |i - j| == 1, ascending"""
    ii = [i for i in range(N) for j in range(N) if abs(i - j) == 1]
    jj = [j for i in range(N) for j in range(N) if abs(i - j) == 1]
    return torch.tensor(ii, device=device), torch.tensor(jj, device=device)


def reproject(poses, disps, intrinsics, ii, jj):
    """projective_transform(poses, disps, intrinsics, ii, jj) -> (coords [B,E,H,W,2], valid [B,E,H,W,1]); poses: the stand-in SE3"""
    coords, valid = _jacobians(poses, disps, intrinsics, ii, jj)[:2]
    return coords, valid


def flow_loss(Ps, disps, poses_est, disps_est, intrinsics, gamma=0.9):
    """-> (loss, epe and v of the last iterate, flattened): Ps / poses_est[i] stand-in SE3s, the rest tensors"""
    ii, jj = chain_edges(disps.shape[1], disps.device)
    coords0, val0 = reproject(Ps, disps, intrinsics, ii, jj)
    val0 = val0 * (disps[:, ii] > 0).to(disps.dtype).unsqueeze(-1)
    n = len(poses_est)
    loss = 0.0
    for i in range(n):
        coords1, val1 = reproject(poses_est[i], disps_est[i], intrinsics, ii, jj)
        v = (val0 * val1).squeeze(-1)
        epe = v * (coords1 - coords0).norm(dim=-1)
        loss = loss + gamma ** (n - i - 1) * epe.mean()
    return loss, epe.reshape(-1), v.reshape(-1)


def metrics(epe, v):
    """the reference's metrics dict from the last iterate's epe and v"""
    e = epe[v > 0.5]
    return {"f_error": float(e.mean()), "1px": float((e < 1.0).float().mean())}        # .float(), as the reference has it
