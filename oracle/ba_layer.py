"""The differentiable dense BA layer -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

A vectorised restatement of the reference's geom/ba.py BA (:31-106), geom/chol.py schur_solve / CholeskySolver (:5-73) and the
Jacobian path of geom/projective_ops.py (iproj, proj, actp, projective_transform: :23-198) on the lietorch and torch_scatter stand-ins
(oracle/shims), on any device and dtype.  Autograd through it is the yardstick for droid_slam_b200.modules.ba_layer's gradients.

Like the reference: valid = (X1.z > 0.2) & (X0.z > 0.2); proj replaces Z < 0.1 by 1; Gij = [-0.1,0,0, 0,0,0,1] on ii == jj edges, with
no gradient through it; depth unknowns are the distinct ii (`unique`); damping H + (ep + lm H) * I before the Schur complement; a failed
Cholesky anywhere in the batch gives dx = 0 and no gradient through the solve (without the reference's print).
"""
import torch

from .shims import lietorch as _lt
from .shims.torch_scatter import scatter_sum

SE3 = _lt.SE3
MIN_DEPTH = 0.2


class _CholeskySolver(torch.autograd.Function):
    """geom/chol.py:5-29: the whole batch in one factorisation; any failure -> zeros and no gradient"""

    @staticmethod
    def forward(ctx, H, b):
        U, info = torch.linalg.cholesky_ex(H)
        ctx.failed = bool((info != 0).any())
        if ctx.failed:
            return torch.zeros_like(b)
        xs = torch.cholesky_solve(b, U)
        ctx.save_for_backward(U, xs)
        return xs

    @staticmethod
    def backward(ctx, grad_x):
        if ctx.failed:
            return None, None
        U, xs = ctx.saved_tensors
        dz = torch.cholesky_solve(grad_x, U)
        return -torch.matmul(xs, dz.transpose(-1, -2)), dz


def _jacobians(poses, disps, intrinsics, ii, jj):
    """projective_transform(jacobian=True): coords [B,E,H,W,2], valid [B,E,H,W,1], Ji / Jj [B,E,H,W,2,6], Jz [B,E,H,W,2,1]"""
    ht, wd = disps.shape[2:]
    dt = disps.dtype
    fx, fy, cx, cy = intrinsics[:, ii, None, None, :].unbind(-1)
    y, x = torch.meshgrid(torch.arange(ht, device=disps.device, dtype=dt), torch.arange(wd, device=disps.device, dtype=dt), indexing="ij")
    d0 = disps[:, ii]
    X0 = torch.stack([(x - cx) / fx, (y - cy) / fy, torch.ones_like(d0), d0], dim=-1)
    Gij = poses[:, jj] * poses[:, ii].inv()
    same = ii == jj
    if bool(same.any()):
        const = torch.as_tensor([-0.1, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0], dtype=dt, device=disps.device)
        data = Gij.data.clone()
        data[:, same] = const
        Gij = SE3(data)
    X1 = Gij[:, :, None, None] * X0
    X, Y, Z, D = X1.unbind(-1)
    o = torch.zeros_like(D)
    Ja = torch.stack([D, o, o, o, Z, -Y, o, D, o, -Z, o, X, o, o, D, Y, -X, o, o, o, o, o, o, o], dim=-1).view(*D.shape, 4, 6)
    fx, fy, cx, cy = intrinsics[:, jj, None, None, :].unbind(-1)
    Zc = torch.where(Z < 0.5 * MIN_DEPTH, torch.ones_like(Z), Z)
    d = 1.0 / Zc
    coords = torch.stack([fx * (X * d) + cx, fy * (Y * d) + cy], dim=-1)
    Jp = torch.stack([fx * d, o, -fx * X * d * d, o, o, fy * d, -fy * Y * d * d, o], dim=-1).view(*D.shape, 2, 4)
    valid = ((X1[..., 2] > MIN_DEPTH) & (X0[..., 2] > MIN_DEPTH)).to(dt).unsqueeze(-1)
    Jj = torch.matmul(Jp, Ja)
    Ji = -Gij[:, :, None, None, None].adjT(Jj)
    Jz0 = torch.zeros_like(X0)
    Jz0[..., -1] = 1.0
    Jz = torch.matmul(Jp, (Gij[:, :, None, None] * Jz0).unsqueeze(-1))
    return coords, valid, Ji, Jj, Jz


def ba(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp=1, ep=0.1, lm=1e-4):
    """BA(target, weight, eta, poses (SE3 stand-in), disps, intrinsics, ii, jj, fixedp) -> (poses', disps'), rig = 1"""
    out = ba_system(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp, ep, lm)
    return out["poses"], out["disps"]


def ba_system(target, weight, eta, poses, disps, intrinsics, ii, jj, fixedp=1, ep=0.1, lm=1e-4):
    """ba() with its reduced system: dict(poses, disps (ba's outputs), S [B,6P,6P] (H + (ep + lm H) I - E Q E^T, both triangles),
    y [B,6P] (v - E Q w), dx [B,6P] (0 when the factor failed anywhere in the batch), dz [B,M,HW]), all differentiable"""
    B, N, ht, wd = disps.shape
    E, D, HW = ii.shape[0], 6, ht * wd
    coords, valid, Ji, Jj, Jz = _jacobians(poses, disps, intrinsics, ii, jj)
    r = (target - coords).view(B, E, -1, 1)
    w = .001 * (valid * weight).view(B, E, -1, 1)
    Ji, Jj = Ji.reshape(B, E, -1, D), Jj.reshape(B, E, -1, D)
    wJiT, wJjT = (w * Ji).transpose(2, 3), (w * Jj).transpose(2, 3)
    Jz = Jz.reshape(B, E, HW, -1)
    Hii, Hij, Hji, Hjj = wJiT @ Ji, wJiT @ Jj, wJjT @ Ji, wJjT @ Jj
    vi, vj = (wJiT @ r).squeeze(-1), (wJjT @ r).squeeze(-1)
    Ei = (wJiT.view(B, E, D, HW, -1) * Jz[:, :, None]).sum(-1)
    Ej = (wJjT.view(B, E, D, HW, -1) * Jz[:, :, None]).sum(-1)
    w, r = w.view(B, E, HW, -1), r.view(B, E, HW, -1)
    wk, Ck = (w * r * Jz).sum(-1), (w * Jz * Jz).sum(-1)
    kx, kk = torch.unique(ii, return_inverse=True)
    M, P = kx.shape[0], N - fixedp
    pi, pj = ii - fixedp, jj - fixedp

    def mat(A, a, b, m):
        v = (a >= 0) & (b >= 0) & (a < P) & (b < m)
        return scatter_sum(A[:, v], a[v] * m + b[v], dim=1, dim_size=P * m)

    def vec(x, a, n):
        v = (a >= 0) & (a < n)
        return scatter_sum(x[:, v], a[v], dim=1, dim_size=n)

    H = mat(Hii, pi, pi, P) + mat(Hij, pi, pj, P) + mat(Hji, pj, pi, P) + mat(Hjj, pj, pj, P)
    Em = mat(Ei, pi, kk, M) + mat(Ej, pj, kk, M)
    v = vec(vi, pi, P) + vec(vj, pj, P)
    C = vec(Ck, kk, M) + eta.view(B, M, HW) + 1e-7
    wv = vec(wk, kk, M)
    H = H.view(B, P, P, D, D).permute(0, 1, 3, 2, 4).reshape(B, P * D, P * D)
    Em = Em.view(B, P, M, D, HW).permute(0, 1, 3, 2, 4).reshape(B, P * D, M * HW)
    Q = (1.0 / C).view(B, M * HW, 1)
    I = torch.eye(P * D, dtype=H.dtype, device=H.device)
    H = H + (ep + lm * H) * I
    v, wv = v.reshape(B, P * D, 1), wv.reshape(B, M * HW, 1)
    Et = Em.transpose(1, 2)
    S = H - Em @ (Q * Et)
    y = v - Em @ (Q * wv)
    dx1 = _CholeskySolver.apply(S, y)
    dz = (Q * (wv - Et @ dx1)).view(B, M, ht, wd)
    dx = dx1.reshape(B, P, D)
    dxa = scatter_sum(dx, torch.arange(P, device=dx.device) + fixedp, dim=1, dim_size=N)
    poses = poses.retr(dxa)
    disps = disps + scatter_sum(dz, kx, dim=1, dim_size=N)
    disps = torch.where(disps > 10, torch.zeros_like(disps), disps)
    return dict(poses=poses, disps=disps.clamp(min=0.0), S=S, y=y.view(B, P * D), dx=dx1.view(B, P * D), dz=dz.view(B, M, HW))


def left_perturbed(data, eps):
    """the data of Exp(eps) X to first order in eps, for X's data [..., 7]: at eps = 0 its value is X's data and its derivative that of
    Exp(eps) X, so autograd with respect to eps gives lietorch's left-tangent gradient (SE3.exp's own derivative is NaN at eps = 0)"""
    t, q = data[..., :3], data[..., 3:]
    tau, phi = eps[..., :3], eps[..., 3:]
    dt = tau + torch.linalg.cross(phi, t)
    v, w = q[..., :3], q[..., 3:]
    dv = 0.5 * (w * phi + torch.linalg.cross(phi, v))
    dw = -0.5 * (phi * v).sum(-1, keepdim=True)
    return torch.cat([t + dt, v + dv, w + dw], dim=-1)
