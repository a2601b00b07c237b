"""Dense bundle adjustment restated from `ba_cuda` (src/droid_kernels.cu:1323-1443) and the kernels it
launches (K1 :185-433, accum :863-1007, EEt6x6 :1010-1065, Ev6x1 :1068-1102, EvT6x1 :1104-1124,
SparseBlock :1126-1228, schur_block :1231-1320, retractions :886-955).

`ba(...)` mutates `poses` and `disps` in place and returns [dx, dz] like the reference.
`dtype=torch.float32` follows the reference's precision split (fp32 kernels, fp64 solve);
`dtype=torch.float64` evaluates the same algebra entirely in fp64 (ground truth for tolerance tests).
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import torch
from .se3 import act_se3, adj_se3, retr_se3
from .geom import edge_transform, pixel_grid, MIN_DEPTH

__all__ = ["ba", "ba_edge_terms", "ba_system", "ba_graph"]


def ba_edge_terms(poses, disps, intrinsics, targets, weights, ii, jj):
    """projective_transform_kernel, src/droid_kernels.cu:185-433, vectorised over edges and pixels.

    Returns dict with Hs [4,E,6,6], vs [2,E,6], Eii,Eij [E,6,HW], Cii,bz [E,HW] (same meaning/layout as
    the reference workspace, :1359-1364), r2 [E,HW], the weighted squared residual wu*ru^2 + wv*rv^2, and
    bz_mag [E,HW], the magnitude of bz's operands wu |Jz_u| (|ru| + |target_u|) + wv |Jz_v| (|rv| + |target_v|)."""
    dt = poses.dtype
    N, ht, wd = disps.shape
    E = ii.shape[0]
    HW = ht * wd
    fx, fy, cx, cy = [intrinsics[k] for k in range(4)]
    tij, qij = edge_transform(poses, ii, jj, stereo_quirk=True)          # :228-258 (Q1)
    u, v = pixel_grid(ht, wd, dt)
    d_i = disps[ii].reshape(E, HW)
    Xi = torch.stack([((u - cx) / fx).expand(E, HW), ((v - cy) / fy).expand(E, HW),
                      torch.ones(E, HW, dtype=dt), d_i], dim=-1)          # :299-302
    t_ = tij[:, None]; q_ = qij[:, None]
    Xj = act_se3(t_, q_, Xi)                                               # :305
    x, y, z, h = Xj.unbind(-1)
    close = z < MIN_DEPTH
    d = torch.where(close, torch.zeros_like(z), 1.0 / torch.where(close, torch.ones_like(z), z))   # :311 (Q2)
    d2 = d * d
    # `.001 * weight` is double*float rounded to float in the kernel (:314-315) (Q4)
    w = (0.001 * weights.reshape(E, 2, HW).double()).to(dt)
    wu = torch.where(close, torch.zeros_like(z), w[:, 0])
    wv = torch.where(close, torch.zeros_like(z), w[:, 1])
    tg = targets.reshape(E, 2, HW)
    ru = tg[:, 0] - (fx * d * x + cx)                                     # :316
    rv = tg[:, 1] - (fy * d * y + cy)
    o = torch.zeros_like(z)
    Jj_u = fx * torch.stack([h * d, o, -x * h * d2, -x * y * d2, 1 + x * x * d2, -y * d], dim=-1)     # :321-326
    Jj_v = fy * torch.stack([o, h * d, -y * h * d2, -1 - y * y * d2, x * y * d2, x * d], dim=-1)      # :354-359
    Jz_u = fx * (tij[:, None, 0] * d - tij[:, None, 2] * (x * d2))                                    # :328
    Jz_v = fy * (tij[:, None, 1] * d - tij[:, None, 2] * (y * d2))                                    # :361
    Cii = wu * Jz_u * Jz_u + wv * Jz_v * Jz_v                            # :329,362
    bz = wu * ru * Jz_u + wv * rv * Jz_v                                  # :330,363
    r2 = wu * ru * ru + wv * rv * rv                                      # weighted squared residual (not in the reference)
    # magnitude of the operands of bz: |w Jz| (|r| + |target|) covers both the residual's subtraction and the sum (not in the reference)
    bz_mag = wu * Jz_u.abs() * (ru.abs() + tg[:, 0].abs()) + wv * Jz_v.abs() * (rv.abs() + tg[:, 1].abs())
    stereo = (ii == jj)[:, None]
    wu = torch.where(stereo, torch.zeros_like(wu), wu)                    # :332,365 (Q1)
    wv = torch.where(stereo, torch.zeros_like(wv), wv)
    Ji_u = -adj_se3(t_, q_, Jj_u)                                         # :334-335
    Ji_v = -adj_se3(t_, q_, Jj_v)
    Ju = torch.cat([Ji_u, Jj_u], dim=-1)                                  # [E,HW,12]
    Jv = torch.cat([Ji_v, Jj_v], dim=-1)
    H = torch.einsum("ep,epn,epm->enm", wu, Ju, Ju) + torch.einsum("ep,epn,epm->enm", wv, Jv, Jv)     # :337-343
    vv = torch.einsum("ep,epn->en", wu * ru, Ju) + torch.einsum("ep,epn->en", wv * rv, Jv)            # :345-347
    Eii = ((wu * Jz_u)[..., None] * Ji_u + (wv * Jz_v)[..., None] * Ji_v).permute(0, 2, 1).contiguous()  # :349,382
    Eij = ((wu * Jz_u)[..., None] * Jj_u + (wv * Jz_v)[..., None] * Jj_v).permute(0, 2, 1).contiguous()
    Hs = torch.stack([H[:, :6, :6], H[:, :6, 6:], H[:, 6:, :6], H[:, 6:, 6:]], dim=0)                 # :416-427 (Q5)
    vs = torch.stack([vv[:, :6], vv[:, 6:]], dim=0)
    return dict(Hs=Hs, vs=vs, Eii=Eii, Eij=Eij, Cii=Cii, bz=bz, r2=r2, bz_mag=bz_mag)


def ba_graph(ii, jj, t0, t1):
    """graph bookkeeping of ba_cuda (:1345-1353): ts, ii_exp, jj_exp, kx (sorted unique), kk_exp."""
    ts = torch.arange(t0, t1, dtype=torch.long)
    ii_exp = torch.cat([ts, ii]); jj_exp = torch.cat([ts, jj])
    kx, kk_exp = torch.unique(ii_exp, sorted=True, return_inverse=True)
    return ts, ii_exp, jj_exp, kx, kk_exp


def _segsum(data, ix, jx):
    """accum_cuda (:957-1007): out[j] = sum_{n: ix[n]==jx[j]} data[n]."""
    out = torch.zeros((jx.shape[0],) + tuple(data.shape[1:]), dtype=data.dtype)
    lut = {int(k): n for n, k in enumerate(jx.tolist())}
    rows = torch.tensor([lut.get(int(k), -1) for k in ix.tolist()], dtype=torch.long)
    m = rows >= 0
    out.index_add_(0, rows[m], data[m])
    return out


def _solve(A, b, lm, ep, P):
    """SparseBlock::solve (:1201-1222): fp64, diag += ep + lm*diag (Q6), zeros when not SPD.
    ep, lm arrive as C floats in the reference (`const float lm, const float ep`)."""
    lm64 = float(torch.tensor(lm, dtype=torch.float32)); ep64 = float(torch.tensor(ep, dtype=torch.float32))
    L = A.clone()
    dg = torch.diagonal(L)
    dg += ep64 + lm64 * dg.clone()
    try:
        ch = torch.linalg.cholesky(L)
        x = torch.cholesky_solve(b[:, None], ch)[:, 0]
        if not bool(torch.isfinite(x).all()):
            raise RuntimeError("non finite")
        return x.reshape(P, 6), True
    except Exception:
        return torch.zeros(P, 6, dtype=A.dtype), False


def ba_system(terms, disps, disps_sens, eta, ii, jj, t0, t1, motion_only, dtype, drop_nonpositive_c=False):
    """Assemble the reduced pose system exactly like ba_cuda/schur_block (:1385-1415, :1231-1320).
    Returns (A64, b64, aux) with A,b in fp64 BEFORE damping.
    drop_nonpositive_c: Q = 0 where C <= 0, the native rule (INTEGRATION.md section 5), instead of the reference's 1/C."""
    P = t1 - t0
    E = ii.shape[0]
    ts, ii_exp, jj_exp, kx, kk_exp = ba_graph(ii, jj, t0, t1)
    Hs, vs = terms["Hs"], terms["vs"]
    A = torch.zeros(P, 6, P, 6, dtype=torch.float64)
    b = torch.zeros(P, 6, dtype=torch.float64)
    ri = (ii - t0).tolist(); rj = (jj - t0).tolist()
    Hd = Hs.double(); vd = vs.double()
    for e in range(E):                                                    # :1387-1392 (rows/cols < 0 dropped)
        i, j = ri[e], rj[e]
        for blk, (a, c) in enumerate(((i, i), (i, j), (j, i), (j, j))):
            if a >= 0 and c >= 0 and a < P and c < P:
                A[a, :, c, :] += Hd[blk, e]
        if 0 <= i < P: b[i] += vd[0, e]
        if 0 <= j < P: b[j] += vd[1, e]
    A = A.reshape(6 * P, 6 * P); b = b.reshape(6 * P)
    aux = dict(kx=kx, kk_exp=kk_exp, ii_exp=ii_exp, jj_exp=jj_exp, ts=ts)
    if motion_only:
        return A, b, aux
    HW = terms["Cii"].shape[1]
    m = (disps_sens[kx].reshape(-1, HW) > 0).to(dtype)                    # :1406 (Q7)
    alpha = torch.tensor(0.05, dtype=torch.float32).to(dtype)             # `const float alpha = 0.05`
    C = _segsum(terms["Cii"], ii, kx) + m * alpha + (1 - m) * eta.reshape(-1, HW).to(dtype)   # :1407
    w = _segsum(terms["bz"], ii, kx) - m * alpha * (disps[kx] - disps_sens[kx]).reshape(-1, HW)  # :1408
    Q = 1.0 / C                                                           # :1409
    if drop_nonpositive_c:
        Q = torch.where(C > 0, Q, torch.zeros_like(Q))
    Ei = _segsum(terms["Eii"], ii, ts)                                    # :1411  [P,6,HW]
    Erows = torch.cat([Ei, terms["Eij"]], dim=0)                         # :1412  [P+E,6,HW]
    pose = (jj_exp - t0)
    # S and bS (K9/K10): aggregate rows per (pose, depth frame), then E Q E^T per depth frame
    S = torch.zeros(P, P, 6, 6, dtype=torch.float64)                      # [pose, pose, 6, 6]
    bS = torch.zeros(P, 6, dtype=torch.float64)
    M = kx.shape[0]
    in_window = (pose >= 0) & (pose < P)                                  # j in [t0,t1) (:1257; j==t1 is UB, Q8)
    for k in range(M):
        rows = torch.nonzero((kk_exp == k) & in_window)[:, 0]
        if rows.numel() == 0:
            continue
        Ek = Erows[rows]                                                  # [R,6,HW]
        G = torch.einsum("rap,p,sbp->rasb", Ek, Q[k], Ek).double()        # fp32 products like K9 (:1039-1046)
        gv = torch.einsum("rap,p->ra", Ek, Q[k] * w[k]).double()          # K10 (:1084-1087)
        pr = pose[rows]
        R = pr.shape[0]
        S.index_put_((pr[:, None].expand(R, R), pr[None, :].expand(R, R)), G.permute(0, 2, 1, 3), accumulate=True)
        bS.index_add_(0, pr, gv)
    aux.update(C=C, w=w, Q=Q, Erows=Erows, pose=pose)
    return A - S.permute(0, 2, 1, 3).reshape(6 * P, 6 * P), b - bS.reshape(6 * P), aux        # :1184-1186, :1415


def ba(poses, disps, intrinsics, disps_sens, targets, weights, eta, ii, jj, t0, t1,
       iterations, lm, ep, motion_only, dtype=torch.float32, return_info=False):
    """ba_cuda, src/droid_kernels.cu:1323-1443.  In-place on `poses`, `disps` (which keep their own dtype)."""
    P = t1 - t0
    N, ht, wd = disps.shape
    HW = ht * wd
    ii = ii.long(); jj = jj.long()
    dx = dz = None
    ok_all = True
    for _ in range(iterations):
        p_ = poses.to(dtype); d_ = disps.to(dtype)
        terms = ba_edge_terms(p_, d_, intrinsics.to(dtype), targets.to(dtype), weights.to(dtype), ii, jj)
        A, b, aux = ba_system(terms, d_, disps_sens.to(dtype), eta, ii, jj, t0, t1, motion_only, dtype)
        x, ok = _solve(A, b, lm, ep, P)
        ok_all = ok_all and ok
        dx = x.to(dtype) if dtype == torch.float64 else x.float()        # :1213-1214
        if not motion_only:
            kx, Q, w, Erows, pose = aux["kx"], aux["Q"], aux["w"], aux["Erows"], aux["pose"]
            valid = (pose > 0) & (pose < P)                               # EvT6x1_kernel :1114 (Q9: pose t0 skipped)
            dw = torch.zeros(Erows.shape[0], HW, dtype=dtype)
            dw[valid] = torch.einsum("nap,na->np", Erows[valid], dx.to(dtype)[pose[valid]])   # :1117-1122
            dz = Q * (w - _segsum(dw, aux["ii_exp"], kx))                 # :1426
            disps[kx] += dz.reshape(-1, ht, wd).to(disps.dtype)           # K8 :942-955
        t_new, q_new = retr_se3(dx.to(dtype), p_[t0:t1, :3], p_[t0:t1, 3:])   # K7 :907-940
        poses[t0:t1] = torch.cat([t_new, q_new], dim=-1).to(poses.dtype)
    out = [dx, dz]
    return (out, ok_all) if return_info else out
