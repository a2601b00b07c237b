"""fp64 values and first-order running error bounds for training's flow loss and upsample_disp's backward (csrc/geom.cu:
flow_edges_kernel, flow_loss_kernel + flow_loss_reduce_kernel, flow_loss_bwd_kernel + flow_pose_grad_kernel, cvx_upsample_bwd_kernel +
cvx_upsample_gather_kernel), in the kernels' own operation order, on geometry_model's R and decide.

Edge transforms.  Gij = Pj Pi^-1 in lie_math.cuh's order: each quaternion normalised on load, g_inv, g_mul, the product normalised
again, stored in fp32.  Per pixel, reproject_pixel: iproj, droid_se3's act_se3, Z < 0.1f -> 1, proj.  Poses and disparities enter as
the fp32 values the kernel reads, so identity rotations and exact translations give exact transforms (bound 0) and the placed
threshold pixels of flow_loss_cases are decided with certainty.

Loss.  sum_s gamma^(n-1-s) / count * sum v |c1 - c0|, v = (z0 > 0.2f) (disps > 0) (z1 > 0.2f).  Each block of 256 pixels is summed in
fp32 by a 5-level warp tree and 7 sequential additions of the warp partials: first order at most BLOCK_DEPTH u sum |term|
(tests/test_flow_loss_stages_cpu.py derives the constant from that structure and checks it on the host).  The fp64 reduction and pow
are charged FP64_SUM 2^-53 of the magnitudes, the final (float) u |loss|.

Disparity gradient, per pixel.  sum over the pixel's out-edges of cs v (Delta / |Delta|) dc1/dd, Delta = c1 - c0.  The direction's
error is at most min(2, 2 |b_Delta| / |Delta|) plus its fp32 roundings, so pixels where c1 ~ c0 get a wide bound and every other pixel
a tight one.  Where the kernel's c1 and c0 come from bit-identical inputs (iterate equal to the ground truth on both frames of the edge
and at the pixel) Delta is exactly 0 and so is the gradient, as torch's norm gives.

Pose gradient, per frame and component.  Each pixel's actp term, the 256-thread block sums (BLOCK_DEPTH), the fp64 chunk sum, then
-Adj(Gij)^T applied in fp64 to the fp32-stored Gij (renormalised on load) for the source frame, + for the target, in edge order; the
bound follows each component's own sum of magnitudes.

cvx_upsample_backward.  The softmax recomputed with expf (2 ulp, CUDA's documented bound) of the rounded logit gap, as the forward
model treats __expf; below 2^-126 a weight is charged its whole value plus 2 subnormal ulps, below 2^-152 (a factor 4 under
round-to-nearest's 2^-150) it is exactly 0.  The mask gradient p_k (g_j d_k - sum_l p_l g_j d_l) with the cancellation in the bracket,
the per-tap partials sum_j g_j p_k, and the gather over at most 9 taps x 8 sub-rows, zero-padded sources excluded.

Decisions (z0, z1 > 0.2f, disps > 0) use decide(): where the fp64 margin exceeds the bound the kernel must decide as fp64 does.  An
ambiguous decision takes fp64's branch and adds the other branch's whole term (value plus bound) to every bound it reaches.  The
Z < 0.1f clamp only fires where z1 < 0.2 surely, so v = 0 there and its gradient is exactly 0 wherever it is finite."""
import math

import torch

import geometry_model as gm
from geometry_model import R, U, decide

BLOCK_DEPTH = 5 + 7          # flow_block_sum / the backward's red[]: 5 warp-tree levels, then 7 of the 8 serial additions round
FP64_SUM = 64                # fp64 reductions and pow, in units of 2^-53 of the magnitudes summed (chunk counts stay below 2^20)
EXPF_ULP = 2                 # CUDA's expf
THREADS = 256


def f32(x, dev=None):
    """the fp32 value the kernel reads, as fp64"""
    return torch.as_tensor(x).to(dev).float().double()


def chain_edges(N):
    """losses.py's chain graph in the kernel's edge order: e -> (i, j)"""
    out = [(0, 1)]
    for e in range(1, 2 * (N - 1)):
        i = (e + 1) >> 1
        out.append((i, i - 1 if e & 1 else i + 1))
    return out


def out_edges(a, N):
    """flow_loss_bwd_kernel's out-edges of frame a, in its order (to a - 1, then to a + 1)"""
    eo = []
    if a > 0:
        eo.append(2 * a - 1)
    if a < N - 1:
        eo.append(0 if a == 0 else 2 * a)
    return eo


def _sum(terms):
    """sequential R sum in the given order, the first term taken as is (0.f + x is exact)"""
    acc = terms[0]
    for t in terms[1:]:
        acc = acc + t
    return acc


def _zero(like):
    return R(torch.zeros_like(like.v))


# ---- SE3 in lie_math.cuh's order ------------------------------------------------------------------------------------------------
def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _rot(q, p):
    uv = [2.0 * x for x in _cross(q, p)]
    c = _cross(q, uv)
    return [p[k] + q[3] * uv[k] + c[k] for k in range(3)]


def _rot_t(q, p):
    return _rot([-q[0], -q[1], -q[2], q[3]], p)


def _qmul(a, b):
    return [a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
            a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0],
            a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3],
            a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]]


def _qnormalize(q):
    s = 1.0 / (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]).sqrt()
    return [x * s for x in q]


def _load(P):
    """Elem::load of [..., 7] data (R components)"""
    return [P[k] for k in range(3)], _qnormalize([P[3 + k] for k in range(4)])


def _inv(t, q):
    qi = [-q[0], -q[1], -q[2], q[3]]
    r = _rot(qi, t)
    return [-x for x in r], qi


def _mul(X, Y):
    r = _rot(X[1], Y[0])
    return [X[0][k] + r[k] for k in range(3)], _qnormalize(_qmul(X[1], Y[1]))


def edge_transforms(P):
    """flow_edges_kernel for one slot: P [B, N, 7] -> (t, q) lists of R [B, E, 1], the fp32 values it stores"""
    P = P.double()
    N = P.shape[1]
    E = chain_edges(N)
    ii = torch.tensor([i for i, _ in E], device=P.device)
    jj = torch.tensor([j for _, j in E], device=P.device)
    Pi = _load([R(P[:, ii, k, None]) for k in range(7)])
    Pj = _load([R(P[:, jj, k, None]) for k in range(7)])
    return _mul(Pj, _inv(*Pi))


def adj_t(t, q, a):
    """g_adjT: (R^T a_tau, R^T (a_phi - t x a_tau))"""
    c = _cross(t, a[:3])
    return _rot_t(q, a[:3]) + _rot_t(q, [a[3 + k] - c[k] for k in range(3)])


# ---- one pixel of reproject_pixel, vectorised over [B, E, HW] ----------------------------------------------------------------------
def _intr(intr, idx):
    """[B, E, 1] R components fx, fy, cx, cy of frames idx"""
    return [R(intr.double()[:, idx, k, None]) for k in range(4)]


def reproject(G, Ki, Kj, d, ht, wd):
    """-> (c (x, y R), X1 (4 R), z R) of reproject_pixel with T = G"""
    u, v = gm.pixels(ht, wd)
    u, v = u.to(d.device)[None], v.to(d.device)[None]
    Xi = [(R(u) - Ki[2]) / Ki[0], (R(v) - Ki[3]) / Ki[1], R(torch.ones_like(d)), R(d)]
    X = gm.act_se3(G[0], G[1], Xi)
    small = X[2].v < gm.REPROJ_SMALL          # the clamp's branch (only where v = 0 surely: checked by the callers)
    Z = X[2].where(~small, R(torch.ones_like(X[2].v)))
    dd = 1.0 / Z
    c = [Kj[0] * (X[0] * dd) + Kj[2], Kj[1] * (X[1] * dd) + Kj[3]]
    return c, X, small


class Flow:
    """the model of one flow-loss case: c = dict(Ps, disps, poses_est, disps_est, intrinsics) (any dtype, fp32 values used), on `dev`"""

    def __init__(self, c, gamma=0.9, grad=1.0, dev="cpu", fp32_inputs=True):
        self.dev = dev
        cast = (lambda t: f32(t, dev)) if fp32_inputs else (lambda t: torch.as_tensor(t).to(dev).double())  # noqa: E731
        self.Ps, self.disps, self.intr = cast(c["Ps"]), cast(c["disps"]), cast(c["intrinsics"])
        self.poses_est = [cast(p) for p in c["poses_est"]]
        self.disps_est = [cast(x) for x in c["disps_est"]]
        self.B, self.N, self.ht, self.wd = self.disps.shape
        self.n = len(self.poses_est)
        self.hw = self.ht * self.wd
        self.edges = chain_edges(self.N)
        self.E = len(self.edges)
        self.ii = torch.tensor([i for i, _ in self.edges], device=dev)
        self.jj = torch.tensor([j for _, j in self.edges], device=dev)
        self.gamma = float(gamma)
        self.grad = float(torch.tensor(grad, dtype=torch.float32)) if fp32_inputs else float(grad)
        self.count = float(self.B * self.E * self.hw)
        self.Ki, self.Kj = _intr(self.intr, self.ii), _intr(self.intr, self.jj)
        G0 = edge_transforms(self.Ps)
        src = self.disps[:, self.ii].reshape(self.B, self.E, -1)
        self.c0, X0, small0 = reproject(G0, self.Ki, self.Kj, src, self.ht, self.wd)
        zd, zs = decide(X0[2], gm.REPROJ_VALID, ">")
        pos = src > 0
        self.v0 = zd & pos
        self.v0_sure = zs | ~pos
        assert not bool((small0 & self.v0 & self.v0_sure).any()), "a sure valid ground-truth pixel takes the Z < 0.1 clamp"
        self.amb = {"v0": int((~self.v0_sure).sum()), "v1": 0, "1px": 0}

    def weight(self, s):
        return self.gamma ** (self.n - 1 - s)

    def iterate(self, s):
        """per-pixel quantities of iterate s: G, c1, X1, v (fp64), v_sure, dx, dy (R) on [B, E, HW]"""
        G = edge_transforms(self.poses_est[s])
        d = self.disps_est[s][:, self.ii].reshape(self.B, self.E, -1)
        c1, X1, small = reproject(G, self.Ki, self.Kj, d, self.ht, self.wd)
        zd, zs = decide(X1[2], gm.REPROJ_VALID, ">")
        v = self.v0 & zd
        sure = (self.v0_sure & zs) | (self.v0_sure & ~self.v0) | (zs & ~zd)
        assert not bool((small & (v | ~sure)).any()), "the Z < 0.1 clamp where v may be 1"
        dx, dy = c1[0] - self.c0[0], c1[1] - self.c0[1]
        # bit-identical inputs through the same code: c1 == c0 exactly
        same_e = (self.poses_est[s] == self.Ps).all(-1)
        same_e = same_e[:, self.ii] & same_e[:, self.jj]
        same = same_e[..., None] & (self.disps_est[s] == self.disps)[:, self.ii].reshape(self.B, self.E, -1)
        zero = R(torch.zeros_like(dx.v))
        dx, dy = dx.where(~same, zero), dy.where(~same, zero)
        return dict(G=G, c1=c1, X1=X1, v=v, sure=sure, dx=dx, dy=dy, small=small)

    # ---- forward ---------------------------------------------------------------------------------------------------------------
    def forward(self):
        """-> dict(loss R, sum R, count (int), below (int, fp64's), below_amb (int), amb)"""
        lv = torch.zeros((), dtype=torch.float64, device=self.dev)
        lb = torch.zeros_like(lv)
        lm = torch.zeros_like(lv)
        for s in range(self.n):
            it = self.iterate(s)
            nrm = (it["dx"] * it["dx"] + it["dy"] * it["dy"]).sqrt()
            vf = it["v"].double()
            epe = nrm * R(vf)
            t_b = torch.where(it["sure"], epe.b, nrm.v.abs() + nrm.b)
            w = self.weight(s) / self.count
            lv = lv + w * epe.v.sum()
            lb = lb + w * (t_b.sum() + BLOCK_DEPTH * U * epe.v.abs().sum())
            lm = lm + w * (epe.v.abs() + t_b).sum()
            self.amb["v1"] += int((~it["sure"]).sum()) if s == self.n - 1 else 0
            if s == self.n - 1:
                m = it["v"]
                ms = it["sure"]
                sv = torch.where(m, epe.v, torch.zeros_like(epe.v)).sum()
                sb = torch.where(m, t_b, torch.zeros_like(t_b)).sum() + BLOCK_DEPTH * U * torch.where(m | ~ms, epe.v.abs(), torch.zeros_like(epe.v)).sum() \
                    + torch.where(~ms, nrm.v.abs() + nrm.b, torch.zeros_like(nrm.v)).sum()
                bd, bs = decide(epe, 1.0, "<")
                self.metric_sum = R(sv, sb + FP64_SUM * 2.0 ** -53 * sv.abs())
                self.count_sure = int((m & ms).sum())
                self.count_amb = int((~ms).sum())
                self.below = int((m & ms & bd).sum())
                self.below_amb = int((~ms | (m & ~bs)).sum())
                self.amb["1px"] = int((m & ~bs).sum())
        lb = lb + FP64_SUM * 2.0 ** -53 * lm
        self.loss = R(lv, lb).f32()
        return self.loss

    # ---- backward ----------------------------------------------------------------------------------------------------------------
    def backward(self):
        """-> (grad_poses_est [n] of R [B, N, 6], grad_disps_est [n] of R [B, N, HW]); 7th pose entries are 0"""
        gd_out, gp_out = [], []
        for s in range(self.n):
            gd, gp = self.backward_iterate(s)
            gd_out.append(gd)
            gp_out.append(gp)
        return gp_out, gd_out

    def backward_iterate(self, s):
        it = self.iterate(s)
        cs = R(torch.tensor(self.grad * self.weight(s) / self.count, dtype=torch.float64, device=self.dev)).f32()
        vf = it["v"].double()
        csv = cs * R(vf)
        dx, dy = it["dx"], it["dy"]
        n64 = torch.sqrt(dx.v * dx.v + dy.v * dy.v)
        r64 = torch.where(n64 == 0, torch.zeros_like(n64), csv.v / n64)
        bD = torch.sqrt(dx.b * dx.b + dy.b * dy.b)
        # the direction Delta / |Delta| and its fp32 roundings (squares, sum, sqrt, division, product: 6 u)
        bu = torch.where(n64 > 0, torch.clamp(2 * bD / n64.clamp(min=1e-300), max=2.0), torch.where(bD > 0, torch.ones_like(n64), torch.zeros_like(n64)))
        bu = bu + torch.where(bu > 0, 6 * U * torch.ones_like(bu), torch.zeros_like(bu))
        ux, uy = dx.v * r64, dy.v * r64                            # cs v Delta / |Delta|, the kernel's order's value
        dirx = torch.where(n64 > 0, dx.v / n64.clamp(min=1e-300), torch.zeros_like(n64)).abs()
        diry = torch.where(n64 > 0, dy.v / n64.clamp(min=1e-300), torch.zeros_like(n64)).abs()
        # exact structure: exact zero direction where Delta is exact
        exactD = (dx.b == 0) & (dy.b == 0)
        gb = lambda dr: torch.where(exactD & (n64 == 0), torch.zeros_like(n64), csv.v.abs() * bu + dr * csv.b + 3 * U * csv.v.abs() * dr)  # noqa: E731
        gcx, gcy = R(ux, gb(dirx)), R(uy, gb(diry))
        T, q = it["G"]
        X = it["X1"]
        small = it["small"]
        one = R(torch.ones_like(X[2].v))
        idz = 1.0 / X[2].where(~small, one)
        fx, fy = self.Kj[0], self.Kj[1]
        gX = gcx * fx * idz
        gY = gcy * fy * idz
        gZ = (-((gcx * fx * X[0] + gcy * fy * X[1]) * idz * idz)).where(~small, _zero(gX))
        gd_e = gX * T[0] + gY * T[1] + gZ * T[2]
        g6 = [gX * X[3], gY * X[3], gZ * X[3], gZ * X[1] - gY * X[2], gX * X[2] - gZ * X[0], gY * X[0] - gX * X[1]]
        # an ambiguous v: fp64's branch, plus the whole term of the other one
        amb = ~it["sure"]
        if bool(amb.any()):
            alt = self._included(s, it, cs)
            gd_e = R(gd_e.v, gd_e.b + torch.where(amb, alt[0].v.abs() + alt[0].b, torch.zeros_like(gd_e.b)))
            g6 = [R(x.v, x.b + torch.where(amb, a.v.abs() + a.b, torch.zeros_like(x.b))) for x, a in zip(g6, alt[1])]
        # disparity gradient: per source frame, its out-edges in order
        gd = []
        for a in range(self.N):
            eo = out_edges(a, self.N)
            gd.append(_sum([gd_e[:, e] for e in eo]))
        gd = R(torch.stack([x.v for x in gd], 1), torch.stack([x.b for x in gd], 1))
        # edge sums: block trees, fp64 chunk sums
        ge = []
        for x in g6:
            mag = x.v.abs().sum(-1)
            ge.append(R(x.v.sum(-1), x.b.sum(-1) + (BLOCK_DEPTH * U + FP64_SUM * 2.0 ** -53) * mag))
        gp = []
        with R.double():
            Gt = [R(t.v[..., 0], t.b[..., 0]) for t in T]
            Gq = _qnormalize([R(x.v[..., 0], x.b[..., 0]) for x in q])
            for f in range(self.N):
                acc = None
                for e, (i, j) in enumerate(self.edges):
                    if i != f and j != f:
                        continue
                    a6 = [x[:, e] for x in ge]
                    if j == f:
                        term = a6
                    else:
                        term = [-y for y in adj_t([x[:, e] for x in Gt], [x[:, e] for x in Gq], a6)]
                    acc = term if acc is None else [p + t for p, t in zip(acc, term)]
                gp.append(acc)
        gp = [R(torch.stack([gp[f][m].v for f in range(self.N)], 1), torch.stack([gp[f][m].b for f in range(self.N)], 1)).f32() for m in range(6)]
        gp = R(torch.stack([x.v for x in gp], -1), torch.stack([x.b for x in gp], -1))
        return gd, gp

    def _included(self, s, it, cs):
        """the per-pixel terms of iterate s with v = 1 wherever v0 may be 1 (for ambiguous decisions' other branch)"""
        dx, dy = it["dx"], it["dy"]
        n64 = torch.sqrt(dx.v * dx.v + dy.v * dy.v)
        u = lambda d: torch.where(n64 > 0, d.v / n64.clamp(min=1e-300), torch.zeros_like(n64))  # noqa: E731
        gcx = R(cs.v * u(dx), cs.v.abs() * 2.0 + cs.b)
        gcy = R(cs.v * u(dy), cs.v.abs() * 2.0 + cs.b)
        T, X = it["G"][0], it["X1"]
        idz = 1.0 / X[2]
        gX, gY = gcx * self.Kj[0] * idz, gcy * self.Kj[1] * idz
        gZ = -((gcx * self.Kj[0] * X[0] + gcy * self.Kj[1] * X[1]) * idz * idz)
        gd = gX * T[0] + gY * T[1] + gZ * T[2]
        return gd, [gX * X[3], gY * X[3], gZ * X[3], gZ * X[1] - gY * X[2], gX * X[2] - gZ * X[0], gY * X[0] - gX * X[1]]


# ---- cvx_upsample's backward ------------------------------------------------------------------------------------------------------
SUB_ZERO = 2.0 ** -152       # below: expf surely returns 0
NORMAL = 2.0 ** -126


def expf(x):
    """R of expf(x) for an R x: EXPF_ULP ulp (<= 2 u each) and the input's bound (e^x moves by b_x relative); subnormal results
    charged their value plus 2 subnormal ulps; surely below 2^-150 exactly 0"""
    e = torch.exp(x.v)
    b = e * (2 * EXPF_ULP * U + x.b)
    sub = e < NORMAL
    b = torch.where(sub, e + 2.0 ** -148, b)
    zero = torch.exp(x.v + x.b) < SUB_ZERO
    e = torch.where(zero, torch.zeros_like(e), e)
    b = torch.where(zero | torch.isnan(x.v) | (x.v == -math.inf), torch.zeros_like(b), b)
    return R(e, b)


def upsample_backward(disps, mask, gout, dev="cpu", fp32_inputs=True):
    """disps [n, ht, wd], mask [n, 576, ht, wd], gout [n, 8ht, 8wd] (an R or a tensor: the cotangent and its bound) ->
    (grad_disps R [n, ht, wd], grad_mask R [n, 576, ht, wd])"""
    n, ht, wd = disps.shape
    hw = ht * wd
    cast = (lambda t: f32(t, dev)) if fp32_inputs else (lambda t: torch.as_tensor(t).to(dev).double())  # noqa: E731
    d = torch.nn.functional.unfold(cast(disps)[:, None], [3, 3], padding=1).view(n, 9, 1, 1, hw)
    m = cast(mask).reshape(n, 9, 8, 8, hw)                                       # [n, k, i, j, pix]
    g = gout if isinstance(gout, R) else R(cast(gout))
    img = lambda t: t.reshape(n, ht, 8, wd, 8).permute(0, 2, 4, 1, 3).reshape(n, 8, 8, hw)  # noqa: E731
    g = R(img(g.v), img(g.b))[:, None]                                              # [n, 1, i, j, pix]
    mx = torch.full_like(m[:, 0], -math.inf)
    for k in range(9):
        mx = torch.fmax(mx, m[:, k])
    x = R(m) - R(mx[:, None])
    e = expf(x)
    den = _sum([e[:, k] for k in range(9)])
    p = e / den[:, None]
    gdk = g * R(d)                                                                   # g_j d_k
    sp = _sum([p[:, k] * gdk[:, k] for k in range(9)])
    gm_ = p * (gdk - sp[:, None])
    P = _sum([g[:, :, :, j] * p[:, :, :, j] for j in range(8)])                     # [n, k, i, pix]
    gmask = R(gm_.v.reshape(n, 576, ht, wd), gm_.b.reshape(n, 576, ht, wd))
    y = torch.arange(ht, device=dev)[:, None].expand(ht, wd).reshape(-1)
    xx = torch.arange(wd, device=dev)[None, :].expand(ht, wd).reshape(-1)
    acc = None
    for k in range(9):
        sy, sx = y - k // 3 + 1, xx - k % 3 + 1
        ok = (sy >= 0) & (sy < ht) & (sx >= 0) & (sx < wd)
        src = (sy.clamp(0, ht - 1) * wd + sx.clamp(0, wd - 1))
        for i in range(8):
            t = P[:, k, i][:, src]
            if acc is None:
                acc = t.where(ok, _zero(t))
                started = ok.clone()
            else:
                nxt = acc + t
                acc = R(torch.where(ok & started, nxt.v, torch.where(ok, t.v, acc.v)), torch.where(ok & started, nxt.b, torch.where(ok, t.b, acc.b)))
                started = started | ok
    gdisps = R(acc.v.reshape(n, ht, wd), acc.b.reshape(n, ht, wd))
    return gdisps, gmask
