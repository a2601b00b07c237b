"""First-order running error bounds for the geometry kernels (csrc/geom.cu) and cvx_upsample, in each kernel's own operation order.

A value the kernel computes in fp32 is carried as R(v, b): v its fp64 restatement, b a bound on |fp32 result - v|.  Every fp32 rounding
is charged u |result| (u = 2^-24), plus 2^-150 below the normal range where the spacing stops shrinking, except where the operands are exact (b = 0) and the fp64 result is an fp32 number: then the fp32
operation returns it exactly, contracted into an FMA or not.  An FMA rounds once and is covered by the two charges of its product and
sum.  Sums, products and quotients propagate the operands' bounds in the usual way (second-order terms of products included; a
quotient whose divisor's bound reaches the divisor has no bound).  The fp64 value v itself is the kernel's expression evaluated in fp64,
in the same order as oracle/geom.py, which the CPU test checks.

Decisions (a comparison of a bounded value with a constant) are `sure` where the fp64 margin exceeds the bound: the kernel must then
decide as fp64 does.  Inside the window either answer is allowed."""
import contextlib
import math

import torch

U = 2.0 ** -24
F32 = lambda x: float(torch.tensor(x, dtype=torch.float32))   # the fp32 literal of the kernel, as an fp64 number

# the kernels' constants, as they compare (fp32 comparisons use the fp32 literal; `(double)z > 0.25` the double one)
PROJ_Z = 0.01                # projmap: Xj[2] > 0.01f; for fp32 z this decides as z > 0.01 (double) does, the reference's literal
MIN_DEPTH = 0.25             # projmap valid, frame_distance: (double)Z > 0.25
REPROJ_SMALL = F32(0.1)      # reproject: Z < 0.5f * 0.2f (== 0.1f) -> Z := 1
REPROJ_VALID = F32(0.2)      # reproject: Z > 0.2f
FRAC = 0.75                  # frame_distance: (double)vv / ((double)t + 1e-8) < 0.75 -> 1000


def _exact(z):
    return torch.isfinite(z) & (z.float().double() == z)


def _charge(z, b):
    """one fp32 rounding of z (bound b before it): u |z|, and half the smallest subnormal (2^-150) below the normal range, where the
    spacing is fixed; nothing for an exact 0 (a product with an exact 0 operand)"""
    tiny = (z.abs() < 2.0 ** -126) & ((z != 0) | (b > 0))
    return U * z.abs() + torch.where(tiny, torch.full_like(z, 2.0 ** -150), torch.zeros_like(z))


class R:
    """fp64 value and first-order bound of an fp32 kernel value.  Inside `with R.double():` each operation is the kernel's fp64
    arithmetic instead: it propagates the operands' bounds and charges 2^-53 |result| for its own rounding, exact operands or not
    (an fp64 FMA may round where the host does not)."""
    __slots__ = ("v", "b")
    u = U

    def __init__(self, v, b=None):
        self.v = torch.as_tensor(v, dtype=torch.float64)
        self.b = torch.zeros_like(self.v) if b is None else torch.as_tensor(b, dtype=torch.float64)

    @staticmethod
    def lift(x):
        return x if isinstance(x, R) else R(x)

    @staticmethod
    @contextlib.contextmanager
    def double():
        R.u = 2.0 ** -53
        try:
            yield
        finally:
            R.u = U

    def f32(self):
        """the kernel's (float) of an fp64 value"""
        return R(self.v, self.b + torch.where(_exact(self.v), torch.zeros_like(self.v), _charge(self.v, self.b)))

    def _rounded(self, z, b, x, y):
        if R.u != U:
            return R(z, b + R.u * z.abs())
        exact = (x.b == 0) & (y.b == 0) & _exact(z)
        return R(z, b + torch.where(exact, torch.zeros_like(z), _charge(z, b)))

    def __add__(self, y):
        y = R.lift(y)
        return self._rounded(self.v + y.v, self.b + y.b, self, y)

    __radd__ = __add__

    def __sub__(self, y):
        y = R.lift(y)
        return self._rounded(self.v - y.v, self.b + y.b, self, y)

    def __rsub__(self, x):
        return R.lift(x) - self

    def __neg__(self):
        return R(-self.v, self.b)

    def __mul__(self, y):
        y = R.lift(y)
        return self._rounded(self.v * y.v, self.v.abs() * y.b + y.v.abs() * self.b + self.b * y.b, self, y)

    __rmul__ = __mul__

    def __truediv__(self, y):
        y = R.lift(y)
        z = self.v / y.v
        room = y.v.abs() - y.b
        b = torch.where(room > 0, (self.b + z.abs() * y.b) / room.clamp(min=1e-300), torch.full_like(z, math.inf))
        b = torch.where(y.b == 0, self.b / y.v.abs(), b)
        return self._rounded(z, b, self, y)

    def __rtruediv__(self, x):
        return R.lift(x) / self

    def sqrt(self):
        z = torch.sqrt(self.v)
        b = self.b / (z + torch.sqrt((self.v - self.b).clamp(min=0)))
        b = torch.where(self.b == 0, torch.zeros_like(z), b)
        return self._rounded(z, b, self, R(0.0))

    def where(self, cond, other):
        other = R.lift(other)
        return R(torch.where(cond, self.v, other.v), torch.where(cond, self.b, other.b))

    def __getitem__(self, i):
        return R(self.v[i], self.b[i])


def decide(x, thr, op):
    """(fp64 decision, sure) for `x op thr` with x an R.  An exact x (b = 0) is the kernel's value, so its decision is sure; so is a
    non-finite one, which the kernel's fp32 evaluation reproduces (NaN compares false in both)."""
    d = x.v > thr if op == ">" else x.v < thr
    margin = (x.v - thr).abs()
    sure = (margin > x.b) | (x.b == 0) | ~torch.isfinite(x.v)
    return d, sure


# ---- SE3 in the order of droid_se3.cuh ---------------------------------------------------------------------------------------
def act_so3(q, X):
    uv0 = 2.0 * (q[1] * X[2] - q[2] * X[1])
    uv1 = 2.0 * (q[2] * X[0] - q[0] * X[2])
    uv2 = 2.0 * (q[0] * X[1] - q[1] * X[0])
    return [X[0] + q[3] * uv0 + (q[1] * uv2 - q[2] * uv1),
            X[1] + q[3] * uv1 + (q[2] * uv0 - q[0] * uv2),
            X[2] + q[3] * uv2 + (q[0] * uv1 - q[1] * uv0)]


def act_se3(t, q, X):
    Y = act_so3(q, X)
    return [Y[0] + X[3] * t[0], Y[1] + X[3] * t[1], Y[2] + X[3] * t[2], X[3]]


def rel_se3(ti, qi, tj, qj):
    q = [-qj[3] * qi[0] + qj[0] * qi[3] - qj[1] * qi[2] + qj[2] * qi[1],
         -qj[3] * qi[1] + qj[1] * qi[3] - qj[2] * qi[0] + qj[0] * qi[2],
         -qj[3] * qi[2] + qj[2] * qi[3] - qj[0] * qi[1] + qj[1] * qi[0],
         qj[3] * qi[3] + qj[0] * qi[0] + qj[1] * qi[1] + qj[2] * qi[2]]
    Y = act_so3(q, ti)
    return [tj[0] - Y[0], tj[1] - Y[1], tj[2] - Y[2]], q


def edge_transform(poses, ii, jj, stereo_quirk):
    """per edge [E, 1] components of (tij, qij); the stereo constant is exact"""
    P = poses.double()
    col = lambda idx, k: R(P[idx, k][:, None])
    t, q = rel_se3([col(ii, k) for k in range(3)], [col(ii, 3 + k) for k in range(4)],
                   [col(jj, k) for k in range(3)], [col(jj, 3 + k) for k in range(4)])
    if stereo_quirk:
        s = (ii == jj)[:, None]
        t = [x.where(~s, R(torch.full_like(x.v, c))) for x, c in zip(t, (F32(-0.1), 0.0, 0.0))]
        q = [x.where(~s, R(torch.full_like(x.v, c))) for x, c in zip(q, (0.0, 0.0, 0.0, 1.0))]
    return t, q


def pixels(ht, wd):
    v, u = torch.meshgrid(torch.arange(ht, dtype=torch.float64), torch.arange(wd, dtype=torch.float64), indexing="ij")
    return u.reshape(1, -1), v.reshape(1, -1)


def backproject(d, K, ht, wd):
    """Xi = ((u - cx) / fx, (v - cy) / fy, 1, d); K: 4 tensors broadcasting against [*, HW]"""
    u, v = pixels(ht, wd)
    fx, fy, cx, cy = [R(k) for k in K]
    return [(R(u) - cx) / fx, (R(v) - cy) / fy, R(torch.ones_like(u)), R(d.double())]


def _K(intr):
    return [intr.double()[..., k] for k in range(4)]


# ---- the kernels ---------------------------------------------------------------------------------------------------------------
def projmap(poses, disps, intr, ii, jj):
    """dict: Z (R), cu / cv (R, the projected branch), u / v (the fallback); all [E, HW]"""
    N, ht, wd = disps.shape
    t, q = edge_transform(poses, ii, jj, False)
    Xi = backproject(disps[ii].reshape(len(ii), -1), _K(intr), ht, wd)
    Xj = act_se3(t, q, Xi)
    fx, fy, cx, cy = [R(k) for k in _K(intr)]
    u, v = pixels(ht, wd)
    return dict(Z=Xj[2], cu=fx * (Xj[0] / Xj[2]) + cx, cv=fy * (Xj[1] / Xj[2]) + cy, u=u, v=v)


def iproj(poses, disps, intr):
    n, ht, wd = disps.shape
    P = poses.double()[:n]
    Xi = backproject(disps.reshape(n, -1), _K(intr), ht, wd)
    Xj = act_se3([R(P[:, k, None]) for k in range(3)], [R(P[:, 3 + k, None]) for k in range(4)], Xi)
    return [Xj[k] / Xj[3] for k in range(3)]


def reproject(poses, disps, intr_pf, ii, jj):
    """dict: Z (R), x / y (R, Z kept), x1 / y1 (R, Z := 1); [E, HW]"""
    N, ht, wd = disps.shape
    t, q = edge_transform(poses, ii, jj, True)
    Ki, Kj = _K(intr_pf[ii][:, None]), [R(k) for k in _K(intr_pf[jj][:, None])]
    Xi = backproject(disps[ii].reshape(len(ii), -1), Ki, ht, wd)
    Xj = act_se3(t, q, Xi)
    d = 1.0 / Xj[2]
    out = dict(Z=Xj[2], x=Kj[0] * (Xj[0] * d) + Kj[2], y=Kj[1] * (Xj[1] * d) + Kj[3])
    out["x1"] = Kj[0] * (Xj[0] * 1.0) + Kj[2]
    out["y1"] = Kj[1] * (Xj[1] * 1.0) + Kj[3]
    return out


def frame_distance(poses, disps, intr, ii, jj, beta):
    """dict per pair: dist (R, where the pair is not 1000), ratio (R, vv / (t + 1e-8)), ambiguous pixel decisions.  The sums' bound:
    each thread adds 2 ceil(hw / 256) terms in sequence, then 5 warp-tree levels and the 8 warp partials; first order the error is
    at most depth u sum |term|.  Sums of terms that are all 0, 1/2 or 1 stay exact (beta in {0, 1/2, 1} and hw < 2^22)."""
    N, ht, wd = disps.shape
    hw = ht * wd
    E = len(ii)
    b32 = R(F32(beta))
    wb = [b32, 1.0 - b32]                    # `beta`, `(1 - beta)` in fp32
    if hw == 0:
        z = torch.zeros(E, dtype=torch.float64)
        return dict(ratio=R(z), dist=R(z), amb=torch.zeros(E, dtype=torch.long), vv=R(z), t=R(z))
    t, q = edge_transform(poses, ii, jj, False)
    K = _K(intr)
    fx, fy, cx, cy = [R(k) for k in K]
    Xi = backproject(disps[ii].reshape(E, -1), K, ht, wd)
    u, v = pixels(ht, wd)
    full = act_se3(t, q, Xi)
    trans = [Xi[0] + Xi[3] * t[0], Xi[1] + Xi[3] * t[1], Xi[2] + Xi[3] * t[2]]
    depth = 2 * -(-hw // 256) + 5 + 8
    acc_v = torch.zeros(E, dtype=torch.float64); acc_b = torch.zeros(E, dtype=torch.float64); acc_m = torch.zeros(E, dtype=torch.float64)
    vv_v = torch.zeros(E, dtype=torch.float64); vv_b = torch.zeros(E, dtype=torch.float64)
    amb = torch.zeros(E, dtype=torch.long)
    for Xj, w in zip((full, trans), wb):
        du = fx * (Xj[0] / Xj[2]) + cx - R(u)
        dv = fy * (Xj[1] / Xj[2]) + cy - R(v)
        d = (du * du + dv * dv).sqrt()
        term = w * d
        ok, sure = decide(Xj[2], MIN_DEPTH, ">")
        inc = ok & sure
        tv = torch.where(inc, term.v, torch.zeros_like(term.v))
        acc_v += tv.sum(1)
        acc_b += torch.where(inc, term.b, torch.zeros_like(term.b)).sum(1) + torch.where(~sure, term.v.abs() + term.b, torch.zeros_like(term.v)).sum(1)
        acc_m += torch.where(inc | ~sure, term.v.abs() + term.b, torch.zeros_like(term.v)).sum(1)
        vv_v += inc.double().sum(1) * w.v
        vv_b += (~sure).double().sum(1) * (w.v.abs() + w.b) + inc.double().sum(1) * w.b
        amb += (~sure).sum(1)
    exact_w = F32(beta) in (0.0, 0.5, 1.0)
    acc = R(acc_v, acc_b + depth * U * acc_m)
    vv = R(vv_v, vv_b + (0.0 if exact_w else depth * U * (vv_v.abs() + vv_b)))
    tot_v = hw * (wb[0].v + wb[1].v)
    tot_b = hw * (wb[0].b + wb[1].b) + (0.0 if exact_w else depth * U * tot_v)
    tt = R(torch.full((E,), float(tot_v), dtype=torch.float64), torch.full((E,), float(tot_b), dtype=torch.float64))
    ratio_v = vv.v / (tt.v + 1e-8)
    ratio_b = (vv.b + ratio_v.abs() * tt.b) / (tt.v + 1e-8 - tt.b).clamp(min=1e-300) + 4 * 2.0 ** -53 * ratio_v.abs()
    return dict(ratio=R(ratio_v, ratio_b), dist=acc / vv, amb=amb, vv=vv, t=tt)


def floor_cells(x):
    """candidate values of __float2int_rd(x32) for x an R: (lo, hi, sure); NaN -> 0 (sure), saturating at +-2^31"""
    lo = torch.floor(x.v - x.b)
    hi = torch.floor(x.v + x.b)
    nan = torch.isnan(x.v)
    lo = torch.where(nan, torch.zeros_like(lo), lo).clamp(-2.0 ** 31, 2.0 ** 31 - 1)
    hi = torch.where(nan, torch.zeros_like(hi), hi).clamp(-2.0 ** 31, 2.0 ** 31 - 1)
    return lo, hi, lo == hi


def depth_filter(poses, disps, intr, ix, thresh):
    """(sure hits, possible hits) per [B, HW]: every neighbour contributes 1 to `sure` if it hits whichever cell floor picks and
    whichever way each comparison within the bound goes, and 1 to `possible` if some admissible choice hits."""
    num, ht, wd = disps.shape
    hw = ht * wd
    B = len(ix)
    D = disps.double().reshape(num, -1)
    K = _K(intr)
    fx, fy, cx, cy = [R(k) for k in K]
    t64 = thresh.double()[:, None]
    sure = torch.zeros(B, hw, dtype=torch.float64)
    poss = torch.zeros(B, hw, dtype=torch.float64)
    amb_cells = 0
    Xi = backproject(D[ix], K, ht, wd)
    for neigh in range(6):
        jx = ix - neigh - 1 if neigh < 3 else ix + neigh
        ok = (jx >= 0) & (jx < num)
        jc = jx.clamp(0, num - 1)
        t, q = edge_transform(poses, ix, jc, False)
        Xj = act_se3(t, q, Xi)
        uj = fx * (Xj[0] / Xj[2]) + cx
        vj = fy * (Xj[1] / Xj[2]) + cy
        dj = Xj[3] / Xj[2]
        idj = 1.0 / dj.v
        idj_b = torch.where(dj.b == 0, torch.zeros_like(idj), dj.b / (dj.v.abs() * (dj.v.abs() - dj.b).clamp(min=0)))
        idj_b = torch.where(dj.v.abs() > dj.b, idj_b, torch.full_like(idj, math.inf))
        idj_b = torch.where(dj.b == 0, torch.zeros_like(idj), idj_b + 2.0 ** -52 * idj.abs())   # + the fp64 division's own rounding
        ulo, uhi, usure = floor_cells(uj)
        vlo, vhi, vsure = floor_cells(vj)
        amb_cells += int((ok[:, None] & ~(usure & vsure)).sum())
        wide = (uhi - ulo > 1) | (vhi - vlo > 1)       # more than two candidate columns or rows: no decision is sure
        s_any = torch.ones(B, hw, dtype=torch.bool)
        p_any = torch.zeros(B, hw, dtype=torch.bool)
        for u0 in (ulo, uhi):
            for v0 in (vlo, vhi):
                inb = (u0 >= 0) & (v0 >= 0) & (u0 < wd - 1) & (v0 < ht - 1)
                uu, vv_ = u0.clamp(0, max(wd - 2, 0)).long(), v0.clamp(0, max(ht - 2, 0)).long()
                hs = torch.zeros(B, hw, dtype=torch.bool)
                hp = torch.zeros(B, hw, dtype=torch.bool)
                for a, c in ((0, 0), (0, 1), (1, 0), (1, 1)):
                    idx = ((vv_ + a) * wd + (uu + c)).clamp(max=hw - 1)
                    dk = torch.gather(D[jc], 1, idx)
                    diff = (idj - 1.0 / dk).abs()
                    hit = diff < t64
                    # the comparison is fp64 on fp64 values of fp32 inputs: only idj carries a bound
                    amb = (diff - t64).abs() < idj_b
                    hs |= hit & ~amb
                    hp |= hit | amb
                s_any &= inb & hs
                p_any |= inb & hp
        ok2 = ok[:, None]
        sure += (ok2 & s_any & ~wide).double()
        poss += (ok2 & (p_any | wide)).double()
    return sure.reshape(B, ht, wd), poss.reshape(B, ht, wd), amb_cells


# ---- cvx_upsample ----------------------------------------------------------------------------------------------------------------
def _taps(disps, mask):
    """d [n, 9, 1, HW] (zero padding) and the fp32 mask values [n, 9, 64, HW]"""
    n, ht, wd = disps.shape
    d = torch.nn.functional.unfold(disps[:, None].double(), [3, 3], padding=1).view(n, 9, 1, ht * wd)
    m = mask.float().double().reshape(n, 9, 64, ht * wd)
    return d, m


def _to_image(x, n, ht, wd):
    """[n, 64 (= i*8 + j), HW] -> [n, 8ht, 8wd]"""
    return x.view(n, 8, 8, ht, wd).permute(0, 3, 1, 4, 2).reshape(n, 8 * ht, 8 * wd)


def cvx_upsample(disps, mask):
    """(fp64 value, bound) [n, 8ht, 8wd].  __expf's documented error, 2 + floor(1.16 |x|) ulp (<= 2u each), plus its input's rounding
    u |x| (x = v_k - max: e^x moves by |x| u relative), gives each weight a relative error delta_k; first order the result moves by at
    most sum_k w_k delta_k |d_k - res|.  Products, the 9-term sums and the division add 10 u sum w_k |d_k| + 10 u |res|.  A tap whose
    exp is below the fp32 normal range may be flushed to 0: delta_k = 1 there."""
    n, ht, wd = disps.shape
    d, m = _taps(disps, mask)
    mx = m.max(1, keepdim=True).values
    x = m - mx
    x_exact = _exact(x)
    w = torch.softmax(m, dim=1)
    res = (w * d).sum(1)
    delta = (2 + torch.floor(1.16 * x.abs())) * 2 * U + torch.where(x_exact, torch.zeros_like(x), U * x.abs())
    delta = torch.where(torch.exp(x) < 2.0 ** -126, torch.ones_like(delta), delta)
    b = (w * delta * (d - res[:, None]).abs()).sum(1) + 10 * U * (w * d.abs()).sum(1) + 10 * U * res.abs()
    return _to_image(res, n, ht, wd), _to_image(b, n, ht, wd)


def cvx_upsample_f32(disps, mask, exp=torch.exp):
    """the kernel's loop in fp32 on the host (max, then den += e, num += e d, res = num / den), with `exp` in place of __expf"""
    n, ht, wd = disps.shape
    d = torch.nn.functional.unfold(disps[:, None].float(), [3, 3], padding=1).view(n, 9, 1, ht * wd)
    m = mask.float().reshape(n, 9, 64, ht * wd)
    mx = torch.full_like(m[:, 0], -math.inf)
    for k in range(9):
        mx = torch.fmax(mx, m[:, k])
    num = torch.zeros_like(mx); den = torch.zeros_like(mx)
    for k in range(9):
        e = exp(m[:, k] - mx)
        den = den + e
        num = num + e * d[:, k]
    return _to_image(num / den, n, ht, wd)
