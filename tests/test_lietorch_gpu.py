"""droid_slam_b200.lietorch on the device (csrc/lie.cu): every forward against the pure-PyTorch stand-in (oracle/shims/lietorch) in fp64,
every backward against the gradient oracle (oracle/lie_grad.py), broadcasting in the kernel at the projective_transform shapes, the
Python API, host synchronisations, and the reprojection of projective_transform rebuilt on the package against the reference's stored
outputs."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from droid_slam_b200 import lietorch as lt  # noqa: E402
from oracle import lie_grad as lg  # noqa: E402
from util import host_syncs  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"
F64, F32 = torch.float64, torch.float32
OPS_FWD = ("exp", "log", "inv", "mul", "adj", "adjT", "Jinv", "act", "act4")
EPS = 1e-6
# fp32: every op is a fixed chain of a few dozen roundings on values of the data's scale, so its error is a small multiple of the unit
# roundoff u = 2^-24 times that scale: 64 u = 3.8e-6 per record, against the stand-in run in fp64 on the same fp32-rounded inputs.  log
# near theta = pi needs nothing more: atan(n / w) is well conditioned for large n / w (its absolute error is about 2 u w / n).  The one
# addition is `conditioning` below, per record, where lietorch's closed forms cancel.
U32 = 2.0 ** -24
BOUND32 = 64 * U32


def G_(group):
    return {"SO3": lt.SO3, "SE3": lt.SE3}[group]


def _tangent(n, K, theta, g):
    """tangents whose rotation part has angle exactly theta (random axes), translation parts O(1)"""
    axis = torch.randn(n, 3, generator=g, dtype=F64)
    phi = axis / axis.norm(dim=-1, keepdim=True) * theta
    return torch.cat([torch.randn(n, 3, generator=g, dtype=F64), phi], -1) if K == 6 else phi


def edge_cases(group, g):
    """tangents and data: angles just below, at and above EPS, near pi, w near 0 of both signs, non-unit quaternions"""
    K = G_(group).manifold_dim
    thetas = [0.5 * EPS, 0.999 * EPS, EPS, 1.001 * EPS, 2 * EPS, 1e-3, 0.3, 1.0, 2.5, math.pi - 1e-3, math.pi - 1e-7]
    a = torch.cat([_tangent(4, K, th, g) for th in thetas])
    X = lg.cls(group).exp(a).data.clone()
    q = X[..., -4:]
    # w near 0 of both signs (|w| a little above and below EPS) and non-unit scales
    w_small = torch.tensor([2e-6, -2e-6, 5e-7, -5e-7], dtype=F64)
    v = torch.randn(4, 3, generator=g, dtype=F64)
    v = v / v.norm(dim=-1, keepdim=True) * (1 - w_small[:, None] ** 2).sqrt()
    extra = torch.cat([v, w_small[:, None]], -1)
    if K == 6:
        extra = torch.cat([torch.randn(4, 3, generator=g, dtype=F64), extra], -1)
    X = torch.cat([X, extra])
    X[-8:, -4:] *= torch.linspace(0.5, 2.0, 8, dtype=F64)[:, None]       # non-unit quaternions (normalised on load)
    return a, X


def shim_fwd(group, op, a, b=None):
    G = lg.cls(group)
    if op == "exp":
        return G.exp(a).data
    X = G(a)
    if op == "log":
        return X.log()
    if op == "inv":
        return X.inv().data
    if op == "mul":
        return (X * G(b)).data
    if op == "act" or op == "act4":
        return X.act(b)
    if op == "Jinv":
        ph = X.log()
        if group == "SO3":
            return (lg.shim._left_jacobian_inverse(ph) @ b[..., None])[..., 0]
        return (lg.left_jacobian_inverse(G, ph) @ b[..., None])[..., 0]
    Ad = lg.adj_matrix(G, a.expand(*torch.broadcast_shapes(a.shape[:-1], b.shape[:-1]), a.shape[-1]))
    M = Ad if op == "adj" else Ad.transpose(-1, -2)
    return (M @ b[..., None])[..., 0]


def native_fwd(group, op, a, b=None):
    G = G_(group)
    if op == "exp":
        return G.exp(a).data
    X = G(a)
    return {"log": lambda: X.log(), "inv": lambda: X.inv().data, "mul": lambda: (X * G(b)).data, "adj": lambda: X.adj(b),
            "adjT": lambda: X.adjT(b), "Jinv": lambda: X.Jinv(b), "act": lambda: X.act(b), "act4": lambda: X.act(b)}[op]()


def operands(group, op, n, g, a=None, X=None):
    G = lg.cls(group)
    K = G.manifold_dim
    if a is None:
        a = _tangent(n, K, 1.0, g) * torch.rand(n, 1, generator=g, dtype=F64)
    if X is None:
        X = G.exp(a).data
    if op == "exp":
        return a, None
    if op in ("log", "inv"):
        return X, None
    b = {"mul": lambda: G.exp(torch.randn(X.shape[0], K, generator=g, dtype=F64)).data, "act": lambda: torch.randn(X.shape[0], 3, generator=g, dtype=F64),
         "act4": lambda: torch.randn(X.shape[0], 4, generator=g, dtype=F64)}.get(op, lambda: torch.randn(X.shape[0], K, generator=g, dtype=F64))()
    return X, b


def check_close(got, want, bound, what):
    """|got - want| <= bound times max(1, the largest entry of want's record); bound: a number or one per record ([..., 1])"""
    scale = want.abs().amax(-1, keepdim=True).clamp(min=1.0)
    r = ((got.detach().double().cpu() - want.cpu()) / scale).abs() / torch.as_tensor(bound, dtype=F64)
    err = float(r.max()) if want.numel() else 0.0
    assert err <= 1.0, (what, "max error / bound", err)
    return err


def conditioning(group, op, A, u, backward=False):
    """the error lietorch's own closed forms carry, per record, where they take the branch at angles t >= EPS and subtract nearly equal
    terms: (1 - cos t) / t^2 in the left Jacobian has an absolute error of u / t^2 against terms of size t |tau| (error u |tau| / t), the
    coefficient (t^2 + 2 cos t - 2) / (2 t^4) of SE3's Q block u / t^4 against terms of size t^2 |tau| (error u |tau| / t^2).  So
    u (1 + |tau|) / t^p with p = 2 where Q enters (SE3: Jinv, the backward of exp and log), else 1; t the rotation angle of the tangent
    (exp) or of log X (log, Jinv).  Below EPS the Taylor branches do not cancel: 0.  Other ops: 0.  The band of 8 fp32 ulps below EPS
    covers a kernel that computes t in fp32 and takes the branch a rounding away."""
    if op not in ("exp", "log", "Jinv"):
        return torch.zeros(A.shape[:-1] + (1,), dtype=F64)
    x = A if op == "exp" else lg.cls(group)(A).log()
    th = x[..., -3:].norm(dim=-1, keepdim=True)
    tau = x[..., :3].norm(dim=-1, keepdim=True) if group == "SE3" else torch.zeros_like(th)
    p = 2 if group == "SE3" and (op == "Jinv" or backward) else 1
    cancels = th >= EPS * (1 - 8 * U32)
    return torch.where(cancels, u * (1 + tau) / th.clamp(min=EPS / 2) ** p, torch.zeros_like(th))


@pytest.mark.parametrize("group", ["SO3", "SE3"])
@pytest.mark.parametrize("op", OPS_FWD)
def test_forward_edge_cases_against_the_stand_in(group, op):
    g = torch.Generator().manual_seed(1)
    a, X = edge_cases(group, g)
    A, B = operands(group, op, 0, g, a=a, X=X)
    want = shim_fwd(group, op, A, B)
    got64 = native_fwd(group, op, A.to(dev), None if B is None else B.to(dev))
    check_close(got64, want, 1e-12 + 16 * conditioning(group, op, A, 2.0 ** -53), (group, op, "fp64"))
    got32 = native_fwd(group, op, A.float().to(dev), None if B is None else B.float().to(dev))
    A32 = A.float().double()
    want32 = shim_fwd(group, op, A32, None if B is None else B.float().double())
    check_close(got32, want32, BOUND32 + 16 * conditioning(group, op, A32, U32), (group, op, "fp32"))


SHAPES = [((), ()), ((0,), (0,)), ((5,), (5,)), ((1,), (6,)), ((6,), (1,)), ((1, 7, 1, 1), (1, 7, 3, 5)), ((1, 7, 3, 5), (1, 7, 1, 1)),
          ((2, 1, 3), (1, 4, 3)), ((2, 1, 1, 2, 1, 1, 2, 1), (1, 2, 3, 1, 1, 2, 1, 2))]


@pytest.mark.parametrize("group", ["SO3", "SE3"])
@pytest.mark.parametrize("op", ["mul", "adj", "adjT", "Jinv", "act", "act4"])
@pytest.mark.parametrize("shapes", SHAPES, ids=[str(s) for s in SHAPES])
def test_forward_broadcast_shapes(group, op, shapes):
    g = torch.Generator().manual_seed(2)
    G = lg.cls(group)
    K = G.manifold_dim
    sa, sb = shapes
    X = G.exp(torch.randn(*sa, K, generator=g, dtype=F64)).data
    db = {"mul": G.embedded_dim, "act": 3, "act4": 4}.get(op, K)
    b = torch.randn(*sb, db, generator=g, dtype=F64)
    if op == "mul":
        b = G.exp(torch.randn(*sb, K, generator=g, dtype=F64)).data
    want = shim_fwd(group, op, X, b) if op != "Jinv" else shim_fwd(group, op, *[t.expand(*torch.broadcast_shapes(sa, sb), t.shape[-1]) for t in (X, b)])
    got = native_fwd(group, op, X.to(dev), b.to(dev))
    assert got.shape == want.shape, (got.shape, want.shape)
    check_close(got, want, 1e-12, (group, op, shapes))


def _backward(group, op, a, b, g):
    """native gradients of op at (a, b) for the upstream gradient g (through the autograd Functions)"""
    G = G_(group)
    a = a.clone().requires_grad_(True)
    b = None if b is None else b.clone().requires_grad_(True)
    if op == "vec":
        out = G(a).vec()
    elif op == "fromvec":
        out = G.InitFromVec(a).data
    else:
        out = native_fwd(group, op, a, b)
    torch.autograd.backward(out, g)
    return a.grad, None if b is None else b.grad


BWD_OPS = ("exp", "log", "inv", "mul", "adj", "adjT", "act", "act4", "vec", "fromvec")


def _upstream(group, op, shape, gen):
    G = lg.cls(group)
    n = {"exp": G.embedded_dim, "inv": G.embedded_dim, "mul": G.embedded_dim, "fromvec": G.embedded_dim, "vec": G.embedded_dim,
         "log": G.manifold_dim, "adj": G.manifold_dim, "adjT": G.manifold_dim, "act": 3, "act4": 4}[op]
    u = torch.randn(*shape, n, generator=gen, dtype=F64)
    if op in lg.GROUP_OUT:
        u[..., G.manifold_dim:] = 0
    return u


@pytest.mark.parametrize("group", ["SO3", "SE3"])
@pytest.mark.parametrize("op", BWD_OPS)
def test_backward_against_the_oracle(group, op):
    gen = torch.Generator().manual_seed(3)
    a, X = edge_cases(group, gen)
    if op == "log":
        # |w| < EPS: the stand-in's log is pi / |v| there, flat in w, so autograd through it is not the log's derivative; lietorch's
        # backward (and this one) uses Jl(log X)^-1 throughout
        w = lg.shim._qnorm(X[..., -4:])[..., 3].abs()
        X = X[w >= EPS]
    A, B = operands(group, op if op not in ("vec", "fromvec") else "log", 0, gen, a=a if op == "exp" else None, X=X)
    u = _upstream(group, op, A.shape[:-1], gen)
    want = lg.autograd_grad(group, op, A, B, u)
    got = _backward(group, op, A.to(dev), None if B is None else B.to(dev), u.to(dev))
    for k, (x, y) in enumerate(zip(got, want)):
        if y is not None:
            check_close(x, y, 1e-10 + 16 * conditioning(group, op, A, 2.0 ** -53, True), (group, op, "fp64", k))
    got32 = _backward(group, op, A.float().to(dev), None if B is None else B.float().to(dev), u.float().to(dev))
    A32 = A.float().double()
    want32 = lg.autograd_grad(group, op, A32, None if B is None else B.float().double(), u.float().double())
    for k, (x, y) in enumerate(zip(got32, want32)):
        if y is not None:
            # a backward is a forward-sized chain plus a Jacobian product: 4x the forward's fixed bound
            check_close(x, y, 4 * BOUND32 + 16 * conditioning(group, op, A32, U32, True), (group, op, "fp32", k))


@pytest.mark.parametrize("group", ["SO3", "SE3"])
@pytest.mark.parametrize("op", ["mul", "adj", "adjT", "act", "act4"])
@pytest.mark.parametrize("shapes", SHAPES[2:], ids=[str(s) for s in SHAPES[2:]])
def test_backward_broadcast_reduction(group, op, shapes):
    gen = torch.Generator().manual_seed(4)
    G = lg.cls(group)
    sa, sb = shapes
    X = G.exp(torch.randn(*sa, G.manifold_dim, generator=gen, dtype=F64)).data
    db = {"mul": G.embedded_dim, "act": 3, "act4": 4}.get(op, G.manifold_dim)
    b = torch.randn(*sb, db, generator=gen, dtype=F64) if op != "mul" else G.exp(torch.randn(*sb, G.manifold_dim, generator=gen, dtype=F64)).data
    u = _upstream(group, op, torch.broadcast_shapes(sa, sb), gen)
    want = lg.autograd_grad(group, op, X, b, u)
    got = _backward(group, op, X.to(dev), b.to(dev), u.to(dev))
    for k, (x, y) in enumerate(zip(got, want)):
        assert x.shape == y.shape
        check_close(x, y, 1e-10, (group, op, shapes, k))


@pytest.mark.parametrize("op", ["act4", "adjT"])
def test_projective_transform_shapes_reduce_per_edge_and_reproducibly(op):
    """E = 512 edges of 48x64 pixels: act4 of Gij [1,E,1,1] on [1,E,ht,wd,4], adjT of Gij [1,E,1,1,1] on the Jacobians [1,E,ht,wd,2,6];
    the per-edge gradient summed in the launch equals the oracle's, and two runs give identical bits"""
    E, ht, wd = 512, 48, 64
    gen = torch.Generator(device=dev).manual_seed(5)
    a = 0.3 * torch.randn(1, E, 6, generator=gen, dtype=F64, device=dev)
    X = lg.shim.SE3.exp(a).data
    if op == "act4":
        Xb, p = X[:, :, None, None], torch.randn(1, E, ht, wd, 4, generator=gen, dtype=F64, device=dev)
    else:
        Xb, p = X[:, :, None, None, None], torch.randn(1, E, ht, wd, 2, 6, generator=gen, dtype=F64, device=dev)
    u = torch.randn(p.shape, generator=gen, dtype=F64, device=dev)
    want = lg.closed_grad("SE3", op, Xb, p, u)                        # the closed forms, held equal to autograd (test_lietorch_cpu.py)
    terms = lg.closed_grad("SE3", op, Xb.expand(*p.shape[:-1], 7), p, u)[0]
    mag = [lg._sum_to(terms.abs(), Xb.shape), want[1].abs()]           # the sum of the summed terms' magnitudes, per edge
    del terms
    # fp32: each term is a fixed chain of roundings (64 u of its magnitude covers it), the per-edge sum adds at most u per term and level
    for dt, bound in ((F64, 1e-10), (F32, 64 * U32)):
        runs = [_backward("SE3", op, Xb.to(dt), p.to(dt), u.to(dt)) for _ in range(2)]
        for k in range(2):
            assert torch.equal(runs[0][k], runs[1][k]), (op, dt, k)
            err = float(((runs[0][k].double() - want[k]).abs() / mag[k].amax(-1, keepdim=True).clamp(min=1.0)).max())
            assert err <= bound, (op, dt, k, err)


def test_python_api_against_the_stand_in_and_the_oracle():
    gen = torch.Generator().manual_seed(6)
    S = lg.shim
    a = 0.5 * torch.randn(3, 4, 6, generator=gen, dtype=F64)
    d = 0.2 * torch.randn(3, 4, 6, generator=gen, dtype=F64)
    P = torch.randn(3, 4, 3, generator=gen, dtype=F64)
    Xs, Xn = S.SE3.exp(a), lt.SE3.exp(a.to(dev))
    check_close(Xn.retr(d.to(dev)).data, Xs.retr(d).data, 1e-12, "retr")
    check_close(Xn.matrix().flatten(-2), Xs.matrix().flatten(-2), 1e-12, "matrix")
    check_close(Xn.translation(), Xs.translation(), 1e-12, "translation")
    check_close((Xn * P.to(dev)), Xs * P, 1e-12, "__mul__ act")
    check_close((Xn * Xn.inv()).data, S.SE3.IdentityLike(Xs).data, 1e-12, "__mul__ mul")
    assert isinstance(Xn * Xn, lt.SE3) and isinstance(Xn[0], lt.SE3) and Xn[:, 1:].shape == (3, 3)
    I = lt.SE3.Identity(2, 3, device=dev, dtype=F64)
    assert torch.equal(I.data.cpu(), S.SE3.Identity(2, 3, dtype=F64).data)
    check_close(lt.SO3(Xn).log(), S.SO3(Xs.data[..., 3:]).log(), 1e-12, "SO3(SE3)")
    check_close(lt.SE3(lt.SO3(Xn)).data, S.SE3(S.SO3(Xs.data[..., 3:])).data, 1e-12, "SE3(SO3)")
    # vec / InitFromVec: gradients through the projector and its pseudo-inverse, against the oracle
    for group, G in (("SE3", lt.SE3), ("SO3", lt.SO3)):
        X = (Xs.data if group == "SE3" else Xs.data[..., 3:]).clone()
        u = torch.randn(X.shape, generator=gen, dtype=F64)
        x = X.to(dev).requires_grad_(True)
        (G(x).vec() * u.to(dev)).sum().backward()
        check_close(x.grad, lg.autograd_grad(group, "vec", X, None, u)[0], 1e-10, ("vec", group))
        K = G.manifold_dim
        u[..., K:] = 0
        x = X.to(dev).requires_grad_(True)
        Y = G.InitFromVec(x)
        check_close(Y.projector().flatten(-2), lg.projector(lg.cls(group), X).flatten(-2), 1e-12, ("projector", group))
        torch.autograd.backward(Y.data, u.to(dev))
        check_close(x.grad, lg.autograd_grad(group, "fromvec", X, None, u)[0], 1e-10, ("fromvec", group))
    # retr's gradient: Exp(d) X with respect to d and X, against the oracle's exp and mul
    dd = d.to(dev).requires_grad_(True)
    xx = Xs.data.to(dev).requires_grad_(True)
    u = torch.randn(3, 4, 7, generator=gen, dtype=F64)
    u[..., 6:] = 0
    torch.autograd.backward(lt.SE3(xx).retr(dd).data, u.to(dev))
    gE, gX = lg.autograd_grad("SE3", "mul", S.SE3.exp(d).data, Xs.data, u)
    check_close(xx.grad, gX, 1e-10, "retr dX")
    check_close(dd.grad, lg.autograd_grad("SE3", "exp", d, None, gE)[0], 1e-10, "retr da")


def test_no_host_synchronisation():
    gen = torch.Generator(device=dev).manual_seed(7)
    X = lt.SE3.exp(0.3 * torch.randn(1, 64, 6, generator=gen, device=dev))
    a = torch.randn(1, 64, 6, generator=gen, device=dev).requires_grad_(True)
    p = torch.randn(1, 64, 8, 8, 4, generator=gen, device=dev).requires_grad_(True)
    x = X.data.clone().requires_grad_(True)
    Xg = lt.SE3(x)
    calls = [lambda: lt.SE3.exp(a), lambda: Xg.log(), lambda: Xg.inv(), lambda: Xg * Xg, lambda: Xg.adj(a), lambda: Xg.adjT(a),
             lambda: Xg.Jinv(a), lambda: Xg[:, :, None, None].act(p), lambda: Xg[:, :, None, None].act(p[..., :3]), lambda: Xg.matrix(),
             lambda: Xg.retr(a), lambda: Xg.vec(), lambda: lt.SE3.InitFromVec(x)]
    for k, f in enumerate(calls):
        n, out = host_syncs(f)
        assert n == 0, ("forward", k, n)
        out = out.data if isinstance(out, lt.LieGroup) else out
        if k == 6:
            continue                                                    # Jinv has no backward
        n, _ = host_syncs(lambda: torch.autograd.backward(out, torch.ones_like(out)))
        assert n == 0, ("backward", k, n)


def test_reprojection_on_the_package_matches_the_reference_projective_transform():
    """projective_transform's reprojection (geom/projective_ops.py:165-198) written here on the package -- inv, mul and act4 with per-edge
    broadcasting -- against the reference's stored outputs, at the tolerance of the reprojection kernel's test on that fixture"""
    import make_reference_python_golden as mk
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "reference_python.pt"))
    for name, poses, disps, intr, ii, jj in mk.reproject_cases():
        P, D, K = lt.SE3(poses[None].to(dev)), disps[None].to(dev), intr[None].to(dev)
        ht, wd = D.shape[2:]
        fx, fy, cx, cy = K[:, ii][..., None, None, :].unbind(-1)
        y, x = torch.meshgrid(torch.arange(ht, device=dev, dtype=F32), torch.arange(wd, device=dev, dtype=F32), indexing="ij")
        X0 = torch.stack([(x - cx) / fx, (y - cy) / fy, torch.ones_like(D[:, ii]), D[:, ii]], -1)
        Gij = P[:, jj.to(dev)] * P[:, ii.to(dev)].inv()
        Gij.data[:, (ii == jj).to(dev)] = torch.tensor([-0.1, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0], device=dev)
        X1 = Gij[:, :, None, None] * X0
        fx, fy, cx, cy = K[:, jj][..., None, None, :].unbind(-1)
        Z = torch.where(X1[..., 2] < 0.1, torch.ones_like(X1[..., 2]), X1[..., 2])
        coords = torch.stack([fx * (X1[..., 0] * (1.0 / Z)) + cx, fy * (X1[..., 1] * (1.0 / Z)) + cy], -1)
        gc = gold["reproject_%s_coords" % name]
        assert coords.shape == gc.shape
        rel = ((coords.cpu() - gc).abs() / gc.abs().clamp(min=1.0)).max()
        assert float(rel) < 1e-4, (name, float(rel))


def test_a_gradient_not_asked_for_is_not_computed():
    """a broadcast operand that needs no gradient (the constant point of translation(), the identity matrix of matrix()) gets none and is
    not reduced: lie_backward returns None for it; the gradient that is asked for equals the one computed with both"""
    from droid_slam_b200 import install
    be = install()
    gen = torch.Generator(device=dev).manual_seed(8)
    X = lg.shim.SE3.exp(0.5 * torch.randn(1, 16, 1, 6, generator=gen, dtype=F64, device=dev)).data
    p = torch.randn(1, 16, 5, 4, generator=gen, dtype=F64, device=dev)
    u = torch.randn(1, 16, 5, 4, generator=gen, dtype=F64, device=dev)
    both = be.lie_backward(lt.ACT4, 3, u, X, p)
    only_x = be.lie_backward(lt.ACT4, 3, u, X, p, True, False)
    only_p = be.lie_backward(lt.ACT4, 3, u, X, p, False, True)
    assert only_x[1] is None and only_p[0] is None
    assert torch.equal(only_x[0], both[0]) and torch.equal(only_p[1], both[1])
    x = X[0, :, 0].clone().requires_grad_(True)
    G = lt.SE3(x)
    torch.autograd.backward(G.translation(), torch.ones(16, 4, dtype=F64, device=dev))
    torch.autograd.backward(G.matrix(), torch.ones(16, 4, 4, dtype=F64, device=dev))
    want = lg.closed_grad("SE3", "act4", X[0, :, 0], torch.tensor([0.0, 0, 0, 1], dtype=F64, device=dev).expand(16, 4), torch.ones(16, 4, dtype=F64, device=dev))[0]
    I = torch.eye(4, dtype=F64, device=dev)
    want = want + sum(lg.closed_grad("SE3", "act4", X[0, :, 0], I[k].expand(16, 4), torch.ones(16, 4, dtype=F64, device=dev))[0] for k in range(4))
    check_close(x.grad, want.cpu(), 1e-12, "translation + matrix gradient")
