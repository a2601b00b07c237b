"""Gradient-convention oracle for the SO3 / SE3 operations of droid_slam_b200.lietorch -- TEST INFRASTRUCTURE ONLY.

lietorch's convention (its CUDA backward kernels): the gradient with respect to a group input X is the left-tangent gradient
d/de L(Exp(e) X) at e = 0, in the first K entries of an N-entry record (rest 0); an upstream gradient g on a group output Y means
dL = g . d for Y -> Exp(d) Y.  Tangent and point inputs get Euclidean gradients.

`autograd_grad` defines every gradient by torch autograd through the pure-PyTorch stand-in (oracle/shims/lietorch) in fp64:
  * a group input X is replaced by Exp1(e) X with e = 0 requiring grad, the product taken by the stand-in.  Exp1(e) = (e_tau, unit(e_phi / 2,
    1)) equals the stand-in's Exp(e) to first order (checked in tests/test_lietorch_cpu.py), which is all a derivative at e = 0 sees; the
    stand-in's own exp is not differentiable at exactly 0 under autograd (its masked small-angle branch takes sqrt'(0)).
  * a group output Y enters the loss as g . psi(Y Y0^-1) with Y0 = Y detached and psi(t, q) = (t, 2 q_xyz): psi(Exp(d)) = d + O(d^2).
  * broadcasting is the stand-in's expand, so autograd sums a broadcast operand's gradient.
`closed_grad` restates the closed forms of lietorch's backward kernels (tests/test_lietorch_cpu.py holds the two equal to 1e-12).
`right` / `transposed`: planted wrong conventions the test must reject."""
import torch

from .shims import lietorch as shim

OPS = ("exp", "log", "inv", "mul", "adj", "adjT", "act", "act4", "vec", "fromvec")
GROUP_OUT = ("exp", "inv", "mul", "fromvec")


def cls(group):
    return {"SO3": shim.SO3, "SE3": shim.SE3}[group]


def exp1(G, e):
    """first-order exponential: (e_tau, unit(e_phi / 2, 1)) [SE3] / unit(e / 2, 1) [SO3]"""
    q = shim._qnorm(torch.cat([0.5 * e[..., -3:], torch.ones_like(e[..., :1])], -1))
    return G(torch.cat([e[..., :3], q], -1) if G is shim.SE3 else q)


def psi(G, Y):
    q = Y.data[..., -4:]
    v = 2.0 * q[..., :3] * torch.sign(q[..., 3:])
    return torch.cat([Y.data[..., :3], v], -1) if G is shim.SE3 else v


def _pad(G, d):
    return torch.cat([d, torch.zeros_like(d[..., :G.embedded_dim - G.manifold_dim])], -1)


def projector_ad(G, X):
    """d (Exp1(e) X).data / de at e = 0, [.., N, K], by autograd"""
    K = G.manifold_dim
    rows = []
    for n in range(G.embedded_dim):
        e = torch.zeros(X.data.shape[:-1] + (K,), dtype=X.dtype, device=X.device, requires_grad=True)
        rows.append(torch.autograd.grad((exp1(G, e) * X).data[..., n].sum(), e)[0])
    return torch.stack(rows, -2)


def autograd_grad(group, op, a, b=None, g=None, perturb="left"):
    """(grad_a, grad_b) of op(a, b) for upstream gradient g, in lietorch's convention, by autograd through the stand-in (fp64 inputs).
    perturb = "right": the planted right-perturbation X Exp(e) instead."""
    G = cls(group)
    K, N = G.manifold_dim, G.embedded_dim

    def group_input(x):
        e = torch.zeros(x.shape[:-1] + (K,), dtype=x.dtype, device=x.device, requires_grad=True)
        X = G(x)
        return e, (exp1(G, e) * X if perturb == "left" else X * exp1(G, e))

    if op == "fromvec":
        P = projector_ad(G, G(a))                                        # [.., N, K]
        Pn = torch.cat([P, torch.zeros_like(P[..., :1]).expand(*P.shape[:-1], N - K)], -1)
        return (g[..., None, :] @ torch.linalg.pinv(Pn))[..., 0, :], None
    if op == "exp":
        x = a.clone().requires_grad_(True)
        wrt, out = [(x, False)], G.exp(x)
    elif op in ("log", "inv", "vec"):
        e, X = group_input(a)
        wrt = [(e, True)]
        out = {"log": lambda: X.log(), "inv": lambda: X.inv(), "vec": lambda: X.data}[op]()
    else:
        e, X = group_input(a)
        if op == "mul":
            f, Y = group_input(b)
            wrt, out = [(e, True), (f, True)], X * Y
        else:
            y = b.clone().requires_grad_(True)
            wrt = [(e, True), (y, False)]
            if G is shim.SO3 and op in ("adj", "adjT"):                  # the stand-in's SO3 has no adj: Adj(X) = R
                out = (X if op == "adj" else X.inv()).act(y)
            else:
                out = {"adj": lambda: X.adj(y), "adjT": lambda: X.adjT(y), "act": lambda: X.act(y), "act4": lambda: X.act(y)}[op]()
    if op in GROUP_OUT:
        Y0 = G(out.data.detach())
        loss = (g[..., :K] * psi(G, out * Y0.inv())).sum()
    else:
        loss = (g * out).sum()
    grads = torch.autograd.grad(loss, [w for w, _ in wrt], allow_unused=True)
    res = []
    for (w, is_group), gr in zip(wrt, grads):
        gr = torch.zeros_like(w) if gr is None else gr
        res.append(_pad(G, gr) if is_group else gr)
    return res[0], (res[1] if len(res) > 1 else None)


# ---- the closed forms of lietorch's backward kernels -----------------------------------------------------------------------------------
def _rotm(q):
    I = torch.eye(3, dtype=q.dtype, device=q.device).expand(*q.shape[:-1], 3, 3)
    return shim._rot(q[..., None, :], I.transpose(-1, -2)).transpose(-1, -2)


def adj_matrix(G, x):
    """Adj(X) [.., K, K]"""
    q = shim._qnorm(x[..., -4:])
    R = _rotm(q)
    if G is shim.SO3:
        return R
    Z = torch.zeros_like(R)
    return torch.cat([torch.cat([R, shim._hat(x[..., :3]) @ R], -1), torch.cat([Z, R], -1)], -2)


def ad_matrix(G, b):
    """ad(b) [.., K, K]: SO3 hat(b); SE3 [[hat(phi), hat(tau)], [0, hat(phi)]]"""
    if G is shim.SO3:
        return shim._hat(b)
    P, U = shim._hat(b[..., 3:]), shim._hat(b[..., :3])
    return torch.cat([torch.cat([P, U], -1), torch.cat([torch.zeros_like(P), P], -1)], -2)


def calc_q(tau, phi):
    th2 = (phi * phi).sum(-1, keepdim=True)[..., None]
    th = th2.sqrt()
    small = th < shim.EPS
    ths = torch.where(small, torch.ones_like(th), th)
    c1 = torch.where(small, 1 / 6 - th2 / 120, (ths - torch.sin(ths)) / ths ** 3)
    c2 = torch.where(small, 1 / 24 - th2 / 720, (ths ** 2 + 2 * torch.cos(ths) - 2) / (2 * ths ** 4))
    c3 = torch.where(small, 1 / 120 - th2 / 2520, (2 * ths - 3 * torch.sin(ths) + ths * torch.cos(ths)) / (2 * ths ** 5))
    P, U = shim._hat(phi), shim._hat(tau)
    return 0.5 * U + c1 * (P @ U + U @ P + P @ U @ P) + c2 * (P @ P @ U + U @ P @ P - 3 * P @ U @ P) + c3 * (P @ U @ P @ P + P @ P @ U @ P)


def left_jacobian(G, a):
    if G is shim.SO3:
        return shim._left_jacobian(a)
    J, Q = shim._left_jacobian(a[..., 3:]), calc_q(a[..., :3], a[..., 3:])
    return torch.cat([torch.cat([J, Q], -1), torch.cat([torch.zeros_like(J), J], -1)], -2)


def left_jacobian_inverse(G, a):
    if G is shim.SO3:
        return shim._left_jacobian_inverse(a)
    Ji, Q = shim._left_jacobian_inverse(a[..., 3:]), calc_q(a[..., :3], a[..., 3:])
    return torch.cat([torch.cat([Ji, -Ji @ Q @ Ji], -1), torch.cat([torch.zeros_like(Ji), Ji], -1)], -2)


def projector(G, x):
    """lietorch's orthogonal projector [.., N, N]"""
    q = shim._qnorm(x[..., -4:])
    v, w = q[..., :3], q[..., 3:]
    I = torch.eye(3, dtype=x.dtype, device=x.device).expand(*x.shape[:-1], 3, 3)
    A = torch.cat([0.5 * (w[..., None] * I - shim._hat(v)), -0.5 * v[..., None, :]], -2)          # 4 x 3
    so3 = torch.cat([A, torch.zeros_like(A[..., :1])], -1)
    if G is shim.SO3:
        return so3
    top = torch.cat([I, -shim._hat(x[..., :3]), torch.zeros_like(I[..., :1])], -1)
    return torch.cat([top, torch.cat([torch.zeros_like(A), so3], -1)], -2)


def _row(g, M):
    return (g[..., None, :] @ M)[..., 0, :]


def closed_grad(group, op, a, b=None, g=None, transposed=False):
    """the closed forms; broadcasting by expand and a sum over broadcast dims.  transposed=True plants a transpose (Adj for Adj^T and
    the like) that the test must reject"""
    G = cls(group)
    K = G.manifold_dim
    T = (lambda M: M.transpose(-1, -2)) if transposed else (lambda M: M)
    if b is not None:
        shape = [max(n, m) for n, m in zip(a.shape[:-1], b.shape[:-1])]
        a_, b_ = a.expand(*shape, a.shape[-1]), b.expand(*shape, b.shape[-1])
    else:
        a_, b_ = a, None
    gk = g[..., :K]
    if op == "exp":
        return _row(gk, T(left_jacobian(G, a_))), None
    if op == "fromvec":
        return _row(g, torch.linalg.pinv(projector(G, a_))), None
    if op == "vec":
        return _row(g, T(projector(G, a_))), None
    Ad = adj_matrix(G, a_)
    if op == "log":
        ga, gb = _row(gk, T(left_jacobian_inverse(G, G(a_).log()))), None
    elif op == "inv":
        ga, gb = -_row(gk, T(adj_matrix(G, G(a_).inv().data))), None
    elif op == "mul":
        ga, gb = gk, _pad(G, _row(gk, T(Ad)))
    elif op == "adj":
        ga, gb = -_row(g, ad_matrix(G, (Ad @ b_[..., None])[..., 0])), _row(g, T(Ad))
    elif op == "adjT":
        ga, gb = -_row(b_, ad_matrix(G, (T(Ad) @ g[..., None])[..., 0])), (T(Ad) @ g[..., None])[..., 0]
    else:                                                                # act / act4
        q = G(a_).act(b_)
        R = _rotm(shim._qnorm(a_[..., -4:]))
        w = b_[..., 3:] if op == "act4" else torch.ones_like(b_[..., :1])
        rot = torch.cross(q[..., :3], g[..., :3], dim=-1)                # g hat(-q)
        ga = torch.cat([g[..., :3] * w, rot], -1) if G is shim.SE3 else rot
        gb = _row(g[..., :3], T(R))
        if op == "act4":
            t = a_[..., :3] if G is shim.SE3 else torch.zeros_like(g[..., :3])
            gb = torch.cat([gb, (g[..., :3] * t).sum(-1, keepdim=True) + g[..., 3:]], -1)
    ga = _pad(G, ga)
    return _sum_to(ga, a.shape), (None if gb is None else _sum_to(gb, b.shape))


def _sum_to(x, shape):
    for d, n in enumerate(shape[:-1]):
        if n == 1 and x.shape[d] != 1:
            x = x.sum(d, keepdim=True)
    return x
