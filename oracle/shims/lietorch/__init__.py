"""Pure-PyTorch stand-in for the `lietorch` package (SE3 group) -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The reference's Python call sites on the path (`droid_slam/depth_video.py`, `geom/projective_ops.py`, `geom/ba.py`, `droid_net.py`)
import `lietorch`, a CUDA extension that cannot be built here (it needs the absent Eigen submodule).  With this package in
sys.modules as `lietorch` (tests/golden/reference.py) those files import UNMODIFIED, which is how `oracle.reproject` (row A5) is
pinned against `pops.projective_transform` itself and how the reference's `geom/ba.py` cross-checks the BA oracle.

Restates the arithmetic of thirdparty/lietorch/lietorch/include/so3.h and se3.h (file:line cited per function) and the Python
wrapper thirdparty/lietorch/lietorch/groups.py:51-231,265-285 (broadcasting per broadcasting.py:9-31).  Data layout
(tx,ty,tz,qx,qy,qz,qw); like the C++ class the quaternion is normalised on load (so3.h:35-37).  Checked with the identities of
thirdparty/lietorch/lietorch/run_tests.py:16-52 in tests/test_shims_cpu.py.
"""
import torch

__all__ = ["SE3", "SO3", "Sim3", "RxSO3", "cat", "stack", "LieGroupParameter"]
EPS = 1e-6   # include/common.h:7


def _cross(a, b):
    return torch.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                        a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], dim=-1)


def _qnorm(q):
    return q / q.norm(dim=-1, keepdim=True)


def _qmul(a, b):
    """Hamilton product, (x,y,z,w) layout (Eigen::Quaternion operator*)"""
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                        aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], dim=-1)


def _qconj(q):
    return torch.cat([-q[..., :3], q[..., 3:]], -1)


def _rot(q, p):
    """so3.h:55-60  p + w*uv + qv x uv, uv = 2 qv x p"""
    qv, w = q[..., :3], q[..., 3:4]
    uv = 2.0 * _cross(qv, p)
    return p + w * uv + _cross(qv, uv)


def _hat(v):
    o = torch.zeros_like(v[..., 0])
    return torch.stack([torch.stack([o, -v[..., 2], v[..., 1]], -1), torch.stack([v[..., 2], o, -v[..., 0]], -1),
                        torch.stack([-v[..., 1], v[..., 0], o], -1)], -2)


def _so3_exp(phi):
    """so3.h:149-166"""
    th2 = (phi * phi).sum(-1, keepdim=True)
    th = th2.sqrt()
    small = th < EPS
    ths = torch.where(small, torch.ones_like(th), th)
    imag = torch.where(small, 0.5 - th2 / 48.0 + th2 * th2 / 3840.0, torch.sin(0.5 * ths) / ths)
    real = torch.where(small, 1.0 - th2 / 8.0 + th2 * th2 / 384.0, torch.cos(0.5 * ths))
    return _qnorm(torch.cat([imag * phi, real], -1))


def _so3_log(q):
    """so3.h:111-147 (atan-based log)"""
    v, w = q[..., :3], q[..., 3:4]
    n2 = (v * v).sum(-1, keepdim=True)
    n = n2.sqrt()
    small = n2 < EPS * EPS
    ns = torch.where(small, torch.ones_like(n), n)
    wz = w.abs() < EPS
    ws = torch.where(wz, torch.ones_like(w), w)
    f_small = 2.0 / ws - (2.0 / 3.0) * n2 / (ws * ws * ws)
    f_wz = torch.where(w > 0, torch.pi / ns, -torch.pi / ns)
    f_gen = 2.0 * torch.atan(ns / ws) / ns
    return torch.where(small, f_small, torch.where(wz, f_wz, f_gen)) * v


def _left_jacobian(phi):
    """so3.h:168-186"""
    th2 = (phi * phi).sum(-1, keepdim=True)[..., None]
    th = th2.sqrt()
    small = th < EPS
    ths = torch.where(small, torch.ones_like(th), th)
    c1 = torch.where(small, 0.5 - th2 / 24.0, (1.0 - torch.cos(ths)) / (ths * ths))
    c2 = torch.where(small, 1.0 / 6.0 - th2 / 120.0, (ths - torch.sin(ths)) / (ths * ths * ths))
    P = _hat(phi)
    I = torch.eye(3, dtype=phi.dtype, device=phi.device).expand_as(P)
    return I + c1 * P + c2 * (P @ P)


def _left_jacobian_inverse(phi):
    """so3.h:188-206"""
    th2 = (phi * phi).sum(-1, keepdim=True)[..., None]
    th = th2.sqrt()
    small = th < EPS
    ths = torch.where(small, torch.ones_like(th), th)
    c2 = torch.where(small, torch.full_like(th, 1.0 / 12.0), (1.0 - ths * torch.cos(0.5 * ths) / (2.0 * torch.sin(0.5 * ths))) / (ths * ths))
    P = _hat(phi)
    I = torch.eye(3, dtype=phi.dtype, device=phi.device).expand_as(P)
    return I - 0.5 * P + c2 * (P @ P)


def _bcast(x, y):
    """broadcasting.py:9-31: same number of dims, sizes equal or 1"""
    assert x.dim() == y.dim(), "lietorch operands need the same number of dimensions"
    shape = [max(n, m) for n, m in zip(x.shape[:-1], y.shape[:-1])]
    return x.expand(*shape, x.shape[-1]), y.expand(*shape, y.shape[-1])


class LieGroup:
    """groups.py:51-231"""

    def __init__(self, data):
        self.data = data

    def __repr__(self):
        return "{}: size={}, device={}, dtype={}".format(self.group_name, self.shape, self.device, self.dtype)

    @property
    def shape(self):
        return self.data.shape[:-1]

    @property
    def device(self):
        return self.data.device

    @property
    def dtype(self):
        return self.data.dtype

    @property
    def tangent_shape(self):
        return self.data.shape[:-1] + (self.manifold_dim,)

    def vec(self):
        return self.data

    @classmethod
    def Identity(cls, *batch_shape, **kwargs):
        if isinstance(batch_shape[0], (tuple, list, torch.Size)):
            batch_shape = tuple(batch_shape[0])
        data = cls.id_elem.to(device=kwargs.get("device", "cpu"), dtype=kwargs.get("dtype", torch.float32))
        return cls(data.repeat(*batch_shape, 1) if len(batch_shape) else data.clone())

    @classmethod
    def IdentityLike(cls, G):
        return cls.Identity(G.shape, device=G.data.device, dtype=G.data.dtype)

    @classmethod
    def InitFromVec(cls, data):
        return cls(data)

    @classmethod
    def Random(cls, *batch_shape, sigma=1.0, **kwargs):
        if isinstance(batch_shape[0], (tuple, list)):
            batch_shape = tuple(batch_shape[0])
        return cls.exp(sigma * torch.randn(tuple(batch_shape) + (cls.manifold_dim,), **kwargs))

    def mul(self, other):
        return self.__class__(self._mul(*_bcast(self.data, other.data)))

    def retr(self, a):
        """Exp(a) * X  (groups.py:153-156)"""
        return self.__class__(self._mul(*_bcast(self.__class__.exp(a).data, self.data)))

    def __mul__(self, other):
        if isinstance(other, LieGroup):
            return self.mul(other)
        if isinstance(other, torch.Tensor):
            return self.act(other)
        return NotImplemented

    def __getitem__(self, index):
        return self.__class__(self.data[index])

    def __setitem__(self, index, item):
        self.data[index] = item.data

    def detach(self):
        return self.__class__(self.data.detach())

    def view(self, dims):
        return self.__class__(self.data.view(tuple(dims) + (self.embedded_dim,)))

    def to(self, *args, **kwargs):
        return self.__class__(self.data.to(*args, **kwargs))

    def cpu(self):
        return self.__class__(self.data.cpu())

    def cuda(self):
        return self.__class__(self.data.cuda())

    def float(self, device=None):
        return self.__class__(self.data.float())

    def double(self, device=None):
        return self.__class__(self.data.double())

    def unbind(self, dim=0):
        return [self.__class__(x) for x in self.data.unbind(dim=dim)]


class SO3(LieGroup):
    group_name, group_id, manifold_dim, embedded_dim = "SO3", 1, 3, 4
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 1.0])

    @classmethod
    def exp(cls, x):
        return cls(_so3_exp(x))

    def log(self):
        return _so3_log(_qnorm(self.data))

    def inv(self):
        return SO3(_qconj(_qnorm(self.data)))

    @staticmethod
    def _mul(a, b):
        return _qnorm(_qmul(_qnorm(a), _qnorm(b)))

    def act(self, p):
        q, p = _bcast(_qnorm(self.data), p)
        if p.shape[-1] == 3:
            return _rot(q, p)
        return torch.cat([_rot(q, p[..., :3]), p[..., 3:]], -1)

    def matrix(self):
        I = torch.eye(4, dtype=self.dtype, device=self.device).view([1] * (self.data.dim() - 1) + [4, 4])
        return SO3(self.data[..., None, :]).act(I).transpose(-1, -2)


class SE3(LieGroup):
    """groups.py:265-285 over se3.h"""
    group_name, group_id, manifold_dim, embedded_dim = "SE3", 3, 6, 7
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])

    def __init__(self, data):
        if isinstance(data, SO3):
            data = torch.cat([torch.zeros_like(data.data[..., :3]), data.data], -1)
        super().__init__(data)

    @staticmethod
    def _split(d):
        return d[..., :3], _qnorm(d[..., 3:7])       # quaternion normalised on load (so3.h:35-37)

    @classmethod
    def exp(cls, x):
        """se3.h:134-142  t = J_l(phi) tau"""
        tau, phi = x[..., :3], x[..., 3:]
        t = (_left_jacobian(phi) @ tau[..., None])[..., 0]
        return cls(torch.cat([t, _so3_exp(phi)], -1))

    def log(self):
        """se3.h:124-132"""
        t, q = self._split(self.data)
        phi = _so3_log(q)
        tau = (_left_jacobian_inverse(phi) @ t[..., None])[..., 0]
        return torch.cat([tau, phi], -1)

    def inv(self):
        """se3.h:36-38"""
        t, q = self._split(self.data)
        qi = _qconj(q)
        return SE3(torch.cat([-_rot(qi, t), qi], -1))

    @staticmethod
    def _mul(a, b):
        """se3.h:45-47  (R1 R2, t1 + R1 t2)"""
        ta, qa = SE3._split(a)
        tb, qb = SE3._split(b)
        return torch.cat([ta + _rot(qa, tb), _qnorm(_qmul(qa, qb))], -1)

    def act(self, p):
        """se3.h:49-56 (act on 3-vectors / homogeneous 4-vectors)"""
        d, p = _bcast(self.data, p)
        t, q = self._split(d)
        if p.shape[-1] == 3:
            return _rot(q, p) + t
        return torch.cat([_rot(q, p[..., :3]) + t * p[..., 3:], p[..., 3:]], -1)

    def _adj_matrix(self, d):
        """se3.h:58-68  [[R, t^ R], [0, R]]"""
        t, q = self._split(d)
        I = torch.eye(3, dtype=d.dtype, device=d.device).expand(*d.shape[:-1], 3, 3)
        R = _rot(q[..., None, :], I.transpose(-1, -2)).transpose(-1, -2)         # columns R e_k
        Z = torch.zeros_like(R)
        return torch.cat([torch.cat([R, _hat(t) @ R], -1), torch.cat([Z, R], -1)], -2)

    def adj(self, a):
        d, a = _bcast(self.data, a)
        return (self._adj_matrix(d) @ a[..., None])[..., 0]

    def adjT(self, a):
        """se3.h:84-86  Adj^T a"""
        d, a = _bcast(self.data, a)
        return (self._adj_matrix(d).transpose(-1, -2) @ a[..., None])[..., 0]

    def matrix(self):
        I = torch.eye(4, dtype=self.dtype, device=self.device).view([1] * (self.data.dim() - 1) + [4, 4])
        return SE3(self.data[..., None, :]).act(I).transpose(-1, -2)

    def translation(self):
        p = torch.as_tensor([0.0, 0.0, 0.0, 1.0], dtype=self.dtype, device=self.device).view([1] * (self.data.dim() - 1) + [4])
        return self.act(p)

    def quaternion(self):
        return self._split(self.data)[1]

    def scale(self, s):
        t, q = self.data.split([3, 4], -1)
        return SE3(torch.cat([t * s.unsqueeze(-1), q], dim=-1))


class Sim3(LieGroup):
    """only the type exists (isinstance checks in geom/projective_ops.py:112); no Sim3 arithmetic is on the path"""
    group_name, group_id, manifold_dim, embedded_dim = "Sim3", 4, 7, 8
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0])


class RxSO3(LieGroup):
    group_name, group_id, manifold_dim, embedded_dim = "RxSO3", 2, 4, 5
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 1.0, 1.0])


class LieGroupParameter(torch.Tensor):
    pass


def cat(group_list, dim):
    return group_list[0].__class__(torch.cat([X.data for X in group_list], dim=dim))


def stack(group_list, dim):
    return group_list[0].__class__(torch.stack([X.data for X in group_list], dim=dim))
