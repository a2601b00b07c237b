"""The `lietorch` API DROID-SLAM and its scripts use, on this package's sm_90a kernels (csrc/lie.cu, droid_backends.lie_forward /
lie_backward): SO3 and SE3 with exp, log, inv, mul, retr, adj, adjT, Jinv, act (3- and 4-vectors), matrix, translation, vec /
InitFromVec, and their gradients in lietorch's convention.

    import droid_slam_b200
    droid_slam_b200.install_dependencies()     # `import lietorch` / `import torch_scatter` now resolve to this package
    from lietorch import SE3

Each operation is a torch.autograd.Function over one kernel launch.  Broadcasting follows lietorch's rule (same rank, each batch size
equal or 1) and happens inside the kernel: no operand is repeated to the output's batch, and the backward sums a broadcast operand's
gradient in the launch.  The gradient with respect to a group element X is the left-tangent gradient d/de L(Exp(e) X) at e = 0 in the
first K entries of its N-entry data record (the rest 0), as lietorch's kernels define it.

What differs from lietorch: arithmetic runs on CUDA tensors only (construction, Identity, indexing, cat / stack work on the CPU; CPU
arithmetic raises); Sim3 and RxSO3 are types with their layouts, construction, indexing, cat / stack, but their arithmetic raises; fp32
results are not bit-identical to lietorch's (Eigen evaluates in another order); quaternion() returns the stored quaternion (lietorch's
groups.py names a Quat op that does not exist)."""
import torch

__all__ = ["LieGroupParameter", "SO3", "RxSO3", "SE3", "Sim3", "cat", "stack"]

# operation codes of include/droid_b200.h (DBA_LIE_*)
EXP, LOG, INV, MUL, ADJ, ADJT, JINV, ACT, ACT4, PROJECTOR, VEC, FROMVEC = range(12)
_BACKEND = None


def _be():
    global _BACKEND
    if _BACKEND is None:
        from .. import install
        _BACKEND = install()
    return _BACKEND


def _no_kernel(entry, why):
    from ..modules import _require
    _require(entry, why)


def _check(cls, name, *tensors):
    """raise for `cls.name` on operands the kernels do not take: a group without kernels, CPU tensors, dtypes other than fp32 / fp64"""
    entry = "%s.%s" % (cls.group_name, name)
    if cls.group_id is None:
        _no_kernel(entry, "%s arithmetic is not implemented (only SO3 and SE3 have kernels)" % cls.group_name)
    for t in tensors:
        if not t.is_cuda:
            _no_kernel(entry, "a %s tensor (the group kernels run on CUDA tensors only)" % t.device)
        if t.dtype not in (torch.float32, torch.float64):
            _no_kernel(entry, "dtype %s (float32 and float64 have kernels)" % t.dtype)


class _Op(torch.autograd.Function):
    """one group operation: forward and backward are one kernel launch each"""

    @staticmethod
    def forward(ctx, op, group, a, b):
        ctx.op, ctx.group = op, group
        ctx.save_for_backward(a, b)
        return _be().lie_forward(op, group, a, b)

    @staticmethod
    def backward(ctx, grad):
        if ctx.op in (JINV, PROJECTOR):
            raise RuntimeError("lietorch: %s has no backward (as in lietorch)" % ("Jinv" if ctx.op == JINV else "projector"))
        a, b = ctx.saved_tensors
        need_a, need_b = ctx.needs_input_grad[2], b is not None and ctx.needs_input_grad[3]
        if not (need_a or need_b):
            return None, None, None, None
        grads = _be().lie_backward(ctx.op, ctx.group, grad, a, b, need_a, need_b)   # an operand needing no gradient is not reduced
        return None, None, grads[0], grads[1] if b is not None else None


class _Embed(torch.autograd.Function):
    """vec() (op VEC) / InitFromVec (op FROMVEC): the identity on the data; the backward maps the gradient through the orthogonal
    projector P of the element (VEC) or its pseudo-inverse (FROMVEC), in one launch"""

    @staticmethod
    def forward(ctx, op, group, x):
        ctx.op, ctx.group = op, group
        ctx.save_for_backward(x)
        return x.view_as(x)

    @staticmethod
    def backward(ctx, grad):
        x, = ctx.saved_tensors
        return None, None, _be().lie_backward(ctx.op, ctx.group, grad, x)[0]


def _bcast_rank(x, y):
    if x.dim() != y.dim():
        raise ValueError("lietorch operands need the same number of dimensions, got %s and %s" % (tuple(x.shape), tuple(y.shape)))


class LieGroup:
    """a batch of group elements: `data` [..., embedded_dim]"""
    group_name, group_id, manifold_dim, embedded_dim, id_elem = None, None, None, None, None

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

    @classmethod
    def _apply(cls, name, op, a, b=None):
        _check(cls, name, *([a] if b is None else [a, b]))
        if b is not None:
            _bcast_rank(a, b)
        return _Op.apply(op, cls.group_id, a, b)

    # ---- construction ----
    @classmethod
    def Identity(cls, *batch_shape, **kwargs):
        if batch_shape and isinstance(batch_shape[0], (tuple, list, torch.Size)):
            batch_shape = tuple(batch_shape[0])
        data = cls.id_elem.to(device=kwargs.get("device", "cpu"), dtype=kwargs.get("dtype", torch.float32))
        return cls(data.repeat(*batch_shape, 1) if len(batch_shape) else data.clone())

    @classmethod
    def IdentityLike(cls, G):
        return cls.Identity(G.shape, device=G.data.device, dtype=G.data.dtype)

    @classmethod
    def InitFromVec(cls, data):
        if not (data.is_cuda or torch.is_grad_enabled() and data.requires_grad):
            return cls(data)
        _check(cls, "InitFromVec", data)
        return cls(_Embed.apply(FROMVEC, cls.group_id, data))

    @classmethod
    def Random(cls, *batch_shape, sigma=1.0, **kwargs):
        if batch_shape and isinstance(batch_shape[0], (tuple, list, torch.Size)):
            batch_shape = tuple(batch_shape[0])
        return cls.exp(sigma * torch.randn(tuple(batch_shape) + (cls.manifold_dim,), **kwargs))

    def vec(self):
        if not (self.data.is_cuda or torch.is_grad_enabled() and self.data.requires_grad):
            return self.data
        _check(type(self), "vec", self.data)
        return _Embed.apply(VEC, self.group_id, self.data)

    # ---- arithmetic ----
    @classmethod
    def exp(cls, x):
        return cls(cls._apply("exp", EXP, x))

    def log(self):
        return self._apply("log", LOG, self.data)

    def inv(self):
        return self.__class__(self._apply("inv", INV, self.data))

    def mul(self, other):
        return self.__class__(self._apply("mul", MUL, self.data, other.data))

    def retr(self, a):
        """Exp(a) * X"""
        return self.__class__(self._apply("retr", MUL, self._apply("retr", EXP, a), self.data))

    def adj(self, a):
        return self._apply("adj", ADJ, self.data, a)

    def adjT(self, a):
        return self._apply("adjT", ADJT, self.data, a)

    def Jinv(self, a):
        return self._apply("Jinv", JINV, self.data, a)

    def act(self, p):
        if p.shape[-1] == 3:
            return self._apply("act", ACT, self.data, p)
        if p.shape[-1] == 4:
            return self._apply("act", ACT4, self.data, p)
        raise ValueError("act takes 3-vectors or homogeneous 4-vectors, got shape %s" % (tuple(p.shape),))

    def projector(self):
        """the orthogonal projector [..., N, N] the gradients of vec() / InitFromVec use"""
        n = self.embedded_dim
        return self._apply("projector", PROJECTOR, self.data).view(*self.shape, n, n)

    def matrix(self):
        """[..., 4, 4]"""
        _check(type(self), "matrix", self.data)
        I = torch.eye(4, dtype=self.dtype, device=self.device).view([1] * (self.data.dim() - 1) + [4, 4])
        return self.__class__(self.data[..., None, :]).act(I).transpose(-1, -2)

    def translation(self):
        """[..., 4]: the homogeneous image of the origin"""
        _check(type(self), "translation", self.data)
        p = torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=self.dtype, device=self.device).view([1] * (self.data.dim() - 1) + [4])
        return self._apply("translation", ACT4, self.data, p)

    def __mul__(self, other):
        if isinstance(other, LieGroup):
            return self.mul(other)
        if isinstance(other, torch.Tensor):
            return self.act(other)
        return NotImplemented

    # ---- data ----
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
    """unit quaternions (qx, qy, qz, qw); tangent 3"""
    group_name, group_id, manifold_dim, embedded_dim = "SO3", 1, 3, 4
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 1.0])

    def __init__(self, data):
        if isinstance(data, SE3):
            data = data.data[..., 3:7]
        super().__init__(data)

    def quaternion(self):
        return self.data


class SE3(LieGroup):
    """(tx, ty, tz, qx, qy, qz, qw); tangent (tau, phi)"""
    group_name, group_id, manifold_dim, embedded_dim = "SE3", 3, 6, 7
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])

    def __init__(self, data):
        if isinstance(data, SO3):
            data = torch.cat([torch.zeros_like(data.data[..., :3]), data.data], -1)
        super().__init__(data)

    def quaternion(self):
        return self.data[..., 3:7]

    def scale(self, s):
        t, q = self.data.split([3, 4], -1)
        return SE3(torch.cat([t * s.unsqueeze(-1), q], dim=-1))


class _NoKernelGroup(LieGroup):
    """a group with its data layout, construction, indexing and cat / stack; every arithmetic method raises"""
    group_id = None

    @classmethod
    def _apply(cls, name, op, a, b=None):
        _check(cls, name, a)

    @classmethod
    def InitFromVec(cls, data):
        return cls(data)

    def vec(self):
        return self.data

    def matrix(self):
        _check(type(self), "matrix")

    def translation(self):
        _check(type(self), "translation")


class RxSO3(_NoKernelGroup):
    """(qx, qy, qz, qw, s); tangent 4.  No kernels."""
    group_name, manifold_dim, embedded_dim = "RxSO3", 4, 5
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 1.0, 1.0])

    def __init__(self, data):
        if isinstance(data, Sim3):
            data = data.data[..., 3:8]
        super().__init__(data)


class Sim3(_NoKernelGroup):
    """(tx, ty, tz, qx, qy, qz, qw, s); tangent 7.  No kernels."""
    group_name, manifold_dim, embedded_dim = "Sim3", 7, 8
    id_elem = torch.as_tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0])

    def __init__(self, data):
        if isinstance(data, SO3):
            d = data.data
            data = torch.cat([torch.zeros_like(d[..., :3]), d, torch.ones_like(d[..., :1])], -1)
        elif isinstance(data, SE3):
            data = torch.cat([data.data, torch.ones_like(data.data[..., :1])], -1)
        elif isinstance(data, RxSO3):
            data = torch.cat([torch.zeros_like(data.data[..., :3]), data.data], -1)
        super().__init__(data)


class LieGroupParameter(torch.Tensor):
    """a tangent-space parameter [..., K] (zeros) over a group element: the element it stands for is group.retr(self)"""
    from torch._C import _disabled_torch_function_impl
    __torch_function__ = _disabled_torch_function_impl

    def __new__(cls, group, requires_grad=True):
        data = torch.zeros(group.tangent_shape, device=group.data.device, dtype=group.data.dtype)
        return torch.Tensor._make_subclass(cls, data, requires_grad)

    def __init__(self, group, requires_grad=True):
        self.group = group

    def retr(self):
        return self.group.retr(self)

    def log(self):
        return self.retr().log()

    def inv(self):
        return self.retr().inv()

    def adj(self, a):
        return self.retr().adj(a)

    def __mul__(self, other):
        if isinstance(other, LieGroupParameter):
            return self.retr() * other.retr()
        return self.retr() * other

    def add_(self, update, alpha):
        self.group = self.group.exp(alpha * update) * self.group

    def __getitem__(self, index):
        return self.retr().__getitem__(index)


def cat(group_list, dim):
    return group_list[0].__class__(torch.cat([X.data for X in group_list], dim=dim))


def stack(group_list, dim):
    return group_list[0].__class__(torch.stack([X.data for X in group_list], dim=dim))
