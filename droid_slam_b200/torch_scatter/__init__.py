"""The two `torch_scatter` reductions DROID-SLAM imports: scatter_sum / scatter_mean(src, index, dim=-1, out=None, dim_size=None) with an
index of src's shape or a 1-D index along `dim` (droid_net.py's GraphAgg, geom/ba.py), on ATen's scatter_add_.  They exist so that the
reference's modules import and its training-side BA runs; under the hooks GraphAgg is native (droid_slam_b200.update.UpdateModule).

dim_size=None reads index.max() back to the host, as torch_scatter does."""
import torch

__all__ = ["scatter_sum", "scatter_mean"]


def _index_along(src, index, dim):
    if index.dim() == src.dim():
        return index
    if index.dim() != 1:
        raise ValueError("torch_scatter: index must have src's rank or be 1-D, got %s for src %s" % (tuple(index.shape), tuple(src.shape)))
    shape = [1] * src.dim()
    shape[dim] = -1
    return index.view(shape).expand_as(src)


def scatter_sum(src, index, dim=-1, out=None, dim_size=None):
    dim = dim % src.dim()
    idx = _index_along(src, index, dim)
    if out is None:
        if dim_size is None:
            dim_size = int(index.max()) + 1 if index.numel() else 0
        shape = list(src.shape)
        shape[dim] = dim_size
        out = torch.zeros(shape, dtype=src.dtype, device=src.device)
    return out.scatter_add_(dim, idx, src)


def scatter_mean(src, index, dim=-1, out=None, dim_size=None):
    dim = dim % src.dim()
    total = scatter_sum(src, index, dim, out, dim_size)
    count = torch.zeros_like(total).scatter_add_(dim, _index_along(src, index, dim), torch.ones_like(src)).clamp_(min=1)
    if total.is_floating_point():
        return total.div_(count)
    return total.div_(count, rounding_mode="floor")
