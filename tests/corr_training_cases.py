"""Inputs of the training-CorrBlock checks, regenerated from seeds, and the reference's CorrBlock formulation on this package's
`droid_backends` (any dtype, any device): the fixture generator (tests/golden/make_corr_training_golden.py), the CPU test that pins
oracle/corr.py to it, the GPU tests and tools/bench_corr_training.py all take them from here."""
import torch
import torch.nn.functional as F

# the fixture's cases: name -> (B, N, C, ht, wd, calls, calls that feed the loss).  17 x 23 drops a row and a column at every level;
# level 3 is at least 2 x 2 everywhere, so the reference's extra pooling pass after level 3 runs
FIXTURE = {
    "odd_17x23": (1, 2, 16, 17, 23, 3, None),
    "batch2_16x20": (2, 2, 16, 16, 20, 2, None),
    "partial_16x24": (1, 2, 16, 16, 24, 3, (0, 2)),
}
SUBSAMPLE = 31        # the fixture stores every 31st element of each level and call output, every 7th of each map gradient


def make_inputs(B, N, ht, wd, calls, seed=0, C=128, dev="cpu"):
    """fmap1, fmap2 [B,N,C,ht,wd] f32, coords of every call [B,N,ht,wd,2] f32 (windows partly and wholly outside every level, a quarter
    of the rows on exact integers), loss weights of every call [B,N,196,ht,wd] f32"""
    g = torch.Generator().manual_seed(seed)
    f1 = torch.randn(B, N, C, ht, wd, generator=g)
    f2 = torch.randn(B, N, C, ht, wd, generator=g)
    coords = []
    for k in range(calls):
        x = torch.rand(B, N, ht, wd, generator=g) * (wd + 16) - 8
        y = torch.rand(B, N, ht, wd, generator=g) * (ht + 16) - 8
        x[..., : max(1, ht // 4), :] = torch.round(x[..., : max(1, ht // 4), :])
        y[..., : max(1, ht // 4), :] = torch.round(y[..., : max(1, ht // 4), :])
        x[..., -1, :] = -40.0 - k
        y[..., :, -1] = ht + 60.0
        coords.append(torch.stack([x, y], dim=-1))
    weights = [torch.randn(B, N, 196, ht, wd, generator=g) for _ in range(calls)]
    return f1.to(dev), f2.to(dev), [c.to(dev) for c in coords], [w.to(dev) for w in weights]


class _Sampler(torch.autograd.Function):
    """the reference's CorrSampler (modules/corr.py:8-22) on this package's corr_index_forward / corr_index_backward"""

    @staticmethod
    def forward(ctx, volume, coords, radius):
        from droid_slam_b200 import install
        ctx.save_for_backward(volume, coords)
        ctx.radius = radius
        return install().corr_index_forward(volume, coords, radius)[0]

    @staticmethod
    def backward(ctx, grad):
        from droid_slam_b200 import install
        volume, coords = ctx.saved_tensors
        return install().corr_index_backward(volume, coords, grad.contiguous(), ctx.radius)[0], None, None


class RefCorrBlock:
    """CorrBlock of modules/corr.py:6-71 in the maps' dtype on the device's droid_backends (fp32: torch.matmul, without tf32 when the
    caller turns it off).  The reference also pools level 3 once more, a result it never uses and that avg_pool2d refuses where level 3
    is one pixel high or wide; that pass is skipped, nothing else differs."""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        batch, num, dim, ht, wd = fmap1.shape
        corr = torch.matmul((fmap1.reshape(batch * num, dim, ht * wd) / 4.0).transpose(1, 2), fmap2.reshape(batch * num, dim, ht * wd) / 4.0)
        corr = corr.reshape(batch * num * ht * wd, 1, ht, wd)
        self.radius, self.corr_pyramid = radius, []
        for i in range(num_levels):
            self.corr_pyramid.append(corr.view(batch * num, ht, wd, ht // 2 ** i, wd // 2 ** i))
            if i < num_levels - 1:
                corr = F.avg_pool2d(corr, 2, stride=2)

    def __call__(self, coords):
        batch, num, ht, wd, _ = coords.shape
        c = coords.permute(0, 1, 4, 2, 3).contiguous().view(batch * num, 2, ht, wd)
        return torch.cat([_Sampler.apply(v, c / 2 ** i, self.radius).view(batch, num, -1, ht, wd) for i, v in enumerate(self.corr_pyramid)], 2)


def run(block_class, f1, f2, coords, weights, used, dtype):
    """(pyramid, outputs of every call, grad fmap1, grad fmap2) of block_class(fmap1, fmap2) looked up at every coords, with the loss
    sum_k (weights[k] * out_k).sum() over the calls in `used` (None: all)"""
    a = f1.to(dtype).requires_grad_(True)
    b = f2.to(dtype).requires_grad_(True)
    blk = block_class(a, b)
    outs = [blk(c) for c in coords]
    loss = sum((weights[k].to(dtype) * outs[k]).sum() for k in (used if used is not None else range(len(coords))))
    g1, g2 = torch.autograd.grad(loss, [a, b])
    return [p.detach() for p in blk.corr_pyramid], [o.detach() for o in outs], g1, g2


def fixture_record(pyr, outs, g1, g2):
    """what the fixture stores of one case's run"""
    rec = {"level%d" % l: v.reshape(-1)[::SUBSAMPLE].clone() for l, v in enumerate(pyr)}
    rec.update({"call%d" % k: o.reshape(-1)[::SUBSAMPLE].clone() for k, o in enumerate(outs)})
    rec.update(grad_fmap1=g1.reshape(-1)[::7].clone(), grad_fmap2=g2.reshape(-1)[::7].clone())
    return rec
