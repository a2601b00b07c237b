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


# the stage checks' cases (tests/test_corr_training_stages_*.py): name -> (n edges, ht, wd, calls); the corner each one reaches is
# checked on the host by tests/test_corr_training_stages_cpu.py
STAGES = {
    "8x8": (3, 8, 8, 2),                     # one source tile, one target block, level 3 is 1x1
    "odd_23x31": (2, 23, 31, 2),             # the floor rule drops a row and a column at every level; partial blocks; HW % 64 = 9
    "portrait_70x43": (2, 70, 43, 2),        # more 8x8 block rows than columns; every level width takes the generic lookup
    "rows8_8x136": (2, 8, 136, 2),           # level 3 is one row 17 wide
    "cols8_136x8": (2, 136, 8, 2),           # level 3 is one column 17 high
    "many_edges_9x13": (300, 9, 13, 2),      # grid.z = 300
    "train_24x48x64": (24, 48, 64, 15),      # the training shape
    "large_60x80": (4, 60, 80, 2),           # longer sums than training: Q = 6370, HW = 4800
}
# committed bounds kappa <= c sqrt(K) per stage (kappa = |native - exact| / (2^-24 A), A the summed magnitude of the terms), set from
# the worst kappa measured on an H100 (tests/test_corr_training_stages_gpu.py) and held below the worst-case model
# (tests/test_corr_training_stages_cpu.py)
KAPPA_PER_SQRT_K = {"volume": 0.6, "g_f1": 0.6, "g_f2": 1.25}


def stage_K(stage, ht, wd):
    """terms per output: 128 channels for the volume, Q for g_f1, HW for g_f2"""
    return {"volume": 128, "g_f1": sum((ht >> l) * (wd >> l) for l in range(4)), "g_f2": ht * wd}[stage]


NONFINITE = ("nan_x", "nan_y", "nan_xy", "inf_x", "inf_y", "inf_xy", "ninf_x", "ninf_y", "ninf_xy")


def stage_cases():
    """[(name, n, ht, wd, calls)] of STAGES"""
    return [(name,) + v for name, v in STAGES.items()]


def special_coords(ht, wd):
    """[(category, x, y)]: half-integers, points exactly on each level's last row and column (at level l the coordinate is scaled by
    2^-l, so (w_l - 1) 2^l lands on w_l - 1), +-1e30 (the floor saturates) and, last, NaN / +inf / -inf in x, in y and in both"""
    inf, nan = float("inf"), float("nan")
    xm, ym = float(wd // 3), float(ht // 3)
    out = [("half", 0.5, 0.5), ("half", wd / 2 + 0.5, ht / 2 - 0.5), ("half", wd - 1.5, ht - 1.5), ("half", -2.5, ym + 0.5)]
    for l in range(4):
        xl, yl = float(((wd >> l) - 1) << l), float(((ht >> l) - 1) << l)
        out += [("last%d" % l, xl, yl), ("last%d" % l, xl, ym), ("last%d" % l, xm, yl)]
    out += [("huge", 1e30, ym), ("huge", -1e30, ym), ("huge", xm, 1e30), ("huge", xm, -1e30), ("huge", 1e30, 1e30)]
    out += [("nan_x", nan, ym), ("nan_y", xm, nan), ("nan_xy", nan, nan), ("inf_x", inf, ym), ("inf_y", xm, inf), ("inf_xy", inf, inf),
            ("ninf_x", -inf, ym), ("ninf_y", xm, -inf), ("ninf_xy", -inf, -inf)]
    return out


def special_pixels(ht, wd, count, seed):
    """`count` distinct source pixels (flat indices) below make_inputs's integer rows, off its last row and last column"""
    y, x = torch.meshgrid(torch.arange(ht // 4, ht - 1), torch.arange(wd - 1), indexing="ij")
    free = (y * wd + x).reshape(-1)
    assert free.numel() >= count, (ht, wd, count)
    return free[torch.randperm(free.numel(), generator=torch.Generator().manual_seed(seed))[:count]]


def stage_inputs(name, seed=0, dev="cpu"):
    """fmap1, fmap2 [n,128,ht,wd] f32; coords of every call [n,2,ht,wd] f32 (the C ABI's layout): make_inputs's coordinates with
    special_coords placed at the same pixels in every call, the non-finite ones on edge 0 only; the lookup gradient of every call
    [n,196,ht,wd] f32 (make_inputs's loss weights); the pixels and categories of the special coordinates"""
    n, ht, wd, calls = STAGES[name]
    f1, f2, coords, weights = make_inputs(1, n, ht, wd, calls, seed=seed)
    spec = special_coords(ht, wd)
    pix = special_pixels(ht, wd, len(spec), seed)
    out = []
    for c in coords:
        c = c[0].permute(0, 3, 1, 2).contiguous()                   # [n, 2, ht, wd]
        flat = c.view(n, 2, ht * wd)
        for (cat, x, y), p in zip(spec, pix.tolist()):
            edges = slice(0, 1) if cat in NONFINITE else slice(None)
            flat[edges, 0, p], flat[edges, 1, p] = x, y
        out.append(c.to(dev))
    return f1[0].to(dev), f2[0].to(dev), out, [w[0].contiguous().to(dev) for w in weights], pix, [s[0] for s in spec]


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
