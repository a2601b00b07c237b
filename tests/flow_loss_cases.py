"""Inputs of the flow loss and upsample_disp test cases (tests/test_flow_loss_*.py, tests/golden/make_flow_loss_golden.py,
tools/bench_flow_loss.py), regenerated from seeds in fp64 on the CPU.  A flow case: dict(Ps [B,N,7], disps [B,N,ht,wd], poses_est /
disps_est (lists of n), intrinsics [B,N,4]); poses are unit-quaternion SE3 data.  An upsample case: dict(disp [B,N,h,w],
mask [B,N,576,h,w], cot [B,N,8h,8w] the cotangent of the loss sum(cot * upsample_disp(disp, mask)))."""
import torch


def _se3(xi):
    half = 0.5 * xi[..., 3:]
    th = half.norm(dim=-1, keepdim=True)
    q = torch.cat([torch.sin(th) / th.clamp_min(1e-12) * half, torch.cos(th)], dim=-1)
    return torch.cat([xi[..., :3], q], dim=-1)


def _compose(a, b):
    """SE3 data a * b (unit quaternions, fp64)"""
    ta, qa, tb, qb = a[..., :3], a[..., 3:], b[..., :3], b[..., 3:]
    va, wa, vb, wb = qa[..., :3], qa[..., 3:], qb[..., :3], qb[..., 3:]
    uv = 2 * torch.linalg.cross(va, tb)
    t = tb + wa * uv + torch.linalg.cross(va, uv) + ta
    v = wa * vb + wb * va + torch.linalg.cross(va, vb)
    w = wa * wb - (va * vb).sum(-1, keepdim=True)
    return torch.cat([t, v, w], -1)


def make_case(B=1, N=7, ht=12, wd=16, n=3, seed=0, motion=0.05, noise=0.02):
    """ground truth with forward motion, iterates converging to it: iterate i perturbed by noise / (1 + i)"""
    g = torch.Generator().manual_seed(seed)
    xi = motion * torch.randn(B, N, 6, generator=g, dtype=torch.float64)
    xi[..., 2] += motion * torch.arange(N, dtype=torch.float64)
    Ps = _se3(xi)
    disps = 0.3 + 0.7 * torch.rand(B, N, ht, wd, generator=g, dtype=torch.float64)
    f = 0.8 * wd
    intr = torch.tensor([f, f, wd / 2 - 0.5, ht / 2 - 0.5], dtype=torch.float64).repeat(B, N, 1)
    intr = intr * (1.0 + 0.02 * torch.arange(N, dtype=torch.float64))[None, :, None]
    poses_est, disps_est = [], []
    for i in range(n):
        s = noise / (1 + i)
        poses_est.append(_compose(_se3(s * torch.randn(B, N, 6, generator=g, dtype=torch.float64)), Ps))
        disps_est.append(disps * (1 + s * torch.randn(B, N, ht, wd, generator=g, dtype=torch.float64)))
    return dict(Ps=Ps, disps=disps, poses_est=poses_est, disps_est=disps_est, intrinsics=intr)


def threshold_case(seed=7, ht=8, wd=12, margin=0.01):
    """N = 2, frame 1 at z = -1 from frame 0 (no rotation): edge 0 -> 1 maps a pixel of disparity d to Z = 1 - d, edge 1 -> 0 to
    Z = 1 + d.  Disparities put Z at margin on each side of 0.1 and of 0.2 (on the ground truth and the iterates), and at 1 - 0.5;
    ground-truth disparities of 0 and below mask val0"""
    g = torch.Generator().manual_seed(seed)
    Ps = torch.tensor([[0, 0, 0, 0, 0, 0, 1], [0, 0, -1, 0, 0, 0, 1]], dtype=torch.float64)[None]
    levels = torch.tensor([0.8 - margin, 0.8 + margin, 0.9 - margin, 0.9 + margin, 0.5], dtype=torch.float64)
    pick = lambda: levels[torch.randint(0, 5, (1, 2, ht, wd), generator=g)]  # noqa: E731
    disps = pick()
    disps[0, :, 0, :3] = torch.tensor([0.0, -0.3, -1e-3], dtype=torch.float64)
    disps_est = [pick(), pick()]
    poses_est = [Ps.clone(), Ps.clone()]
    f = 0.8 * wd
    intr = torch.tensor([f, f, wd / 2 - 0.5, ht / 2 - 0.5], dtype=torch.float64).repeat(1, 2, 1)
    return dict(Ps=Ps, disps=disps, poses_est=poses_est, disps_est=disps_est, intrinsics=intr)


def cases():
    """name -> flow inputs: the fixture's cases (small maps)"""
    out = {}
    out["train_n3"] = make_case(seed=1)
    out["batch2_n2"] = make_case(B=2, N=3, n=2, ht=9, wd=11, seed=2)
    out["n2_frames2"] = make_case(N=2, n=1, seed=3)
    out["thresholds"] = threshold_case()
    eq = make_case(N=3, n=2, seed=4)
    eq["poses_est"][0] = eq["Ps"].clone()                     # iterate 0 equals the ground truth where its disparity does: c1 == c0
    eq["disps_est"][0][..., ::2] = eq["disps"][..., ::2]
    neg = make_case(N=3, n=2, seed=5)
    neg["disps"][..., :4, :] = -neg["disps"][..., :4, :]      # ground-truth disparities below 0 and at 0: val0 = 0
    neg["disps"][..., 4, :] = 0.0
    out["exact_equal"] = eq
    out["zero_negative_gt"] = neg
    return out


def upsample_case(B=1, N=1, ht=5, wd=6, seed=0, kind="random"):
    """kind: random logits, tied (all 9 taps equal), dominant (one tap far above the rest)"""
    g = torch.Generator().manual_seed(seed)
    disp = 0.2 + torch.rand(B, N, ht, wd, generator=g, dtype=torch.float64)
    mask = 2.0 * torch.randn(B, N, 576, ht, wd, generator=g, dtype=torch.float64)
    if kind == "tied":
        mask = torch.full_like(mask, 0.75)
    elif kind == "dominant":
        mask = mask.view(B, N, 9, 64, ht, wd)
        mask[:, :, 4] += 40.0
        mask = mask.reshape(B, N, 576, ht, wd)
    cot = torch.randn(B, N, 8 * ht, 8 * wd, generator=g, dtype=torch.float64)
    return dict(disp=disp, mask=mask, cot=cot)


def upsample_cases():
    """name -> upsample inputs: the fixture's cases (maps of a few pixels: the mask gradient is 576 values per pixel)"""
    return {"random": upsample_case(seed=11), "batch2": upsample_case(B=2, N=2, ht=3, wd=2, seed=12),
            "ht1": upsample_case(ht=1, wd=5, seed=13), "wd1": upsample_case(ht=4, wd=1, seed=14),
            "tied": upsample_case(ht=3, wd=3, seed=15, kind="tied"), "dominant": upsample_case(ht=4, wd=4, seed=16, kind="dominant")}
