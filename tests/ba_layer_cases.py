"""Inputs of the dense BA layer's test cases (tests/test_ba_layer_*.py, tests/golden/make_ba_layer_golden.py, tools/bench_ba_layer.py),
regenerated from seeds in fp64 on the CPU.  Each case: dict(target, weight, eta, poses [B,N,7], disps, intrinsics, ii, jj, fixedp,
chain) -- chain = 2: two chained calls with a loss on both outputs."""
import torch


def radius_graph(N, rad=2):
    """train.py:92-94: every i -> j with i != j and |i - j| <= rad"""
    ii = [i for i in range(N) for j in range(N) if i != j and abs(i - j) <= rad]
    jj = [j for i in range(N) for j in range(N) if i != j and abs(i - j) <= rad]
    return torch.tensor(ii), torch.tensor(jj)


def make_inputs(ii, jj, N, ht=12, wd=16, B=1, fixedp=2, seed=0, motion=0.05, weight_scale=1.0, near=False):
    g = torch.Generator().manual_seed(seed)
    E = ii.shape[0]
    xi = motion * torch.randn(B, N, 6, generator=g, dtype=torch.float64)
    xi[..., 2] += motion * torch.arange(N, dtype=torch.float64)          # forward motion along the sequence
    half = 0.5 * xi[..., 3:]
    th = half.norm(dim=-1, keepdim=True)
    q = torch.cat([torch.sin(th) / th.clamp_min(1e-12) * half, torch.cos(th)], dim=-1)
    poses = torch.cat([xi[..., :3], q], dim=-1)
    disps = 0.3 + 0.7 * torch.rand(B, N, ht, wd, generator=g, dtype=torch.float64)
    if near:                                                            # points close to / behind the camera: Z < 0.2 and Z < 0.1
        disps[..., : ht // 3, :] = 0.5 + 11.5 * torch.rand(B, N, ht // 3, wd, generator=g, dtype=torch.float64)
        poses[..., 2] += torch.linspace(-0.9, 0.9, N, dtype=torch.float64)
    f = 0.8 * wd
    intr = torch.tensor([f, f, wd / 2 - 0.5, ht / 2 - 0.5], dtype=torch.float64).repeat(B, N, 1)
    intr = intr * (1.0 + 0.02 * torch.arange(N, dtype=torch.float64))[None, :, None]
    y, x = torch.meshgrid(torch.arange(ht, dtype=torch.float64), torch.arange(wd, dtype=torch.float64), indexing="ij")
    target = torch.stack([x, y], -1).expand(B, E, ht, wd, 2) + 1.5 * torch.randn(B, E, ht, wd, 2, generator=g, dtype=torch.float64)
    weight = weight_scale * torch.rand(B, E, ht, wd, 2, generator=g, dtype=torch.float64)
    M = int(torch.unique(ii).numel())
    eta = 1e-3 + 0.05 * torch.rand(B, M, ht, wd, generator=g, dtype=torch.float64)
    return dict(target=target.contiguous(), weight=weight, eta=eta, poses=poses, disps=disps, intrinsics=intr, ii=ii.clone(),
                jj=jj.clone(), fixedp=fixedp, chain=1)


def cases():
    """name -> inputs: the fixture's cases (12 x 16 maps).  The training graph (22 edges) once; the other cases on an 8-edge graph that
    also has an edge out of a fixed frame (0 -> 3), a frame with no out-edge (5) and an ii == jj edge (4 -> 4), which keeps the stored
    gradients of target and weight (one map per edge) small"""
    out = {}
    ii, jj = radius_graph(7)
    out["train_graph"] = make_inputs(ii, jj, 7, seed=1)
    ii2, jj2 = torch.tensor([0, 1, 2, 3, 4, 6, 4, 2]), torch.tensor([3, 2, 3, 4, 5, 5, 4, 6])
    out["fixed_out_noout_selfedge"] = make_inputs(ii2, jj2, 7, seed=2)
    out["near_plane_crossings"] = make_inputs(ii2, jj2, 7, seed=3, motion=0.3, near=True)
    out["batch2"] = make_inputs(ii2, jj2, 7, B=2, seed=4)
    neg = make_inputs(ii2, jj2, 7, seed=5, weight_scale=1.0)
    neg["weight"] = neg["weight"] - 0.9                                 # mostly negative weights: an indefinite system
    out["indefinite"] = neg
    ch = make_inputs(ii2, jj2, 7, seed=6)
    ch["chain"] = 2
    out["chained"] = ch
    return out


def loss_weights(B, N, ht, wd, seed=99):
    """fixed random cotangents: loss = sum(a * poses'.log()) ... built on the outputs' data directly (poses' [B,N,7], disps')"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, N, 7, generator=g, dtype=torch.float64), torch.randn(B, N, ht, wd, generator=g, dtype=torch.float64)
