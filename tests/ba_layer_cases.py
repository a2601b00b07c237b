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


def seeded_graph(N, E, rad, seed, lo=0):
    """E edges i -> j among frames [lo, N), i != j, |i - j| <= rad, the highest of a seeded score: a per-source part (so that some
    sources keep all their candidates and others lose them all) plus a smaller per-pair part.  Edges come in score order, not sorted."""
    g = torch.Generator().manual_seed(seed)
    src = torch.rand(N, generator=g, dtype=torch.float64)
    pairs = [(i, j) for i in range(lo, N) for j in range(lo, N) if i != j and abs(i - j) <= rad]
    score = torch.tensor([src[i] for i, _ in pairs], dtype=torch.float64) + 0.3 * torch.rand(len(pairs), generator=g, dtype=torch.float64)
    keep = torch.argsort(score, descending=True)[:E].tolist()
    return torch.tensor([pairs[k][0] for k in keep]), torch.tensor([pairs[k][1] for k in keep])


def hub_graph():
    """9 frames: frame 4 has 12 out-edges (to every frame, itself included, and again to 3, 5 and 7); the other frames a radius-1
    chain that skips frame 4"""
    ii = [4] * 12 + [0, 1, 1, 2, 2, 3, 5, 6, 6, 7, 7, 8]
    jj = [0, 1, 2, 3, 4, 5, 6, 7, 8, 5, 3, 7] + [1, 0, 2, 1, 3, 2, 6, 5, 7, 6, 8, 7]
    return torch.tensor(ii), torch.tensor(jj)


def domain_cases():
    """name -> inputs: the corners of the layer's domain (N - fixedp up to 20, fixedp = 0 and N - 1, N > 64 with gaps in the source
    set, B = 4 with element 2 failing, a 12-out-edge hub with duplicate and ii == jj edges, maps from 3 x 5 to 60 x 80, points at and
    behind the camera at 20 pose unknowns).  tests/test_ba_layer_cpu.py checks that each reaches the corner it is named for."""
    out = {}
    ii, jj = radius_graph(22)
    # long edges from every other frame to the fixed frame 0: without them the radius-2 chain of 20 pose unknowns drifts in a weak
    # x-translation / y-rotation mode (S near condition 1e4), and the fp32 oracle's error on the card reaches 1e-3
    star_i, star_j = torch.arange(3, 22, 2), torch.zeros(10, dtype=torch.long)
    out["p20_48x64"] = make_inputs(torch.cat([ii, star_i]), torch.cat([jj, star_j]), 22, ht=48, wd=64, seed=41)
    gi, gj = seeded_graph(22, 60, 3, seed=42)
    ch = make_inputs(torch.cat([gi, star_i]), torch.cat([gj, star_j]), 22, ht=60, wd=80, seed=42)
    ch["eta"] = ch["eta"] + 1.0         # keeps every disparity of the 4 calls off the clamp at 0, where fp32 and fp64 gradients part
    ch["chain"] = 4
    out["p20_60x80_chain4"] = ch
    out["fixedp0"] = make_inputs(*radius_graph(6), 6, fixedp=0, seed=43)
    out["p1"] = make_inputs(*radius_graph(7), 7, fixedp=6, seed=44)
    # every free frame is on some edge: a pose unknown with none has dx = 0 exactly, where the oracle's Exp has no derivative
    out["many_fixed_gaps"] = make_inputs(*seeded_graph(70, 60, 3, seed=53, lo=40), 70, ht=9, wd=13, fixedp=55, seed=45)
    g24 = seeded_graph(7, 24, 3, seed=57)
    out["train24_batch4"] = make_inputs(*g24, 7, ht=48, wd=64, B=4, seed=46)
    fail = make_inputs(*g24, 7, B=4, seed=47)
    fail["weight"][2] = fail["weight"][2] - 0.9                          # element 2 indefinite, the others not
    out["batch4_third_fails"] = fail
    out["hub_duplicates"] = make_inputs(*hub_graph(), 9, ht=17, wd=23, B=2, seed=48)
    out["tiny_3x5"] = make_inputs(*radius_graph(7), 7, ht=3, wd=5, seed=49)
    out["near_plane_p20"] = make_inputs(*radius_graph(22), 22, ht=24, wd=32, seed=50, near=True)
    return out


def loss_weights(B, N, ht, wd, seed=99):
    """fixed random cotangents: loss = sum(a * poses'.log()) ... built on the outputs' data directly (poses' [B,N,7], disps')"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, N, 7, generator=g, dtype=torch.float64), torch.randn(B, N, ht, wd, generator=g, dtype=torch.float64)
