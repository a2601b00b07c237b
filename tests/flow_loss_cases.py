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


# ---- the stage cases of tests/test_flow_loss_stages_*.py -----------------------------------------------------------------------------
GRID = 2.0 ** -24                   # the fp32 spacing of disparities in [0.5, 1): z = 1 - d is exact there (Sterbenz)
PLACED_STEPS = (-64, -8, -2, -1, 0, 1, 2, 8, 64)


def placed_threshold_case(seed=41, ht=8, wd=12, n=2):
    """N = 2, frame 1 at z = -1 from frame 0 with identity rotations, so every transform and z is exact in fp32: edge 0 -> 1 maps a
    pixel of disparity d to z = 1 - d, edge 1 -> 0 to z = 1 + d.  Frame 0's disparities (ground truth and iterates) sit a few fp32
    steps either side of 1 - 0.2f, so z0 and z1 straddle 0.2f by 1 to 64 steps; frame 1's iterate disparities sit around -0.8 (z1
    around 0.2 on edge 1 -> 0).  Also: ground-truth disparities of 0, -0 and -0.3; iterate pixels behind the camera (z = -0.5) on
    each edge; iterates equal to the ground truth elsewhere (c1 == c0 bit for bit)."""
    g = torch.Generator().manual_seed(seed)
    Ps = torch.tensor([[0, 0, 0, 0, 0, 0, 1], [0, 0, -1, 0, 0, 0, 1]], dtype=torch.float64)[None]
    base = float(torch.tensor(0.8, dtype=torch.float32))
    lv0 = torch.tensor([base + k * GRID for k in PLACED_STEPS], dtype=torch.float64)            # z = 1 - d around 0.2
    lv1 = -lv0                                                                                 # z = 1 + d around 0.2
    hw = ht * wd
    disps = 0.3 + 0.5 * torch.rand(1, 2, hw, generator=g, dtype=torch.float64)
    disps[0, 0] = lv0[torch.randint(0, len(lv0), (hw,), generator=g)]
    disps[0, 0, :3] = torch.tensor([0.0, -0.0, -0.3], dtype=torch.float64)
    disps[0, 1, :3] = torch.tensor([0.0, -0.0, -0.3], dtype=torch.float64)
    disps_est = []
    for s in range(n):
        d = disps.clone()
        pick = torch.rand(2, hw, generator=g) < 0.7
        d[0, 0][pick[0]] = lv0[torch.randint(0, len(lv0), (int(pick[0].sum()),), generator=g)]
        d[0, 1][pick[1]] = lv1[torch.randint(0, len(lv1), (int(pick[1].sum()),), generator=g)]
        d[0, 0, 3 + s] = 1.5                                                                   # z1 = -0.5 on edge 0 -> 1
        d[0, 1, 3 + s] = -1.5                                                                  # z1 = -0.5 on edge 1 -> 0
        disps_est.append(d.view(1, 2, ht, wd))
    f = 0.8 * wd
    intr = torch.tensor([f, f, wd / 2 - 0.5, ht / 2 - 0.5], dtype=torch.float64).repeat(1, 2, 1)
    return dict(Ps=Ps, disps=disps.view(1, 2, ht, wd), poses_est=[Ps.clone() for _ in range(n)], disps_est=disps_est, intrinsics=intr)


def _stage_flow():
    out = {}
    shapes = {"N2_B1_n1_1x1": (1, 2, 1, 1, 1), "N3_B2_n3_1x300": (2, 3, 1, 300, 3), "N7_B4_n1_300x1": (4, 7, 300, 1, 1),
              "N33_B1_n3_hw255": (1, 33, 15, 17, 3), "N2_B2_n15_hw256": (2, 2, 16, 16, 15), "N3_B1_n3_hw257": (1, 3, 1, 257, 3),
              "N7_B1_n3_hw513": (1, 7, 27, 19, 3), "N7_B2_n3_37x53": (2, 7, 37, 53, 3), "N3_B4_n3_13x11": (4, 3, 13, 11, 3),
              "train_N7_B1_n15_384x512": (1, 7, 384, 512, 15)}
    for k, (name, (B, N, ht, wd, n)) in enumerate(shapes.items()):
        out[name] = lambda B=B, N=N, ht=ht, wd=wd, n=n, k=k: dict(case=make_case(B=B, N=N, ht=ht, wd=wd, n=n, seed=100 + k))
    out["placed_thresholds"] = lambda: dict(case=placed_threshold_case())
    out.update(_stage_structure())
    return out


def _stage_structure():
    out = {}
    eq = make_case(N=3, n=2, ht=20, wd=24, seed=120)
    eq["poses_est"][0] = eq["Ps"].clone()
    eq["disps_est"][0][..., ::3] = eq["disps"][..., ::3]                                    # c1 == c0 bit for bit on these columns
    out["exact_equal"] = dict(case=eq)
    zt = make_case(N=4, n=2, ht=12, wd=16, seed=121)
    for P in [zt["Ps"]] + zt["poses_est"]:
        P[..., :3] = 0.0                                                                       # no translation: dc1/dd = 0
    out["zero_translation"] = dict(case=zt)
    nv = make_case(N=3, n=2, ht=12, wd=16, seed=122)
    nv["disps"][..., 2:5, :] = -nv["disps"][..., 2:5, :]                                       # every edge of these pixels has v = 0
    out["no_valid_rows"] = dict(case=nv)
    ne = make_case(N=4, n=3, ht=12, wd=16, seed=123)
    ne["disps_est"][1][0, 2, 5, 7] = float("nan")
    ne["disps_est"][2][0, 1, 3, 3] = float("inf")
    out["nonfinite_iterate"] = dict(case=ne)
    ng = make_case(N=4, n=2, ht=12, wd=16, seed=124)
    ng["disps"][0, 1, 6, 9] = float("nan")
    ng["disps"][0, 3, 2, 2] = float("inf")
    out["nonfinite_ground_truth"] = dict(case=ng)
    for k, (gamma, grad) in enumerate([(0.5, 0.05), (1.0, -2.5), (0.0, 1.0), (0.9, 0.0)]):
        out["gamma%g_grad%g" % (gamma, grad)] = dict(case=make_case(B=2, N=3, ht=9, wd=13, n=3, seed=130 + k), gamma=gamma, grad=grad)
    out = {k: (lambda v=v: v) for k, v in out.items()}
    qs = make_case(B=2, N=5, ht=11, wd=14, n=3, seed=140)
    g = torch.Generator().manual_seed(141)
    for P in [qs["Ps"]] + qs["poses_est"]:
        P[..., 3:] *= 0.5 + 1.5 * torch.rand(*P.shape[:-1], 1, generator=g, dtype=torch.float64)   # |q| in [0.5, 2]
    out["quaternions_scaled"] = lambda: dict(case=qs)
    return out


def _stage_upsample():
    out = {}
    for k, (name, (B, N, ht, wd)) in enumerate({"up_1x1": (1, 1, 1, 1), "up_1x9": (1, 2, 1, 9), "up_7x1": (2, 1, 7, 1),
                                                 "up_13x17": (1, 2, 13, 17), "up_43x70": (1, 1, 43, 70), "up_44x69": (1, 1, 44, 69),
                                                 "up_train_7x48x64": (1, 7, 48, 64)}.items()):
        out[name] = lambda B=B, N=N, ht=ht, wd=wd, k=k: upsample_case(B=B, N=N, ht=ht, wd=wd, seed=200 + k)
    out.update({k: (lambda v=v: v) for k, v in _stage_upsample_edges().items()})
    return out


def _stage_upsample_edges():
    out = {}
    s20 = upsample_case(ht=9, wd=11, seed=210)
    s20["mask"] *= 10.0                                                                        # N(0, 20)
    out["up_sigma20"] = s20
    out["up_tied"] = upsample_case(ht=5, wd=6, seed=211, kind="tied")
    out["up_dominant"] = upsample_case(ht=5, wd=6, seed=212, kind="dominant")
    ni = upsample_case(ht=4, wd=5, seed=213)
    v = ni["mask"].view(1, 1, 9, 64, 4, 5)
    v[:, :, 2, :, 1, 1] = float("-inf")                                                        # one -inf tap
    v[:, :, [0, 3, 7], 9, 2, 3] = float("-inf")
    v[:, :, :, 5, 3, 4] = float("-inf")                                                        # all -inf: NaN
    out["up_neginf"] = ni
    uf = upsample_case(ht=6, wd=7, seed=214)
    v = uf["mask"].view(1, 1, 9, 64, 6, 7)
    gaps = torch.linspace(80.0, 112.0, 64 * 42, dtype=torch.float64).view(64, 6, 7)
    v[:, :, 4] = 0.0
    v[:, :, :4] = -gaps
    v[:, :, 5:] = -gaps - 0.37                                                                 # gaps straddling expf's underflow
    out["up_underflow"] = uf
    nf = upsample_case(ht=4, wd=5, seed=215)
    v = nf["mask"].view(1, 1, 9, 64, 4, 5)
    v[:, :, 3, 10, 1, 2] = float("nan")
    v[:, :, 6, 20, 2, 4] = float("inf")
    out["up_nan_inf"] = nf
    nc = upsample_case(ht=5, wd=6, seed=216)
    nc["cot"][0, 0, 8 * 2 + 3, 8 * 4 + 5] = float("nan")                                       # one sub-pixel of grad_out
    out["up_nan_cot"] = nc
    return out


# name -> builder of dict(case, gamma=0.9, grad=1.0): the flow cases (the training-size one is built only when asked for)
STAGES = _stage_flow()
UPSAMPLE_STAGES = _stage_upsample()           # name -> builder of an upsample case


def upsample_stage(name):
    return UPSAMPLE_STAGES[name]()


def stage(name):
    """the flow case `name` with its arguments: dict(case, gamma, grad)"""
    return {"gamma": 0.9, "grad": 1.0, **STAGES[name]()}
