"""Seeded inputs for the geometry kernels (csrc/geom.cu: projmap, reproject, motion_features, graph_writeback, frame_distance,
depth_filter, iproj) and cvx_upsample at their edges.  Nothing is stored: every case is regenerated from its seed.  Each case names
the corner it reaches; tests/test_geometry_stages_cpu.py checks that it does.

Frames whose transformed depth must land on a threshold use an identity rotation and a translation along z: Z = 1 + d tz with tz = -1
and d = 1 - Z on the 2^-24 grid, so d, d tz and 1 + d tz are all fp32 numbers and the contracted and the uncontracted evaluation give
the same Z.  Below 0.5 that grid is as fine as 1 + d tz gets in fp32, so thresholds that are not on it (0.01, 0.1f, 0.2f) are straddled
by the grid points next to them."""
import torch

GRID = 2.0 ** -24
F32 = lambda x: float(torch.tensor(x, dtype=torch.float32))
# Z targets around each threshold: on it (where the grid has it) and 1, 2, 3, 8, 64, 2048 and 4096 grid steps to either side
STEPS = (0, 1, 2, 3, 8, 64, 2048, 4096)
THRESHOLDS = {"projmap_z": 0.01, "reproject_small": F32(0.1), "reproject_valid": F32(0.2), "min_depth": 0.25}

SHAPES = {"s1x1": (1, 1), "s1x7": (1, 7), "s7x1": (7, 1), "hw255": (15, 17), "hw256": (16, 16), "hw257": (1, 257),
          "s43x70": (43, 70), "s48x64": (48, 64), "s60x80": (60, 80)}
BETAS = (0.0, 0.3, 0.7, 1.0)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def random_poses(n, g, t_scale=0.5, rot=0.3, qnorm=0.03):
    """translations ~ t_scale N(0,1), rotations of angle ~ rot, quaternions scaled by 1 +- qnorm (not renormalised, as BA leaves them)"""
    axis = torch.randn(n, 3, generator=g)
    axis = axis / axis.norm(dim=1, keepdim=True)
    ang = rot * torch.rand(n, 1, generator=g)
    q = torch.cat([axis * torch.sin(ang / 2), torch.cos(ang / 2)], 1)
    q = q * (1 + qnorm * (2 * torch.rand(n, 1, generator=g) - 1))
    return torch.cat([t_scale * torch.randn(n, 3, generator=g), q], 1).float()


def identity_poses(n):
    p = torch.zeros(n, 7)
    p[:, 6] = 1
    return p


def intrinsics_for(ht, wd, g):
    return torch.tensor([0.9 * max(wd, 2) + 0.37, 0.85 * max(ht, 2) + 0.21, (wd - 1) / 2 + 0.13, (ht - 1) / 2 - 0.17]) * \
        (1 + 0.05 * torch.rand(4, generator=g))


def base_case(name, ht, wd, n, seed, n_edges=12, stereo=2):
    g = _gen(seed)
    K = intrinsics_for(ht, wd, g).float()
    Kpf = (K[None] * (1 + 0.1 * (2 * torch.rand(n, 4, generator=g) - 1))).float()   # per-frame intrinsics, Ki != Kj
    ii = torch.randint(0, n, (n_edges,), generator=g)
    jj = (ii + torch.randint(1, max(n, 2), (n_edges,), generator=g)) % n
    jj[:stereo] = ii[:stereo]                                   # stereo edges ii == jj
    return dict(name=name, poses=random_poses(n, g), disps=(0.05 + 1.5 * torch.rand(n, ht, wd, generator=g)).float(), intr=K, intr_pf=Kpf,
                ii=ii, jj=jj, df_ix=torch.arange(n), df_thresh=(0.02 + 0.3 * torch.rand(n, generator=g)).float(), betas=BETAS,
                placed={})


def threshold_targets():
    """(Z values, threshold name per value): the 2^-24 grid points at STEPS from each threshold; every Z is an fp32 number and
    1 - Z is one too"""
    zs, names = [], []
    for name, thr in THRESHOLDS.items():
        base = round(thr / GRID)
        for s in STEPS:
            for z in sorted({(base - s) * GRID, (base + s) * GRID}):
                zs.append(z); names.append(name)
    return torch.tensor(zs, dtype=torch.float64), names


def thresholds_case():
    """Frame 0 (identity) to frame 1 (t = (0, 0, -1)): Z = 1 - d, full and translation-only alike, at every threshold.  Frame 1 has
    a rotation and a non-unit quaternion so the reverse edge and the random pixels are generic.  16 x 16 pixels."""
    g = _gen(11)
    c = base_case("thresholds", 16, 16, 3, 11)
    P = identity_poses(3)
    P[1, 2] = -1.0
    P[2] = random_poses(1, g)[0]
    z, names = threshold_targets()
    d = c["disps"].clone()
    k = len(z)
    d0 = (0.5 + 0.5 * torch.rand(256, generator=g)).double()
    d0 = torch.round(d0 / GRID) * GRID
    d0[:k] = 1 - z
    d[0] = d0.float().view(16, 16)
    assert torch.equal(d[0].reshape(-1)[:k].double(), 1 - z)
    c.update(poses=P, disps=d, ii=torch.tensor([0, 0, 1, 2, 0]), jj=torch.tensor([1, 2, 0, 0, 0]), target_z=z, target_names=names)
    c["intr_pf"][:] = c["intr"]                                  # a shared camera: Z does not depend on it anyway
    return c


def three_quarters_case():
    """frame_distance at a valid fraction of exactly 3/4 (pair 0 -> 1: 192 of 256 pixels at Z = 0.75, 64 at Z = 0.125, in both the
    full and the translation-only point) and one valid pixel more (pair 2 -> 1)"""
    c = base_case("fd_three_quarters", 16, 16, 3, 12)
    P = identity_poses(3)
    P[1, 2] = -1.0
    d = torch.full((3, 16, 16), 0.25)
    d.view(3, -1)[:, 192:] = 0.875
    d[2].view(-1)[192] = 0.25
    c.update(poses=P, disps=d, ii=torch.tensor([0, 2]), jj=torch.tensor([1, 1]))
    return c


def empty_case():
    """hw = 0: frame_distance gives 1000 for every pair (the reference's valid / (total + 1e-8) = 0); the other kernels write nothing"""
    c = base_case("empty", 0, 5, 3, 13, n_edges=4, stereo=0)
    return c


def depth_cells_case():
    """depth_filter projections onto chosen cells: ix = 0 identity; neighbours 3, 4, 5 translated by (1,0,0), (0,1,0), (1,1,0), no
    rotation, fx = fy = 1, cx = cy = 0, so uj = u + d (frame 3), vj = v + d (frame 4) or both (frame 5), exactly.  Pixel columns of
    row 0 carry d = target - u for: integer columns, the last accepted cell (u0 = wd - 2), the first rejected one (wd - 1), just below
    0, and beyond +-2^31.  Rows use t = inf (every in-range cell hits), t = 0 (nothing hits) and t = 0.3."""
    ht, wd = 6, 12
    c = base_case("df_cells", ht, wd, 6, 14)
    P = identity_poses(6)
    P[3, 0] = 1.0
    P[4, 1] = 1.0
    P[5, 0] = 1.0; P[5, 1] = 1.0
    g = _gen(14)
    d = (0.5 + torch.rand(6, ht, wd, generator=g)).float()
    targets = [3.0, 5.0, wd - 2 + 0.5, wd - 2.0, wd - 1.0, wd - 1 + 2.0 ** -20, -2.0 ** -20, -0.5, 3.0e9, -3.0e9, 1.0 + 2.0 ** -20, wd - 2 + 0.9990234375]
    u = torch.arange(wd, dtype=torch.float64)
    for r in range(ht):
        tgt = torch.tensor(targets, dtype=torch.float64)
        if r % 2:
            tgt = tgt.flip(0)
        d[0, r] = (tgt - u).float()
    c.update(poses=P, disps=d, intr=torch.tensor([1.0, 1.0, 0.0, 0.0]), df_ix=torch.tensor([0, 0, 0]),
             df_thresh=torch.tensor([float("inf"), 0.0, 0.3]), row_targets=targets)
    c["intr_pf"] = c["intr"][None].repeat(6, 1)
    return c


def nan_projection_case():
    """depth_filter's Z == 0, X == Y == 0 pixel: frame 3 (identity) -> neighbour 2 (t = (0,0,-1)) at pixel (cx, cy) = (2, 1) with
    d = 1: Xj = (0, 0, 0, 1), so uj = vj = 0/0 = NaN and dj = 1/0 = inf.  The target disparities in cell (0,0) of frame 2 are 4 > 1/t
    (t = 0.5): 1/dj = 0 lies within t of 1/4, so a kernel that maps NaN to cell 0 counts the pixel."""
    ht, wd = 4, 5
    c = base_case("df_nan", ht, wd, 4, 15)
    P = identity_poses(4)
    P[2, 2] = -1.0
    P[1, :3] = torch.tensor([0.3, -0.2, 0.1])
    d = c["disps"].clone()
    d[3, 1, 2] = 1.0
    d[2, :2, :2] = 4.0
    c.update(poses=P, disps=d, intr=torch.tensor([2.0, 2.0, 2.0, 1.0]), df_ix=torch.tensor([3, 3]), df_thresh=torch.tensor([0.5, 0.2]),
             ii=torch.tensor([3, 2]), jj=torch.tensor([2, 3]), nan_pixel=(3, 1, 2))
    c["intr_pf"] = c["intr"][None].repeat(4, 1)
    return c


def neighbours_case(num):
    """depth_filter with num frames (1..7): every ix from 0 to num - 1, so the neighbour set -1,-2,-3,+3,+4,+5 is clipped at both
    ends; thresholds differ per row and include 0 and inf"""
    c = base_case("df_num%d" % num, 5, 6, num, 20 + num, n_edges=3, stereo=1)
    g = _gen(40 + num)
    c["poses"] = random_poses(num, g, t_scale=0.05, rot=0.05)
    th = (0.05 + 0.5 * torch.rand(num, generator=g)).float()
    th[0] = float("inf")
    if num > 1:
        th[-1] = 0.0
    c.update(df_ix=torch.arange(num), df_thresh=th)
    return c


def nonfinite_case():
    """NaN, +-inf, 0 and negative disparities, on frame 1 only"""
    c = base_case("nonfinite", 9, 13, 4, 16)
    d = c["disps"].clone()
    vals = [float("nan"), float("inf"), -float("inf"), 0.0, -0.5, -3.0, -1e-3]
    for k, v in enumerate(vals):
        d[1].view(-1)[7 * k:7 * k + 7] = v
    c.update(disps=d, ii=torch.tensor([1, 1, 0, 2, 1, 3]), jj=torch.tensor([0, 1, 1, 1, 2, 1]), df_ix=torch.arange(4))
    return c


def many_edges_case():
    """grid.x above 65535: 70 000 edges, 70 000 depth_filter rows and 70 000 iproj frames, on a 2x3 map"""
    n = 70000
    g = _gen(17)
    c = base_case("many_edges", 2, 3, n, 17, n_edges=n, stereo=0)
    c["jj"][::97] = c["ii"][::97]
    c["df_thresh"] = (0.02 + 0.3 * torch.rand(n, generator=g)).float()
    return c


def cases():
    out = {}
    for k, (ht, wd) in SHAPES.items():
        out[k] = base_case(k, ht, wd, 8, 100 + len(out))
    for f in (thresholds_case, three_quarters_case, empty_case, depth_cells_case, nan_projection_case, nonfinite_case):
        c = f()
        out[c["name"]] = c
    for num in range(1, 8):
        c = neighbours_case(num)
        out[c["name"]] = c
    return out


CASES = ["s1x1", "s1x7", "s7x1", "hw255", "hw256", "hw257", "s43x70", "s48x64", "s60x80", "thresholds", "fd_three_quarters", "empty",
         "df_cells", "df_nan", "nonfinite"] + ["df_num%d" % n for n in range(1, 8)]


def case(name):
    if name == "many_edges":
        return many_edges_case()
    return cases()[name]


# ---- write-back -----------------------------------------------------------------------------------------------------------------
def writeback_case(name, ht, wd, seed, n_rows, n_graph, n_inactive, n_src, n_frames, n_ba_frames, edge_index):
    """inputs of dba_graph_writeback / dba_motion_features: `edge_index` is 'perm' (a permutation of graph edges), 'repeat' (edges
    named twice, for motion_features' reads) or None (identity)"""
    g = _gen(seed)
    if edge_index == "perm":
        ei = torch.randperm(n_graph, generator=g)[:n_rows]
    elif edge_index == "repeat":
        ei = torch.randint(0, n_graph, (n_rows,), generator=g)
        ei[1] = ei[0]
    else:
        ei = None
    return dict(name=name, ht=ht, wd=wd, n_graph=n_graph, n_inactive=n_inactive, edge_index=ei,
                delta=torch.randn(n_rows, ht, wd, 2, generator=g), weight=torch.rand(n_rows, ht, wd, 2, generator=g),
                coords=(wd * torch.rand(n_rows, ht, wd, 2, generator=g)), eta=torch.rand(n_src, ht, wd, generator=g),
                src_frames=torch.randperm(n_frames, generator=g)[:n_src], n_frames=n_frames,
                ba_frames=torch.randint(0, n_frames, (n_ba_frames,), generator=g), ep=0.1 * float(torch.rand(1, generator=g)) + 1e-3,
                target=wd * torch.rand(n_graph, ht, wd, 2, generator=g))


WRITEBACK = {
    "wb_perm_257": dict(ht=1, wd=257, seed=50, n_rows=5, n_graph=9, n_inactive=3, n_src=2, n_frames=6, n_ba_frames=4, edge_index="perm"),
    "wb_null_43x70": dict(ht=43, wd=70, seed=51, n_rows=4, n_graph=4, n_inactive=0, n_src=3, n_frames=5, n_ba_frames=5, edge_index=None),
    "wb_rows_only_7x1": dict(ht=7, wd=1, seed=52, n_rows=3, n_graph=6, n_inactive=2, n_src=0, n_frames=4, n_ba_frames=0, edge_index="perm"),
    "wb_damping_only_16x16": dict(ht=16, wd=16, seed=53, n_rows=0, n_graph=3, n_inactive=1, n_src=4, n_frames=6, n_ba_frames=3, edge_index=None),
}


def writeback(name):
    return writeback_case(name, **WRITEBACK[name])


# ---- cvx_upsample ---------------------------------------------------------------------------------------------------------------
def upsample_case(name):
    """(disps [n, ht, wd] fp32, mask [n, 576, ht, wd], what it reaches)"""
    shapes = {"up_equal": (2, 5, 7), "up_dominant": (2, 6, 5), "up_ties": (1, 4, 9), "up_f16_extremes": (2, 5, 6), "up_neginf": (1, 6, 7),
              "up_nan_inf": (1, 5, 5), "up_ht1": (2, 1, 9), "up_wd1": (2, 9, 1), "up_random_48x64": (2, 48, 64), "up_random_43x70": (1, 43, 70)}
    n, ht, wd = shapes[name]
    g = _gen(60 + sorted(shapes).index(name))
    d = (0.05 + 2 * torch.rand(n, ht, wd, generator=g)).float()
    m = (4 * torch.randn(n, 9, 64, ht, wd, generator=g))
    dt = torch.float16
    if name == "up_equal":
        m = m[:, :1].expand_as(m).clone()                 # all nine taps equal: the exact 9-tap mean, zero padding included
    elif name == "up_dominant":
        k = torch.randint(0, 9, (n, 1, 64, ht, wd), generator=g)
        m = torch.full_like(m, -65504.0).scatter_(1, k, 65504.0)     # one tap at the fp16 maximum, the rest at its negative
    elif name == "up_ties":
        m = torch.full_like(m, -float("inf"))
        m[:, 2] = 1.5; m[:, 6] = 1.5                      # two equal taps, the others -inf (fp32 masks)
        dt = torch.float32
    elif name == "up_f16_extremes":
        m = torch.where(torch.rand(m.shape, generator=g) < 0.3, torch.sign(m) * 65504.0, m)
    elif name == "up_neginf":
        dt = torch.float32
        m = torch.where(torch.rand(m.shape, generator=g) < 0.3, torch.full_like(m, -float("inf")), m)
        m[:, :, :, 0, :] = -float("inf")                  # every tap of row 0
    elif name == "up_nan_inf":
        dt = torch.float32
        m[:, 4, :, 1, 1] = float("nan")
        m[:, 0, :, 2, 3] = float("inf")
        m[:, 1:3, :, 3, 0] = float("inf")
    elif name.startswith("up_random"):
        dt = torch.float16 if name.endswith("48x64") else torch.float32
    return d, m.reshape(n, 576, ht, wd).to(dt).contiguous()


UPSAMPLE = ["up_equal", "up_dominant", "up_ties", "up_f16_extremes", "up_neginf", "up_nan_inf", "up_ht1", "up_wd1", "up_random_48x64",
            "up_random_43x70"]
