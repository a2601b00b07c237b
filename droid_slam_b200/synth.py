"""Synthetic factor graphs of the shapes BASELINE.json names (SURVEY.md section 8d "Synthetic inputs").

Everything is generated on the CPU with fixed seeds (torch.Generator) and returned as a dict of CPU tensors; callers
move what they need to the GPU.  Pure PyTorch, no dependency on the oracle or on the native extension.
"""
import math
import torch
import torch.nn.functional as F

__all__ = ["CONFIGS", "make_graph", "make_scene", "reproject", "make_corr_inputs", "se3_exp", "se3_mul"]

# name -> (edges, frames, ht, wd, stereo, ba iterations, lm, ep)
CONFIGS = {
    "c1_plumbing": dict(E=24, N=8, ht=48, wd=64, stereo=False, itrs=3, lm=1e-4, ep=0.1),
    "c2_frontend": dict(E=128, N=25, ht=48, wd=64, stereo=False, itrs=2, lm=1e-4, ep=0.1),
    "metric": dict(E=512, N=72, ht=48, wd=64, stereo=False, itrs=2, lm=1e-4, ep=0.1),
    "c3_global": dict(E=2048, N=400, ht=48, wd=64, stereo=False, itrs=10, lm=1e-5, ep=1e-2),
    "c4_stereo": dict(E=256, N=64, ht=48, wd=64, stereo=True, itrs=2, lm=1e-4, ep=0.1),
    "c5_stress": dict(E=4096, N=500, ht=72, wd=96, stereo=False, itrs=2, lm=1e-4, ep=0.1),
}


# ---- minimal SE3 (tx,ty,tz,qx,qy,qz,qw), double precision, only for scene generation ---------------------------
def _qmul(a, b):
    ax, ay, az, aw = a.unbind(-1); bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx,
                        aw * bz + ax * by - ay * bx + az * bw,
                        aw * bw - ax * bx - ay * by - az * bz], dim=-1)


def _qrot(q, v):
    qv, qw = q[..., :3], q[..., 3:4]
    uv = 2.0 * torch.cross(qv, v, dim=-1)
    return v + qw * uv + torch.cross(qv, uv, dim=-1)


def se3_exp(xi):
    """xi [...,6] (tau, phi) -> pose [...,7]."""
    tau, phi = xi[..., :3], xi[..., 3:]
    th = phi.norm(dim=-1, keepdim=True)
    small = th < 1e-6
    ths = torch.where(small, torch.ones_like(th), th)
    q = torch.cat([torch.where(small, 0.5 * phi, torch.sin(0.5 * ths) / ths * phi), torch.where(small, torch.ones_like(th), torch.cos(0.5 * ths))], -1)
    a = torch.where(small, 0.5 * torch.ones_like(th), (1 - torch.cos(ths)) / ths ** 2)
    b = torch.where(small, torch.ones_like(th) / 6, (ths - torch.sin(ths)) / ths ** 3)
    c1 = torch.cross(phi, tau, dim=-1)
    t = tau + a * c1 + b * torch.cross(phi, c1, dim=-1)
    return torch.cat([t, q], -1)


def se3_mul(A, B):
    """A * B (apply B first)."""
    return torch.cat([_qrot(A[..., 3:], B[..., :3]) + A[..., :3], _qmul(A[..., 3:], B[..., 3:])], -1)


def se3_inv(A):
    qi = torch.cat([-A[..., 3:6], A[..., 6:7]], -1)
    return torch.cat([-_qrot(qi, A[..., :3]), qi], -1)


def reproject(poses, disps, intr, ii, jj):
    """pixel coordinates of frame ii's pixels in frame jj; poses are world->camera (like DROID). [E,ht,wd,2], depth z."""
    E = ii.shape[0]
    N, ht, wd = disps.shape
    fx, fy, cx, cy = [float(v) for v in intr]
    v, u = torch.meshgrid(torch.arange(ht, dtype=poses.dtype), torch.arange(wd, dtype=poses.dtype), indexing="ij")
    X = torch.stack([(u - cx) / fx, (v - cy) / fy, torch.ones_like(u)], -1).expand(E, ht, wd, 3)
    d = disps[ii].to(poses.dtype)[..., None]
    G = se3_mul(poses[jj], se3_inv(poses[ii]))
    stereo = (ii == jj)
    if bool(stereo.any()):
        G = G.clone()
        G[stereo] = torch.tensor([-0.1, 0, 0, 0, 0, 0, 1], dtype=poses.dtype)
    Y = _qrot(G[:, None, None, 3:], X) + d * G[:, None, None, :3]
    z = Y[..., 2].clamp(min=1e-3)
    return torch.stack([fx * Y[..., 0] / z + cx, fy * Y[..., 1] / z + cy], -1), Y[..., 2]


def _smooth_noise(g, n, ht, wd):
    low = torch.randn(n, 1, max(2, ht // 8), max(2, wd // 8), generator=g, dtype=torch.float64)
    return F.interpolate(low, size=(ht, wd), mode="bilinear", align_corners=True)[:, 0]


def make_graph(E, N, stereo=False, seed=0, t0=1):
    """radius-2 neighbourhood edges in both directions + random loop closures with |i-j|>2 until E edges;
    stereo graphs add one (i,i) edge per frame first.  Edge order is shuffled deterministically (the reference's
    edge lists are not sorted either).  Returns ii, jj (int64)."""
    g = torch.Generator().manual_seed(1234 + seed)
    edges = []
    if stereo:
        edges += [(i, i) for i in range(N)]
    for dlt in (1, 2):          # all radius-1 edges first: truncation to E keeps an out-edge for every frame
        for i in range(N):
            for j in (i - dlt, i + dlt):
                if 0 <= j < N:
                    edges.append((i, j))
    edges = edges[:E] if len(edges) > E else edges
    have = set(edges)
    # loop closures between covisible frames: 2 < |i-j| <= span, the span grows only when the near pairs are exhausted
    span = 12
    while len(edges) < E:
        cand = [(i, j) for i in range(N) for j in range(N) if 2 < abs(i - j) <= span and (i, j) not in have]
        if not cand:
            if span >= N:
                break
            span = min(N, span * 2)
            continue
        order = torch.randperm(len(cand), generator=g).tolist()
        for k in order[:E - len(edges)]:
            have.add(cand[k]); edges.append(cand[k])
        span = min(N, span * 2)
    perm = torch.randperm(len(edges), generator=g)
    ii = torch.tensor([edges[k][0] for k in perm.tolist()], dtype=torch.long)
    jj = torch.tensor([edges[k][1] for k in perm.tolist()], dtype=torch.long)
    return ii, jj


def make_scene(cfg="metric", seed=0, rgbd=False, device="cpu", **over):
    """Full BA problem for a named config: dict with poses, disps, disps_sens, intrinsics, targets, weights, eta, ii, jj,
    t0, t1, itrs, lm, ep, plus the ground truth (poses_gt, disps_gt).
    device: where the per-pixel tensors are generated (default CPU; a CUDA device draws from that device's seeded generator -- a
    different but equally deterministic scene, used for the stress config whose 8192-edge scene takes minutes on the host)."""
    c = dict(CONFIGS[cfg]) if isinstance(cfg, str) else dict(cfg)
    c.update(over)
    E, N, ht, wd = c["E"], c["N"], c["ht"], c["wd"]
    if str(device) != "cpu":
        return _make_scene_on_device(c, seed, rgbd, torch.device(device))
    g = torch.Generator().manual_seed(1234 + seed)
    intr = torch.tensor([0.8 * 320 / 8 * (wd / 64), 0.8 * 320 / 8 * (wd / 64), wd / 2 - 0.5, ht / 2 - 0.5], dtype=torch.float64)
    k = torch.arange(N, dtype=torch.float64)[:, None]
    xi = k * torch.tensor([0.05, 0.0, 0.02, 0.0, 0.01, 0.0], dtype=torch.float64) + 0.01 * torch.randn(N, 6, generator=g, dtype=torch.float64)
    poses_gt = se3_exp(xi)
    disps_gt = (1.0 + 0.3 * _smooth_noise(g, N, ht, wd)).clamp(0.1, 4.0)
    if c.get("graph") is not None:                       # explicit edge list (ii, jj) instead of the generated sliding-window graph
        ii, jj = (torch.as_tensor(x, dtype=torch.long) for x in c["graph"])
    else:
        ii, jj = make_graph(E, N, stereo=c.get("stereo", False), seed=seed)
    E = ii.shape[0]
    t0 = c.get("t0", 1); t1 = c.get("t1", N)
    coords, z_true = reproject(poses_gt, disps_gt, intr, ii, jj)
    targets = coords + 0.5 * torch.randn(E, ht, wd, 2, generator=g, dtype=torch.float64)
    weights = torch.rand(E, ht, wd, 2, generator=g, dtype=torch.float64)
    weights = torch.where(torch.rand(E, ht, wd, 2, generator=g) < 0.1, torch.zeros_like(weights), weights)
    # like the update operator, give no confidence to points that are not observable from the target frame
    visible = (z_true > 0.5) & (coords[..., 0] > -wd) & (coords[..., 0] < 2 * wd) & (coords[..., 1] > -ht) & (coords[..., 1] < 2 * ht)
    weights = weights * visible[..., None].to(weights.dtype)
    targets = torch.where(visible[..., None], targets, torch.zeros_like(targets))
    kx = torch.unique(torch.cat([torch.arange(t0, t1), ii]))
    M = kx.shape[0]
    eta = 0.2 * 0.01 * F.softplus(torch.randn(M, ht, wd, generator=g, dtype=torch.float64)) + 1e-7
    poses = se3_mul(se3_exp(0.02 * torch.randn(N, 6, generator=g, dtype=torch.float64)), poses_gt)
    poses[:t0] = poses_gt[:t0]
    disps = disps_gt * torch.exp(0.1 * torch.randn(N, ht, wd, generator=g, dtype=torch.float64))
    if rgbd:
        mask = torch.rand(N, ht, wd, generator=g) < 0.5
        disps_sens = torch.where(mask, disps_gt, torch.zeros_like(disps_gt))
    else:
        disps_sens = torch.zeros_like(disps_gt)
    f32 = lambda x: x.float().contiguous()
    return dict(cfg=c, poses=f32(poses), disps=f32(disps), disps_sens=f32(disps_sens), intrinsics=f32(intr),
                targets=f32(targets.permute(0, 3, 1, 2)), weights=f32(weights.permute(0, 3, 1, 2)), eta=f32(eta),
                ii=ii, jj=jj, t0=t0, t1=t1, itrs=c["itrs"], lm=c["lm"], ep=c["ep"], M=M,
                poses_gt=f32(poses_gt), disps_gt=f32(disps_gt), coords_gt=f32(coords))


def _make_scene_on_device(c, seed, rgbd, dev):
    """make_scene with the per-pixel work on a CUDA device (same construction, device-side random streams); returns CPU-free tensors
    on `dev` except ii/jj (CPU, like make_scene)"""
    E, N, ht, wd = c["E"], c["N"], c["ht"], c["wd"]
    g = torch.Generator(device=dev).manual_seed(1234 + seed)
    f64 = dict(dtype=torch.float64, device=dev)
    intr = torch.tensor([0.8 * 320 / 8 * (wd / 64), 0.8 * 320 / 8 * (wd / 64), wd / 2 - 0.5, ht / 2 - 0.5], **f64)
    k = torch.arange(N, **f64)[:, None]
    xi = k * torch.tensor([0.05, 0.0, 0.02, 0.0, 0.01, 0.0], **f64) + 0.01 * torch.randn(N, 6, generator=g, **f64)
    poses_gt = se3_exp(xi)
    low = torch.randn(N, 1, max(2, ht // 8), max(2, wd // 8), generator=g, **f64)
    disps_gt = (1.0 + 0.3 * F.interpolate(low, size=(ht, wd), mode="bilinear", align_corners=True)[:, 0]).clamp(0.1, 4.0)
    if c.get("graph") is not None:
        ii, jj = (torch.as_tensor(x, dtype=torch.long) for x in c["graph"])
    else:
        ii, jj = make_graph(E, N, stereo=c.get("stereo", False), seed=seed)
    E = ii.shape[0]
    t0 = c.get("t0", 1); t1 = c.get("t1", N)
    iid, jjd = ii.to(dev), jj.to(dev)
    # reprojection in edge chunks (the [E,ht,wd,3] fp64 intermediates of 8192 edges at 72x96 would not fit comfortably at once)
    coords = torch.empty(E, ht, wd, 2, **f64); z_true = torch.empty(E, ht, wd, **f64)
    fx, fy, cx, cy = [float(v) for v in intr]
    v, u = torch.meshgrid(torch.arange(ht, **f64), torch.arange(wd, **f64), indexing="ij")
    Xn = torch.stack([(u - cx) / fx, (v - cy) / fy, torch.ones_like(u)], -1)
    for s0 in range(0, E, 512):
        sl = slice(s0, min(E, s0 + 512))
        G = se3_mul(poses_gt[jjd[sl]], se3_inv(poses_gt[iid[sl]]))
        st = iid[sl] == jjd[sl]
        if bool(st.any()):
            G = G.clone(); G[st] = torch.tensor([-0.1, 0, 0, 0, 0, 0, 1], **f64)
        Y = _qrot(G[:, None, None, 3:], Xn.expand(G.shape[0], ht, wd, 3)) + disps_gt[iid[sl]][..., None] * G[:, None, None, :3]
        z = Y[..., 2].clamp(min=1e-3)
        coords[sl] = torch.stack([fx * Y[..., 0] / z + cx, fy * Y[..., 1] / z + cy], -1); z_true[sl] = Y[..., 2]
    targets = coords + 0.5 * torch.randn(E, ht, wd, 2, generator=g, **f64)
    weights = torch.rand(E, ht, wd, 2, generator=g, **f64)
    weights = torch.where(torch.rand(E, ht, wd, 2, generator=g, device=dev) < 0.1, torch.zeros_like(weights), weights)
    visible = (z_true > 0.5) & (coords[..., 0] > -wd) & (coords[..., 0] < 2 * wd) & (coords[..., 1] > -ht) & (coords[..., 1] < 2 * ht)
    weights = weights * visible[..., None].to(weights.dtype)
    targets = torch.where(visible[..., None], targets, torch.zeros_like(targets))
    kx = torch.unique(torch.cat([torch.arange(t0, t1), ii]))
    M = kx.shape[0]
    eta = 0.2 * 0.01 * F.softplus(torch.randn(M, ht, wd, generator=g, **f64)) + 1e-7
    poses = se3_mul(se3_exp(0.02 * torch.randn(N, 6, generator=g, **f64)), poses_gt)
    poses[:t0] = poses_gt[:t0]
    disps = disps_gt * torch.exp(0.1 * torch.randn(N, ht, wd, generator=g, **f64))
    if rgbd:
        disps_sens = torch.where(torch.rand(N, ht, wd, generator=g, device=dev) < 0.5, disps_gt, torch.zeros_like(disps_gt))
    else:
        disps_sens = torch.zeros_like(disps_gt)
    f32 = lambda x: x.float().contiguous()
    return dict(cfg=c, poses=f32(poses), disps=f32(disps), disps_sens=f32(disps_sens), intrinsics=f32(intr),
                targets=f32(targets.permute(0, 3, 1, 2)), weights=f32(weights.permute(0, 3, 1, 2)), eta=f32(eta),
                ii=ii, jj=jj, t0=t0, t1=t1, itrs=c["itrs"], lm=c["lm"], ep=c["ep"], M=M,
                poses_gt=f32(poses_gt), disps_gt=f32(disps_gt), coords_gt=f32(coords))


def make_corr_inputs(scene, dtype=torch.float16, seed=0, channels=128, device="cpu", levels=4, edge_chunk=32):
    """feature maps ~ N(0,1), the 4-level correlation pyramid built with the reference formula (modules/corr.py:63-71,
    24-38) and lookup coordinates = true reprojection + U(-2,2)  (~3 % of windows cross the border).
    Returns (pyramid list of [E,ht,wd,ht/2^l,wd/2^l], coords [E,2,ht,wd] float32, fmaps [N,C,ht,wd])."""
    g = torch.Generator().manual_seed(4321 + seed)
    c = scene["cfg"]
    N, ht, wd = c["N"], c["ht"], c["wd"]
    ii, jj = scene["ii"], scene["jj"]
    E = ii.shape[0]
    fmaps = torch.randn(N, channels, ht, wd, generator=g).to(device=device, dtype=dtype)
    coords = scene["coords_gt"] + (4 * torch.rand(E, ht, wd, 2, generator=g) - 2).to(scene["coords_gt"].device)
    coords = coords.permute(0, 3, 1, 2).contiguous().to(device)
    pyr = [torch.empty(E, ht, wd, ht // 2 ** l, wd // 2 ** l, dtype=dtype, device=device) for l in range(levels)]
    for s in range(0, E, edge_chunk):
        e = slice(s, min(E, s + edge_chunk))
        f1 = fmaps[ii[e].to(device)].reshape(-1, channels, ht * wd) / 4.0
        f2 = fmaps[jj[e].to(device)].reshape(-1, channels, ht * wd) / 4.0
        corr = torch.matmul(f1.transpose(1, 2), f2)
        n = corr.shape[0]
        corr = corr.reshape(n * ht * wd, 1, ht, wd)
        for l in range(levels):
            pyr[l][e] = corr.view(n, ht, wd, ht // 2 ** l, wd // 2 ** l)
            if l + 1 < levels:
                corr = F.avg_pool2d(corr, 2, stride=2)
    return pyr, coords, fmaps


# ---- update operator (SURVEY section 8a row A6): weights with the reference's state_dict names and shapes (droid_net.py:79-109,
# modules/gru.py:9-17, droid_net.py:46-57), drawn from a seed so that the reference module, the oracle and the mirror share them
UPDATE_SHAPES = {
    "corr_encoder.0": (128, 196, 1), "corr_encoder.2": (128, 128, 3),
    "flow_encoder.0": (128, 4, 7), "flow_encoder.2": (64, 128, 3),
    "weight.0": (128, 128, 3), "weight.2": (2, 128, 3),
    "delta.0": (128, 128, 3), "delta.2": (2, 128, 3),
    "gru.convz": (128, 448, 3), "gru.convr": (128, 448, 3), "gru.convq": (128, 448, 3), "gru.w": (128, 128, 1),
    "gru.convz_glo": (128, 128, 1), "gru.convr_glo": (128, 128, 1), "gru.convq_glo": (128, 128, 1),
    "agg.conv1": (128, 128, 3), "agg.conv2": (128, 128, 3), "agg.eta.0": (1, 128, 3), "agg.upmask.0": (576, 128, 1),
}


def make_update_weights(seed=0, dtype=torch.float32):
    """He-scaled random weights + small biases for every conv of the update operator, keyed like UpdateModule.state_dict()."""
    g = torch.Generator().manual_seed(4321 + seed)
    w = {}
    for name, (co, ci, k) in UPDATE_SHAPES.items():
        w[name + ".weight"] = (torch.randn(co, ci, k, k, generator=g) * (1.0 / (ci * k * k)) ** 0.5).to(dtype)
        w[name + ".bias"] = (0.1 * torch.randn(co, generator=g)).to(dtype)
    return w


def make_encoder_weights(seed=0, output_dim=128):
    """He-scaled random weights (fan_out, like the reference's init, extractor.py:166-168) + nonzero biases for every conv of a
    BasicEncoder (extractor.py:118-181), keyed like its state_dict()."""
    g = torch.Generator().manual_seed(8765 + seed)
    shapes = {"conv1": (32, 3, 7), "conv2": (output_dim, 128, 1)}
    for layer, cin, p in ((1, 32, 32), (2, 32, 64), (3, 64, 128)):
        shapes["layer%d.0.conv1" % layer] = (p, cin, 3)
        for name in ("layer%d.0.conv2" % layer, "layer%d.1.conv1" % layer, "layer%d.1.conv2" % layer):
            shapes[name] = (p, p, 3)
        if layer > 1:
            shapes["layer%d.0.downsample.0" % layer] = (p, cin, 1)
    w = {}
    for name, (co, ci, k) in shapes.items():
        w[name + ".weight"] = torch.randn(co, ci, k, k, generator=g) * math.sqrt(2.0 / (co * k * k))
        w[name + ".bias"] = 0.1 * torch.randn(co, generator=g)
    return w


def make_update_inputs(E=5, ht=6, wd=8, seed=0, n_src=3):
    """net/inp/corr/flow of E edges at ht x wd and source-frame indices ii with n_src distinct (unsorted) values."""
    g = torch.Generator().manual_seed(99 + seed)
    net = torch.tanh(torch.randn(1, E, 128, ht, wd, generator=g))
    inp = torch.relu(torch.randn(1, E, 128, ht, wd, generator=g))
    corr = torch.randn(1, E, 196, ht, wd, generator=g)
    flow = 4.0 * torch.randn(1, E, 4, ht, wd, generator=g)
    ii = torch.randint(0, n_src, (E,), generator=g) * 3 + 2          # unsorted, non-contiguous frame numbers
    return net, inp, corr, flow, ii


def make_frames(n, H, W, cams=1, seed=0, still=0.5, move=6.0, margin=32):
    """n synthetic camera frames, uint8 [n,cams,3,H,W]: one smooth random texture seen through a camera that pans by a bounded random
    walk, each frame's step either small (up to `still` pixels) or large (up to `move` pixels) at random; camera k of a rig looks 8k
    pixels to the right of camera 0.  Inputs for MotionFilter.track with frames on both sides of its motion threshold."""
    g = torch.Generator().manual_seed(9137 + seed)
    hh, ww = H + 2 * margin, W + 2 * margin + 8 * (cams - 1)
    coarse = torch.rand(1, 3, hh // 16 + 2, ww // 16 + 2, generator=g)
    fine = torch.rand(1, 3, hh // 4 + 2, ww // 4 + 2, generator=g)
    tex = 0.7 * F.interpolate(coarse, size=(hh, ww), mode="bilinear", align_corners=False)[0] \
        + 0.3 * F.interpolate(fine, size=(hh, ww), mode="bilinear", align_corners=False)[0]
    tex = (255 * tex).round().clamp(0, 255).to(torch.uint8)
    out = torch.empty(n, cams, 3, H, W, dtype=torch.uint8)
    pos = torch.zeros(2)
    for k in range(n):
        size = still if float(torch.rand(1, generator=g)) < 0.5 else move
        pos = (pos + size * (2 * torch.rand(2, generator=g) - 1)).clamp(-margin, margin)
        y, x = margin + int(round(float(pos[0]))), margin + int(round(float(pos[1])))
        for c in range(cams):
            out[k, c] = tex[:, y:y + H, x + 8 * c:x + 8 * c + W]
    return out
