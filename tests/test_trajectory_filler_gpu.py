"""The native trajectory filler: droid_backends.fill_interpolate / pose_only_ba against fp64, pose_only_ba against the general ba, and
modules.fill_trajectory / install_trajectory_filler_hook against the reference's control flow (oracle/trajectory_filler.py) on the
native operators.  Stand-ins for DepthVideo, FactorGraph and PoseTrajectoryFiller are built from seeds; the reference tree is not read."""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle.shims import lietorch  # noqa: E402  (pure torch: runs the reference's SE3 arithmetic on CUDA tensors in fp32)
import droid_slam_b200  # noqa: E402
import oracle  # noqa: E402
import oracle.encoder as oenc  # noqa: E402
from oracle import trajectory_filler as otf  # noqa: E402
from droid_slam_b200 import modules, synth  # noqa: E402
import factor_graph_stubs as fs  # noqa: E402
from util import host_syncs, syncs_not_counted  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def be():
    return droid_slam_b200.install()


def _keyframe_poses(n, g, step=0.15):
    xi = step * torch.randn(n, 6, generator=g, dtype=torch.float64)
    xi[:, :3] += 0.2 * torch.arange(n, dtype=torch.float64)[:, None]
    return lietorch.SE3.exp(xi).data


# ---- fill_interpolate ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ["unsorted", "sorted"])
def test_fill_interpolate_against_fp64(be, order):
    g = torch.Generator().manual_seed(0)
    N = 9
    P = _keyframe_poses(N, g)
    ts = torch.randperm(40, generator=g)[:N].double().sort().values
    if order == "unsorted":
        ts = ts[torch.randperm(N, generator=g)]
    tq = torch.cat([ts - 1e-4, ts, ts + 0.5, torch.tensor([-2.0, float(ts.max()) + 3.0, float(ts.min()) - 0.25])])
    t0, t1, G = be.fill_interpolate(P.float().to(DEV), ts.float().to(DEV), tq.float().to(DEV))
    w0, w1, G64 = otf.interpolate(P, ts.float().double(), tq.float().double().tolist(), lietorch.SE3)
    _, _, G32 = otf.interpolate(P.float(), ts.float(), tq.float().tolist(), lietorch.SE3)
    assert torch.equal(t0.cpu(), w0) and torch.equal(t1.cpu(), w1)
    assert int((w0 == -1).sum()) >= 2 and int((w0 == w1).sum()) >= 1
    scale = 1 + G64[:, :3].norm(dim=1)
    err = (G.cpu().double() - G64).abs().amax(dim=1)
    err32 = (G32.double() - G64).abs().amax(dim=1)
    # frames inside their bracket (t0 >= 0, ts[t0] <= t <= ts[t1]): 1e-6 (1 + |t|)
    tsf, tqf = ts.float().double(), tq.float().double()
    inside = (w0 >= 0) & (w1 > w0) & (tsf[w0.clamp(min=0)] <= tqf) & (tqf <= tsf[w1])
    if order == "sorted":
        assert int(inside.sum()) >= 2 * (N - 1)
    assert bool((err[inside] <= 1e-6 * scale[inside]).all()), float((err / scale)[inside].max())
    # extrapolated frames (t0 = -1, after the last keyframe, or outside ts[t0]..ts[t1] with an unsorted ts) take tangent steps of many
    # times the bracket, where lietorch's own fp32 formulas (oracle/shims) lose up to a few 1e-5: 1e-6 (1 + |t|) or 4x that error
    out = ~inside
    assert bool((err[out] <= 1e-6 * scale[out] + 4 * err32[out]).all()), (float((err / scale)[out].max()), float((err32 / scale)[out].max()))


# ---- pose_only_ba --------------------------------------------------------------------------------------------------------------------
def _filler_ba_case(F, ht, wd, two, seed, zero_frame=None):
    """K keyframes (fixed, frames 0..K-1) and F optimised frames (K..K+F-1), each with one edge from keyframe t0 (and one from t0 + 1 when
    `two`), in the filler's order: all t0 edges, then the t1 edges"""
    g = torch.Generator().manual_seed(seed)
    K = 6
    kf = _keyframe_poses(K, g)
    t0 = torch.randint(0, K - 1, (F,), generator=g)
    a = torch.rand(F, 1, generator=g, dtype=torch.float64)
    xi = torch.cat([0.05 * torch.randn(F, 6, generator=g, dtype=torch.float64)], 1)
    fr = (lietorch.SE3.exp(xi) * lietorch.SE3(kf[t0])).data
    fr[:, :3] += a * (kf[t0 + 1, :3] - kf[t0, :3])
    poses = torch.cat([kf, fr]).float()
    disps = (0.4 + 0.6 * torch.rand(K, ht, wd, generator=g))
    intr = torch.tensor([0.9 * wd, 0.9 * wd, wd / 2.0, ht / 2.0])
    k = torch.arange(F)
    ii = torch.cat([t0, t0 + 1]) if two else t0
    jj = (torch.cat([k, k]) if two else k) + K
    E = ii.numel()
    coords, _ = oracle.reproject(poses, torch.cat([disps, torch.ones(F, ht, wd)]), intr[None].repeat(K + F, 1), ii, jj)
    gt = lietorch.SE3(poses.double()).data.clone()
    targets = (coords + 1.5 * torch.randn(coords.shape, generator=g)).permute(0, 3, 1, 2).contiguous()
    weights = torch.rand(E, 2, ht, wd, generator=g)
    if zero_frame is not None:
        weights[jj == K + zero_frame] = 0
    return dict(poses=poses, disps=disps, intr=intr, ii=ii, jj=jj, targets=targets, weights=weights, t0=K, t1=K + F, gt=gt)


def _fp64_block_system(c, poses):
    terms = oracle.ba_edge_terms(poses.double(), c["disps"].double(), c["intr"].double(), c["targets"].double(), c["weights"].double(),
                                 c["ii"], c["jj"])
    A, b, _ = oracle.ba_system(terms, c["disps"].double(), None, None, c["ii"], c["jj"], c["t0"], c["t1"], True, torch.float64)
    F = c["t1"] - c["t0"]
    blocks = torch.stack([A[6 * f:6 * f + 6, 6 * f:6 * f + 6] for f in range(F)])
    chi2 = torch.zeros(F, dtype=torch.float64).index_add_(0, c["jj"] - c["t0"], terms["r2"].double().sum(1))
    return blocks, b.view(F, 6), chi2


CASES = [(1, 3, 5, False), (16, 30, 40, True), (16, 43, 70, False), (16, 48, 64, True), (300, 48, 64, True), (5, 30, 40, True)]


@pytest.mark.parametrize("F,ht,wd,two", CASES)
def test_pose_only_ba_each_iteration_against_fp64(be, F, ht, wd, two):
    c = _filler_ba_case(F, ht, wd, two, seed=F + ht, zero_frame=2 if F == 5 else None)
    P = c["poses"].to(DEV)
    args = [x.to(DEV) for x in (c["disps"], c["intr"], c["targets"], c["weights"], c["ii"], c["jj"])]
    lm64, ep64 = float(torch.tensor(1e-4)), float(torch.tensor(0.1))
    for it in range(3):
        before = P.cpu().clone()
        status, dx, sys_ = be.pose_only_ba(P, *args, c["t0"], c["t1"], 1, 1e-4, 0.1, True, True)
        after = P.cpu()
        H, b, chi2 = _fp64_block_system(c, before)
        Hn, bn = sys_.cpu()[:, :36].view(-1, 6, 6), sys_.cpu()[:, 36:]
        d = torch.diagonal(H, dim1=1, dim2=2).clamp(min=1e-30)
        eH = ((Hn - H).abs() / (d[:, :, None] * d[:, None, :]).sqrt()).amax()
        eb = ((bn - b).abs() / (d * chi2[:, None]).clamp(min=1e-30).sqrt()).amax()
        assert eH <= 1e-5 and eb <= 1e-5, (it, float(eH), float(eb))
        # the solve against fp64 on the native block, damped as dba_ba damps
        Hd = Hn.clone()
        Hd.diagonal(dim1=1, dim2=2).add_(ep64 + lm64 * Hn.diagonal(dim1=1, dim2=2))
        x = torch.linalg.solve(Hd, bn[..., None])[..., 0]
        if F == 5:
            assert torch.equal(dx.cpu()[2], torch.zeros(6)), "a frame without weight has H = b = 0: its dx must be exactly 0"
        ex = float((dx.cpu().double() - x).abs().max()) / max(float(x.abs().max()), 1e-30)
        assert ex <= 1e-6, (it, ex)
        # the retraction of the native dx, fp64
        tq = oracle.retr_se3(dx.cpu().double(), before[c["t0"]:, :3].double(), before[c["t0"]:, 3:].double())
        want = torch.cat(tq, -1)
        er = ((after[c["t0"]:].double() - want).abs().amax(1) / (1 + want[:, :3].norm(dim=1))).max()
        assert er <= 1e-6, (it, float(er))
        assert torch.equal(after[:c["t0"]], before[:c["t0"]])
        assert int(status.cpu()) == 0


@pytest.mark.parametrize("F,ht,wd,two", [(16, 30, 40, True), (16, 48, 64, False), (300, 48, 64, True)])
def test_pose_only_ba_against_general_motion_only_ba(be, F, ht, wd, two):
    c = _filler_ba_case(F, ht, wd, two, seed=7 + F)
    dev_args = [x.to(DEV) for x in (c["disps"], c["intr"], c["targets"], c["weights"], c["ii"], c["jj"])]
    Pa, Pb = c["poses"].to(DEV), c["poses"].to(DEV)
    be.pose_only_ba(Pa, *dev_args, c["t0"], c["t1"], 2, 1e-4, 0.1, True, True)
    n = Pb.shape[0]
    disps_all = torch.cat([c["disps"], torch.ones(n - c["disps"].shape[0], ht, wd)]).to(DEV)
    be.ba(Pb, disps_all, c["intr"].to(DEV), torch.zeros_like(disps_all), dev_args[2], dev_args[3], torch.ones(1, device=DEV), dev_args[4],
          dev_args[5], c["t0"], c["t1"], 2, 1e-4, 0.1, True)
    dt = (Pa[:, :3] - Pb[:, :3]).norm(dim=1).max()
    assert float(dt) <= 1e-4 * float(Pb[:, :3].norm(dim=1).max()), float(dt)
    assert float((Pa[:, 3:] - Pb[:, 3:]).abs().max()) <= 1e-4


def test_pose_only_ba_bits_do_not_depend_on_the_batch(be):
    c = _filler_ba_case(16, 30, 40, True, seed=3)
    full = c["poses"].to(DEV)
    be.pose_only_ba(full, *[x.to(DEV) for x in (c["disps"], c["intr"], c["targets"], c["weights"], c["ii"], c["jj"])], c["t0"], c["t1"], 2, 1e-4, 0.1, True, True)
    K, f = c["t0"], 5
    sel = torch.nonzero(c["jj"] == K + f)[:, 0]
    one = torch.cat([c["poses"][:K], c["poses"][K + f:K + f + 1]]).to(DEV)
    be.pose_only_ba(one, c["disps"].to(DEV), c["intr"].to(DEV), c["targets"][sel].to(DEV), c["weights"][sel].to(DEV), c["ii"][sel].to(DEV),
                    torch.full((sel.numel(),), K, dtype=torch.long, device=DEV), K, K + 1, 2, 1e-4, 0.1, True, True)
    assert torch.equal(one[K], full[K + f])


@pytest.mark.parametrize("bad", ["source_in_window", "target_outside", "negative"])
def test_pose_only_ba_structure_violation_raises_with_poses_untouched(be, bad):
    c = _filler_ba_case(4, 30, 40, True, seed=1)
    ii, jj = c["ii"].clone(), c["jj"].clone()
    if bad == "source_in_window":
        ii[3] = c["t0"] + 1
    elif bad == "target_outside":
        jj[5] = c["t0"] - 1
    else:
        ii[0] = -1
    P = c["poses"].to(DEV)
    before = P.clone()
    with pytest.raises(RuntimeError, match="no pose was changed"):
        be.pose_only_ba(P, c["disps"].to(DEV), c["intr"].to(DEV), c["targets"].to(DEV), c["weights"].to(DEV), ii.to(DEV), jj.to(DEV),
                        c["t0"], c["t1"], 2, 1e-4, 0.1, True, True)
    assert torch.equal(P, before)


# ---- the whole filler --------------------------------------------------------------------------------------------------------------------
HT, WD = 16, 24


class FVideo:
    """DepthVideo's buffers, counter, __setitem__ (depth_video.py:70-113) and geometry on the native kernels"""

    def __init__(self, B, N, seed):
        g = torch.Generator().manual_seed(seed)
        s = synth.make_scene(dict(E=4, N=N, ht=HT, wd=WD, itrs=2, lm=1e-4, ep=0.1), seed=seed)
        self.counter = types.SimpleNamespace(value=N)
        self.tstamp = torch.zeros(B, device=DEV)
        self.tstamp[:N] = (3.0 * torch.arange(N) + torch.rand(N, generator=g)).to(DEV)
        self.images = torch.zeros(B, 3, 8 * HT, 8 * WD, dtype=torch.uint8, device=DEV)
        self.poses = torch.zeros(B, 7, device=DEV)
        self.poses[:, 6] = 1
        self.poses[:N] = s["poses"].to(DEV)
        self.poses[B - 1] = s["poses"][N // 2].to(DEV)          # the slot a frame before keyframe 0 reads (index -1)
        self.disps = torch.ones(B, HT, WD, device=DEV)
        self.disps[:N] = s["disps"].to(DEV)
        self.disps[B - 1] = s["disps"][N // 2].to(DEV)
        self.disps_sens = torch.zeros_like(self.disps)
        self.intrinsics = torch.zeros(B, 4, device=DEV)
        self.intrinsics[:N] = s["intrinsics"].to(DEV)
        self.intrinsics[B - 1] = s["intrinsics"].to(DEV)
        self.fmaps = torch.randn(B, 1, 128, HT, WD, generator=g).half().to(DEV)
        self.nets = torch.tanh(torch.randn(B, 128, HT, WD, generator=g)).half().to(DEV)
        self.inps = torch.relu(torch.randn(B, 128, HT, WD, generator=g)).half().to(DEV)

    def state(self):
        return [t.clone() for t in (self.tstamp, self.images, self.poses, self.disps, self.intrinsics, self.fmaps, self.nets, self.inps)]

    def __setitem__(self, index, item):
        self.tstamp[index] = item[0]
        self.images[index] = item[1]
        self.poses[index] = item[2]
        self.disps[index] = item[3]
        self.intrinsics[index] = item[5]
        self.fmaps[index] = item[6]

    def reproject(self, ii, jj):
        return modules.reproject(self.poses, self.disps, self.intrinsics, ii, jj)

    def ba(self, target, weight, eta, ii, jj, t0=1, t1=None, itrs=2, lm=1e-4, ep=0.1, motion_only=False):
        with syncs_not_counted():
            droid_slam_b200.install().ba(self.poses, self.disps, self.intrinsics[0], self.disps_sens, target, weight, eta, ii, jj, t0, t1,
                                         itrs, lm, ep, motion_only)


class FGraph:
    """FactorGraph.add_factors (factor_graph.py:95-150, volume corr) and update on modules.update (the general ba).  Negative source
    indices are taken modulo the buffer, as the reference's tensor indexing does (its ba kernel would read out of bounds)."""

    def __init__(self, video, update_op):
        self.video, self.update_op, self.upsample = video, update_op, False
        z = torch.zeros(0, dtype=torch.long, device=DEV)
        self.ii, self.jj, self.age, self.ii_inac, self.jj_inac = z, z, z, z, z
        y, x = torch.meshgrid(torch.arange(HT, device=DEV).float(), torch.arange(WD, device=DEV).float(), indexing="ij")
        self.coords0 = torch.stack([x, y], dim=-1)
        self.damping = 1e-6 * torch.ones_like(video.disps)
        self.target = torch.zeros(1, 0, HT, WD, 2, device=DEV)
        self.weight = torch.zeros_like(self.target)
        self.net = self.inp = self.corr = None

    def add_factors(self, ii, jj):
        ii = ii % self.video.poses.shape[0]
        if len(self.ii) > 0:
            keep = ~((ii[:, None] == self.ii) & (jj[:, None] == self.jj)).any(dim=-1)
            ii, jj = ii[keep], jj[keep]
        if ii.shape[0] == 0:
            return
        v = self.video
        self.ii, self.jj = torch.cat([self.ii, ii]), torch.cat([self.jj, jj])
        self.age = torch.cat([self.age, torch.zeros_like(ii)])
        net, inp = v.nets[ii][None], v.inps[ii][None]
        self.net = net if self.net is None else torch.cat([self.net, net], 1)
        self.inp = inp if self.inp is None else torch.cat([self.inp, inp], 1)
        self.corr = fs.CorrBlock(v.fmaps[self.ii, 0][None], v.fmaps[self.jj, 0][None])       # the same volumes as CorrBlock.cat
        target = v.reproject(ii, jj)[0]
        self.target = torch.cat([self.target, target], 1)
        self.weight = torch.cat([self.weight, torch.zeros_like(target)], 1)

    def update(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
        modules.update(self, t0, t1, itrs, use_inactive, EP, motion_only)


def _encoder_class():
    ns = types.SimpleNamespace(BasicEncoder=type("BasicEncoder", (oenc.BasicEncoder,), {}))
    modules.install_encoder_hook(ns)
    return ns.BasicEncoder


def _filler(video):
    fnet = _encoder_class()(output_dim=128, norm_fn="instance")
    fnet.load_state_dict(synth.make_encoder_weights(0, 128))
    return types.SimpleNamespace(fnet=fnet.to(DEV).eval(), update=fs.update_op(DEV), video=video,
                                 MEAN=torch.as_tensor([0.485, 0.456, 0.406], device=DEV)[:, None, None],
                                 STDV=torch.as_tensor([0.229, 0.224, 0.225], device=DEV)[:, None, None])


def _stream(video, T, seed):
    """frames at, between and after keyframes, one before keyframe 0, T frames (not a multiple of 16)"""
    g = torch.Generator().manual_seed(seed)
    N = video.counter.value
    kts = video.tstamp[:N].cpu().tolist()
    ts = [kts[0] - 1.5, kts[0], kts[2], kts[-1] + 2.0] + sorted((torch.rand(T - 4, generator=g) * (kts[-1] - kts[0]) + kts[0]).tolist())
    intr = video.intrinsics[0].cpu() * 8.0
    return [(t, torch.randint(0, 255, (1, 3, 8 * HT, 8 * WD), generator=g, dtype=torch.uint8).to(DEV), intr) for t in ts]


def test_fill_trajectory_against_the_reference_flow(be, monkeypatch):
    video = FVideo(64, 8, seed=11)
    filler = _filler(video)
    stream = _stream(video, 37, seed=2)
    monkeypatch.setattr(modules, "_filler_frame_budget", lambda *a: 16)         # the reference's batches, to compare edge lists
    native_edges, fill_batch = [], modules._fill_batch

    def recording(*a):
        out = fill_batch(*a)
        native_edges.append(out[1])
        return out

    monkeypatch.setattr(modules, "_fill_batch", recording)
    before = video.state()
    with torch.no_grad():
        got = modules.fill_trajectory(filler, stream)
    after = video.state()
    assert all(torch.equal(a, b) for a, b in zip(before, after)), "the native filler modified the video"
    with torch.no_grad():
        want, edges = otf.fill(filler, stream, FGraph, lietorch.SE3)
    assert got.shape == want.shape == (37, 7)
    # the hook's t0 / t1 and edge lists against the reference flow's, batch by batch (the hook's frame B + k is the reference's N + k)
    B, N = video.poses.shape[0], video.counter.value
    t0, t1, _ = otf.interpolate(video.poses[:N].cpu(), video.tstamp[:N].cpu(), [s[0] for s in stream], lietorch.SE3)
    assert len(native_edges) == len(edges) == 3
    for k, ((ii, jj), (n0, n1, nii, njj)) in enumerate(zip(edges, native_edges)):
        assert torch.equal(n0, t0[16 * k:16 * k + 16]) and torch.equal(n1, t1[16 * k:16 * k + 16]), k
        assert torch.equal(nii, ii.cpu()) and torch.equal(njj - B + N, jj.cpu()), k
    assert int((t0 == -1).sum()) == 1 and int((t0 == t1).sum()) >= 1
    dt = (got[:, :3] - want[:, :3]).norm(dim=1).max()
    assert float(dt) <= 1e-4 * float(want[:, :3].norm(dim=1).max()), float(dt)


def test_fill_trajectory_bits_do_not_depend_on_the_batch_size(be, monkeypatch):
    video = FVideo(64, 8, seed=12)
    filler = _filler(video)
    stream = _stream(video, 40, seed=3)
    out = []
    for budget in (16, 1000):
        monkeypatch.setattr(modules, "_filler_frame_budget", lambda *a, b=budget: b)
        with torch.no_grad():
            out.append(modules.fill_trajectory(filler, stream))
    assert torch.equal(out[0], out[1])


def test_fill_trajectory_host_syncs_per_batch(be, monkeypatch):
    monkeypatch.setattr(modules, "_filler_frame_budget", lambda *a: 8)
    video = FVideo(64, 8, seed=13)
    filler = _filler(video)
    stream = _stream(video, 20, seed=4)
    with torch.no_grad():
        modules.fill_trajectory(filler, stream)          # warm-up: packs the weights once
        n, _ = host_syncs(lambda: modules.fill_trajectory(filler, stream))
    assert n <= 3, n                                     # three batches of at most 8 frames


def _filler_class():
    class PoseTrajectoryFiller:
        def __init__(self, filler):
            self.__dict__.update(vars(filler))

        def __call__(self, image_stream):
            return "reference"
    return PoseTrajectoryFiller


def test_filler_hook_strict_and_fallback(be, monkeypatch):
    PoseTrajectoryFiller = _filler_class()
    video = FVideo(64, 8, seed=14)
    mod = types.SimpleNamespace(PoseTrajectoryFiller=PoseTrajectoryFiller, SE3=lietorch.SE3)
    modules.install_trajectory_filler_hook(mod)
    f = PoseTrajectoryFiller(_filler(video))
    out = f(_stream(video, 5, seed=5))
    assert isinstance(out, lietorch.SE3) and out.data.shape == (5, 7)
    f.update = torch.nn.Identity()
    with pytest.raises(RuntimeError, match="not droid_slam_b200.update.UpdateModule"):
        f([])
    f = PoseTrajectoryFiller(_filler(video))
    f.fnet = oenc.BasicEncoder(output_dim=128, norm_fn="instance").to(DEV)
    with pytest.raises(RuntimeError, match="install_encoder_hook"):
        f([])
    mod2 = types.SimpleNamespace(PoseTrajectoryFiller=_filler_class(), SE3=lietorch.SE3)
    modules.install_trajectory_filler_hook(mod2, strict=False)
    g = mod2.PoseTrajectoryFiller(_filler(video))
    checks, check = [], modules._filler_unsupported
    monkeypatch.setattr(modules, "_filler_unsupported", lambda *a: checks.append(a) or check(*a))
    assert isinstance(g(_stream(video, 5, seed=5)), lietorch.SE3)
    assert len(checks) == 1                               # native: the readiness check ran once for the call
    g.video = types.SimpleNamespace(**{k: (t.cpu() if isinstance(t, torch.Tensor) else t) for k, t in vars(video).items()})
    assert g([]) == "reference"
