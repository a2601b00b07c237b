"""Stand-in for the reference's `droid_async` module and the classes its backend process runs on, for the native DroidAsync backend
(tests/test_async_cpu.py, tests/test_async_gpu.py).  One importable module, so that every hook installed on it can be re-installed by
name in a spawned process: CorrBlock / AltCorrBlock (install_corr_volume_hook / install_alt_corr_hook take this module), UpdateModule
and DroidNet (install_update_module_hook), FactorGraph (install_factor_graph_hook, install_proximity_hook), DepthVideo
(install_depth_video_hook), and droid_async's globals backend_process, load_network, DroidAsyncBackend (install_async_hook).

DepthVideo holds the reference's buffers as CUDA tensors (handed to a spawned process through CUDA IPC, as the reference's shared
buffers are) with counter / ready as multiprocessing Values.  DroidAsyncBackend marks the frames [0, counter) dirty and records the
iteration count and whether the network's update operator is the native one; it runs no BA (BA is not bit-reproducible on large graphs,
DESIGN §5, so the tests compare the hand-over).  Built from seeds with synth and the lietorch stand-in; the reference tree is not read."""
import multiprocessing
import sys
from collections import OrderedDict

import torch

import droid_slam_b200
from droid_slam_b200 import modules, synth
from oracle.shims.lietorch import SE3


class CorrBlock:
    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        raise NotImplementedError


class AltCorrBlock:
    def __init__(self, fmaps, num_levels=4, radius=3):
        raise NotImplementedError

    def __call__(self, coords, ii, jj):
        raise NotImplementedError


class UpdateModule(torch.nn.Module):
    """the reference's operator: install_update_module_hook replaces this global"""

    def forward(self, *args):
        raise NotImplementedError


class DroidNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.update = UpdateModule()


class FactorGraph:
    def update(self, *args, **kwargs):
        raise NotImplementedError

    def update_lowmem(self, *args, **kwargs):
        raise NotImplementedError

    def add_proximity_factors(self, *args, **kwargs):
        raise NotImplementedError


class DepthVideo:
    """DepthVideo's buffers (depth_video.py:17-60) on `device`, counter / ready / lock as the reference's (multiprocessing Values)"""

    def __init__(self, buffer, ht, wd, stereo=False, device="cuda", ctx=None):
        ctx = ctx or multiprocessing.get_context("spawn")
        cams = 2 if stereo else 1
        self.counter, self.ready, self.stereo = ctx.Value("i", 0), ctx.Value("i", 0), stereo
        z = dict(device=device)
        self.tstamp = torch.zeros(buffer, **z)
        self.images = torch.zeros(buffer, cams, 3, 8 * ht, 8 * wd, dtype=torch.uint8, **z)
        self.dirty = torch.zeros(buffer, dtype=torch.bool, **z)
        self.poses = torch.zeros(buffer, 7, **z)
        self.poses[:, 6] = 1.0
        self.disps = torch.ones(buffer, ht, wd, **z)
        self.disps_sens = torch.zeros(buffer, ht, wd, **z)
        self.disps_up = torch.zeros(buffer, 8 * ht, 8 * wd, **z)
        self.intrinsics = torch.zeros(buffer, 4, **z)
        self.fmaps = torch.zeros(buffer, cams, 128, ht, wd, dtype=torch.half, **z)
        self.nets = torch.zeros(buffer, 128, ht, wd, dtype=torch.half, **z)
        self.inps = torch.zeros(buffer, 128, ht, wd, dtype=torch.half, **z)
        self.record = torch.zeros(2, dtype=torch.long, **z)        # DroidAsyncBackend: iterations, native update operator (1)

    def get_lock(self):
        return self.counter.get_lock()


def make_videos(buffer, ht, wd, mode, t0, t1, dev1="cuda", dev2="cuda", seed=0):
    """(video1 on dev1, video2 on dev2) as a backend round finds them: video1's keyframes [0, t1) filled; video2's fragment
    [t0-10, t0-1) is video1's seen through a random Sim(3), with noise.  mode: mono, rgbd (sensor depth on every keyframe), rgbd_last
    (one sensor depth in the buffer's last frame only) or stereo"""
    stereo = mode == "stereo"
    v1, v2 = DepthVideo(buffer, ht, wd, stereo, dev1), DepthVideo(buffer, ht, wd, stereo, dev2)
    g = torch.Generator().manual_seed(seed)
    front = SE3.exp(torch.cumsum(0.05 * torch.randn(buffer, 6, generator=g), 0)).data
    moved = front.clone()
    moved[:, :3] *= 0.5 + torch.rand((), generator=g)
    back = (SE3.exp(0.5 * torch.randn(1, 6, generator=g)) * SE3(moved)).data + 1e-3 * torch.randn(buffer, 7, generator=g)
    v1.poses[:t1] = front[:t1].to(dev1)
    v2.poses[:t0] = back[:t0].to(dev2)
    v1.disps[:t1] = (0.2 + torch.rand(t1, ht, wd, generator=g)).to(dev1)
    v2.disps[:t0] = (0.2 + torch.rand(t0, ht, wd, generator=g)).to(dev2)
    if mode == "rgbd":
        v1.disps_sens[:t1] = (torch.rand(t1, ht, wd, generator=g) * (torch.rand(t1, ht, wd, generator=g) > 0.2)).to(dev1)
    elif mode == "rgbd_last":
        v1.disps_sens[buffer - 1, ht // 2, wd // 2] = 0.5      # one sensor depth, in the buffer's last frame: outside [t0, t1)
    gd = torch.Generator(dev1).manual_seed(seed + 1)
    v1.images[:t1] = torch.randint(0, 256, v1.images[:t1].shape, generator=gd, dtype=torch.uint8, device=dev1)
    v1.tstamp[:t1] = torch.arange(t1, dtype=torch.float32, device=dev1) * 2.0
    v1.intrinsics[:t1] = torch.tensor([60.0, 60.0, 4.0 * wd, 4.0 * ht], device=dev1)
    for k in ("fmaps", "nets", "inps"):
        t = getattr(v1, k)
        t[:t1] = torch.randn(t[:t1].shape, generator=gd, device=dev1).half()
    v1.counter.value = t1
    v2.counter.value = t0 + 2 if t0 else 0
    return v1, v2


def write_checkpoint(path, seed=0):
    """a DROID-style checkpoint (`module.`-prefixed keys) holding random update-operator weights"""
    torch.save(OrderedDict(("module.update." + k, v) for k, v in synth.make_update_weights(seed).items()), path)


def load_network(weights, device="cuda:0"):
    """droid_async.load_network's steps on DroidNet: module. prefix dropped, loaded, moved, eval"""
    net = DroidNet()
    net.load_state_dict(OrderedDict((k.replace("module.", ""), v) for k, v in torch.load(weights).items()))
    return net.to(device=device).eval()


class DroidAsyncBackend:
    def __init__(self, net, video, args):
        self.net, self.video = net, video

    def __call__(self, steps=12, normalize=True):
        from droid_slam_b200.update import UpdateModule as Native
        t = self.video.counter.value
        self.video.dirty[:t] = True
        self.video.record[0] = steps
        self.video.record[1] = int(isinstance(self.net.update, Native))


REFERENCE_CALLS = []


def backend_process(args, depth_video1, depth_video2, device="cuda"):
    """the reference's backend_process stand-in: records that it ran"""
    REFERENCE_CALLS.append(device)


def install_backend_hooks(strict=True):
    """every hook the native backend needs, on this module"""
    this = sys.modules[__name__]
    modules.install_update_module_hook(this)
    modules.install_alt_corr_hook(this)
    modules.install_factor_graph_hook(FactorGraph)
    modules.install_proximity_hook(FactorGraph)
    modules.install_depth_video_hook(DepthVideo)
    modules.install_async_hook(this, strict=strict)


def report_hooks(backend, queue):
    """spawned-process target: the stand-ins' methods before and after backend.prepare() re-installs the carried hooks"""
    def where():
        this = sys.modules[__name__]
        return {"UpdateModule": this.UpdateModule.__module__, "AltCorrBlock.__init__": AltCorrBlock.__init__.__module__,
                "FactorGraph.update_lowmem": FactorGraph.update_lowmem.__module__,
                "FactorGraph.add_proximity_factors": FactorGraph.add_proximity_factors.__module__,
                "DepthVideo.reproject": getattr(DepthVideo, "reproject", None).__module__ if hasattr(DepthVideo, "reproject") else None}
    before = where()
    backend.prepare()
    queue.put((before, where(), droid_slam_b200.install().__name__))
