"""Stub DepthVideo / FactorGraph objects on the GPU for the native FactorGraph.update / update_lowmem (tests/test_factor_graph_gpu.py,
__graft_entry__.smoke).  They carry the attributes the reference methods read and run the native operators: the reprojection and
upsampling kernels (droid_slam_b200.modules.reproject / upsample), droid_backends.ba, the native CorrBlock / AltCorrBlock (the corr
hooks installed on stand-in classes) and droid_slam_b200.update.UpdateModule.  Built from seeds with synth; the reference tree is not read.

droid_backends.ba accumulates its systems with fp64 atomics (csrc/ba.cu), so on large graphs its result is not bit-reproducible from one
call to the next.  To compare two paths bit for bit, the first one's video logs every ba call (`ba_log`) and the second one's replays
them (`ba_replay`) after checking that its ba inputs are bit-identical."""
import types

import torch

import droid_slam_b200
from droid_slam_b200 import modules, synth
from droid_slam_b200.update import UpdateModule
from util import syncs_not_counted


def _corr_classes():
    class CorrBlock:
        def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
            raise NotImplementedError

        def __call__(self, coords):
            raise NotImplementedError

    class AltCorrBlock:
        def __init__(self, fmaps, num_levels=4, radius=3):
            raise NotImplementedError

        def __call__(self, coords, ii, jj):
            raise NotImplementedError

    m = types.SimpleNamespace(CorrBlock=CorrBlock, AltCorrBlock=AltCorrBlock)
    modules.install_corr_volume_hook(m, fused_lookup=True)
    modules.install_alt_corr_hook(m)
    return m.CorrBlock, m.AltCorrBlock


CorrBlock, AltCorrBlock = _corr_classes()      # update_lowmem resolves AltCorrBlock in the graph class's module, as factor_graph.py does


class _Counter:
    def __init__(self, v):
        self.value = v


class Video:
    """DepthVideo's attributes and geometric methods on the native kernels"""

    def __init__(self, n, rig, ht, wd, seed, dev="cuda"):
        g = torch.Generator().manual_seed(seed)
        s = synth.make_scene(dict(E=4, N=n, ht=ht, wd=wd, itrs=2, lm=1e-4, ep=0.1), seed=seed)
        self.counter = _Counter(n)
        self.poses = s["poses"].to(dev)
        self.disps = s["disps"].to(dev)
        self.disps_sens = torch.zeros_like(self.disps)
        self.disps_up = torch.zeros(n, 8 * ht, 8 * wd, device=dev)
        self.intrinsics = s["intrinsics"][None].repeat(n, 1).contiguous().to(dev)
        self.dirty = torch.zeros(n, dtype=torch.bool, device=dev)
        self.fmaps = torch.randn(n, rig, 128, ht, wd, generator=g).half().to(dev)
        self.nets = torch.tanh(torch.randn(n, 128, ht, wd, generator=g)).half().to(dev)
        self.inps = torch.relu(torch.randn(n, 128, ht, wd, generator=g)).half().to(dev)
        self.stereo = rig == 2
        self.ba_log = None        # a list: every ba call's inputs and resulting poses / disps are appended
        self.ba_replay = None     # a list as ba_log made: ba checks that its inputs are bit-identical and replays the results

    def reproject(self, ii, jj):
        return modules.reproject(self.poses, self.disps, self.intrinsics, ii, jj)

    def upsample(self, ix, mask):
        modules.upsample(self.disps, self.disps_up, ix, mask)

    def ba(self, target, weight, eta, ii, jj, t0=1, t1=None, itrs=2, lm=1e-4, ep=0.1, motion_only=False):
        if t1 is None:
            t1 = max(int(ii.max()), int(jj.max())) + 1
        args = (target, weight, eta, ii, jj, t0, t1, itrs, lm, ep, motion_only)
        if self.ba_replay is not None:
            want, poses, disps = self.ba_replay.pop(0)
            differ = [k for k, a, b in zip(("target", "weight", "eta", "ii", "jj"), args, want) if not torch.equal(a, b)]
            assert not differ and args[5:] == want[5:], ("ba inputs differ", differ, args[5:], want[5:])
            self.poses.copy_(poses)
            self.disps.copy_(disps)
            return
        with syncs_not_counted():                      # ba's own status reads are not the update's
            droid_slam_b200.install().ba(self.poses, self.disps, self.intrinsics[0], self.disps_sens, target, weight, eta, ii, jj, t0, t1,
                                         itrs, lm, ep, motion_only)
        self.disps.clamp_(min=0.001)
        if self.ba_log is not None:
            self.ba_log.append((tuple(a.clone() if isinstance(a, torch.Tensor) else a for a in args), self.poses.clone(), self.disps.clone()))


_UPDATE_OPS = {}


def update_op(dev="cuda"):
    if dev not in _UPDATE_OPS:
        op = UpdateModule().to(dev)
        op.load_state_dict(synth.make_update_weights(0))
        _UPDATE_OPS[dev] = op
    return _UPDATE_OPS[dev]


class Graph:
    """FactorGraph's attributes: edges (ii, jj), inactive edges, net / inp from the video, a native CorrBlock, noisy targets"""

    def __init__(self, video, edges, inactive, upsample=False, seed=0, op=None, volume=True):
        g = torch.Generator().manual_seed(seed + 1)
        dev = video.poses.device
        n, rig, _, ht, wd = video.fmaps.shape
        self.video, self.upsample = video, upsample
        self.update_op = op if op is not None else update_op(dev)
        self.ii = torch.tensor([e[0] for e in edges], dtype=torch.long, device=dev)
        self.jj = torch.tensor([e[1] for e in edges], dtype=torch.long, device=dev)
        y, x = torch.meshgrid(torch.arange(ht, device=dev).float(), torch.arange(wd, device=dev).float(), indexing="ij")
        self.coords0 = torch.stack([x, y], dim=-1)
        self.age = (torch.arange(len(edges), dtype=torch.long) % 3).to(dev)
        self.net = video.nets[self.ii][None]
        self.inp = video.inps[self.ii][None]
        c = (self.ii == self.jj).long() if rig == 2 else torch.zeros_like(self.ii)
        # the correlation volume of update(); update_lowmem does not read it
        self.corr = CorrBlock(video.fmaps[self.ii, 0][None], video.fmaps[self.jj, c][None]) if volume else None
        self.damping = (1e-6 + 1e-3 * torch.rand(n, ht, wd, generator=g)).to(dev)
        coords = video.reproject(self.ii, self.jj)[0]
        self.target = coords + (0.5 * torch.randn(coords.shape, generator=g)).to(dev)
        self.weight = torch.rand(coords.shape, generator=g).to(dev)
        shape = (1, len(inactive), ht, wd, 2)
        self.ii_inac = torch.tensor([e[0] for e in inactive], dtype=torch.long, device=dev)
        self.jj_inac = torch.tensor([e[1] for e in inactive], dtype=torch.long, device=dev)
        ci = video.reproject(self.ii_inac, self.jj_inac)[0] if inactive else torch.zeros(shape, device=dev)
        self.target_inac = ci + (0.5 * torch.randn(shape, generator=g)).to(dev)
        self.weight_inac = torch.rand(shape, generator=g).to(dev)


def neighbourhood(lo, hi, r, closures=(), stereo=False):
    """edges i -> j with 0 < |i - j| <= r among frames lo..hi-1 (every frame a source), then `closures`; stereo adds (i, i) first"""
    e = [(i, i) for i in range(lo, hi)] if stereo else []
    e += [(i, j) for i in range(lo, hi) for j in range(i - r, i + r + 1) if j != i and lo <= j < hi]
    return e + list(closures)


def state(graph):
    v = graph.video
    return {"net": graph.net, "target": graph.target, "weight": graph.weight, "damping": graph.damping, "age": graph.age,
            "poses": v.poses, "disps": v.disps, "disps_up": v.disps_up, "dirty": v.dirty}


def differing(a, b):
    """names of the state entries that are not torch.equal"""
    return [k for k in a if not torch.equal(a[k], b[k])]


def compare(run_a, make_a, run_b, make_b):
    """run_a on make_a() logging BA, run_b on make_b() replaying it -> (state a, state b)"""
    ga, gb = make_a(), make_b()
    ga.video.ba_log = []
    sa = run_a(ga)
    gb.video.ba_replay = ga.video.ba_log
    sb = run_b(gb)
    assert gb.video.ba_replay == [], "the second path made fewer ba calls"
    return sa, sb
