"""Golden vectors for FactorGraph.update / update_lowmem from the reference's own methods, run UNMODIFIED in this container:

    python tests/golden/make_factor_graph_golden.py        -> tests/golden/factor_graph.pt

`FactorGraph.update` and `FactorGraph.update_lowmem` (droid_slam/factor_graph.py:214-330) are called as unbound functions on a stub graph
and a stub video that carry exactly the attributes the methods read.  The stubs run CPU restatements of the operators: oracle.reproject
(DepthVideo.reproject), oracle.corr lookups (CorrBlock / AltCorrBlock), oracle.update_module_forward (the update operator),
oracle.ba (DepthVideo.ba) and oracle.cvx_upsample (DepthVideo.upsample).  Inputs are regenerated from seeds by `cases()`; only the final
graph state (target, weight, damping, age) and the video's poses, disps and dirty flags are stored, and for the large net and
disps_up the SHA-256 of their bytes (`digest`), which is equal exactly when the tensors are bit-identical.
"""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle  # noqa: E402
from droid_slam_b200 import synth  # noqa: E402
from make_proximity_golden import import_reference_factor_graph  # noqa: E402,F401

HT, WD, CH = 16, 18, 128        # the smallest maps the reference's 4-level pyramids take (its last avg_pool2d needs 2 rows)
DIGESTED = ("net", "disps_up")


def _frontend_edges(n, lo, r=2):
    """radius-r neighbourhood of frames lo..n-1 (every frame a source)"""
    return [(i, j) for i in range(lo, n) for j in range(i - r, i + r + 1) if j != i and lo <= j < n]


def cases():
    """(name, method, kwargs, frames, rig, active edges, inactive edges, upsample)"""
    fe = _frontend_edges(9, 3)
    inac = [(i, j) for i in range(0, 6) for j in (i - 1, i + 1) if 0 <= j < 6]
    back = _frontend_edges(12, 0, 1) + [(0, 9), (10, 2), (3, 11)]
    stereo = [(i, i) for i in range(10)] + _frontend_edges(10, 0, 1)[::2]
    # sources 8..11 see only frames <= 7: the reference's chunks range(0, 8, 8) stop at source frame 7
    quirk = [(i, j) for i in range(8) for j in (i - 1, i + 1) if 0 <= j < 8] + [(8, 7), (9, 7), (10, 6), (11, 5), (9, 4)]
    return [
        ("update_inac_t0none", "update", dict(use_inactive=True), 9, 1, fe, inac, True),
        ("update_t0_given", "update", dict(t0=4, t1=9, use_inactive=False), 9, 1, fe, inac, False),
        ("update_motion_only", "update", dict(use_inactive=True, motion_only=True, itrs=1), 9, 1, fe, inac, True),
        ("lowmem_rig1_inac", "update_lowmem", dict(use_inactive=True, steps=2), 12, 1, back, inac, True),
        ("lowmem_rig1", "update_lowmem", dict(use_inactive=False, steps=1, itrs=1), 12, 1, back, inac, False),
        ("lowmem_rig2_inac", "update_lowmem", dict(use_inactive=True, steps=1), 10, 2, stereo, inac, False),
        ("lowmem_quirk", "update_lowmem", dict(use_inactive=False, steps=1), 12, 1, quirk, [], False),
    ]


class _Counter:
    def __init__(self, v):
        self.value = v


class Video:
    """the attributes of DepthVideo that update / update_lowmem read, on CPU operators"""

    def __init__(self, n, rig, seed):
        g = torch.Generator().manual_seed(seed)
        s = synth.make_scene(dict(E=4, N=n, ht=HT, wd=WD, itrs=2, lm=1e-4, ep=0.1), seed=seed)
        self.counter = _Counter(n)
        self.poses = s["poses"].clone()
        self.disps = s["disps"].clone()
        self.disps_sens = torch.zeros_like(self.disps)
        self.disps_up = torch.zeros(n, 8 * HT, 8 * WD)
        self.intrinsics = s["intrinsics"][None].repeat(n, 1).contiguous()
        self.dirty = torch.zeros(n, dtype=torch.bool)
        self.fmaps = torch.randn(n, rig, CH, HT, WD, generator=g)
        self.nets = torch.tanh(torch.randn(n, CH, HT, WD, generator=g))
        self.inps = torch.relu(torch.randn(n, CH, HT, WD, generator=g))
        self.stereo = rig == 2

    def reproject(self, ii, jj):
        coords, valid = oracle.reproject(self.poses, self.disps, self.intrinsics, ii, jj)
        return coords[None], valid[None]

    def ba(self, target, weight, eta, ii, jj, t0=1, t1=None, itrs=2, lm=1e-4, ep=0.1, motion_only=False):
        if t1 is None:
            t1 = max(int(ii.max()), int(jj.max())) + 1
        oracle.ba(self.poses, self.disps, self.intrinsics[0], self.disps_sens, target, weight, eta, ii, jj, t0, t1, itrs, lm, ep, motion_only)
        self.disps.clamp_(min=0.001)

    def upsample(self, ix, mask):
        up = oracle.cvx_upsample(self.disps[ix].unsqueeze(-1), mask)
        self.disps_up[ix] = up.reshape(-1, 8 * HT, 8 * WD)


class CorrBlock:
    """CorrBlock (modules/corr.py:14-50) on oracle.corr"""

    def __init__(self, fmap1, fmap2):
        self.pyramid = oracle.corr_pyramid(fmap1, fmap2)

    def __call__(self, coords):
        return oracle.corr_block_lookup(self.pyramid, coords)


class AltCorrBlock:
    """AltCorrBlock (modules/corr.py:85-117) on oracle.corr"""

    def __init__(self, fmaps, num_levels=4, radius=3):
        self.pyramid = oracle.fmap_pyramid(fmaps, num_levels)
        self.radius = radius

    def __call__(self, coords, ii, jj):
        return oracle.altcorr_block_lookup(self.pyramid, coords, ii, jj, self.radius)


class UpdateOp:
    def __init__(self, weights):
        self.w = weights

    def __call__(self, net, inp, corr, flow, ii, jj):
        return oracle.update_module_forward(self.w, net.float(), inp.float(), corr.float(), flow, ii)


class Graph:
    """the attributes of FactorGraph that update / update_lowmem read"""

    def __init__(self, video, update_op, edges, inactive, upsample, seed, corr_block=CorrBlock):
        g = torch.Generator().manual_seed(seed + 1)
        self.video, self.update_op, self.upsample = video, update_op, upsample
        self.ii = torch.tensor([e[0] for e in edges], dtype=torch.long)
        self.jj = torch.tensor([e[1] for e in edges], dtype=torch.long)
        E = len(edges)
        y, x = torch.meshgrid(torch.arange(HT).float(), torch.arange(WD).float(), indexing="ij")
        self.coords0 = torch.stack([x, y], dim=-1)
        self.age = torch.arange(E, dtype=torch.long) % 3
        self.net = video.nets[self.ii][None].clone()
        self.inp = video.inps[self.ii][None].clone()
        rig = video.fmaps.shape[1]
        c = (self.ii == self.jj).long() if rig == 2 else torch.zeros_like(self.ii)
        self.corr = corr_block(video.fmaps[self.ii, 0][None], video.fmaps[self.jj, c][None])
        self.damping = 1e-6 + 1e-3 * torch.rand(video.disps.shape, generator=g)
        coords, _ = video.reproject(self.ii, self.jj)
        self.target = coords + 0.5 * torch.randn(coords.shape, generator=g)
        self.weight = torch.rand(coords.shape, generator=g)
        self.ii_inac = torch.tensor([e[0] for e in inactive], dtype=torch.long)
        self.jj_inac = torch.tensor([e[1] for e in inactive], dtype=torch.long)
        shape = (1, len(inactive), HT, WD, 2)
        ci = video.reproject(self.ii_inac, self.jj_inac)[0] if inactive else torch.zeros(shape)
        self.target_inac = ci + 0.5 * torch.randn(shape, generator=g)
        self.weight_inac = torch.rand(shape, generator=g)


def make(case, seed=0):
    """fresh (graph, kwargs) of one case on CPU operators"""
    name, method, kw, n, rig, edges, inactive, ups = case
    video = Video(n, rig, seed)
    return Graph(video, UpdateOp(synth.make_update_weights(0)), edges, inactive, ups, seed), dict(kw)


def state(graph):
    v = graph.video
    return {"net": graph.net, "target": graph.target, "weight": graph.weight, "damping": graph.damping, "age": graph.age,
            "poses": v.poses, "disps": v.disps, "disps_up": v.disps_up, "dirty": v.dirty}


def digest(t):
    return torch.tensor(list(hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).digest()), dtype=torch.uint8)


def stored(st):
    """state -> what the fixture keeps of it"""
    return {k: (digest(t) if k in DIGESTED else t.clone()) for k, t in st.items()}


def run_reference(fg, case):
    graph, kw = make(case)
    if case[1] == "update":
        fg.FactorGraph.update(graph, **kw)
    else:
        fg.AltCorrBlock = AltCorrBlock            # the name update_lowmem resolves in its module
        fg.FactorGraph.update_lowmem(graph, **kw)
    return stored(state(graph))


def main(out=None):
    fg = import_reference_factor_graph()
    gold = {}
    for case in cases():
        for k, t in run_reference(fg, case).items():
            gold[case[0] + "/" + k] = t
        print("%-22s done" % case[0])
    torch.save(gold, out or os.path.join(ROOT, "tests", "golden", "factor_graph.pt"))


if __name__ == "__main__":
    main()
