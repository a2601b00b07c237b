"""Golden vectors for PoseTrajectoryFiller.__call__ / __fill from the reference's own methods, run UNMODIFIED in this container:

    python tests/golden/make_trajectory_filler_golden.py        -> tests/golden/trajectory_filler.pt

`PoseTrajectoryFiller.__call__` (droid_slam/trajectory_filler.py:86-110, with `__fill`, :42-84) runs on a filler built with
`object.__new__` (device "cpu"), whose `video` is a CPU stand-in with DepthVideo's buffers and `__setitem__` semantics
(depth_video.py:70-113), `fnet` the oracle's BasicEncoder and `update` the oracle's update operator.  `__fill` builds the reference's
own `FactorGraph` (factor_graph.py, imported unmodified; only its device argument is "cpu") whose `add_factors` / `update` run as
written on CPU stand-ins of CorrBlock (oracle.corr, with `cat`), DepthVideo.reproject (oracle.reproject) and DepthVideo.ba (oracle.ba).
`__fill` hard-codes "cuda" (`torch.as_tensor(..., device="cuda")`, `.cuda()`): while it runs here, and only here, both are redirected
to the CPU.  Only the results are stored: per case the returned poses, every batch's graph edges (ii, jj) as `update` sees them, and
the video's poses / tstamps / counter afterwards.  tests/test_trajectory_filler_cpu.py holds oracle/trajectory_filler.py to them.
"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle  # noqa: E402
import oracle.encoder as oenc  # noqa: E402
from droid_slam_b200 import synth  # noqa: E402
from make_proximity_golden import import_reference_factor_graph  # noqa: E402
import make_factor_graph_golden as mk  # noqa: E402
from reference import cuda_on_cpu, reference_modules  # noqa: E402

HT, WD = mk.HT, mk.WD
BUFFER = 48


def cases():
    """(name, keyframes, frame stamps): keyframes are stamped 3k + jitter.  Frames at, between and after keyframes, after the last one
    (one edge), before keyframe 0 (t0 = -1), and streams whose length is not a multiple of 16."""
    return [
        ("mixed_19", 6, [-1.5, 0.0, 0.4, 1.0, 3.0, 3.2, 4.7, 6.0, 6.1, 7.9, 9.0, 9.5, 11.0, 12.0, 12.5, 14.9, 15.2, 16.0, 17.5]),
        ("after_last_5", 5, [12.1, 13.0, 14.5, 20.0, 2.2]),
        ("before_first_17", 4, [-3.0, -0.5] + [0.5 * k for k in range(15)]),
    ]


class Video:
    """DepthVideo's buffers (depth_video.py:13-38, device cpu), __setitem__ (:70-113) and the geometric methods __fill's graph calls"""

    def __init__(self, n_kf, seed):
        g = torch.Generator().manual_seed(seed)
        s = synth.make_scene(dict(E=4, N=n_kf, ht=HT, wd=WD, itrs=2, lm=1e-4, ep=0.1), seed=seed)
        self.counter = mk._Counter(n_kf)
        self.ht, self.wd = 8 * HT, 8 * WD
        self.tstamp = torch.zeros(BUFFER)
        self.tstamp[:n_kf] = 3.0 * torch.arange(n_kf) + 0.2 * torch.rand(n_kf, generator=g)
        self.images = torch.zeros(BUFFER, 3, 8 * HT, 8 * WD, dtype=torch.uint8)
        self.poses = torch.zeros(BUFFER, 7)
        self.poses[:, 6] = 1
        self.poses[:n_kf] = s["poses"]
        self.poses[-1] = s["poses"][n_kf // 2]          # the slot a frame before keyframe 0 reads (index -1)
        self.disps = torch.ones(BUFFER, HT, WD)
        self.disps[:n_kf] = s["disps"]
        self.disps[-1] = s["disps"][n_kf // 2]
        self.disps_sens = torch.zeros_like(self.disps)
        self.intrinsics = torch.zeros(BUFFER, 4)
        self.intrinsics[:n_kf] = s["intrinsics"]
        self.intrinsics[-1] = s["intrinsics"]
        self.fmaps = torch.randn(BUFFER, 1, 128, HT, WD, generator=g)
        self.nets = torch.tanh(torch.randn(BUFFER, 128, HT, WD, generator=g))
        self.inps = torch.relu(torch.randn(BUFFER, 128, HT, WD, generator=g))

    def __setitem__(self, index, item):
        self.tstamp[index] = item[0]
        self.images[index] = item[1]
        if item[2] is not None:
            self.poses[index] = item[2]
        if item[3] is not None:
            self.disps[index] = item[3]
        if item[5] is not None:
            self.intrinsics[index] = item[5]
        if len(item) > 6:
            self.fmaps[index] = item[6]

    reproject = mk.Video.reproject
    ba = mk.Video.ba


class CorrBlock(mk.CorrBlock):
    """CorrBlock (modules/corr.py:14-71) on oracle.corr, with `cat` (:63-71)"""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        super().__init__(fmap1.float(), fmap2.float())

    def cat(self, other):
        out = object.__new__(CorrBlock)
        out.pyramid = [torch.cat([a, b], 0) for a, b in zip(self.pyramid, other.pyramid)]
        return out


def encoder():
    enc = oenc.BasicEncoder(output_dim=128, norm_fn="instance")
    enc.load_state_dict(synth.make_encoder_weights(0, 128))
    return enc.eval()


def filler_parts(seed, n_kf):
    """(video, fnet, update operator, MEAN, STDV) of one case"""
    mean = torch.as_tensor([0.485, 0.456, 0.406])[:, None, None]
    stdv = torch.as_tensor([0.229, 0.224, 0.225])[:, None, None]
    return Video(n_kf, seed), encoder(), mk.UpdateOp(synth.make_update_weights(0)), mean, stdv


def stream(seed, video, stamps):
    g = torch.Generator().manual_seed(seed + 100)
    intr = video.intrinsics[0] * 8.0
    return [(t, torch.randint(0, 255, (1, 3, 8 * HT, 8 * WD), generator=g, dtype=torch.uint8), intr.clone()) for t in stamps]


def import_reference_trajectory_filler():
    """the reference's trajectory_filler module; its FactorGraph is the unmodified class of factor_graph.py (CorrBlock -> the stand-in)"""
    fg = import_reference_factor_graph()
    fg.CorrBlock = CorrBlock
    with reference_modules("trajectory_filler", stubs={"factor_graph": fg, "droid_net": types.SimpleNamespace(DroidNet=None)}) as (tf,):
        pass

    class FactorGraph(fg.FactorGraph):
        def __init__(self, video, update_op):
            super().__init__(video, update_op, device="cpu")

        def update(self, *a, **k):
            video_edges.append((self.ii.clone(), self.jj.clone()))
            return fg.FactorGraph.update(self, *a, **k)

    video_edges = []
    tf.FactorGraph = FactorGraph
    return tf, video_edges


def run_reference(tf, edges_log, case, seed=0):
    name, n_kf, stamps = case
    video, fnet, update, mean, stdv = filler_parts(seed, n_kf)
    f = object.__new__(tf.PoseTrajectoryFiller)
    f.cnet, f.fnet, f.update, f.count, f.video, f.device, f.MEAN, f.STDV = None, fnet, update, 0, video, "cpu", mean, stdv
    edges_log.clear()
    with cuda_on_cpu():
        out = tf.PoseTrajectoryFiller.__call__(f, stream(seed, video, stamps))
    edges = []
    for k in range(0, len(edges_log), 6):           # six updates per batch see the same edges
        assert all(torch.equal(edges_log[k][0], e[0]) for e in edges_log[k:k + 6])
        edges.append(edges_log[k])
    return out.data, edges, video


def stored(poses, edges, video):
    gold = {"poses": poses.clone(), "n_batches": torch.tensor(len(edges)), "video_poses": video.poses.clone(),
            "video_tstamp": video.tstamp.clone(), "counter": torch.tensor(video.counter.value)}
    for k, (ii, jj) in enumerate(edges):
        gold["ii%d" % k], gold["jj%d" % k] = ii.clone(), jj.clone()
    return gold


def main(out=None):
    tf, log = import_reference_trajectory_filler()
    gold = {}
    for case in cases():
        with torch.no_grad():
            for k, t in stored(*run_reference(tf, log, case)).items():
                gold[case[0] + "/" + k] = t
        print("%-18s done" % case[0])
    torch.save(gold, out or os.path.join(ROOT, "tests", "golden", "trajectory_filler.pt"))


if __name__ == "__main__":
    main()
