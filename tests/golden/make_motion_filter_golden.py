"""Golden vectors for MotionFilter.track from the reference's own method, run UNMODIFIED in this container:

    python tests/golden/make_motion_filter_golden.py        -> tests/golden/motion_filter.pt

`MotionFilter.track` (droid_slam/motion_filter.py:50-91) runs on a filter built with `object.__new__` (device "cpu") whose `video` is
the reference's own DepthVideo (depth_video.py, imported unmodified; device "cpu"), `fnet` / `cnet` the oracle's BasicEncoder and
`update` the oracle's update operator; the module's CorrBlock is the CPU stand-in on oracle.corr.  Substituted for the import only:
lietorch (oracle/shims), droid_net (a stub: the filter's networks are given), droid_backends (not called on this path).  `track` and
the video's setter hard-code ".cuda()": while a case runs here, and only here, it is redirected to the CPU.

Cases: mono, stereo and RGB-D streams of synth.make_frames; each case's thresh is the median of a dry run's statistics (thresh = inf:
every frame probed against the first), so that the stream has keyframes and skipped frames.  Stored per case: every frame's statistic
(NaN for the first frame), decision and count, thresh, and the final filter state (net, inp, fmap, count) and video state (counter and
the first counter slots of tstamp, images, poses, disps, disps_sens, intrinsics, fmaps, nets, inps); the large tensors as the SHA-256 of
their bytes, which is equal exactly when the tensors are bit-identical.
tests/test_motion_filter_cpu.py holds oracle/motion_filter.py to them.
"""
import math
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle.encoder as oenc  # noqa: E402
from droid_slam_b200 import synth  # noqa: E402
import make_factor_graph_golden as mk  # noqa: E402
from reference import cuda_on_cpu, reference_modules  # noqa: E402

HT, WD = mk.HT, mk.WD          # feature maps; frames 8x that
BUFFER = 16
VIDEO_STATE = ("tstamp", "images", "poses", "disps", "disps_sens", "intrinsics", "fmaps", "nets", "inps")
FILTER_STATE = ("net", "inp", "fmap")
DIGESTED = ("images", "fmaps", "nets", "inps")       # and the filter state: stored as the SHA-256 of their bytes (mk.digest)


def cases():
    """(name, cameras, with depth, frames, seed)"""
    return [("mono", 1, False, 9, 0), ("stereo", 2, False, 8, 1), ("rgbd", 1, True, 8, 2)]


def stream(case):
    """[(tstamp, image uint8 [cams,3,H,W], depth [H,W] or None, intrinsics [4])] of one case"""
    name, cams, with_depth, n, seed = case
    frames = synth.make_frames(n, 8 * HT, 8 * WD, cams, seed)
    g = torch.Generator().manual_seed(seed + 50)
    intr = torch.tensor([0.9 * 8 * WD, 0.9 * 8 * WD, 4.0 * WD, 4.0 * HT])
    out = []
    for k in range(n):
        depth = None
        if with_depth:
            depth = 0.5 + 4 * torch.rand(8 * HT, 8 * WD, generator=g)
            depth[torch.rand(8 * HT, 8 * WD, generator=g) < 0.2] = 0.0          # missing depth stays 0
        out.append((float(k), frames[k], depth, intr.clone()))
    return out


class UpdateOp(mk.UpdateOp):
    """the update operator as the filter calls it: update(net, inp, corr) -> net, delta, weight"""

    def __call__(self, net, inp, corr, flow=None, ii=None, jj=None):
        return super().__call__(net, inp, corr, flow, ii, jj)


def encoders():
    fnet = oenc.BasicEncoder(output_dim=128, norm_fn="instance")
    fnet.load_state_dict(synth.make_encoder_weights(0, 128))
    cnet = oenc.BasicEncoder(output_dim=256, norm_fn="none")
    cnet.load_state_dict(synth.make_encoder_weights(1, 256))
    return fnet.eval(), cnet.eval()


def filter_parts(thresh):
    """the attributes of a MotionFilter on the CPU (motion_filter.py:22-37) but the video"""
    fnet, cnet = encoders()
    return dict(fnet=fnet, cnet=cnet, update=UpdateOp(synth.make_update_weights(0)), thresh=thresh, device="cpu", count=0,
                MEAN=torch.as_tensor([0.485, 0.456, 0.406])[:, None, None], STDV=torch.as_tensor([0.229, 0.224, 0.225])[:, None, None])


class Video:
    """DepthVideo's buffers (depth_video.py:13-41) and `append` (:78-109, :133-135) on any device, for runs that may not read the
    reference tree"""

    def __init__(self, stereo, device="cpu", ht=8 * HT, wd=8 * WD, buffer=BUFFER):
        self.counter = types.SimpleNamespace(value=0)
        self.tstamp = torch.zeros(buffer, device=device)
        self.images = torch.zeros(buffer, 3, ht, wd, dtype=torch.uint8, device=device)
        self.poses = torch.zeros(buffer, 7, device=device)
        self.poses[:, 6] = 1
        self.disps = torch.ones(buffer, ht // 8, wd // 8, device=device)
        self.disps_sens = torch.zeros(buffer, ht // 8, wd // 8, device=device)
        self.intrinsics = torch.zeros(buffer, 4, device=device)
        self.fmaps = torch.zeros(buffer, 2 if stereo else 1, 128, ht // 8, wd // 8, dtype=torch.half, device=device)
        self.nets = torch.zeros(buffer, 128, ht // 8, wd // 8, dtype=torch.half, device=device)
        self.inps = torch.zeros(buffer, 128, ht // 8, wd // 8, dtype=torch.half, device=device)
        self.device = device

    def append(self, *item):
        index = self.counter.value
        self.counter.value = index + 1
        self.tstamp[index] = item[0]
        self.images[index] = item[1]
        if item[2] is not None:
            self.poses[index] = item[2]
        if item[3] is not None:
            self.disps[index] = item[3]
        if item[4] is not None:
            depth = item[4][3::8, 3::8].to(self.device)
            self.disps_sens[index] = torch.where(depth > 0, 1.0 / depth, depth)
        if item[5] is not None:
            self.intrinsics[index] = item[5]
        self.fmaps[index] = item[6]
        self.nets[index] = item[7]
        self.inps[index] = item[8]


class CorrBlock(mk.CorrBlock):
    """CorrBlock (modules/corr.py:14-50) on oracle.corr, with the reference's constructor signature"""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        super().__init__(fmap1.float(), fmap2.float())


def import_reference():
    """the reference's motion_filter and depth_video modules, imported unmodified on stubs; the filter's CorrBlock is the stand-in"""
    stubs = {"droid_net": types.SimpleNamespace(DroidNet=None, cvx_upsample=None), "droid_backends": types.ModuleType("droid_backends")}
    with reference_modules("motion_filter", "depth_video", stubs=stubs) as (mf, dv):
        mf.CorrBlock = CorrBlock
        return mf, dv


def run_reference(mf, dv, case, thresh):
    """-> per-frame (statistic, keyframe, count) lists, the filter and the video"""
    name, cams = case[0], case[1]
    f = object.__new__(mf.MotionFilter)
    for k, v in filter_parts(thresh).items():
        setattr(f, k, v)
    f.video = dv.DepthVideo([8 * HT, 8 * WD], buffer=BUFFER, stereo=cams == 2, device="cpu")
    stats = []
    probe = f.update

    def recording(net, inp, corr):
        out = probe(net, inp, corr)
        stats.append(out[1].norm(dim=-1).mean().item())
        return out

    f.update = recording
    rows = []
    with cuda_on_cpu(), torch.no_grad():
        for tstamp, image, depth, intr in stream(case):
            n_before, n_stats = f.video.counter.value, len(stats)
            f.track(tstamp, image, depth, intr)
            stat = stats[-1] if len(stats) > n_stats else math.nan
            rows.append((stat, f.video.counter.value > n_before, f.count))
    f.update = probe
    return rows, f, f.video


def stored(rows, thresh, filt, video):
    gold = {"stat": torch.tensor([r[0] for r in rows], dtype=torch.float64), "keyframe": torch.tensor([r[1] for r in rows]),
            "count": torch.tensor([r[2] for r in rows]), "thresh": torch.tensor(thresh, dtype=torch.float64),
            "counter": torch.tensor(video.counter.value), "filter_count": torch.tensor(filt.count)}
    n = video.counter.value
    for k in VIDEO_STATE:
        t = getattr(video, k)[:n]
        gold["video_" + k] = mk.digest(t) if k in DIGESTED else t.clone()
    for k in FILTER_STATE:
        gold["filter_" + k] = mk.digest(getattr(filt, k))
    return gold


def dry_run_thresh(mf, dv, case):
    """the median of the statistics of every frame probed against the first (thresh = inf), taken half way between the two middle
    statistics so that no statistic of the dry run ties with it"""
    rows, _, _ = run_reference(mf, dv, case, math.inf)
    s = sorted(r[0] for r in rows[1:])
    return 0.5 * (s[len(s) // 2 - 1] + s[len(s) // 2])


def main(out=None):
    mf, dv = import_reference()
    gold = {}
    for case in cases():
        thresh = dry_run_thresh(mf, dv, case)
        rows, filt, video = run_reference(mf, dv, case, thresh)
        for k, t in stored(rows, thresh, filt, video).items():
            gold[case[0] + "/" + k] = t
        print("%-8s thresh %.6f  keyframes %s" % (case[0], thresh, "".join("K" if r[1] else "." for r in rows)))
    torch.save(gold, out or os.path.join(ROOT, "tests", "golden", "motion_filter.pt"))


if __name__ == "__main__":
    main()
