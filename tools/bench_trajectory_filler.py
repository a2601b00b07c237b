"""Time the native trajectory filler (droid_slam_b200.modules.fill_trajectory) against the reference's control flow in 16-frame batches
(oracle/trajectory_filler.py: per-frame bracket search on the host, fnet, two add_factors, 6 x FactorGraph.update(motion_only=True))
running on the hooked native operators (native encoder, CorrBlock, reprojection, modules.update with the general droid_backends.ba).
The lietorch calls of that flow run on the pure-torch stand-in (oracle/shims), the only lietorch available here.

Synthetic video: 100 keyframes stamped 10 frames apart, a stream of 1000 frames, at 384x512 and 352x552 input (48x64 and 44x69 feature
maps).  Each whole stream timed, the two paths alternating, median over --reps rounds after --warmup runs of each.  The host-sync count
per stream includes BA's status reads.

    python tools/bench_trajectory_filler.py [--reps 3] [--warmup 1] [--frames 1000] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.shims import lietorch  # noqa: E402
import droid_slam_b200  # noqa: E402
import oracle.encoder as oenc  # noqa: E402
from oracle import trajectory_filler as otf  # noqa: E402
from droid_slam_b200 import modules, synth  # noqa: E402
from droid_slam_b200.update import UpdateModule  # noqa: E402
from util import card, host_syncs, timed  # noqa: E402

DEV = "cuda"
KEYFRAMES = 100
SIZES = [(384, 512), (352, 552)]


class Video:
    """DepthVideo's buffers, counter and __setitem__ (depth_video.py:13-113) with its geometry on the native kernels"""

    def __init__(self, H, W, n_kf, buffer, seed=0):
        ht, wd = H // 8, W // 8
        g = torch.Generator().manual_seed(seed)
        s = synth.make_scene(dict(E=4, N=n_kf, ht=ht, wd=wd, itrs=2, lm=1e-4, ep=0.1), seed=seed)
        self.counter = types.SimpleNamespace(value=n_kf)
        self.tstamp = torch.zeros(buffer, device=DEV)
        self.tstamp[:n_kf] = (10.0 * torch.arange(n_kf)).to(DEV)
        self.images = torch.zeros(buffer, 3, H, W, dtype=torch.uint8, device=DEV)
        self.poses = torch.zeros(buffer, 7, device=DEV)
        self.poses[:, 6] = 1
        self.poses[:n_kf] = s["poses"].to(DEV)
        self.disps = torch.ones(buffer, ht, wd, device=DEV)
        self.disps[:n_kf] = s["disps"].to(DEV)
        self.disps_sens = torch.zeros_like(self.disps)
        self.intrinsics = torch.zeros(buffer, 4, device=DEV)
        self.intrinsics[:n_kf] = s["intrinsics"].to(DEV)
        self.fmaps = torch.randn(buffer, 1, 128, ht, wd, generator=g).half().to(DEV)
        self.nets = torch.tanh(torch.randn(buffer, 128, ht, wd, generator=g)).half().to(DEV)
        self.inps = torch.relu(torch.randn(buffer, 128, ht, wd, generator=g)).half().to(DEV)

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
        droid_slam_b200.install().ba(self.poses, self.disps, self.intrinsics[0], self.disps_sens, target, weight, eta, ii, jj, t0, t1,
                                     itrs, lm, ep, motion_only)
        self.disps.clamp_(min=0.001)


def _hooked_classes():
    """BasicEncoder under install_encoder_hook; CorrBlock under install_corr_volume_hook with the reference's `cat` (modules/corr.py:63-71)"""
    class CorrBlock:
        def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
            raise NotImplementedError

        def __call__(self, coords):
            raise NotImplementedError

        def cat(self, other):
            for i in range(self.num_levels):
                self.corr_pyramid[i] = torch.cat([self.corr_pyramid[i], other.corr_pyramid[i]], 0)
            return self

    ns = types.SimpleNamespace(CorrBlock=CorrBlock, BasicEncoder=type("BasicEncoder", (oenc.BasicEncoder,), {}))
    modules.install_corr_volume_hook(ns, fused_lookup=True)
    modules.install_encoder_hook(ns)
    return ns.CorrBlock, ns.BasicEncoder


def make(H, W, frames, CorrBlock, BasicEncoder):
    video = Video(H, W, KEYFRAMES, KEYFRAMES + 20)
    fnet = BasicEncoder(output_dim=128, norm_fn="instance")
    fnet.load_state_dict(synth.make_encoder_weights(0, 128))
    op = UpdateModule().to(DEV)
    op.load_state_dict(synth.make_update_weights(0))
    filler = types.SimpleNamespace(fnet=fnet.to(DEV).eval(), update=op, video=video,
                                   MEAN=torch.as_tensor([0.485, 0.456, 0.406], device=DEV)[:, None, None],
                                   STDV=torch.as_tensor([0.229, 0.224, 0.225], device=DEV)[:, None, None])
    g = torch.Generator().manual_seed(1)
    span = 10.0 * (KEYFRAMES - 1)
    intr = video.intrinsics[0].cpu() * 8.0
    stream = [(span * k / frames, torch.randint(0, 255, (1, 3, H, W), generator=g, dtype=torch.uint8).to(DEV), intr) for k in range(frames)]
    return filler, stream


def native(filler, stream, _):
    return modules.fill_trajectory(filler, stream)


def reference_flow(filler, stream, CorrBlock):
    graph = lambda v, op: otf.FillerGraph(v, op, CorrBlock, modules.update, device=DEV)
    return otf.fill(filler, stream, graph, lietorch.SE3)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_trajectory_filler needs a CUDA device")
    CorrBlock, BasicEncoder = _hooked_classes()
    rows = []
    with torch.no_grad():
        for H, W in SIZES:
            filler, stream = make(H, W, args.frames, CorrBlock, BasicEncoder)
            paths = [("native", native), ("reference flow", reference_flow)]
            for _, fn in paths:
                for _ in range(args.warmup):
                    fn(filler, stream, CorrBlock)
            times = {p: [] for p, _ in paths}
            for r in range(args.reps):
                for p, fn in (paths if r % 2 == 0 else paths[::-1]):
                    times[p].append(timed(lambda: fn(filler, stream, CorrBlock))[0])
            n_sync = {p: host_syncs(lambda: fn(filler, stream, CorrBlock))[0] for p, fn in paths}
            got, want = native(filler, stream, None), reference_flow(filler, stream, CorrBlock)
            dt = float((got[:, :3] - want[:, :3]).norm(dim=1).max()) / float(want[:, :3].norm(dim=1).max())
            n = len(stream)
            row = dict(input="%dx%d" % (H, W), frames=n, keyframes=KEYFRAMES,
                       native_ms_per_frame=statistics.median(times["native"]) / n,
                       reference_flow_ms_per_frame=statistics.median(times["reference flow"]) / n,
                       native_syncs=n_sync["native"], reference_flow_syncs=n_sync["reference flow"], max_translation_diff_rel=dt)
            row["speedup"] = row["reference_flow_ms_per_frame"] / row["native_ms_per_frame"]
            rows.append(row)
            print("%-8s %d frames  native %7.3f ms/frame (%d syncs)  reference flow %7.3f ms/frame (%d syncs)  %.2fx  (poses differ by %.1e "
                  "of the translation norm)" % (row["input"], n, row["native_ms_per_frame"], row["native_syncs"], row["reference_flow_ms_per_frame"],
                                                row["reference_flow_syncs"], row["speedup"], dt), flush=True)
            del filler, stream
            torch.cuda.empty_cache()
    info = card()
    print("card: %s" % ", ".join("%s=%s" % kv for kv in info.items()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=info, rows=rows, reps=args.reps, warmup=args.warmup), f, indent=1)


if __name__ == "__main__":
    main()
