"""Time the native motion filter (droid_slam_b200.modules.track) against the reference's control flow (oracle/motion_filter.py: a
pageable upload, the flip and three fp32 passes of ATen normalisation, fnet, CorrBlock, the update operator and `.item()`) running on
the same hooked native operators (encoders under install_encoder_hook, CorrBlock under install_corr_volume_hook with the fused lookup,
droid_slam_b200.update.UpdateModule).

Synthetic stream: synth.make_frames, 1000 frames of one camera at 384x512 and at 352x552 (48x64 and 44x69 feature maps), held on the
host as a camera delivers them; thresh is set by bisection on the native path over the whole stream, aiming at a third of the frames as
keyframes (the count is not monotonic in thresh, so the count reached is reported).  Each pass runs the whole stream on a fresh filter and video; the two paths alternate, median over --reps passes
after --warmup passes of each.  Per frame: wall time (every frame waits for its own statistic, so this is what a caller sees), event
time and host synchronisations.  The two paths must make the same keyframe decisions.

    python tools/bench_motion_filter.py [--reps 3] [--warmup 1] [--frames 1000] [--json out.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import droid_slam_b200  # noqa: E402
import oracle.encoder as oenc  # noqa: E402
from oracle import motion_filter as omf  # noqa: E402
from droid_slam_b200 import modules, synth  # noqa: E402
from droid_slam_b200.update import UpdateModule  # noqa: E402
from make_motion_filter_golden import Video  # noqa: E402  (DepthVideo's buffers and append)
from util import card, host_syncs, timed  # noqa: E402

DEV = "cuda"
SIZES = [(384, 512), (352, 552)]
KEYFRAME_SHARE = 1 / 3


def _hooked_classes():
    class CorrBlock:
        def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
            raise NotImplementedError

        def __call__(self, coords):
            raise NotImplementedError

    ns = types.SimpleNamespace(CorrBlock=CorrBlock, BasicEncoder=type("BasicEncoder", (oenc.BasicEncoder,), {}))
    modules.install_corr_volume_hook(ns, fused_lookup=True)
    modules.install_encoder_hook(ns)
    return ns.CorrBlock, ns.BasicEncoder


class Parts:
    """the networks of one MotionFilter, shared by every pass"""

    def __init__(self, BasicEncoder):
        self.fnet = BasicEncoder(output_dim=128, norm_fn="instance")
        self.fnet.load_state_dict(synth.make_encoder_weights(0, 128))
        self.cnet = BasicEncoder(output_dim=256, norm_fn="none")
        self.cnet.load_state_dict(synth.make_encoder_weights(1, 256))
        self.fnet, self.cnet = self.fnet.to(DEV).eval(), self.cnet.to(DEV).eval()
        self.update = UpdateModule().to(DEV)
        self.update.load_state_dict(synth.make_update_weights(0))

    def filter(self, H, W, n, thresh):
        return types.SimpleNamespace(fnet=self.fnet, cnet=self.cnet, update=self.update, video=Video(False, DEV, H, W, n), thresh=thresh,
                                     device=DEV, count=0, MEAN=torch.as_tensor([0.485, 0.456, 0.406], device=DEV)[:, None, None],
                                     STDV=torch.as_tensor([0.229, 0.224, 0.225], device=DEV)[:, None, None])


def native(filt, stream, _):
    out = []
    for t, image, depth, intr in stream:
        modules.track(filt, t, image, depth, intr)
        out.append(filt.video.counter.value)
    return out


def reference_flow(filt, stream, CorrBlock):
    out = []
    for t, image, depth, intr in stream:
        omf.track(filt, t, image, depth, intr, corr_block=CorrBlock)
        out.append(filt.video.counter.value)
    return out


def calibrate(parts, H, W, stream, share):
    """thresh giving about `share` keyframes over the stream (bisection on the native path)"""
    lo, hi = 0.0, 1.0
    while native(parts.filter(H, W, len(stream), hi), stream, None)[-1] > share * len(stream):
        hi *= 2
    for _ in range(7):
        mid = 0.5 * (lo + hi)
        kf = native(parts.filter(H, W, len(stream), mid), stream, None)[-1]
        lo, hi = (mid, hi) if kf > share * len(stream) else (lo, mid)
    return 0.5 * (lo + hi)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_motion_filter needs a CUDA device")
    CorrBlock, BasicEncoder = _hooked_classes()
    parts = Parts(BasicEncoder)
    rows = []
    with torch.no_grad():
        for H, W in SIZES:
            frames = synth.make_frames(args.frames, H, W, 1, seed=H)
            intr = torch.tensor([0.9 * W, 0.9 * W, W / 2.0, H / 2.0])
            stream = [(float(k), frames[k], None, intr) for k in range(args.frames)]
            thresh = calibrate(parts, H, W, stream, KEYFRAME_SHARE)
            paths = [("native", native), ("reference flow", reference_flow)]
            fresh = lambda: parts.filter(H, W, len(stream), thresh)
            for _, fn in paths:
                for _ in range(args.warmup):
                    fn(fresh(), stream, CorrBlock)
            wall, event, decisions = {p: [] for p, _ in paths}, {p: [] for p, _ in paths}, {}
            for r in range(args.reps):
                for p, fn in (paths if r % 2 == 0 else paths[::-1]):
                    filt = fresh()
                    e, w, decisions[p] = timed(lambda: fn(filt, stream, CorrBlock))
                    wall[p].append(w)
                    event[p].append(e)
            assert decisions["native"] == decisions["reference flow"], "the two flows made different keyframe decisions"
            n_sync = {}
            for p, fn in paths:
                filt = fresh()
                n_sync[p] = host_syncs(lambda: fn(filt, stream, CorrBlock))[0]
            n = len(stream)
            row = dict(input="%dx%d" % (H, W), frames=n, keyframes=decisions["native"][-1], thresh=thresh)
            for p, key in (("native", "native"), ("reference flow", "reference_flow")):
                row[key + "_wall_ms_per_frame"] = statistics.median(wall[p]) / n
                row[key + "_event_ms_per_frame"] = statistics.median(event[p]) / n
                row[key + "_syncs_per_frame"] = n_sync[p] / n
            row["speedup_wall"] = row["reference_flow_wall_ms_per_frame"] / row["native_wall_ms_per_frame"]
            rows.append(row)
            print("%-8s %d frames, %d keyframes  native %6.3f ms/frame wall, %6.3f event, %.2f syncs  reference flow %6.3f wall, %6.3f event, "
                  "%.2f syncs  %.2fx" % (row["input"], n, row["keyframes"], row["native_wall_ms_per_frame"], row["native_event_ms_per_frame"],
                                          row["native_syncs_per_frame"], row["reference_flow_wall_ms_per_frame"],
                                          row["reference_flow_event_ms_per_frame"], row["reference_flow_syncs_per_frame"], row["speedup_wall"]),
                  flush=True)
            del frames, stream
            torch.cuda.empty_cache()
    info = card()
    print("card: %s" % ", ".join("%s=%s" % kv for kv in info.items()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=info, rows=rows, reps=args.reps, warmup=args.warmup), f, indent=1)


if __name__ == "__main__":
    main()
