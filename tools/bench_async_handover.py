"""Time one DroidAsync backend round's hand-over (reference droid_slam/droid_async.py:54-119): the native round
(droid_slam_b200.modules.handover_round: slice copies + droid_backends.fragment_handover + one stream synchronisation) against the
reference's flow on the same tensors (torch.any, full-buffer clones of poses and disps, align_pose_fragements and the re-anchoring on the
lietorch stand-in, the seven slice copies, then a synchronisation so that both end with the work done).

    python tools/bench_async_handover.py --reps 20 --warmup 3 [--json out.json]

Shapes: buffers of 512 and 1024 keyframes at 48x64 and 44x69 feature maps (384x512 and 352x552 images), a round with t0 = 300 and 64
new keyframes, mono (the scale aligned) and RGB-D (sensor depth on every keyframe); both videos on cuda:0, and frontend on cuda:0 with
backend on cuda:1 when two GPUs are visible.  Host clock around each round (each ends in a synchronisation), the two paths alternating,
median over --reps rounds after --warmup of each.  The reference's lietorch is a CUDA extension; the stand-in runs the same group
operations as ATen kernels, so the reference-flow figure is an estimate of the reference's launch chain, not a run of it."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from droid_slam_b200 import modules  # noqa: E402
from oracle.async_backend import SE3, align_pose_fragments  # noqa: E402
import async_stubs  # noqa: E402
from util import card, host_syncs  # noqa: E402


def reference_round(front, back, t0, t1, device):
    """The reference's hand-over flow (droid_async.py:59-119) on the lietorch stand-in: the host read of any(disps_sens), clones of the
    frontend's whole poses and disps buffers under the lock, the alignment as separate group operations, the re-anchoring and the
    slice copies under the lock again, then a synchronisation so that the round's work is done when the clock stops."""
    keep_scale = not back.stereo and not bool(torch.any(front.disps_sens))
    with front.get_lock():
        poses, disps = front.poses.clone().to(device), front.disps.clone().to(device)
    if t0 == 0:
        dG, s = SE3.IdentityLike(SE3(back.poses[[0]])), 1.0
    else:
        dG, s = align_pose_fragments(poses[t0 - 10:t0 - 1], back.poses[t0 - 10:t0 - 1])
        s = s if keep_scale else 1.0
        poses[..., :3] *= s
    with front.get_lock():
        back.poses[t0:t1] = (dG * SE3(poses[t0:t1])).data
        back.disps[t0:t1] = disps[t0:t1] / s
        for k in ("disps_sens", "images", "tstamp", "intrinsics", "fmaps", "nets", "inps"):
            getattr(back, k)[t0:t1] = getattr(front, k)[t0:t1].to(device)
    torch.cuda.synchronize(device)


def native_round(video1, video2, t0, t1, device):
    modules.handover_round(video1, video2, t0, t1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_async_handover: no CUDA device")
    t0, t1 = 300, 364
    placements = [("cuda:0", "cuda:0")] + ([("cuda:0", "cuda:1")] if torch.cuda.device_count() > 1 else [])
    rows = []
    print(card())
    with torch.no_grad():
        for dev1, dev2 in placements:
            for buffer, ht, wd in ((512, 48, 64), (512, 44, 69), (1024, 48, 64), (1024, 44, 69)):
                for mode in ("mono", "rgbd"):
                    v1, v2 = async_stubs.make_videos(buffer, ht, wd, mode, t0, t1, dev1, dev2, seed=1)
                    poses2, disps2 = v2.poses.clone(), v2.disps.clone()
                    paths = [("native", native_round), ("reference flow", reference_round)]
                    times = {p: [] for p, _ in paths}
                    for r in range(args.warmup + args.reps):
                        for p, fn in paths:
                            v2.poses.copy_(poses2)
                            v2.disps.copy_(disps2)
                            torch.cuda.synchronize(dev2)
                            a = time.perf_counter()
                            fn(v1, v2, t0, t1, dev2)
                            b = time.perf_counter()
                            if r >= args.warmup:
                                times[p].append(1e3 * (b - a))
                    n_sync = {p: host_syncs(lambda: fn(v1, v2, t0, t1, dev2))[0] for p, fn in paths}
                    row = dict(frontend=dev1, backend=dev2, buffer=buffer, ht=ht, wd=wd, mode=mode,
                               native_ms=statistics.median(times["native"]), reference_flow_ms=statistics.median(times["reference flow"]),
                               native_syncs=n_sync["native"], reference_flow_syncs=n_sync["reference flow"])
                    row["speedup"] = row["reference_flow_ms"] / row["native_ms"]
                    rows.append(row)
                    print("%s->%s buffer %4d %dx%d %-4s  native %7.3f ms (%d sync)  reference flow %7.3f ms (%d syncs)  %.1fx" % (
                        dev1, dev2, buffer, ht, wd, mode, row["native_ms"], row["native_syncs"], row["reference_flow_ms"],
                        row["reference_flow_syncs"], row["speedup"]), flush=True)
                    del v1, v2, poses2, disps2
                    torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
