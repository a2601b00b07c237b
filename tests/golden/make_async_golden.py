"""Golden vectors for DroidAsync's frontend -> backend hand-over from the reference's own code, run UNMODIFIED in this container:

    python tests/golden/make_async_golden.py        -> tests/golden/async_backend.pt

  * `align_pose_fragements` (droid_slam/align.py) imported unmodified on the lietorch stand-in (oracle/shims), run on each case's
    fragments in fp32 and in fp64 (the fp32 poses converted).
  * One pass of the unmodified `backend_process` (droid_slam/droid_async.py:37-130) per case: `ready = 1` (the last round, so the
    `while` loop runs once), video2's counter preset to t0 + 2 and video1's to t1, device "cpu" (its torch.cuda.set_device call is made a
    no-op while the pass runs).  `load_network` and `DroidAsyncBackend` are recording stubs: the backend records the iteration count
    and video2's counter it was called with, and changes nothing.  The modules droid_async.py imports but this function does not use
    (droid_net, depth_video, motion_filter, droid_frontend, droid_backend, trajectory_filler) are empty stand-ins for the import.

Cases (buffer 40, 4x6 maps, images and features at that size with 2 feature channels as the hand-over only copies them, t1 = 36): mono (t0 = 28, the scale is aligned), rgbd (t0 = 28, one nonzero sensor depth: the scale is
discarded, dG stays the one from the scaled poses), stereo (t0 = 28, the scale is discarded), t0 = 0 (identity, s = 1).  The frontend's
fragment is the backend's one seen through a random Sim(3) with noise, as when the backend has moved the map.  Stored per case: the
inputs, the alignment in fp32 and fp64, the back buffers after the pass and the stubs' records.
tests/test_async_cpu.py holds oracle/async_backend.py to them.
"""
import os
import sys
import threading
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle.shims.lietorch import SE3  # noqa: E402
from reference import reference_modules  # noqa: E402

BUFFER, HT, WD, T1 = 40, 4, 6, 36
BUFFERS = ("poses", "disps", "disps_sens", "images", "tstamp", "intrinsics", "fmaps", "nets", "inps")


def cases():
    """(name, t0, stereo, rgbd, seed)"""
    return [("mono", 28, False, False, 0), ("rgbd", 28, False, True, 1), ("stereo", 28, True, False, 2), ("t0_zero", 0, False, False, 3)]


def videos(case):
    """(front, back) dicts of the BUFFERS on the CPU for one case"""
    name, t0, stereo, rgbd, seed = case
    g = torch.Generator().manual_seed(seed)
    cams = 2 if stereo else 1

    def video():
        return {"poses": torch.zeros(BUFFER, 7), "disps": torch.ones(BUFFER, HT, WD), "disps_sens": torch.zeros(BUFFER, HT, WD),
                "images": torch.zeros(BUFFER, cams, 3, HT, WD, dtype=torch.uint8), "tstamp": torch.zeros(BUFFER),
                "intrinsics": torch.zeros(BUFFER, 4), "fmaps": torch.zeros(BUFFER, cams, 2, HT, WD, dtype=torch.float16),
                "nets": torch.zeros(BUFFER, 2, HT, WD, dtype=torch.float16), "inps": torch.zeros(BUFFER, 2, HT, WD, dtype=torch.float16)}

    front, back = video(), video()
    xi = torch.cumsum(0.15 * torch.randn(BUFFER, 6, generator=g), 0)
    front["poses"][:] = SE3.exp(xi).data
    sim = SE3.exp(0.5 * torch.randn(1, 6, generator=g))
    scale = 0.5 + torch.rand((), generator=g)
    moved = front["poses"].clone()
    moved[:, :3] *= scale
    back["poses"][:] = (sim * SE3(moved)).data + 1e-3 * torch.randn(BUFFER, 7, generator=g)
    back["poses"][t0:] = 0.0
    back["poses"][t0:, 6] = 1.0
    front["disps"][:] = 0.2 + torch.rand(BUFFER, HT, WD, generator=g)
    back["disps"][:] = 0.2 + torch.rand(BUFFER, HT, WD, generator=g)
    if rgbd:
        front["disps_sens"][BUFFER - 1, 2, 1] = 0.7          # outside [t0, t1): the reference's any() spans the whole buffer
    front["images"][:] = torch.randint(0, 256, front["images"].shape, generator=g, dtype=torch.uint8)
    front["tstamp"][:] = torch.arange(BUFFER, dtype=torch.float32) * 1.5
    front["intrinsics"][:] = torch.rand(BUFFER, 4, generator=g) * 50
    for k in ("fmaps", "nets", "inps"):
        front[k][:] = torch.randn(front[k].shape, generator=g).half()
    return front, back


class _Value:
    def __init__(self, v):
        self.value = v
        self._lock = threading.Lock()

    def get_lock(self):
        return self._lock


class Video(types.SimpleNamespace):
    """DepthVideo's attributes backend_process touches: the buffers, counter / ready values, stereo and get_lock"""

    def __init__(self, buffers, counter, stereo):
        super().__init__(**{k: v.clone() for k, v in buffers.items()})
        self.counter, self.ready, self.stereo = _Value(counter), _Value(0), stereo

    def get_lock(self):
        return self.counter.get_lock()


def import_reference():
    """(droid_async, align) imported unmodified; the modules droid_async.py imports but backend_process does not use are empty stand-ins"""
    stubs = {}
    for name, cls in (("droid_net", "DroidNet"), ("depth_video", "DepthVideo"), ("motion_filter", "MotionFilter"),
                      ("droid_frontend", "DroidFrontend"), ("droid_backend", "DroidAsyncBackend"), ("trajectory_filler", "PoseTrajectoryFiller")):
        stubs[name] = types.ModuleType(name)
        setattr(stubs[name], cls, type(cls, (), {}))
    with reference_modules("droid_async", "align", stubs=stubs) as modules:
        return modules


def run_backend_process(droid_async, case, front, back):
    """one pass of the unmodified backend_process -> (video2's buffers, the stubs' records)"""
    name, t0, stereo, rgbd, seed = case
    video1 = Video(front, T1, stereo)
    video2 = Video(back, t0 + 2, stereo)
    video2.ready.value = 1
    record = {}

    class Backend:
        def __init__(self, net, video, args):
            record["net"] = net

        def __call__(self, steps, normalize=True):
            record["steps"], record["normalize"], record["counter2"] = steps, normalize, video2.counter.value

    saved = (droid_async.load_network, droid_async.DroidAsyncBackend, torch.cuda.set_device, torch.get_num_threads())
    droid_async.load_network = lambda weights, device="cuda:0": ("net", weights, device)
    droid_async.DroidAsyncBackend = Backend
    torch.cuda.set_device = lambda device: None
    try:
        droid_async.backend_process(types.SimpleNamespace(weights="droid.pth"), video1, video2, device="cpu")
    finally:
        droid_async.load_network, droid_async.DroidAsyncBackend, torch.cuda.set_device, threads = saved
        torch.set_num_threads(threads)
    return {k: getattr(video2, k) for k in BUFFERS}, {"steps": record["steps"], "normalize": record["normalize"],
                                                      "counter2": record["counter2"], "net": record["net"]}


def main():
    out = {}
    droid_async, align = import_reference()
    for case in cases():
        name, t0, stereo, rgbd, seed = case
        front, back = videos(case)
        entry = {"case": case, "front": front, "back": back, "t1": T1}
        if t0 > 0:
            for dt, tag in ((torch.float32, "fp32"), (torch.float64, "fp64")):
                dG, s = align.align_pose_fragements(front["poses"][t0 - 10:t0 - 1].to(dt), back["poses"][t0 - 10:t0 - 1].to(dt))
                entry["align_" + tag] = (dG.data.clone(), s.clone())
        entry["after"], entry["record"] = run_backend_process(droid_async, case, front, back)
        out[name] = entry
        print(name, "s(fp64) =", float(entry["align_fp64"][1]) if t0 > 0 else 1.0, entry["record"])
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "async_backend.pt")
    torch.save(out, path)
    print("wrote", path)


if __name__ == "__main__":
    main()
