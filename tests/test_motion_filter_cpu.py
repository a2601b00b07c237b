"""MotionFilter.track without a GPU: the restatement (oracle/motion_filter.py), on a stand-in of DepthVideo, bit for bit against what the
unmodified reference method computed with the reference's own DepthVideo (tests/golden/motion_filter.pt), and the C ABI of the frame
ingest (exported, arguments rejected before any launch)."""
import ctypes
import math
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from oracle import motion_filter as omf  # noqa: E402
from droid_slam_b200 import c_api  # noqa: E402
import make_motion_filter_golden as mmf  # noqa: E402

CASES = {c[0]: c for c in mmf.cases()}


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "motion_filter.pt"))


def _run_oracle(case, thresh):
    filt = types.SimpleNamespace(video=mmf.Video(case[1] == 2), **mmf.filter_parts(thresh))
    rows = []
    for tstamp, image, depth, intr in mmf.stream(case):
        n_before = filt.video.counter.value
        stat = omf.track(filt, tstamp, image, depth, intr, corr_block=mmf.CorrBlock)
        rows.append((math.nan if stat is None else stat, filt.video.counter.value > n_before, filt.count))
    return mmf.stored(rows, thresh, filt, filt.video)


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_matches_the_reference_filter(gold, name):
    """every frame's statistic, decision and count, and the final filter and video state, bit for bit"""
    got = _run_oracle(CASES[name], float(gold[name + "/thresh"]))
    for k, t in got.items():
        want = gold[name + "/" + k]
        assert t.dtype == want.dtype and t.shape == want.shape, (name, k)
        assert torch.equal(t, want) if k != "stat" else torch.equal(t.nan_to_num(-1.0), want.nan_to_num(-1.0)), (name, k)


def test_cases_exercise_the_reference_behaviours(gold):
    for name, case in CASES.items():
        kf, stat, thresh = gold[name + "/keyframe"], gold[name + "/stat"], float(gold[name + "/thresh"])
        assert bool(kf[0]) and math.isnan(float(stat[0]))                          # the first frame is always a keyframe
        assert bool(kf[1:].any()) and not bool(kf[1:].all()), name                  # frames on both sides of thresh
        assert torch.equal(kf[1:], stat[1:] > thresh), name                          # strict >
        assert int(gold[name + "/counter"]) == int(kf.sum())
        count = gold[name + "/count"]
        assert all(int(count[k]) == (0 if kf[k] and k else int(count[k - 1]) + 1 if k else 0) for k in range(len(kf))), name
    # the first frame writes channel 0 of the context features broadcast over the video's 128 channels, the identity and disparity 1
    filt = types.SimpleNamespace(video=mmf.Video(False), **mmf.filter_parts(math.inf))
    t, image, depth, intr = mmf.stream(CASES["mono"])[0]
    omf.track(filt, t, image, depth, intr, corr_block=mmf.CorrBlock)
    v = filt.video
    assert torch.equal(v.nets[0], filt.net[0, 0].half().expand(128, -1, -1)) and torch.equal(v.inps[0], filt.inp[0, 0].half().expand(128, -1, -1))
    assert torch.equal(v.poses[0], torch.tensor(omf.IDENTITY)) and bool((v.disps[0] == 1).all())
    assert torch.equal(v.intrinsics[0], intr / 8) and torch.equal(v.images[0], image[0])
    # RGB-D: the video keeps 1 / depth at [3::8, 3::8], 0 where the depth is missing
    ds = gold["rgbd/video_disps_sens"]
    assert bool((ds == 0).any()) and bool((ds > 0).any())


def test_capi_frame_ingest_symbol_and_argument_checks():
    L = c_api.load()
    assert "dba_encoder_forward_frames" in c_api.SYMBOLS and hasattr(L, "dba_encoder_forward_frames")
    f = c_api.FrameFormat(1, (ctypes.c_float * 3)(0.485, 0.456, 0.406), (ctypes.c_float * 3)(0.229, 0.224, 0.225))
    assert L.dba_encoder_forward_frames(None, ctypes.byref(f)) == 1                   # null args
    args = ctypes.cast(ctypes.c_void_p(8), ctypes.POINTER(c_api.EncoderArgs))           # a dummy pointer: the null format is refused first
    assert L.dba_encoder_forward_frames(args, None) == 1 and b"frame format" in L.dba_last_error()
