"""The native motion filter: the frame ingest (droid_backends.encoder_forward_frames) against encoder_forward on the frames ATen
normalises, and modules.track / install_motion_filter_hook against the reference's control flow (oracle/motion_filter.py) on the same
native operators.  Stand-ins for DepthVideo and MotionFilter are built from seeds; the reference tree is not read."""
import math
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import droid_slam_b200  # noqa: E402
import oracle.encoder as oenc  # noqa: E402
from oracle import motion_filter as omf  # noqa: E402
from droid_slam_b200 import modules, synth  # noqa: E402
from droid_slam_b200.encoder import pack_encoder_weights  # noqa: E402
import factor_graph_stubs as fs  # noqa: E402
import make_motion_filter_golden as mmf  # noqa: E402
from util import host_syncs  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
MEAN = (0.485, 0.456, 0.406)
STDV = (0.229, 0.224, 0.225)


@pytest.fixture(scope="module")
def be():
    return droid_slam_b200.install()


def _aten_normalised(frames, bgr=True):
    """the reference's normalisation (motion_filter.py:62-63) on the device: fp32 [n,3,H,W]"""
    mean = torch.as_tensor(MEAN, device=DEV)[:, None, None]
    stdv = torch.as_tensor(STDV, device=DEV)[:, None, None]
    x = frames[:, [2, 1, 0]] if bgr else frames
    return (x / 255.0).sub_(mean).div_(stdv)


def _frames(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.randint(0, 256, (n, 3, H, W), generator=g, dtype=torch.uint8)
    f[:, :, :2, :] = 0                                     # the extremes of the range
    f[:, :, -2:, :] = 255
    return f.to(DEV)


def test_aten_normalisation_is_what_the_ingest_restates():
    """on CUDA, x / 255.0 multiplies by the fp32 reciprocal and .div_(STDV) is an IEEE division: the two roundings the kernel makes"""
    x = torch.arange(256, device=DEV, dtype=torch.uint8)
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(255.0, dtype=torch.float32)
    assert torch.equal(x / 255.0, x.float() * inv.to(DEV))
    y = (x / 255.0)[None].repeat(3, 1) - torch.as_tensor(MEAN, device=DEV)[:, None]
    s = torch.as_tensor(STDV, device=DEV)[:, None]
    assert torch.equal(y / s, (y.double() / s.double()).float())      # correctly rounded: fp64 division rounded once to fp32


@pytest.mark.parametrize("H,W", [(384, 512), (352, 552)])
@pytest.mark.parametrize("n", [1, 2, 16])
@pytest.mark.parametrize("norm_fn,od,code", [("instance", 128, 1), ("none", 256, 0)])
def test_ingest_bit_identical_to_encoder_forward_on_aten_frames(be, H, W, n, norm_fn, od, code):
    packed = pack_encoder_weights(synth.make_encoder_weights(code, od), norm_fn, od, DEV)
    frames = _frames(n, H, W, seed=n + H)
    want = be.encoder_forward(_aten_normalised(frames), packed, code, od)
    got = be.encoder_forward_frames(frames, packed, code, od, True, list(MEAN), list(STDV))
    assert got.dtype == torch.float16 and got.shape == (n, od, H // 8, W // 8)
    assert torch.equal(got, want)
    if n == 2:                                             # frames already in RGB order
        rgb = be.encoder_forward_frames(frames, packed, code, od, False, list(MEAN), list(STDV))
        assert torch.equal(rgb, be.encoder_forward(_aten_normalised(frames, bgr=False), packed, code, od))


def test_ingest_argument_checks(be):
    packed = pack_encoder_weights(synth.make_encoder_weights(0, 128), "instance", 128, DEV)
    frames = _frames(1, 64, 64, seed=0)
    with pytest.raises(RuntimeError, match="frames must be UInt8|must be Byte|UInt8"):
        be.encoder_forward_frames(frames.float(), packed, 1, 128, True, list(MEAN), list(STDV))
    with pytest.raises(RuntimeError, match="mean and std must hold 3 values"):
        be.encoder_forward_frames(frames, packed, 1, 128, True, list(MEAN[:2]), list(STDV))
    with pytest.raises(RuntimeError, match="multiples of 8"):
        be.encoder_forward_frames(frames[..., :60].contiguous(), packed, 1, 128, True, list(MEAN), list(STDV))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        be.encoder_forward_frames(frames.cpu(), packed, 1, 128, True, list(MEAN), list(STDV))


# ---- the whole filter ---------------------------------------------------------------------------------------------------------------------
def _encoder_class():
    ns = types.SimpleNamespace(BasicEncoder=type("BasicEncoder", (oenc.BasicEncoder,), {}))
    modules.install_encoder_hook(ns)
    return ns.BasicEncoder


_ENC = _encoder_class()


def _filter(video, thresh):
    """a MotionFilter's attributes (motion_filter.py:22-37) on the native operators"""
    fnet = _ENC(output_dim=128, norm_fn="instance")
    fnet.load_state_dict(synth.make_encoder_weights(0, 128))
    cnet = _ENC(output_dim=256, norm_fn="none")
    cnet.load_state_dict(synth.make_encoder_weights(1, 256))
    return types.SimpleNamespace(fnet=fnet.to(DEV).eval(), cnet=cnet.to(DEV).eval(), update=fs.update_op(DEV), video=video, thresh=thresh,
                                 device=DEV, count=0, MEAN=torch.as_tensor(MEAN, device=DEV)[:, None, None],
                                 STDV=torch.as_tensor(STDV, device=DEV)[:, None, None])


def _stream(n, H, W, cams, depth, seed):
    frames = synth.make_frames(n, H, W, cams, seed)
    g = torch.Generator().manual_seed(seed + 7)
    intr = torch.tensor([0.9 * W, 0.9 * W, W / 2.0, H / 2.0])
    out = []
    for k in range(n):
        d = None
        if depth:
            d = 0.5 + 4 * torch.rand(H, W, generator=g)
            d[torch.rand(H, W, generator=g) < 0.2] = 0.0
        out.append((float(k), frames[k], d, intr.clone()))
    return out


def _oracle(filt, stream):
    rows = []
    for t, image, depth, intr in stream:
        stat = omf.track(filt, t, image, depth, intr, corr_block=fs.CorrBlock)
        rows.append((stat, filt.video.counter.value, filt.count))
    return rows


def _state(filt):
    v, n = filt.video, filt.video.counter.value
    out = {k: getattr(v, k)[:n] for k in ("tstamp", "images", "poses", "disps", "disps_sens", "intrinsics", "fmaps", "nets", "inps")}
    out.update(net=filt.net, inp=filt.inp, fmap=filt.fmap, count=torch.tensor(filt.count), counter=torch.tensor(n))
    return out


def _reference_run(stream, H, W, cams):
    """(thresh, filter, per-frame rows) of the reference flow with a thresh that gives keyframes and skipped frames: quantiles of a dry
    run's statistics (every frame against the first), half way between neighbours, the median first"""
    rows = _oracle(_filter(mmf.Video(cams == 2, DEV, H, W, len(stream)), math.inf), stream)
    s = sorted(r[0] for r in rows[1:])
    for k in (len(s) // 2, 3 * len(s) // 4, len(s) // 4, len(s) - 1, 1):
        thresh = 0.5 * (s[k - 1] + s[k])
        filt = _filter(mmf.Video(cams == 2, DEV, H, W, len(stream)), thresh)
        rows = _oracle(filt, stream)
        keyframes = [b[1] > a[1] for a, b in zip(rows, rows[1:])]
        if any(keyframes) and not all(keyframes):
            return thresh, filt, rows
    raise AssertionError("no thresh splits the stream")


@pytest.mark.parametrize("H,W", [(384, 512), (352, 552)])
@pytest.mark.parametrize("kind", ["mono", "stereo", "rgbd"])
def test_track_bit_identical_to_the_reference_flow(be, H, W, kind):
    cams = 2 if kind == "stereo" else 1
    stream = _stream(10, H, W, cams, kind == "rgbd", seed=H + cams)
    thresh, want_f, rows = _reference_run(stream, H, W, cams)
    got_f = _filter(mmf.Video(cams == 2, DEV, H, W, len(stream)), thresh)
    got_rows = []
    for t, image, depth, intr in stream:
        modules.track(got_f, t, image, depth, intr)
        got_rows.append((got_f.video.counter.value, got_f.count))
    assert got_rows == [r[1:] for r in rows]
    keyframes = [b[0] > a[0] for a, b in zip([(0, 0)] + got_rows[:-1], got_rows)][1:]
    assert any(keyframes) and not all(keyframes), keyframes               # frames on both sides of thresh
    want, got = _state(want_f), _state(got_f)
    bad = [k for k in want if not (got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]))]
    assert not bad, bad


def test_track_one_host_read_per_frame(be):
    H, W = 384, 512
    stream = _stream(12, H, W, 1, True, seed=5)
    filt = _filter(mmf.Video(False, DEV, H, W, len(stream)), _reference_run(stream, H, W, 1)[0])
    for t, image, depth, intr in stream[:3]:                 # warm-up: packs the weights, reads MEAN / STDV once
        modules.track(filt, t, image, depth, intr)
    kf0 = filt.video.counter.value
    n, _ = host_syncs(lambda: [modules.track(filt, t, image, depth, intr) for t, image, depth, intr in stream[3:]])
    assert n <= len(stream) - 3, n
    assert filt.video.counter.value > kf0                    # keyframes were appended inside the counted window


def _filter_class():
    class MotionFilter:
        def __init__(self, filt):
            self.__dict__.update(vars(filt))

        def track(self, tstamp, image, depth=None, intrinsics=None):
            return "reference"
    return MotionFilter


def test_motion_filter_hook_strict_and_fallback(be, monkeypatch):
    H, W = 384, 512
    stream = _stream(2, H, W, 1, False, seed=9)
    t, image, depth, intr = stream[0]
    mod = types.SimpleNamespace(MotionFilter=_filter_class())
    modules.install_motion_filter_hook(mod)
    f = mod.MotionFilter(_filter(mmf.Video(False, DEV, H, W, 4), 1.0))
    assert f.track(t, image, depth, intr) is None and f.video.counter.value == 1
    f.update = torch.nn.Identity()
    with pytest.raises(RuntimeError, match="not droid_slam_b200.update.UpdateModule"):
        f.track(t, image, depth, intr)
    for name in ("fnet", "cnet"):
        f = mod.MotionFilter(_filter(mmf.Video(False, DEV, H, W, 4), 1.0))
        setattr(f, name, oenc.BasicEncoder(output_dim=128, norm_fn="instance").to(DEV))
        with pytest.raises(RuntimeError, match="filter.%s .*install_encoder_hook" % name):
            f.track(t, image, depth, intr)
    f = mod.MotionFilter(_filter(mmf.Video(False, "cpu", H, W, 4), 1.0))
    with pytest.raises(RuntimeError, match="video.tstamp is not a CUDA tensor"):
        f.track(t, image, depth, intr)
    f = mod.MotionFilter(_filter(mmf.Video(False, DEV, H, W, 4), 1.0))
    with pytest.raises(RuntimeError, match="multiples of 8"):
        f.track(t, image[..., :508], depth, intr)
    with pytest.raises(RuntimeError, match="no correlation volume kernel"):
        f.track(t, image[..., :56, :], depth, intr)
    mod2 = types.SimpleNamespace(MotionFilter=_filter_class())
    modules.install_motion_filter_hook(mod2, strict=False)
    g = mod2.MotionFilter(_filter(mmf.Video(False, DEV, H, W, 4), 1.0))
    checks, check = [], modules._motion_filter_unsupported
    monkeypatch.setattr(modules, "_motion_filter_unsupported", lambda *a: checks.append(a) or check(*a))
    assert g.track(t, image, depth, intr) is None and g.video.counter.value == 1
    assert len(checks) == 1                                  # native: the readiness check ran once for the call
    g = mod2.MotionFilter(_filter(mmf.Video(False, "cpu", H, W, 4), 1.0))
    assert g.track(t, image, depth, intr) == "reference"


def test_filler_results_unchanged_by_the_ingest(be, monkeypatch):
    """fill_trajectory with fnet on the frame ingest against the same call with the reference's ATen normalisation and the hooked
    fnet under autocast, which it replaced: the same poses bit for bit"""
    import test_trajectory_filler_gpu as tfg
    video = tfg.FVideo(64, 8, seed=21)
    filler = tfg._filler(video)
    stream = tfg._stream(video, 21, seed=6)
    with torch.no_grad():
        got = modules.fill_trajectory(filler, stream)

    def aten(be_, enc, frames, norm):
        x = (frames.flip(1) / 255.0).sub_(filler.MEAN).div_(filler.STDV)
        with torch.autocast("cuda", enabled=True):
            return enc(x[None])[0]

    monkeypatch.setattr(modules, "_encode_frames", aten)
    with torch.no_grad():
        want = modules.fill_trajectory(filler, stream)
    assert torch.equal(got, want)
