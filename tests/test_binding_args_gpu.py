"""The argument contract of `droid_backends`: every tensor argument of every entry point is checked for device, dtype, layout and
shape before anything is launched.  For each entry point one small valid call runs first; then each tensor argument in turn is
replaced by a CPU tensor, a wrong dtype, a non-contiguous view (where the kernel reads the raw layout) and wrongly shaped tensors
(among them every extent the binding now checks against the others), and the call must raise a RuntimeError that names the argument.
The in-place entry points must leave their outputs untouched when they raise, which shows that nothing was launched."""
import re

import pytest
import torch

from droid_slam_b200 import synth
from droid_slam_b200.encoder import pack_encoder_weights
from droid_slam_b200.update import PACKED_ORDER, pack_update_weights

pytestmark = pytest.mark.gpu
DEV = "cuda"
N, HT, WD, E = 4, 8, 8, 3


def _f(*shape, fill=None):
    g = torch.Generator().manual_seed(sum(shape) + len(shape))
    t = torch.full(shape, float(fill)) if fill is not None else torch.rand(*shape, generator=g)
    return t.to(DEV)


def _i(*v):
    return torch.tensor(v, dtype=torch.int64, device=DEV)


def _poses(n=N):
    p = torch.zeros(n, 7)
    p[:, 6] = 1
    p[:, :3] = 0.05 * torch.arange(n, dtype=torch.float32)[:, None]
    return p.to(DEV)


def _intr(n=None):
    k = torch.tensor([8.0, 8.0, 4.0, 4.0])
    return (k if n is None else k.repeat(n, 1)).to(DEV)


def _noncontig(t):
    """same values and shape, strides of a view"""
    v = t.new_empty(tuple(t.shape) + (2,))[..., 0]
    v.copy_(t)
    assert not v.is_contiguous()
    return v


def _wrong_dtype(t):
    return t.to(torch.int32) if t.is_floating_point() else t.float()


# Each case: (entry point, builder of the positional arguments, {argument name: (position, checks)}, in-place outputs).  A position is
# an index into the arguments or (index, k) for element k of a list argument.  checks: "d" the dtype is checked, "c" contiguity is
# required, and a list of functions making wrongly shaped tensors from the valid one.
def _ba_args():
    return [_poses(), _f(N, HT, WD, fill=1), _intr(), _f(N, HT, WD, fill=0), 4 * _f(E, 2, HT, WD), _f(E, 2, HT, WD, fill=0.5),
            _f(1, HT, WD, fill=1), _i(0, 1, 2), _i(1, 2, 3), 1, 4, 1, 1e-4, 0.1, False]


def _geom_args():
    return [_poses(), _f(N, HT, WD, fill=1), _intr(), _i(0, 1, 2), _i(1, 2, 3)]


def _wb_args():
    # delta, weight, coords, edge_index, target, weight_out, ba_target, ba_weight, n_inactive, eta, src_frames, damping, ba_frames, ba_damping, ep
    return [_f(E, HT, WD, 2), _f(E, HT, WD, 2), _f(E, HT, WD, 2), _i(2, 0, 1), _f(E, HT, WD, 2), _f(E, HT, WD, 2), _f(E + 1, 2, HT, WD),
            _f(E + 1, 2, HT, WD), 1, _f(2, HT, WD), _i(0, 3), _f(N, HT, WD), _i(0, 1, 2), _f(3, HT, WD), 1e-7]


def _pose_only_args():
    return [_poses(), _f(N, HT, WD, fill=1), _intr(), 4 * _f(E, 2, HT, WD), _f(E, 2, HT, WD, fill=0.5), _i(0, 1, 0), _i(2, 3, 3), 2, 4, 2,
            1e-4, 0.1, True, False]


def _corr_volume_args():
    return [_f(2, 128, HT, WD).half(), _f(2, 128, HT, WD).half(), _i(0, 1), _i(1, 0), False]


def _corr_lookup_args(be):
    return [be.corr_volume_pyramid(*_corr_volume_args()), 8 * _f(2, 2, HT, WD), False]


def _altcorr_args():
    return [_f(1, 2, 8, HT, WD), _f(1, 2, 8, HT, WD), 8 * _f(1, 2, 2, HT, WD), _i(0, 1), _i(1, 0), 3]


def _alt_lookup_args(be):
    return [be.altcorr_pyramid(_f(1, 2, 8, HT, WD).half(), 4), 8 * _f(1, 2, 2, HT, WD), _i(0, 1), _i(1, 0), 3]


def _update_args():
    net, inp, corr, flow, ii = synth.make_update_inputs(E=E, ht=HT, wd=WD, seed=0, n_src=2)
    net, inp, corr = (t[0].half().contiguous().to(DEV) for t in (net, inp, corr))
    flow = flow[0].contiguous().to(DEV)
    seg = torch.unique(ii, return_inverse=True)[1].to(DEV)
    pk = pack_update_weights(synth.make_update_weights(0), DEV)
    return [net, inp, corr, flow, seg, 2, [pk[k] for k in PACKED_ORDER], False]


def _encoder_args():
    packed = [t.to(DEV) for t in pack_encoder_weights(synth.make_encoder_weights(0, 128), "instance", 128)]
    return [_f(1, 3, 16, 16), packed, 1, 128]


def _conv_args():
    return [_f(2, HT, WD, 64).half(), _f(2, HT, WD, 32).half(), _f(9, 64, 128).half(), _f(64), 3, True]


def _shorter(t):
    return t[:-1].contiguous()


def _longer(t):
    return torch.cat([t, t[:1]]).contiguous()


def _last_minus_one(t):
    return t[..., :-1].contiguous()


GEOM = {"poses": (0, "dc", [lambda t: t[:, :6].contiguous()]), "disps": (1, "dc", [lambda t: t.flatten(1)]),
        "intrinsics": (2, "dc", [lambda t: t[:3].contiguous()]), "ii": (3, "dc", []), "jj": (4, "dc", [_shorter])}

CASES = {
    "ba": (_ba_args, {"poses": (0, "dc", [lambda t: t[:, :6].contiguous()]), "disps": (1, "dc", [lambda t: t.flatten(1)]),
                      "intrinsics": (2, "dc", [lambda t: t[:3].contiguous()]), "disps_sens": (3, "dc", [_last_minus_one]),
                      "targets": (4, "dc", [_shorter, _last_minus_one]), "weights": (5, "dc", [_shorter, _last_minus_one]),
                      "eta": (6, "d", [_last_minus_one]), "ii": (7, "dc", []), "jj": (8, "dc", [_longer])}, (0, 1)),
    "frame_distance": (lambda: _geom_args() + [0.5], GEOM, ()),
    "projmap": (_geom_args, GEOM, ()),
    "iproj": (lambda: _geom_args()[:3], {"poses": (0, "dc", [_shorter, lambda t: t[:, :6].contiguous()]),
                                         "disps": (1, "dc", [lambda t: t.flatten(1)]), "intrinsics": (2, "dc", [lambda t: t[:3].contiguous()])}, ()),
    "depth_filter": (lambda: _geom_args()[:3] + [_i(0, 1, 2, 3), _f(4, fill=0.05)],
                     {"poses": (0, "dc", [lambda t: t[:, :6].contiguous()]), "disps": (1, "dc", [lambda t: t.flatten(1)]),
                      "intrinsics": (2, "dc", [lambda t: t[:3].contiguous()]), "ix": (3, "dc", []), "thresh": (4, "dc", [_shorter])}, ()),
    "corr_index_forward": (lambda: [_f(2, HT, WD, HT, WD), 8 * _f(2, 2, HT, WD), 3],
                           {"volume": (0, "c", [lambda t: t.flatten(3)]), "coords": (1, "dc", [_last_minus_one, _shorter])}, ()),
    "corr_index_backward": (lambda: [_f(2, HT, WD, HT, WD), 8 * _f(2, 2, HT, WD), _f(2, 7, 7, HT, WD), 3],
                            {"volume": (0, "c", [lambda t: t.flatten(3)]), "coords": (1, "dc", [_last_minus_one, _shorter]),
                             "corr_grad": (2, "dc", [_last_minus_one, _shorter, lambda t: t.half()])}, ()),
    "altcorr_forward": (_altcorr_args, {"fmap1": (0, "c", [_last_minus_one, lambda t: t[:0].contiguous()]),
                                        "fmap2": (1, "dc", [lambda t: t[:, :, :4].contiguous(), lambda t: t[:0].contiguous(), lambda t: t.half()]),
                                        "coords": (2, "dc", [lambda t: t[0]]), "ii": (3, "d", [_longer]), "jj": (4, "d", [_shorter])}, ()),
    "altcorr_backward": (lambda: _altcorr_args()[:3] + [_f(1, 2, 7, 7, HT, WD)] + _altcorr_args()[3:],
                         {"fmap1": (0, "c", [_last_minus_one, lambda t: t[:0].contiguous()]),
                          "fmap2": (1, "dc", [lambda t: t[:, :, :4].contiguous(), lambda t: t[:0].contiguous(), lambda t: t.half()]),
                          "coords": (2, "dc", [lambda t: t[0], lambda t: t.flatten(3)]), "corr_grad": (3, "c", [_last_minus_one]),
                          "ii": (4, "d", [_shorter]), "jj": (5, "d", [_shorter])}, ()),
    "corr_volume_pyramid": (_corr_volume_args, {"fmap1": (0, "dc", [lambda t: t[0]]), "fmap2": (1, "dc", [lambda t: t[:, :64].contiguous()]),
                                                "ii": (2, "dc", []), "jj": (3, "dc", [_longer])}, ()),
    "corr_lookup_pyramid": (_corr_lookup_args, {"pyramid[0]": ((0, 0), "dc", [_last_minus_one]), "pyramid[2]": ((0, 2), "dc", [_last_minus_one]),
                                                "pyramid[3]": ((0, 3), "dc", [_shorter]), "coords": (1, "dc", [_last_minus_one, _shorter])}, ()),
    "altcorr_pyramid": (lambda: [_f(1, 2, 8, HT, WD).half(), 4], {"fmaps": (0, "dc", [lambda t: t[0]])}, ()),
    "altcorr_lookup_pyramid": (_alt_lookup_args, {"pyramid[0]": ((0, 0), "c", [lambda t: t[0]]), "pyramid[1]": ((0, 1), "dc", [_last_minus_one]),
                                                  "pyramid[3]": ((0, 3), "dc", [_shorter]), "coords": (1, "dc", [_last_minus_one]),
                                                  "ii": (2, "d", [_longer]), "jj": (3, "d", [_shorter])}, ()),
    "reproject": (lambda: [_poses(), _f(N, HT, WD, fill=1), _intr(N), _i(0, 1, 2), _i(1, 2, 3)],
                  {"poses": (0, "dc", []), "disps": (1, "dc", [lambda t: t.flatten(1)]), "intrinsics": (2, "dc", [lambda t: t[:, :3].contiguous()]),
                   "ii": (3, "dc", []), "jj": (4, "dc", [_shorter])}, ()),
    "motion_features": (lambda: [_poses(), _f(N, HT, WD, fill=1), _intr(N), _i(0, 1, 2), _i(1, 2, 3), _f(E, HT, WD, 2), _i(2, 1)],
                        {"poses": (0, "dc", []), "disps": (1, "dc", [lambda t: t.flatten(1)]),
                         "intrinsics": (2, "dc", [lambda t: t[:, :3].contiguous()]), "ii": (3, "dc", []), "jj": (4, "dc", [_shorter]),
                         "target": (5, "dc", [_shorter, _last_minus_one]), "edge_index": (6, "dc", [])}, ()),
    "graph_writeback": (_wb_args, {"delta": (0, "dc", [_last_minus_one]), "weight": (1, "dc", [_shorter]), "coords": (2, "dc", [_longer]),
                                   "edge_index": (3, "dc", [_shorter]), "target": (4, "dc", [_last_minus_one]), "weight_out": (5, "dc", [_shorter]),
                                   "ba_target": (6, "dc", [_last_minus_one]), "ba_weight": (7, "dc", [_shorter]), "eta": (9, "dc", [_last_minus_one]),
                                   "src_frames": (10, "dc", [_longer]), "damping": (11, "dc", [lambda t: t.flatten(1)]),
                                   "ba_frames": (12, "dc", []), "ba_damping": (13, "dc", [_shorter])}, (4, 5, 6, 7, 11, 13)),
    "fill_interpolate": (lambda: [_poses(), torch.arange(N, dtype=torch.float32, device=DEV), _f(5) * N],
                         {"poses": (0, "dc", [lambda t: t[:, :6].contiguous()]), "tstamps": (1, "dc", [_shorter, _longer]),
                          "t": (2, "dc", [lambda t: t[None]])}, ()),
    "pose_only_ba": (_pose_only_args, {"poses": (0, "dc", [lambda t: t[:, :6].contiguous()]), "disps": (1, "dc", [lambda t: t.flatten(1)]),
                                       "intrinsics": (2, "dc", [lambda t: t[:3].contiguous()]), "targets": (3, "dc", [_shorter, _last_minus_one]),
                                       "weights": (4, "dc", [_shorter]), "ii": (5, "dc", []), "jj": (6, "dc", [_longer])}, (0,)),
    "update_forward": (_update_args, {"net": (0, "c", [lambda t: t[:, :64].contiguous()]), "inp": (1, "c", [_shorter, _last_minus_one]),
                                      "corr": (2, "c", [lambda t: t[:, :128].contiguous()]), "flow": (3, "", [_shorter]),
                                      "seg": (4, "d", [_shorter]), "packed[0]": ((6, 0), "dc", [lambda t: t[:, :64].contiguous()]),
                                      "packed[5]": ((6, 5), "dc", [_last_minus_one]), "packed[11]": ((6, 11), "dc", [_shorter]),
                                      "packed[12]": ((6, 12), "dc", [_shorter]), "packed[24]": ((6, 24), "dc", [_last_minus_one]),
                                      "packed[26]": ((6, 26), "dc", [_longer])}, ()),
    "encoder_forward": (_encoder_args, {"images": (0, "dc", [lambda t: t[:, :2].contiguous()]),
                                        "packed_weights[3]": ((1, 3), "dc", [_last_minus_one]), "packed_weights[20]": ((1, 20), "dc", [_shorter])}, ()),
    "conv_nhwc": (_conv_args, {"src0": (0, "dc", [lambda t: t[0]]), "src1": (1, "dc", [lambda t: t[:, :, :-1].contiguous(), _shorter]),
                               "wpk": (2, "dc", [lambda t: t[..., :64].contiguous(), _shorter]), "bias": (3, "dc", [_shorter])}, ()),
    "cvx_upsample": (lambda: [_f(2, HT, WD), _f(2, 576, HT, WD).half()],
                     {"disps": (0, "dc", [lambda t: t.flatten(1)]), "mask": (1, "dc", [lambda t: t[:, :575].contiguous()])}, ()),
    "proximity_edges": (lambda: [_f(36, fill=5.0), 0, 0, 6, _i(0, 1), _i(1, 2), 2, 2, 16.0, -1, False],
                        {"d": (0, "dc", [_shorter]), "ii_known": (4, "dc", []), "jj_known": (5, "dc", [_longer])}, ()),
}

def _get(args, pos):
    return args[pos[0]][pos[1]] if isinstance(pos, tuple) else args[pos]


def _set(args, pos, value):
    if isinstance(pos, tuple):
        args[pos[0]] = list(args[pos[0]])
        args[pos[0]][pos[1]] = value
    else:
        args[pos] = value


def _bad_calls(name):
    _, tensors, inplace = CASES[name]
    for arg, (pos, flags, shapes) in tensors.items():
        for kind, make in [("cpu", lambda t: t.cpu())] + ([("dtype", _wrong_dtype)] if "d" in flags else []) + \
                          ([("noncontiguous", _noncontig)] if "c" in flags else []) + [("shape%d" % k, f) for k, f in enumerate(shapes)]:
            yield "%s-%s-%s" % (name, arg, kind), name, arg, pos, make, inplace


BAD = [c for n in CASES for c in _bad_calls(n)]


def _build(be, name):
    build = CASES[name][0]
    return build(be) if build in (_corr_lookup_args, _alt_lookup_args) else build()


@pytest.mark.parametrize("name", sorted(CASES))
def test_valid_call_runs(backends, name):
    args = _build(backends, name)
    getattr(backends, name)(*args)
    torch.cuda.synchronize()


@pytest.mark.parametrize("case", BAD, ids=[c[0] for c in BAD])
def test_bad_argument_raises_before_any_launch(backends, case):
    _, name, arg, pos, make, inplace = case
    args = _build(backends, name)
    bad = make(_get(args, pos))
    _set(args, pos, bad)
    before = [_get(args, p).clone() for p in inplace]
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match=re.escape(name + ": " + arg + " ")):
        getattr(backends, name)(*args)
    torch.cuda.synchronize()
    for p, b in zip(inplace, before):
        assert torch.equal(_get(args, p), b), "argument %d changed although the call raised" % p


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("name", sorted(CASES))
def test_tensor_on_another_device_raises(backends, name):
    _, tensors, _ = CASES[name]
    for arg, (pos, _, _) in list(tensors.items())[1:]:   # the first tensor argument sets the device
        args = _build(backends, name)
        _set(args, pos, _get(args, pos).to("cuda:1"))
        with pytest.raises(RuntimeError, match=re.escape(name + ": " + arg + " must be on cuda:0")):
            getattr(backends, name)(*args)
