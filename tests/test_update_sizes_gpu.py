"""The update operator (csrc/update_op.cu) at feature widths that are not a multiple of 8, where its convolutions run the row-flattened
tiles of csrc/conv_engine.cuh: 1/8 of ETH3D through the reference's eval script (43x70), raw EuRoC through demo.py (44x69), 16:9 video
through demo.py (41x73) and a tiny 9x13.  Tolerances are those of tests/test_update_gpu.py and of the other stages' own tests; the
single convolutions at these widths are held to fp64 in tests/test_tensor_core_fp64_gpu.py."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import oracle
import oracle.encoder as oenc
from droid_slam_b200 import c_api, synth
from droid_slam_b200.encoder import pack_encoder_weights
from droid_slam_b200.update import PACKED_ORDER, UpdateModule, _taps, pack_update_weights

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from update_emul import emulate  # noqa: E402
from util import ptr, rel_err, stream  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [(43, 70), (44, 69), (41, 73), (9, 13)]
TOL = dict(net=1e-2, delta=2e-2, weight=1e-2, eta=2e-4, upmask=2e-2)


def _conv_case(E, ht, wd, c0, c1, ks, n, seed):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(E, ht, wd, c0, generator=g).half()
    x1 = torch.randn(E, ht, wd, c1, generator=g).half() if c1 else None
    cuse0 = 196 if c0 == 200 else c0
    ctot = cuse0 + c1
    w = (torch.randn(n, ctot, ks, ks, generator=g) * (1.0 / (ctot * ks * ks)) ** 0.5).half()
    b = 0.1 * torch.randn(n, generator=g)
    parts = [_taps(w[:, :cuse0].float(), 64 * ((cuse0 + 63) // 64))]
    if c1:
        parts.append(_taps(w[:, cuse0:].float(), 64 * ((c1 + 63) // 64)))
    return x0, x1, w, b, torch.cat(parts, 2).half().contiguous(), cuse0


def _conv_native(backends, x0, x1, wpk, b, ks, n, relu):
    E, ht, wd, c0 = x0.shape
    if c0 == 200:        # a 196-channel source on a 200-element row pitch: the C ABI directly
        L = c_api.load()
        xd, wd_, bd = x0.to(DEV), wpk.to(DEV), b.to(DEV)
        out = torch.full((E, ht, wd, n), float("nan"), dtype=torch.float16, device=DEV)
        c_api.check(L.dba_conv_nhwc(ptr(xd), 196, 200, None, 0, 0, ptr(wd_), ptr(bd), ptr(out), n, E, ht, wd, ks, n, int(relu), stream()), "conv_nhwc")
        return out
    return backends.conv_nhwc(x0.to(DEV), x1.to(DEV) if x1 is not None else None, wpk.to(DEV), b.to(DEV), ks, relu)


@pytest.mark.parametrize("c0,c1,ks,n", [(128, 0, 3, 128), (128, 320, 3, 256), (128, 0, 3, 384), (256, 0, 1, 64)])
def test_row_flattened_tiles_equal_rectangular_tiles_bit_for_bit(backends, c0, c1, ks, n):
    """width 69 (row-flattened) against the same input zero-padded to width 72 (32-wide rectangular tiles): with 'same' zero padding
    columns 0..68 are the same sums, accumulated in the same order (K block, dx, dy, k16) whatever the tiling"""
    E, ht = 6, 44
    x0, x1, _, b, wpk, _ = _conv_case(E, ht, 69, c0, c1, ks, n, 17 + n)
    pad = lambda t: None if t is None else F.pad(t, (0, 0, 0, 3))
    got = _conv_native(backends, x0, x1, wpk, b, ks, n, True)
    wide = _conv_native(backends, pad(x0), pad(x1), wpk, b, ks, n, True)
    torch.cuda.synchronize()
    assert torch.equal(got, wide[:, :, :69])


def _run(E, ht, wd, seed, n_src, with_flow=True, with_agg=True):
    w = synth.make_update_weights(0)
    net, inp, corr, flow, ii = synth.make_update_inputs(E=E, ht=ht, wd=wd, seed=seed, n_src=n_src)
    mod = UpdateModule().to(DEV)
    mod.load_state_dict(w)
    with torch.no_grad():
        got = mod(net.half().to(DEV), inp.half().to(DEV), corr.half().to(DEV), flow.to(DEV) if with_flow else None, ii.to(DEV) if with_agg else None)
    torch.cuda.synchronize()
    ref = oracle.update_module_forward(w, net.half().float(), inp.half().float(), corr.half().float(), flow if with_flow else None, ii if with_agg else None)
    return got, ref, (w, net, inp, corr, flow, ii)


def _check(got, ref, names):
    assert len(got) == len(names)
    for k, a, b in zip(names, got, ref):
        assert tuple(a.shape) == tuple(b.shape), (k, a.shape, b.shape)
        err = float((a.float().cpu() - b).abs().max())
        assert err < TOL[k], (k, err)


@pytest.mark.parametrize("ht,wd", SIZES)
def test_update_module_matches_oracle_at_odd_widths(ht, wd):
    got, ref, _ = _run(6, ht, wd, seed=ht + wd, n_src=3)
    _check(got, ref, ("net", "delta", "weight", "eta", "upmask"))
    assert got[0].dtype == torch.float16 and got[1].dtype == torch.float32 and got[2].dtype == torch.float32
    assert got[3].dtype == torch.float32 and got[4].dtype == torch.float16
    assert got[4].is_contiguous()


@pytest.mark.parametrize("ht,wd", SIZES)
def test_update_module_without_flow_and_aggregation_at_odd_widths(ht, wd):
    got, ref, _ = _run(4, ht, wd, seed=9, n_src=2, with_flow=False, with_agg=False)     # MotionFilter.track's call
    _check(got, ref, ("net", "delta", "weight"))


def test_update_module_matches_packed_weight_emulation_tightly_at_44x69():
    got, _, (w, net, inp, corr, flow, ii) = _run(5, 44, 69, seed=2, n_src=3)
    uniq, seg = torch.unique(ii, return_inverse=True)
    em = emulate(pack_update_weights(w), net[0].half(), inp[0].half(), corr[0].half(), flow[0], seg, uniq.numel(), round16=True)
    assert float((got[0][0].permute(0, 2, 3, 1).float().cpu() - em[0]).abs().max()) < 4e-3
    assert float((got[1][0].cpu() - em[1]).abs().max()) < 4e-3
    assert float((got[3][0].cpu() - em[3]).abs().max()) < 1e-4


def test_channels_last_state_round_trip_at_41x73():
    w = synth.make_update_weights(0)
    net, inp, corr, flow, ii = synth.make_update_inputs(E=4, ht=41, wd=73, seed=3, n_src=2)
    mod = UpdateModule().to(DEV)
    mod.load_state_dict(w)
    with torch.no_grad():
        o1 = mod(net.half().to(DEV), inp.half().to(DEV), corr.half().to(DEV), flow.to(DEV), ii.to(DEV))
        o2 = mod(o1[0], inp.half().to(DEV), corr.half().to(DEV), flow.to(DEV), ii.to(DEV))               # channels-last view straight back in
        o2b = mod(o1[0].contiguous(), inp.to(DEV), corr.half().to(DEV), flow.to(DEV), ii.to(DEV))        # NCHW copy, f32 context features
    torch.cuda.synchronize()
    assert torch.equal(o2[0], o2b[0]) and torch.equal(o2[1], o2b[1]) and torch.equal(o2[3], o2b[3])
    r1 = oracle.update_module_forward(w, net.half().float(), inp.half().float(), corr.half().float(), flow, ii)
    r2 = oracle.update_module_forward(w, r1[0], inp.half().float(), corr.half().float(), flow, ii)
    assert float((o2[0].float().cpu() - r2[0]).abs().max()) < 2e-2


def test_update_forward_reads_nothing_it_did_not_write_at_43x70():
    """dba_update_forward on a NaN-filled workspace and NaN-filled outputs: every output finite and equal to a call on a zeroed workspace
    (a partial-sum slot or tile that no kernel writes would carry the NaN through)"""
    E, ht, wd, n_src = 6, 43, 70, 3
    L = c_api.load()
    pk = pack_update_weights(synth.make_update_weights(0), DEV)
    W = c_api.UpdateWeights(*[pk[k].data_ptr() for k in PACKED_ORDER])
    net, inp, corr, flow, ii = synth.make_update_inputs(E=E, ht=ht, wd=wd, seed=5, n_src=n_src)
    net, inp, corr = (t[0].half().contiguous().to(DEV) for t in (net, inp, corr))
    flow = flow[0].contiguous().to(DEV)
    seg = torch.unique(ii, return_inverse=True)[1].to(DEV)
    nbytes = L.dba_update_workspace_bytes(E, n_src, ht, wd)

    def call(fill):
        ws = torch.full((nbytes // 4 + 64,), fill, dtype=torch.float32, device=DEV)
        wsp = (ws.data_ptr() + 255) // 256 * 256
        outs = [torch.full(s, float("nan"), dtype=dt, device=DEV) for s, dt in (((E, ht, wd, 128), torch.float16), ((E, ht, wd, 2), torch.float32),
                                                                                 ((E, ht, wd, 2), torch.float32), ((n_src, ht, wd), torch.float32),
                                                                                 ((n_src, 576, ht, wd), torch.float16))]
        a = c_api.UpdateArgs(E, ht, wd, net.data_ptr(), c_api.DBA_F16, 0, inp.data_ptr(), c_api.DBA_F16, corr.data_ptr(), c_api.DBA_F16,
                             flow.data_ptr(), seg.data_ptr(), n_src, ctypes.pointer(W), *[o.data_ptr() for o in outs], wsp, nbytes,
                             torch.cuda.current_stream().cuda_stream)
        c_api.check(L.dba_update_forward(ctypes.byref(a)), "update_forward")
        torch.cuda.synchronize()
        return outs

    nan_run, zero_run = call(float("nan")), call(0.0)
    for a, b in zip(nan_run, zero_run):
        assert bool(torch.isfinite(a).all())
        assert torch.equal(a, b)


def test_update_forward_cuda_graph_replays_bit_identically_at_41x73(backends):
    E, ht, wd, n_src = 5, 41, 73, 3
    mod = UpdateModule().to(DEV)
    mod.load_state_dict(synth.make_update_weights(0))
    net, inp, corr, flow, ii = synth.make_update_inputs(E=E, ht=ht, wd=wd, seed=11, n_src=n_src)
    net, inp, corr = (t[0].half().contiguous().to(DEV) for t in (net, inp, corr))
    flow = flow[0].contiguous().to(DEV)
    seg = torch.unique(ii, return_inverse=True)[1].to(DEV)
    packed = mod.packed_weights(torch.device(DEV))

    def step():
        return backends.update_forward(net, inp, corr, flow, seg, n_src, packed, False)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = [t.clone() for t in step()]
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for o in outs:
        o.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs, eager))


def _oracle_pyramid(f1, f2):
    """oracle.corr_pyramid plus level 3 as the 2x2 mean of level 2 (the reference pools once more after the last level)"""
    pyr = oracle.corr_pyramid(f1, f2, 3)
    E, ht, wd, h2, w2 = pyr[2].shape
    l3 = F.avg_pool2d(pyr[2].reshape(E * ht * wd, 1, h2, w2), 2, stride=2)
    return pyr + [l3.view(E, ht, wd, h2 // 2, w2 // 2)]


def test_native_chain_at_eth3d_size(backends):
    """ETH3D through the reference's eval script: 344x560 images, 43x70 feature maps.  Every stage against the oracle on the previous
    stage's native output: encoders, correlation pyramid + fused lookup, update operator, bundle adjustment."""
    N, H, W = 4, 344, 560
    ht, wd = H // 8, W // 8
    s = synth.make_scene(dict(E=10, N=N, ht=ht, wd=wd, stereo=False, itrs=2, lm=1e-4, ep=0.1), seed=3)
    ii, jj = s["ii"], s["jj"]
    E = ii.shape[0]
    assert torch.equal(torch.unique(ii), torch.arange(N))        # every frame is a source: the update's eta rows are BA's frames
    # encoders (tolerance of tests/test_encoder_gpu.py)
    images = torch.randn(1, N, 3, H, W, generator=torch.Generator().manual_seed(6)).to(DEV)
    feats = {}
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        for name, norm_fn, od, seed in (("fnet", "instance", 128, 0), ("cnet", "none", 256, 1)):
            sd = synth.make_encoder_weights(seed, od)
            sdd = {k: v.to(DEV) for k, v in sd.items()}
            with torch.no_grad():
                got = backends.encoder_forward(images[0], pack_encoder_weights(sd, norm_fn, od, DEV), 1 if norm_fn == "instance" else 0, od)
                ref = oenc.encoder_forward(sdd, images, norm_fn)[0]
                with torch.autocast("cuda", dtype=torch.float16):
                    ac = oenc.encoder_forward(sdd, images, norm_fn)[0].float()
            assert got.shape == (N, od, ht, wd)
            e_nat, e_ac = float((got.float() - ref).abs().max()), float((ac - ref).abs().max())
            assert e_nat <= 2 * e_ac + 1e-3 * float(ref.abs().max()), (name, e_nat, e_ac)
            feats[name] = got
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    # correlation pyramid on the native fnet maps (tests/test_corr_sizes_gpu.py) and the fused lookup, bit for bit against the oracle
    fm = feats["fnet"]
    pyr = backends.corr_volume_pyramid(fm, fm, ii.to(DEV), jj.to(DEV))
    ref = _oracle_pyramid(fm[None, ii.to(DEV)].float().cpu(), fm[None, jj.to(DEV)].float().cpu())
    for l in range(4):
        assert pyr[l].shape == ref[l].shape
        assert float((pyr[l].float().cpu() - ref[l]).abs().max()) < 2e-2 + 2e-3 * float(ref[l].abs().max()), l
    coords = s["coords_gt"]                                      # [E, ht, wd, 2]
    corr = backends.corr_lookup_pyramid(pyr, coords.permute(0, 3, 1, 2).contiguous().to(DEV))
    want = oracle.corr_block_lookup([v.cpu() for v in pyr], coords[None], 3)[0]
    assert torch.equal(corr.cpu(), want.reshape(corr.shape).to(corr.dtype))
    # update operator on the native context features and correlation features (tests/test_update_gpu.py)
    cnet = feats["cnet"][ii.to(DEV)]
    net, inp = torch.tanh(cnet[:, :128].float()).half()[None], torch.relu(cnet[:, 128:].float()).half()[None]
    flow = 2.0 * torch.randn(1, E, 4, ht, wd, generator=torch.Generator().manual_seed(8))
    w = synth.make_update_weights(0)
    mod = UpdateModule().to(DEV)
    mod.load_state_dict(w)
    with torch.no_grad():
        upd = mod(net, inp, corr[None], flow.to(DEV), ii.to(DEV))
    torch.cuda.synchronize()
    uref = oracle.update_module_forward(w, net.float().cpu(), inp.float().cpu(), corr[None].float().cpu(), flow, ii)
    # The bounds of tests/test_update_gpu.py are set for inputs of magnitude <= 1; real correlation and context features are larger, and
    # so is the f16 rounding of the chain.  Each output may therefore also reach twice the error of the reference's own f16 execution
    # (the oracle under autocast) on the same inputs.
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        uac = oracle.update_module_forward({k: v.to(DEV) for k, v in w.items()}, net, inp, corr[None], flow.to(DEV), ii.to(DEV))
    for k, a, b, c in zip(("net", "delta", "weight", "eta", "upmask"), upd, uref, uac):
        assert tuple(a.shape) == tuple(b.shape), (k, a.shape, b.shape)
        e_nat, e_ac = float((a.float().cpu() - b).abs().max()), float((c.float().cpu() - b).abs().max())
        print("update %s: native err %.3e, oracle-autocast err %.3e" % (k, e_nat, e_ac))
        assert e_nat < max(TOL[k], 2 * e_ac), (k, e_nat, e_ac)
    # bundle adjustment on the native update's targets, confidences and damping (tests/test_fullsize_gpu.py)
    targets = (coords + upd[1][0].cpu()).permute(0, 3, 1, 2).contiguous()
    weights = upd[2][0].cpu().permute(0, 3, 1, 2).contiguous()
    eta = upd[3][0].cpu().contiguous()
    P, D = s["poses"].to(DEV), s["disps"].to(DEV)
    backends.ba(P, D, s["intrinsics"].to(DEV), s["disps_sens"].to(DEV), targets.to(DEV), weights.to(DEV), eta.to(DEV), ii.to(DEV), jj.to(DEV),
                s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    P64, D64 = s["poses"].double(), s["disps"].double()
    oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], targets, weights, eta, ii, jj, s["t0"], s["t1"], 2, s["lm"], s["ep"], False, dtype=torch.float64)
    torch.cuda.synchronize()
    assert rel_err(P, P64, floor=1.0) < 1e-4 and rel_err(D, D64, floor=1.0) < 1e-4, (rel_err(P, P64, floor=1.0), rel_err(D, D64, floor=1.0))
