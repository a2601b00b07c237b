"""The native feature / context encoders (droid_backends.encoder_forward, dba_encoder_forward, install_encoder_hook) against the fp32
oracle (oracle/encoder.py) on the GPU.  Tolerance per output: err(native) <= 2 err(oracle under autocast) + 1e-3 max|ref|, both errors
against the fp32 oracle on the same input, so the native path is no worse than the reference's own f16 execution."""
import ctypes
import types

import pytest
import torch

import oracle.encoder as oenc
from droid_slam_b200 import c_api, synth
from droid_slam_b200.encoder import pack_encoder_weights

pytestmark = pytest.mark.gpu

ENCODERS = {"fnet": ("instance", 128), "cnet": ("none", 256)}


@pytest.fixture
def no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _images(n, H, W, seed, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(1, n, 3, H, W, generator=g) + shift


def _compare(backends, name, n, H, W, shift=0.0, dtype=torch.float32, seed=0):
    norm_fn, od = ENCODERS[name]
    sd = synth.make_encoder_weights(seed, od)
    sdd = {k: v.cuda() for k, v in sd.items()}
    x = _images(n, H, W, seed + 1, shift).to("cuda", dtype)
    with torch.no_grad():
        ref = oenc.encoder_forward(sdd, x.float(), norm_fn)
        with torch.autocast("cuda", dtype=torch.float16):
            ac = oenc.encoder_forward(sdd, x, norm_fn)
        got = backends.encoder_forward(x[0].contiguous(), pack_encoder_weights(sd, norm_fn, od, "cuda"), 1 if norm_fn == "instance" else 0, od)
    assert got.shape == (n, od, H // 8, W // 8) and got.dtype == torch.float16
    assert torch.isfinite(got).all()
    e_nat = float((got.float() - ref[0]).abs().max())
    e_ac = float((ac.float() - ref).abs().max())
    scale = float(ref.abs().max())
    print("%s n=%d %dx%d shift=%g %s: native err %.3e, oracle-autocast err %.3e, max|ref| %.3e" % (name, n, H, W, shift, dtype, e_nat, e_ac, scale))
    assert e_nat <= 2 * e_ac + 1e-3 * scale, (e_nat, e_ac, scale)


@pytest.mark.parametrize("name", ["fnet", "cnet"])
@pytest.mark.parametrize("n,H,W", [(1, 384, 512), (16, 384, 512), (1, 352, 552), (1, 240, 320), (2, 64, 96)])
def test_encoder_matches_oracle(backends, no_tf32, name, n, H, W):
    _compare(backends, name, n, H, W)


@pytest.mark.parametrize("name", ["fnet", "cnet"])
def test_encoder_mean_shifted_input_matches_oracle(backends, no_tf32, name):
    """images + 40: every instance norm sees |mean| >> std over up to 49 152 pixels"""
    _compare(backends, name, 1, 384, 512, shift=40.0)


@pytest.mark.parametrize("name", ["fnet", "cnet"])
def test_encoder_f16_images_match_oracle(backends, no_tf32, name):
    _compare(backends, name, 2, 240, 320, dtype=torch.float16)


def test_encoder_argument_validation_launches_nothing(capi):
    H, W = 64, 96
    pk = pack_encoder_weights(synth.make_encoder_weights(0, 128), "instance", 128, "cuda")
    wt = c_api.EncoderWeights()
    for k in range(14):
        wt.w[k], wt.b[k] = pk[k].data_ptr(), pk[14 + k].data_ptr()
    img = torch.randn(1, 3, H, W, device="cuda")
    out = torch.full((1, 128, H // 8, W // 8), 7.0, device="cuda", dtype=torch.float16)
    nbytes = capi.dba_encoder_workspace_bytes(1, H, W, 128)
    assert nbytes > 0 and capi.dba_encoder_workspace_bytes(1, H + 1, W, 128) == 0 and capi.dba_encoder_workspace_bytes(1, H, W, 64) == 0
    ws = torch.empty(nbytes + 256, device="cuda", dtype=torch.uint8)
    wsp = (ws.data_ptr() + 255) // 256 * 256

    def args(**over):
        a = c_api.EncoderArgs(img.data_ptr(), c_api.DBA_F32, 1, H, W, ctypes.pointer(wt), 1, 128, out.data_ptr(), wsp, nbytes, None)
        for k, v in over.items():
            setattr(a, k, v)
        return a

    torch.cuda.synchronize()
    assert capi.dba_encoder_forward(ctypes.byref(args(H=H - 1))) == 1
    assert capi.dba_encoder_forward(ctypes.byref(args(workspace_bytes=nbytes - 1))) == 3
    assert capi.dba_encoder_forward(ctypes.byref(args(images=None))) == 1
    assert capi.dba_encoder_forward(None) == 1
    wt.w[3] = None
    assert capi.dba_encoder_forward(ctypes.byref(args())) == 1
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()), "a rejected call wrote its output"
    wt.w[3] = pk[3].data_ptr()
    assert capi.dba_encoder_forward(ctypes.byref(args())) == 0
    torch.cuda.synchronize()
    assert not bool((out == 7.0).all())


def test_encoder_cuda_graph_replays_bit_identically(backends):
    H, W = 240, 320
    x = torch.randn(1, 3, H, W, device="cuda")
    pf = pack_encoder_weights(synth.make_encoder_weights(0, 128), "instance", 128, "cuda")
    pc = pack_encoder_weights(synth.make_encoder_weights(1, 256), "none", 256, "cuda")
    eager = (backends.encoder_forward(x, pf, 1, 128), backends.encoder_forward(x, pc, 0, 256))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        backends.encoder_forward(x, pf, 1, 128)
        backends.encoder_forward(x, pc, 0, 256)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = (backends.encoder_forward(x, pf, 1, 128), backends.encoder_forward(x, pc, 0, 256))
    for _ in range(2):
        for o in outs:
            o.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(outs, eager))


def test_encoder_hook_on_standin():
    from droid_slam_b200.modules import install_encoder_hook
    ns = types.SimpleNamespace(BasicEncoder=type("BasicEncoder", (oenc.BasicEncoder,), {}))
    install_encoder_hook(ns)
    fnet = ns.BasicEncoder(output_dim=128, norm_fn="instance").cuda().eval()
    fnet.load_state_dict(synth.make_encoder_weights(0, 128))
    cnet = ns.BasicEncoder(output_dim=256, norm_fn="none").cuda().eval()
    cnet.load_state_dict(synth.make_encoder_weights(1, 256))
    images = torch.randn(2, 3, 64, 96, device="cuda")
    with torch.no_grad():
        with torch.autocast("cuda", enabled=True):
            f, c = fnet(images[None]), cnet(images[None])
        assert f.shape == (1, 2, 128, 8, 12) and f.dtype == torch.float16
        assert c.shape == (1, 2, 256, 8, 12) and c.dtype == torch.float16
        f32 = fnet(images[None])
        assert f32.dtype == torch.float32 and torch.equal(f32, f.float())
        with pytest.raises(RuntimeError, match="multiples of 8"):
            fnet(torch.randn(1, 1, 3, 60, 96, device="cuda"))
    with pytest.raises(RuntimeError, match="requires grad"):
        fnet(images[None].clone().requires_grad_(True))
    # the hook changed only the subclass
    assert oenc.BasicEncoder.forward is not ns.BasicEncoder.forward
