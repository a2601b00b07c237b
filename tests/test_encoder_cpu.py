"""CPU checks of the native feature / context encoders: the fp32 oracle against the reference's own outputs (tests/golden/encoder.pt),
the packed weight layout of pack_encoder_weights (gather K order included) against F.conv2d, the hook's strict / fallback selection and
grad guard, and the C-ABI symbols."""
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

import oracle.encoder as oenc
from droid_slam_b200 import c_api, synth
from droid_slam_b200.encoder import ENCODER_CONVS, pack_encoder_weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import reference  # noqa: E402


def test_oracle_matches_reference_golden():
    g = torch.load(os.path.join(ROOT, "tests", "golden", "encoder.pt"))
    assert len(g["cases"]) == 6
    for c in g["cases"]:
        sd = synth.make_encoder_weights(c["weight_seed"], c["output_dim"])
        got = oenc.encoder_forward(sd, c["images"], c["norm_fn"])
        err = float((got - c["out"]).abs().max())
        assert err <= 1e-4 * float(c["out"].abs().max()) + 1e-5, (c["name"], tuple(c["images"].shape), err)


def _im2col_stem(x):
    """[n,3,H,W] -> [n,H/2,W/2,147], K = (dy*7 + dx)*3 + c"""
    u = F.unfold(x, 7, padding=3, stride=2)                      # [n, 3*49 (c, dy, dx), L]
    n, _, L = u.shape
    return u.view(n, 3, 49, L).permute(0, 3, 2, 1).reshape(n, x.shape[2] // 2, x.shape[3] // 2, 147)


def _gather_s2(x):
    """[n,C,h,w] -> [n,h/2,w/2,9C], K = (dy*3 + dx)*C + c"""
    n, C, h, w = x.shape
    u = F.unfold(x, 3, padding=1, stride=2)                      # [n, C*9 (c, dy, dx), L]
    return u.view(n, C, 9, -1).permute(0, 3, 2, 1).reshape(n, h // 2, w // 2, 9 * C)


def _conv_taps(x, wk, ci):
    """3x3 'same' convolution from packed [9][N][Kpad] weights: sum over taps of the shifted channels-last input"""
    n, C, h, w = x.shape
    xp = F.pad(x, (1, 1, 1, 1)).permute(0, 2, 3, 1)
    out = 0
    for t in range(9):
        dy, dx = divmod(t, 3)
        out = out + xp[:, dy:dy + h, dx:dx + w, :] @ wk[t, :, :ci].T
    return out


@pytest.mark.parametrize("norm_fn,od", [("instance", 128), ("none", 256)])
def test_packed_weights_reproduce_conv2d(norm_fn, od):
    sd = synth.make_encoder_weights(3, od)
    pk = pack_encoder_weights(sd, norm_fn, od)
    assert len(pk) == 28 and all(t.dtype == torch.float16 for t in pk[:14]) and all(t.dtype == torch.float32 for t in pk[14:])
    W = [t.float() for t in pk[:14]]
    B = pk[14:]
    q = lambda t: t.half().float()                               # the packed operands are f16
    g = torch.Generator().manual_seed(0)
    tol = lambda ref: 1e-4 * float(ref.abs().max()) + 1e-5
    # conv1 7x7/2 over the im2col rows
    x = torch.randn(2, 3, 16, 24, generator=g)
    ref = F.conv2d(x, q(sd["conv1.weight"]), sd["conv1.bias"], stride=2, padding=3).permute(0, 2, 3, 1)
    got = _im2col_stem(x) @ W[0][0, :, :147].T + B[0]
    assert W[0][0, :, 147:].abs().max() == 0 and float((got - ref).abs().max()) <= tol(ref)
    # 3x3 stride-1 convolutions
    for k, name in enumerate(ENCODER_CONVS):
        if name in ("conv1", "conv2", "layer2.0.conv1", "layer3.0.conv1"):
            continue
        w = sd[name + ".weight"]
        x = torch.randn(1, w.shape[1], 6, 10, generator=g)
        ref = F.conv2d(x, q(w), sd[name + ".bias"], padding=1).permute(0, 2, 3, 1)
        got = _conv_taps(x, W[k], w.shape[1]) + B[k]
        assert W[k].shape[2] % 64 == 0 and W[k][:, :, w.shape[1]:].abs().sum() == 0
        assert float((got - ref).abs().max()) <= tol(ref), name
    # stride-2 blocks: conv1 3x3/2 | downsample 1x1/2 as one GEMM over the gathered taps
    for k, blk in ((5, "layer2.0"), (9, "layer3.0")):
        w1, wd = sd[blk + ".conv1.weight"], sd[blk + ".downsample.0.weight"]
        P, C = w1.shape[0], w1.shape[1]
        x = torch.randn(1, C, 12, 20, generator=g)
        got = _gather_s2(x) @ W[k][0, :, :9 * C].T + B[k]
        r1 = F.conv2d(x, q(w1), sd[blk + ".conv1.bias"], stride=2, padding=1).permute(0, 2, 3, 1)
        r2 = F.conv2d(x, q(wd), sd[blk + ".downsample.0.bias"], stride=2).permute(0, 2, 3, 1)
        assert float((got[..., :P] - r1).abs().max()) <= tol(r1) and float((got[..., P:] - r2).abs().max()) <= tol(r2), blk
        assert W[k][0, :, 9 * C:].abs().sum() == 0
    # conv2 1x1
    x = torch.randn(1, 128, 3, 5, generator=g)
    ref = F.conv2d(x, q(sd["conv2.weight"]), sd["conv2.bias"]).permute(0, 2, 3, 1)
    got = x.permute(0, 2, 3, 1) @ W[13][0].T + B[13]
    assert float((got - ref).abs().max()) <= tol(ref)


def test_pack_rejects_encoders_without_kernel():
    with pytest.raises(ValueError):
        pack_encoder_weights(synth.make_encoder_weights(0, 128), "batch", 128)
    with pytest.raises(ValueError):
        pack_encoder_weights(synth.make_encoder_weights(0, 128), "instance", 256)


def _extractor_module():
    """the reference's modules.extractor where the reference tree exists, else a namespace around a subclass of the oracle's stand-in;
    either way a fresh class, so patching it leaves other tests alone"""
    if reference.present("droid_slam", "modules", "extractor.py"):
        with reference.reference_modules("modules.extractor") as (m,):
            return m
    return types.SimpleNamespace(BasicEncoder=type("BasicEncoder", (oenc.BasicEncoder,), {}))


def test_hook_strict_and_fallback_selection():
    from droid_slam_b200.modules import install_encoder_hook
    x = torch.randn(1, 1, 3, 32, 48)
    ref_mod = _extractor_module()
    fnet = ref_mod.BasicEncoder(output_dim=128, norm_fn="instance").eval()
    fnet.load_state_dict(synth.make_encoder_weights(0, 128))
    with torch.no_grad():
        want = fnet(x)
    install_encoder_hook(ref_mod, strict=False)
    with torch.no_grad():
        assert torch.equal(fnet(x), want)                        # CPU input: the reference's forward runs
    strict_mod = _extractor_module()
    install_encoder_hook(strict_mod)
    for enc, inp, why in ((strict_mod.BasicEncoder(128, "instance"), x, "CUDA"), (strict_mod.BasicEncoder(128, "batch"), x, "norm_fn"),
                          (strict_mod.BasicEncoder(128, "instance", dropout=0.1), x, "dropout"),
                          (strict_mod.BasicEncoder(128, "instance", multidim=True), x, "multidim")):
        with pytest.raises(RuntimeError, match=why):
            enc(inp)


def test_hook_grad_guard(monkeypatch):
    from droid_slam_b200 import modules
    m = _extractor_module()
    modules.install_encoder_hook(m)
    monkeypatch.setattr(modules, "_encoder_unsupported", lambda enc, x: None)
    enc = m.BasicEncoder(128, "instance")
    with pytest.raises(RuntimeError, match="requires grad"):
        enc(torch.randn(1, 1, 3, 32, 48, requires_grad=True))


def test_capi_encoder_symbols_and_workspace():
    L = c_api.load()
    assert hasattr(L, "dba_encoder_forward") and hasattr(L, "dba_encoder_workspace_bytes")
    assert L.dba_encoder_workspace_bytes(1, 384, 512, 128) > 0
    assert L.dba_encoder_workspace_bytes(16, 384, 512, 256) > L.dba_encoder_workspace_bytes(1, 384, 512, 256)
    for bad in ((0, 64, 96, 128), (1, 60, 96, 128), (1, 64, 90, 128), (1, 64, 96, 64)):
        assert L.dba_encoder_workspace_bytes(*bad) == 0, bad
    assert L.dba_encoder_forward(None) == 1
