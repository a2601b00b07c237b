"""Row A6 on the GPU: the tensor-core update operator (csrc/update_op.cu) against the CPU oracle (oracle/update.py, pinned bit-exactly
against the reference's own UpdateModule).  The channels-last convolution building block is held to fp64 on every tiling route in
tests/test_tensor_core_fp64_gpu.py.

Tolerance: the reference runs this operator under fp16 autocast (factor_graph.py:214): activations and weights are f16, accumulation
fp32.  The oracle is fp32 end to end, so the comparison bound is the f16 rounding of ~10 chained layers: 1e-2 absolute on values of
magnitude <= 1 (observed ~2e-3), 2e-2 on the flow revision (magnitude ~1, K = 1152 sums)."""
import os
import sys

import pytest
import torch

import oracle
from droid_slam_b200 import synth
from droid_slam_b200.update import UpdateModule, pack_update_weights

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from update_emul import emulate  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(E, ht, wd, seed, n_src, with_flow=True, with_agg=True):
    w = synth.make_update_weights(0)
    net, inp, corr, flow, ii = synth.make_update_inputs(E=E, ht=ht, wd=wd, seed=seed, n_src=n_src)
    mod = UpdateModule().to(DEV)
    mod.load_state_dict(w)
    args = [net.half().to(DEV), inp.half().to(DEV), corr.half().to(DEV)]
    with torch.no_grad():
        got = mod(*args, flow.to(DEV) if with_flow else None, ii.to(DEV) if with_agg else None)
    torch.cuda.synchronize()
    ref = oracle.update_module_forward(w, net.half().float(), inp.half().float(), corr.half().float(), flow if with_flow else None, ii if with_agg else None)
    return got, ref, (w, net, inp, corr, flow, ii)


@pytest.mark.parametrize("E,ht,wd,n_src", [(6, 16, 64, 3), (5, 24, 32, 4), (3, 10, 40, 2), (4, 48, 64, 2)])
def test_update_module_matches_oracle(E, ht, wd, n_src):
    got, ref, _ = _run(E, ht, wd, seed=E, n_src=n_src)
    assert len(got) == 5
    tol = dict(net=1e-2, delta=2e-2, weight=1e-2, eta=2e-4, upmask=2e-2)
    for k, a, b in zip(("net", "delta", "weight", "eta", "upmask"), got, ref):
        assert tuple(a.shape) == tuple(b.shape), (k, a.shape, b.shape)
        err = float((a.float().cpu() - b).abs().max())
        assert err < tol[k], (k, err)
    assert got[0].dtype == torch.float16 and got[1].dtype == torch.float32 and got[4].dtype == torch.float16
    assert got[4].is_contiguous()                      # cvx_upsample views it (droid_net.py:25)


def test_update_module_without_flow_and_aggregation():
    got, ref, _ = _run(4, 16, 64, seed=9, n_src=2, with_flow=False, with_agg=False)     # MotionFilter.track's call (motion_filter.py:81)
    assert len(got) == 3
    for k, a, b, tol in zip(("net", "delta", "weight"), got, ref, (1e-2, 2e-2, 1e-2)):
        assert float((a.float().cpu() - b).abs().max()) < tol, k


def test_update_module_accepts_its_own_channels_last_state_and_f32_inputs():
    w = synth.make_update_weights(0)
    net, inp, corr, flow, ii = synth.make_update_inputs(E=4, ht=16, wd=64, seed=3, n_src=2)
    mod = UpdateModule().to(DEV)
    mod.load_state_dict(w)
    with torch.no_grad():
        o1 = mod(net.half().to(DEV), inp.half().to(DEV), corr.half().to(DEV), flow.to(DEV), ii.to(DEV))
        # second iteration: the returned hidden state (a channels-last view) goes straight back in
        o2 = mod(o1[0], inp.half().to(DEV), corr.half().to(DEV), flow.to(DEV), ii.to(DEV))
        o2b = mod(o1[0].contiguous(), inp.to(DEV), corr.half().to(DEV), flow.to(DEV), ii.to(DEV))       # NCHW copy, f32 context features
    torch.cuda.synchronize()
    assert torch.equal(o2[0], o2b[0]) and torch.equal(o2[1], o2b[1]) and torch.equal(o2[3], o2b[3])
    r1 = oracle.update_module_forward(w, net.half().float(), inp.half().float(), corr.half().float(), flow, ii)
    r2 = oracle.update_module_forward(w, r1[0], inp.half().float(), corr.half().float(), flow, ii)
    assert float((o2[0].float().cpu() - r2[0]).abs().max()) < 2e-2


def test_update_module_matches_packed_weight_emulation_tightly():
    """against the same dataflow on the same f16-rounded weights / activations (tests/update_emul.py): only accumulation order and
    the tanh.approx-based gates differ"""
    got, _, (w, net, inp, corr, flow, ii) = _run(5, 16, 64, seed=2, n_src=3)
    uniq, seg = torch.unique(ii, return_inverse=True)
    em = emulate(pack_update_weights(w), net[0].half(), inp[0].half(), corr[0].half(), flow[0], seg, uniq.numel(), round16=True)
    assert float((got[0][0].permute(0, 2, 3, 1).float().cpu() - em[0]).abs().max()) < 4e-3
    assert float((got[1][0].cpu() - em[1]).abs().max()) < 4e-3
    assert float((got[3][0].cpu() - em[3]).abs().max()) < 1e-4


def test_update_module_rejects_cpu_tensors():
    mod = UpdateModule()
    net, inp, corr, flow, ii = synth.make_update_inputs(E=2, ht=8, wd=8, seed=0, n_src=1)
    with pytest.raises(RuntimeError):
        mod(net, inp, corr, flow, ii)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_cvx_upsample_kernel_matches_oracle(backends, dtype):
    """DepthVideo.upsample's cvx_upsample (reference droid_net.py:21-42) in one kernel; f16 masks as the update operator emits them"""
    g = torch.Generator().manual_seed(5)
    n, ht, wd = 5, 48, 64
    d = torch.rand(n, ht, wd, generator=g) + 0.1
    m = (2.0 * torch.randn(n, 576, ht, wd, generator=g)).to(dtype)
    got = backends.cvx_upsample(d.to(DEV), m.to(DEV))
    ref = oracle.cvx_upsample(d[..., None], m.float())[..., 0]
    assert got.shape == (n, 8 * ht, 8 * wd)
    assert float((got.cpu() - ref).abs().max()) < 2e-6
    from droid_slam_b200.modules import upsample
    up = torch.zeros(8, 8 * ht, 8 * wd, device=DEV)
    ix = torch.tensor([1, 3, 4, 6, 7], device=DEV)
    disps = torch.zeros(8, ht, wd, device=DEV); disps[ix] = d.to(DEV)
    upsample(disps, up, ix, m.to(DEV)[None])
    assert torch.equal(up[ix], got) and float(up[0].abs().max()) == 0.0
