"""Row A6 (update operator) on CPU: the oracle against golden vectors produced by the reference module itself
(tests/golden/make_update_golden.py); the host side (droid_slam_b200/update.py): parameter names, and the packed weight layout + kernel
dataflow (restated in tests/update_emul.py on the packed tensors) against the oracle.  The kernels themselves: tests/test_update_gpu.py."""
import os
import sys

import pytest
import torch

import oracle
from droid_slam_b200 import synth
from droid_slam_b200.update import UpdateModule, pack_update_weights, PACKED_ORDER

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from update_emul import emulate  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_update_golden as mk  # noqa: E402
CASES = (("a", dict(E=5, ht=6, wd=8, seed=0, n_src=3)), ("b", dict(E=7, ht=5, wd=9, seed=1, n_src=4)))
NAMES = ("net", "delta", "weight", "eta", "upmask")


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "update_module.pt"))


@pytest.fixture(scope="module")
def weights():
    return synth.make_update_weights(0)


@pytest.mark.parametrize("name,kw", CASES)
def test_update_oracle_matches_reference_module(gold, weights, name, kw):
    net, inp, corr, flow, ii = synth.make_update_inputs(**kw)
    out = oracle.update_module_forward(weights, net, inp, corr, flow, ii)
    for k, t in zip(NAMES, out):
        if k == "upmask":                                                   # stored as a seeded quarter of the elements
            assert tuple(t.shape) == gold["%s_upmask_shape" % name]
            t, g = t.reshape(-1)[mk.upmask_sample_index(t.numel())], gold["%s_upmask_sample" % name]
        else:
            g = gold["%s_%s" % (name, k)]
        assert t.shape == g.shape
        assert torch.allclose(t, g, rtol=1e-5, atol=1e-6), (k, float((t - g).abs().max()))      # observed: bit-identical
    out = oracle.update_module_forward(weights, net, inp, corr, None, None)
    assert len(out) == 3
    for k, t in zip(NAMES[:3], out):
        assert torch.allclose(t, gold["%s_noflow_%s" % (name, k)], rtol=1e-5, atol=1e-6)


def test_update_module_has_the_reference_parameter_names(gold, weights):
    mod = UpdateModule()
    assert sorted(mod.state_dict().keys()) == gold["state_dict_keys"]          # a DROID checkpoint's update.* entries load as they are
    assert mod.load_state_dict(weights, strict=True) is not None
    for k, v in mod.state_dict().items():
        assert v.shape == weights[k].shape


def test_update_module_has_no_cpu_path(weights):
    mod = UpdateModule()
    net, inp, corr, flow, ii = synth.make_update_inputs(E=2, ht=8, wd=8, seed=0, n_src=1)
    with pytest.raises(RuntimeError):
        mod(net, inp, corr, flow, ii)


def test_packed_weights_layout(weights):
    pk = pack_update_weights(weights)
    assert tuple(pk.keys()) == PACKED_ORDER
    shapes = dict(w_corr0=(1, 128, 256), w_corr2=(9, 128, 128), w_flow0=(1, 128, 256), w_flow2=(9, 64, 128), w_gate=(1, 128, 128),
                  w_zr=(9, 256, 448), w_q=(9, 128, 448), w_stem=(9, 384, 128), w_heads=(1, 64, 256), w_agg2=(9, 128, 128), w_eta=(1, 32, 128),
                  w_upmask=(1, 576, 128), w_glo=(384, 128), b_glo=(384,), b_heads=(4,), b_eta=(1,), b_zr=(256,), b_stem=(384,), b_zero=(64,))
    for k, sh in shapes.items():
        assert tuple(pk[k].shape) == sh, k
    for i, k in enumerate(PACKED_ORDER):
        assert pk[k].dtype == (torch.float16 if i < 12 else torch.float32) and pk[k].is_contiguous()


@pytest.mark.parametrize("name,kw", CASES)
def test_packed_dataflow_matches_oracle(weights, name, kw):
    """the kernel sequence of csrc/update_op.cu, restated with torch on the packed weights, reproduces the reference operator up to the
    f16 rounding of the weights"""
    net, inp, corr, flow, ii = synth.make_update_inputs(**kw)
    uniq, seg = torch.unique(ii, return_inverse=True)
    pk = pack_update_weights(weights)
    got = emulate(pk, net[0], inp[0], corr[0], flow[0], seg, uniq.numel())
    ref = oracle.update_module_forward(weights, net, inp, corr, flow, ii)
    refs = [ref[0][0].permute(0, 2, 3, 1), ref[1][0], ref[2][0], ref[3][0], ref[4][0]]
    for k, a, b in zip(NAMES, got, refs):
        assert a.shape == b.shape and float((a - b).abs().max()) < 2e-3, (k, float((a - b).abs().max()))
    got3 = emulate(pk, net[0], inp[0], corr[0], None, None, 0)                 # flow=None, ii=None like MotionFilter.track's call
    ref3 = oracle.update_module_forward(weights, net, inp, corr)
    for a, b in zip(got3, [ref3[0][0].permute(0, 2, 3, 1), ref3[1][0], ref3[2][0]]):
        assert float((a - b).abs().max()) < 2e-3


def test_cvx_upsample_oracle_matches_reference_function(gold):
    """oracle.cvx_upsample vs the output of the reference's own cvx_upsample (droid_net.py:21-35, stored by make_update_golden.py)"""
    g = torch.Generator().manual_seed(321)
    d = torch.rand(3, 6, 10, 1, generator=g) + 0.2
    m = 2.0 * torch.randn(3, 576, 6, 10, generator=g)
    out = oracle.cvx_upsample(d, m)
    assert out.shape == gold["cvx_upsample"].shape == (3, 48, 80, 1)
    assert torch.allclose(out, gold["cvx_upsample"], rtol=1e-6, atol=1e-7)
    assert torch.equal(oracle.upsample_disp(d[None, ..., 0], m[None]), out[None, ..., 0])
