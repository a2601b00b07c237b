"""The update operator's ConvGRU on the GPU (droid_slam_b200.modules.conv_gru, csrc/gru_train.cu): forward and every gradient against
autograd through the oracle (oracle/update.py conv_gru_forward) in fp64, no less accurate than the oracle in fp32 on cuDNN without TF32;
bit-identical reruns, no host synchronisation, what the forward keeps, NaN propagation and the strict policy on CUDA tensors."""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from conv_gru_cases import ConvGRU, load_params, make_cotangent, make_inputs, make_params, run_chain  # noqa: E402
from droid_slam_b200 import modules  # noqa: E402
from oracle.update import conv_gru_forward  # noqa: E402
from util import host_syncs  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
FULL = lambda name, t: t  # noqa: E731
# A measure at fp32's unit roundoff is as exact as an fp32 result can be; where the fp32 oracle happens to be exact (a 1x1 image's
# sums of one term) twice its measure would be zero, so the bound never goes below this.
FLOOR = 2.0 ** -24


def _native(params):
    """the stand-in ConvGRU on the device with `params` (fp64 dict) in fp32 -> (module, {name: leaf})"""
    m = load_params(ConvGRU().to(DEV), params)
    return m, dict(m.named_parameters())


def _run_all(b, h, w, calls, seed, grads=True):
    """(native, oracle fp32 without TF32, oracle fp64) results of run_chain on the same seeded chain"""
    params = make_params(seed)
    net, _ = make_inputs(b, h, w, 100 * seed)
    ins = [make_inputs(b, h, w, 100 * seed + 1 + k)[1] for k in range(calls)]
    cots = [make_cotangent(b, h, w, 100 * seed + 50 + k) for k in range(calls)]
    res = []
    for kind in ("native", torch.float32, torch.float64):
        dt = torch.float32 if kind == "native" else kind
        x = lambda t: t.to(DEV, dt)  # noqa: E731
        n, i, c = x(net), [[x(t) for t in call] for call in ins], [x(t) for t in cots]
        if kind == "native":
            m, leaves = _native(params)
            fwd = lambda hh, *xs: modules.conv_gru(m, hh, *xs)  # noqa: E731
        else:
            leaves = {k: x(v).requires_grad_(True) for k, v in params.items()}
            fwd = lambda hh, *xs: conv_gru_forward(leaves, hh, *xs, prefix="")  # noqa: E731
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            res.append(run_chain(fwd, leaves, n, i, c, keep=FULL))
    return res


def _flat(r):
    out = [("out%d" % k, o) for k, o in enumerate(r["outs"])] + [("grad_net", r["grad_net"])]
    out += [("grad_%s[%d]" % (n, k), g) for k, call in enumerate(r["grad_inputs"]) for n, g in zip(("inp", "corr", "flow"), call)]
    return out + [("grad_" + n, g) for n, g in r["grad_params"].items()]


def _rel(x, x64):
    return float((x.double() - x64).abs().max()) / max(float(x64.abs().max()), 1e-300)


def _check(nat, f32, f64):
    worst = []
    for (name, a), (_, b), (_, c) in zip(_flat(nat), _flat(f32), _flat(f64)):
        assert torch.isfinite(a).all(), name
        en, e32 = _rel(a, c), _rel(b, c)
        worst.append((en / max(e32, FLOOR), name, en, e32))
        assert en <= max(2 * e32, FLOOR), (name, en, e32)
    return max(worst)


@pytest.mark.parametrize("b,h,w,calls", [(22, 48, 64, 1), (24, 48, 64, 1), (1, 1, 1, 1), (3, 5, 7, 1), (2, 37, 53, 1), (4, 12, 16, 3)],
                         ids=["b22_48x64", "b24_48x64", "b1_1x1", "b3_5x7", "b2_37x53_tail", "chain3_b4_12x16"])
def test_forward_and_every_gradient_against_fp64(b, h, w, calls):
    _check(*_run_all(b, h, w, calls, seed=7))


def test_parameter_gradients_when_only_parameters_require_grad():
    params = make_params(3)
    net, ins = make_inputs(2, 9, 11, 30)
    cot = make_cotangent(2, 9, 11, 31)
    res = []
    for kind in ("native", torch.float32, torch.float64):
        dt = torch.float32 if kind == "native" else kind
        n, i, c = net.to(DEV, dt), [t.to(DEV, dt) for t in ins], cot.to(DEV, dt)
        if kind == "native":
            m, leaves = _native(params)
            out = modules.conv_gru(m, n, *i)
        else:
            leaves = {k: v.to(DEV, dt).requires_grad_(True) for k, v in params.items()}
            with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
                out = conv_gru_forward(leaves, n, *i, prefix="")
        assert out.requires_grad
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            g = torch.autograd.grad((out * c).sum(), [leaves[k] for k in modules.CONV_GRU_PARAMS])
        res.append([out.detach()] + list(g))
    for k, (a, b, c) in enumerate(zip(*res)):
        en, e32 = _rel(a, c), _rel(b, c)
        assert en <= max(2 * e32, FLOOR), (k, en, e32)


def _call(m, net, ins, cot):
    out = modules.conv_gru(m, net, *ins)
    return [out] + list(torch.autograd.grad(out, [net] + ins + list(m.parameters()), cot))


def test_reruns_give_the_same_bits():
    m, _ = _native(make_params(4))
    net, ins = make_inputs(3, 9, 11, 40)
    net, ins = net.to(DEV).float().requires_grad_(True), [t.to(DEV).float().requires_grad_(True) for t in ins]
    cot = make_cotangent(3, 9, 11, 41).to(DEV).float()
    first, second = _call(m, net, ins, cot), _call(m, net, ins, cot)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    out = modules.conv_gru(m, net, *ins)
    g1 = torch.autograd.grad(out, net, cot, retain_graph=True)[0]
    g2 = torch.autograd.grad(out, net, cot)[0]
    assert torch.equal(g1, g2) and torch.equal(g1, first[1])


def test_no_host_synchronisation():
    m, _ = _native(make_params(5))
    net, ins = make_inputs(4, 12, 16, 50)
    net, ins = net.to(DEV).float().requires_grad_(True), [t.to(DEV).float().requires_grad_(True) for t in ins]
    cot = make_cotangent(4, 12, 16, 51).to(DEV).float()
    _call(m, net, ins, cot)                                           # warm-up: the first call loads the kernels
    out = {}
    n_fwd, _ = host_syncs(lambda: out.setdefault("y", modules.conv_gru(m, net, *ins)))
    n_bwd, _ = host_syncs(lambda: torch.autograd.grad(out["y"], [net] + ins + list(m.parameters()), cot))
    with torch.no_grad():
        n_ng, _ = host_syncs(lambda: modules.conv_gru(m, net, *ins))
    assert (n_fwd, n_bwd, n_ng) == (0, 0, 0)


def test_saved_state_is_at_most_384_channels_and_per_edge_vectors():
    m, leaves = _native(make_params(6))
    b, h, w = 3, 10, 13
    net, ins = make_inputs(b, h, w, 60)
    net, ins = net.to(DEV).float().requires_grad_(True), [t.to(DEV).float().requires_grad_(True) for t in ins]
    saved = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append(t) or t, lambda t: t):
        out = modules.conv_gru(m, net, *ins)
    own = {t.data_ptr() for t in [net] + ins + list(leaves.values())}
    extra = sum(t.numel() * t.element_size() for t in saved if t.data_ptr() not in own)
    assert extra <= (384 * h * w + 128) * b * 4, extra
    assert len(saved) >= 4 + 14                                          # the inputs and parameters are kept by reference
    with torch.no_grad():
        saved.clear()
        with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append(t) or t, lambda t: t):
            y = modules.conv_gru(m, net, *ins)
        assert saved == [] and not y.requires_grad and torch.equal(y, out.detach())


def test_nan_in_one_corr_pixel_gives_the_oracles_nan_set():
    params = make_params(8)
    net, ins = make_inputs(2, 9, 11, 80)
    ins[1][1, 5, 4, 6] = float("nan")
    m, _ = _native(params)
    with torch.no_grad():
        got = modules.conv_gru(m, net.to(DEV).float(), *[t.to(DEV).float() for t in ins])
        want = conv_gru_forward({k: v.to(DEV) for k, v in params.items()}, net.to(DEV), *[t.to(DEV) for t in ins], prefix="")
    assert bool(torch.isnan(want).any()) and torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(torch.isnan(got[0]), torch.zeros_like(got[0], dtype=torch.bool))


def test_strict_policy_on_cuda_tensors():
    gru = types.ModuleType("gru")
    gru.ConvGRU = type("ConvGRU", (ConvGRU,), {})
    modules.install_conv_gru_hook(gru)
    m = load_params(gru.ConvGRU().to(DEV), make_params(9))
    net, ins = make_inputs(2, 5, 6, 90)
    net, ins = net.to(DEV).float(), [t.to(DEV).float() for t in ins]
    with torch.no_grad():
        assert torch.equal(m(net, *ins), modules.conv_gru(m, net, *ins))
        assert torch.equal(m(net.transpose(2, 3).contiguous().transpose(2, 3), *ins), m(net, *ins))   # non-contiguous: copied
    msg = "ConvGRU.forward has no kernel for this call: "
    with pytest.raises(RuntimeError, match=msg + "net must be a CUDA float32"):
        m(net.double(), *ins)
    with pytest.raises(RuntimeError, match=msg + r"inputs\[1\] must be a CUDA float32"):
        m(net, ins[0], ins[1].cpu(), ins[2])
    with pytest.raises(RuntimeError, match=msg + "CUDA autocast is enabled"):
        with torch.autocast("cuda", dtype=torch.float16):
            m(net, *ins)
    with pytest.raises(RuntimeError, match=msg + "net and inputs must be 4-d with 128"):
        m(net, ins[0], ins[1], ins[1])
    with pytest.raises(RuntimeError, match=msg + r"net and the inputs disagree in \(b, h, w\)"):
        m(net, ins[0], ins[1][:1], ins[2])
    cpu_params = load_params(gru.ConvGRU(), make_params(9))
    with pytest.raises(RuntimeError, match=msg + "convz.weight must be a CUDA float32"):
        cpu_params(net, *ins)
    modules.install_conv_gru_hook(gru, strict=False)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        ref = m(net, *ins)                                              # the reference's forward (here the oracle's) under autocast
        want = ConvGRU.forward(m, net, *ins)
    assert torch.equal(ref, want)
