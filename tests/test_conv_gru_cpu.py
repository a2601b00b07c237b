"""The update operator's ConvGRU without a GPU: the oracle (oracle/update.py conv_gru_forward) against the fixture of the reference's
own module (tests/golden/conv_gru.pt), the library's exports of the new entry points, and the hook's strict policy on CPU tensors."""
import ctypes
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import reference  # noqa: E402
from conv_gru_cases import CASES, ConvGRU, case_inputs, load_params, make_inputs, make_params, run_chain  # noqa: E402
from droid_slam_b200 import c_api, modules  # noqa: E402
from oracle.update import conv_gru_forward  # noqa: E402

GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "conv_gru.pt"), weights_only=False)


def _close(a, b, tol):
    a, b = a.double(), b.double()
    return float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_reference_conv_gru(name):
    params, net, ins, cots = case_inputs(name)
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    got = run_chain(lambda h, *x: conv_gru_forward(leaves, h, *x, prefix=""), leaves, net, ins, cots)
    want = GOLDEN[name]
    assert len(got["outs"]) == len(want["outs"]) == CASES[name][3]
    for a, b in zip(got["outs"], want["outs"]):
        assert _close(a, b, 1e-12), name
    assert _close(got["grad_net"], want["grad_net"], 1e-12), name
    for ga, gb in zip(got["grad_inputs"], want["grad_inputs"]):
        for a, b in zip(ga, gb):
            assert _close(a, b, 1e-12), name
    assert set(got["grad_params"]) == set(want["grad_params"]) == set(modules.CONV_GRU_PARAMS)
    for k, a in got["grad_params"].items():
        assert _close(a, want["grad_params"][k], 1e-12), (name, k)


@pytest.mark.skipif(not reference.present("droid_slam"), reason="reference tree not present")
def test_generator_import_leaves_sys_path_and_sys_modules_alone():
    import make_conv_gru_golden
    path, before = list(sys.path), set(sys.modules)
    assert make_conv_gru_golden.import_reference() is not None
    assert sys.path == path
    added = {m for m in set(sys.modules) - before if m.split(".")[0] in ("lietorch", "torch_scatter", "modules")}
    assert not added, sorted(added)


def test_library_exports_the_conv_gru_entry_points():
    L = ctypes.CDLL(c_api.lib_path())
    for name in ("dba_conv_gru_workspace_bytes", "dba_conv_gru_forward", "dba_conv_gru_backward"):
        assert hasattr(L, name) and name in c_api.TRAINING_PROTOTYPES, name
    lib = c_api.load()
    assert lib.dba_conv_gru_workspace_bytes(0, 48, 64, 0) == 0 and lib.dba_conv_gru_workspace_bytes(2, 0, 64, 1) == 0
    assert lib.dba_conv_gru_workspace_bytes(24, 48, 64, 0) == 24 * 384 * 4        # the per-edge vectors
    assert lib.dba_conv_gru_workspace_bytes(24, 48, 64, 1) > 24 * 384 * 48 * 64 * 4  # the pre-activation gradients and more


def _module():
    return load_params(ConvGRU().float(), make_params(0))


def test_strict_policy_on_cpu_tensors():
    gru = types.ModuleType("gru")
    calls = []

    def forward(self, net, *inputs):
        calls.append("forward")
        return "reference"

    RefGRU = type("ConvGRU", (ConvGRU,), {"forward": forward})        # the reference's class name, its forward a marker
    gru.ConvGRU = RefGRU
    modules.install_conv_gru_hook(gru)
    m = load_params(RefGRU().float(), make_params(0))
    net, ins = make_inputs(1, 3, 4, 0)
    net, ins = net.float(), [t.float() for t in ins]
    msg = "ConvGRU.forward has no kernel for this call: "
    with pytest.raises(RuntimeError, match=msg + "net must be a CUDA float32"):
        m(net, *ins)
    with pytest.raises(RuntimeError, match=msg + r"net and inputs must be 4-d with 128 / \(128, 128, 64\) channels"):
        m(net, ins[0], ins[1], ins[1])
    with pytest.raises(RuntimeError, match=msg + r"net and inputs must be 4-d"):
        m(net, *ins[:2])
    with pytest.raises(RuntimeError, match=msg + r"net and the inputs disagree in \(b, h, w\)"):
        m(net, ins[0], ins[1], ins[2][:, :, :2])
    with pytest.raises(RuntimeError, match=msg + "an empty batch"):
        m(net[:0], *[t[:0] for t in ins])
    small = RefGRU(128, 256)
    with pytest.raises(RuntimeError, match=msg + r"the module is not ConvGRU\(128, 320\)"):
        small(net, *ins)
    with pytest.raises(RuntimeError, match=msg + "net must be a CUDA float32"):
        modules.conv_gru(m, net, *ins)                      # called directly: the same words
    assert calls == []
    for _ in range(2):                                      # a second install still reaches the reference's forward
        modules.install_conv_gru_hook(gru, strict=False)
    assert m(net, *ins) == "reference" and calls == ["forward"]
    entry = [e for e in modules.hook_registry() if e["installer"] == "install_conv_gru_hook"][-1]
    assert entry["kwargs"] == {"strict": False} and entry["target"] == repr(gru)


def test_stand_in_module_matches_the_oracle():
    """the tests' stand-in ConvGRU has the reference class's parameter names and the oracle's forward"""
    m = _module().double()
    assert [n for n, _ in m.named_parameters()] == list(modules.CONV_GRU_PARAMS)
    net, ins = make_inputs(1, 2, 3, 0)
    want = conv_gru_forward({k: v for k, v in m.named_parameters()}, net, *ins, prefix="")
    assert torch.equal(m(net, *ins), want)
