"""Training's flow loss and upsample_disp without a GPU: the oracles (oracle/flow_loss.py, oracle/upsample.py) against the fixture of
the reference's own functions (tests/golden/flow_loss.pt), the fixture generator's import, the training header's prototypes against
c_api.TRAINING_PROTOTYPES and the library's exports, and the hooks' strict policy on CPU tensors."""
import ctypes
import os
import re
import subprocess
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import reference  # noqa: E402
from droid_slam_b200 import c_api, modules  # noqa: E402
from droid_slam_b200 import lietorch as lt  # noqa: E402
from flow_loss_cases import cases, upsample_cases  # noqa: E402
from oracle import ba_layer as oba, flow_loss as ofl, upsample as oup  # noqa: E402
from test_oracle_cpu import _c_kind, _py_kind  # noqa: E402

GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "flow_loss.pt"), weights_only=False)
HEADER = os.path.join(ROOT, "include", "droid_b200_training.h")


def oracle_flow(c, dtype=torch.float64, dev="cpu"):
    """loss, metrics and gradients through oracle/flow_loss.py, in the fixture's form"""
    to = lambda t: t.to(dev, dtype)  # noqa: E731
    n = len(c["poses_est"])
    d = [to(x).requires_grad_(True) for x in c["disps_est"]]
    eps = [torch.zeros(*p.shape[:-1], 6, dtype=dtype, device=dev, requires_grad=True) for p in c["poses_est"]]
    P = [oba.SE3(oba.left_perturbed(to(p), e)) for p, e in zip(c["poses_est"], eps)]
    loss, epe, v = ofl.flow_loss(oba.SE3(to(c["Ps"])), to(c["disps"]), P, d, to(c["intrinsics"]))
    g = torch.autograd.grad(loss, d + eps)
    gp = [torch.cat([x, torch.zeros_like(x[..., :1])], -1) for x in g[n:]]
    return dict(loss=loss.detach(), metrics=ofl.metrics(epe.detach(), v), grad_disps_est=list(g[:n]), grad_poses_est=gp)


def _close(a, b, tol):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    nan = torch.isnan(b)
    assert torch.equal(torch.isnan(a), nan)
    return float((a[~nan] - b[~nan]).abs().max()) <= tol * max(1.0, float(b[~nan].abs().max())) if (~nan).any() else True


@pytest.mark.parametrize("name", sorted(cases()))
def test_oracle_reproduces_the_reference_flow_loss(name):
    want, got = GOLDEN["flow"][name], oracle_flow(cases()[name])
    assert _close(got["loss"], want["loss"], 1e-12), name
    for k in ("f_error", "1px"):
        assert _close(got["metrics"][k], want["metrics"][k], 1e-12), (name, k)
    for k in ("grad_disps_est", "grad_poses_est"):
        for i, (a, b) in enumerate(zip(got[k], want[k])):
            assert _close(a, b, 1e-12), (name, k, i)


@pytest.mark.parametrize("name", sorted(upsample_cases()))
def test_oracle_reproduces_the_reference_upsample_disp(name):
    c, want = upsample_cases()[name], GOLDEN["upsample"][name]
    disp, mask = c["disp"].clone().requires_grad_(True), c["mask"].clone().requires_grad_(True)
    loss = (c["cot"] * oup.upsample_disp(disp, mask)).sum()
    gd, gm = torch.autograd.grad(loss, [disp, mask])
    assert _close(loss.detach(), want["loss"], 1e-12) and _close(gd, want["grad_disp"], 1e-12) and _close(gm, want["grad_mask"], 1e-12)


def test_fixture_covers_the_edges():
    """the threshold case puts pixels on both sides of Z = 0.1 and 0.2; no-valid and NaN metrics are what the reference gives"""
    c = cases()["thresholds"]
    z = 1.0 - c["disps_est"][0][0, 0]                    # edge 0 -> 1 of iterate 0
    for t in (0.1, 0.2):
        assert bool(((z - t).abs() < 0.02).any() & (z < t).any() & (z > t).any()), t
    assert bool((cases()["zero_negative_gt"]["disps"] <= 0).any())


@pytest.mark.skipif(not reference.present("droid_slam"), reason="reference tree not present")
def test_generator_import_leaves_sys_path_and_sys_modules_alone():
    import make_flow_loss_golden
    names = {"lietorch", "torch_scatter", "droid_backends", "geom", "modules", "droid_net"}
    path, before = list(sys.path), set(sys.modules)
    assert make_flow_loss_golden.import_reference() is not None
    assert sys.path == path
    added = {m for m in set(sys.modules) - before if m.split(".")[0] in names}
    assert not added, sorted(added)


def test_training_prototypes_match_header(tmp_path):
    src, aux = tmp_path / "protos.c", tmp_path / "protos.txt"
    src.write_text('#include "droid_b200_training.h"\n')
    subprocess.run(["gcc", "-fsyntax-only", "-I", os.path.dirname(HEADER), "-aux-info", str(aux), str(src)], check=True)
    header = {}
    for line in aux.read_text().splitlines():
        m = re.search(r"droid_b200_training\.h:\d+:\w+ \*/ extern (.*?)\s*\b(dba_\w+) \((.*)\);$", line)
        if m:
            header[m.group(2)] = (m.group(1), m.group(3).split(", "))
    assert set(header) == set(c_api.TRAINING_PROTOTYPES), set(header) ^ set(c_api.TRAINING_PROTOTYPES)
    assert not set(header) & set(c_api.PROTOTYPES)
    for name, (ret, params) in header.items():
        restype, argtypes = c_api.TRAINING_PROTOTYPES[name]
        assert _c_kind(ret) == _py_kind(restype), name
        assert [_c_kind(p) for p in params] == [_py_kind(a) for a in argtypes], name
    L = ctypes.CDLL(c_api.lib_path())
    assert all(hasattr(L, name) for name in header)
    assert c_api.load().dba_flow_loss_workspace_bytes(1, 1, 8, 8, 1) == 0          # N < 2: no call to size


def test_strict_policy_on_cpu_tensors():
    c = cases()["train_n3"]
    f = lambda t: t.float()  # noqa: E731
    args = (lt.SE3(f(c["Ps"])), f(c["disps"]), [lt.SE3(f(p)) for p in c["poses_est"]], [f(d) for d in c["disps_est"]], f(c["intrinsics"]), None)
    calls = []
    losses = types.ModuleType("losses")
    losses.flow_loss = lambda *a, **k: calls.append("flow_loss") or "reference"
    net = types.ModuleType("droid_net")
    net.upsample_disp = lambda *a, **k: calls.append("upsample_disp") or "reference"
    modules.install_flow_loss_hook(losses)
    modules.install_upsample_disp_hook(net)
    with pytest.raises(RuntimeError, match="flow_loss has no kernel for this call: Ps must be a CUDA float32"):
        losses.flow_loss(*args)
    with pytest.raises(RuntimeError, match="upsample_disp has no kernel for this call: disp must be a CUDA float32"):
        net.upsample_disp(torch.zeros(1, 2, 3, 4), torch.zeros(1, 2, 576, 3, 4))
    for _ in range(2):                                     # a second install still reaches the reference's function
        modules.install_flow_loss_hook(losses, strict=False)
        modules.install_upsample_disp_hook(net, strict=False)
    assert losses.flow_loss(*args) == "reference" and net.upsample_disp(torch.zeros(1, 2, 3, 4), None) == "reference"
    assert calls == ["flow_loss", "upsample_disp"]
