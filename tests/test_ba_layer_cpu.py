"""The dense BA layer without a GPU: the oracle (oracle/ba_layer.py) against the reference's stored outputs and gradients
(tests/golden/ba_layer.pt, fp64), the fixture against the reference itself where its sources are present, the exported C ABI, the
binding's rejections and the hook under droid_net (registry entry, strict / fallback)."""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from ba_layer_cases import cases  # noqa: E402
from oracle import ba_layer as oba  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ba_layer.pt")
REF = os.environ.get("DROID_REFERENCE_ROOT", "/root/reference")


def _golden():
    return torch.load(GOLDEN)


def test_oracle_matches_reference_fixture():
    import make_ba_layer_golden as mk
    gold = _golden()
    for name, c in cases().items():
        got = mk.run(lambda *a, **k: oba.ba(*a, **k), oba.SE3, c)
        assert len(got) == len(gold[name]), name
        for i, (u, v) in enumerate(zip(got, gold[name])):
            err = float((u - v).abs().max()) / max(float(v.abs().max()), 1e-300)
            assert err < 1e-12, (name, i, err)


def test_indefinite_case_fails_and_keeps_only_the_dz_path():
    gold = _golden()["indefinite"]
    c = cases()["indefinite"]
    # dx = 0: the poses come back as Exp(0) X
    X = oba.SE3.exp(torch.zeros(1, 7, 6, dtype=torch.float64)) * oba.SE3(c["poses"])
    assert float((gold[0] - X.data).abs().max()) < 1e-15
    # gradients still reach target, weight, eta and disps through dz = Q w
    assert all(float(g.abs().max()) > 0 for g in (gold[2], gold[3], gold[4], gold[6]))


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "droid_slam", "geom")), reason="the reference's sources are not present")
def test_fixture_reproduces_from_the_reference():
    import make_ba_layer_golden as mk
    now, gold = mk.generate(), _golden()
    for name in gold:
        for u, v in zip(now[name], gold[name]):
            assert torch.equal(u, v), name


def test_c_abi_exports_the_layer():
    from droid_slam_b200 import c_api
    names = ("dba_ba_layer_workspace_bytes", "dba_ba_layer_forward", "dba_ba_layer_backward")
    assert all(n in c_api.SYMBOLS for n in names)
    import droid_slam_b200
    lib = droid_slam_b200.capi()
    for n in names:
        assert hasattr(lib, n), n


def _inputs(dev="cpu"):
    c = cases()["train_graph"]
    return [c[k].to(dev, torch.float32) for k in ("target", "weight", "eta", "poses", "disps", "intrinsics")] + [c["ii"], c["jj"]]


def test_binding_rejects_cpu_tensors():
    import droid_slam_b200
    be = droid_slam_b200.install()
    args = _inputs()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        be.ba_layer_forward(*args, 2, 0.1, 1e-4, True)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        be.ba_layer_backward(torch.zeros(1, 7, 7), torch.zeros(1, 7, 12, 16), *args, 2, 0.1, 1e-4, torch.zeros(1, 30, 30, dtype=torch.float64),
                             torch.zeros(1, 30, dtype=torch.float64), torch.zeros(1, 7, 192, dtype=torch.float64), torch.zeros(2, dtype=torch.int32))


def _droid_net_module():
    m = types.ModuleType("fake_droid_net")
    calls = []

    def BA(*a, **k):
        calls.append((a, k))
        return oba.ba(*a, **k)

    m.BA = BA
    return m, calls


def test_hook_registry_and_strict_policy():
    from droid_slam_b200 import modules
    m, calls = _droid_net_module()
    sys.modules[m.__name__] = m
    try:
        modules.install_ba_layer_hook(m)
        e = [h for h in modules.hook_registry() if h["installer"] == "install_ba_layer_hook"][-1]
        assert (e["module"], e["kwargs"], e["transferable"]) == ("fake_droid_net", {"strict": True}, True)
        c = cases()["train_graph"]
        args = (c["target"], c["weight"], c["eta"], oba.SE3(c["poses"]), c["disps"], c["intrinsics"], c["ii"], c["jj"])
        with pytest.raises(RuntimeError, match="BA has no kernel for this call: "):
            m.BA(*args, fixedp=2)                                   # CPU fp64: no native path
        assert not calls
        modules.install_ba_layer_hook(m, strict=False)              # fallback: the reference's BA, on the CPU stand-in
        P, D = m.BA(*args, fixedp=2)
        assert len(calls) == 1
        gold = _golden()["train_graph"]
        assert float((P.data - gold[0]).abs().max()) < 1e-12 and float((D - gold[1]).abs().max()) < 1e-12
        assert [h["kwargs"] for h in modules.hook_registry() if h["installer"] == "install_ba_layer_hook"] == [{"strict": False}]
    finally:
        del sys.modules[m.__name__]
        modules._HOOKS[:] = [h for h in modules._HOOKS if h["installer"] != "install_ba_layer_hook"]


@pytest.mark.parametrize("why,edit", [
    ("poses must be SE3", lambda a, k: (a[:3] + (a[3].data,) + a[4:], k)),
    ("CUDA float32", lambda a, k: (a, k)),
    ("rig", lambda a, k: (a, dict(k, rig=2))),
    ("fixedp", lambda a, k: (a, dict(k, fixedp=7))),
])
def test_unsupported_reasons(why, edit):
    from droid_slam_b200 import modules
    c = cases()["train_graph"]
    a = (c["target"], c["weight"], c["eta"], oba.SE3(c["poses"]), c["disps"], c["intrinsics"], c["ii"], c["jj"])
    a, k = edit(a, dict(fixedp=2))
    assert why in modules._ba_layer_unsupported(*a, **k)


def test_near_plane_case_covers_both_depth_branches_and_both_crossings():
    """the near-plane case has pixels with 0.1 <= Z < 0.2 (invalid, no clamp) and Z < 0.1 (clamped to 1), and updated disparities above
    10 and below 0 before the where / clamp"""
    c = cases()["near_plane_crossings"]
    P = oba.SE3(c["poses"])
    ht, wd = c["disps"].shape[2:]
    fx, fy, cx, cy = c["intrinsics"][:, c["ii"], None, None, :].unbind(-1)
    y, x = torch.meshgrid(torch.arange(ht, dtype=torch.float64), torch.arange(wd, dtype=torch.float64), indexing="ij")
    d0 = c["disps"][:, c["ii"]]
    X0 = torch.stack([(x - cx) / fx, (y - cy) / fy, torch.ones_like(d0), d0], -1)
    Z = ((P[:, c["jj"]] * P[:, c["ii"]].inv())[:, :, None, None] * X0)[..., 2]
    assert int(((Z >= 0.1) & (Z < 0.2)).sum()) > 0 and int((Z < 0.1).sum()) > 0
    seen = {}
    where = torch.where

    def spy(cond, a, b):
        seen["pre"] = b
        return where(cond, a, b)

    torch.where = spy
    try:
        oba.ba(c["target"], c["weight"], c["eta"], P, c["disps"], c["intrinsics"], c["ii"], c["jj"], fixedp=c["fixedp"])
    finally:
        torch.where = where
    assert int((seen["pre"] > 10).sum()) > 0 and int((seen["pre"] < 0).sum()) > 0
