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

from ba_layer_cases import cases, domain_cases  # noqa: E402
from oracle import ba_layer as oba  # noqa: E402
import reference  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ba_layer.pt")


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


@pytest.mark.skipif(not reference.present("droid_slam", "geom"), reason="the reference's sources are not present")
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


def _assert_near_plane_bands(c):
    """pixels with 0.1 <= Z < 0.2 (invalid, no clamp) and Z < 0.1 (clamped to 1), and updated disparities above 10 and below 0 before
    the where / clamp"""
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


def test_near_plane_case_covers_both_depth_branches_and_both_crossings():
    """the near-plane case has pixels with 0.1 <= Z < 0.2 (invalid, no clamp) and Z < 0.1 (clamped to 1), and updated disparities above
    10 and below 0 before the where / clamp"""
    _assert_near_plane_bands(cases()["near_plane_crossings"])


def _facts(c):
    B, N, ht, wd = c["disps"].shape
    ii, jj = c["ii"], c["jj"]
    P = N - c["fixedp"]
    n = 6 * P
    src = torch.unique(ii)
    pairs = list(zip(ii.tolist(), jj.tolist()))
    return dict(B=B, N=N, HW=ht * wd, P=P, n=n, E=len(pairs), outdeg=torch.bincount(ii, minlength=N),
                src=src.tolist(), dup=len(pairs) - len(set(pairs)), self_edges=int((ii == jj).sum()))


def test_domain_cases_reach_their_corners():
    """each of domain_cases() reaches the corner of the layer's domain it is named for"""
    d = {name: _facts(c) for name, c in domain_cases().items()}
    for name in ("p20_48x64", "p20_60x80_chain4", "near_plane_p20"):
        f = d[name]
        # bal_factor_kernel at its largest: n = 120, P^2 = 400 blocks over 256 threads (the shared memory it launches with is read
        # from the launch itself, tests/test_ba_layer_domain_gpu.py test_p20_factor_and_lambda_x_launch_with_the_full_system)
        assert (f["P"], f["n"]) == (20, 120) and f["P"] ** 2 > 256, name
    assert d["p20_48x64"]["HW"] == 48 * 64 and 85 <= d["p20_48x64"]["E"] <= 95
    f = d["p20_60x80_chain4"]
    assert f["HW"] % 128 == 64 and domain_cases()["p20_60x80_chain4"]["chain"] == 4
    assert int(f["outdeg"].max()) >= 5 and int((f["outdeg"] == 0).sum()) > 0
    assert (d["fixedp0"]["P"], d["fixedp0"]["N"]) == (6, 6)
    f = d["p1"]
    assert f["P"] == 1 and sum(1 for s in f["src"] if s < 6) >= 5          # one pose unknown; the other sources are fixed frames
    f, c = d["many_fixed_gaps"], domain_cases()["many_fixed_gaps"]
    assert f["N"] > 64 and f["P"] == 15 and max(f["src"]) >= 64
    assert f["src"] != list(range(f["src"][0], f["src"][0] + len(f["src"])))  # the ii -> k map has gaps above its first source
    assert len([s for s in range(40, 70) if s not in f["src"]]) >= 5 and int((c["jj"] < 55).sum()) > 0
    touched = set(c["ii"].tolist()) | set(c["jj"].tolist())
    assert all(s in touched for s in range(55, 70))                           # every pose unknown is on some edge
    f = d["train24_batch4"]
    assert (f["B"], f["E"], f["P"]) == (4, 24, 5) and int(f["outdeg"].max()) >= 5 and int((f["outdeg"] == 0).sum()) > 0
    f = d["hub_duplicates"]
    assert f["B"] == 2 and int(f["outdeg"].max()) == 12 and f["dup"] >= 2 and f["self_edges"] == 1
    assert d["tiny_3x5"]["HW"] == 15 < 32
    # the chained case keeps every disparity off the clamp at 0 (fp64, all 4 calls), by far more than D's fp32 error (~1e-6 of 2)
    c = domain_cases()["p20_60x80_chain4"]
    P, D = oba.SE3(c["poses"]), c["disps"]
    for _ in range(c["chain"]):
        P, D = oba.ba(c["target"], c["weight"], c["eta"], P, D, c["intrinsics"], c["ii"], c["jj"], fixedp=c["fixedp"])
        assert float(D.min()) > 0.05


def test_batch4_third_fails_fails_in_element_2_only():
    c = domain_cases()["batch4_third_fails"]
    S = oba.ba_system(c["target"], c["weight"], c["eta"], oba.SE3(c["poses"]), c["disps"], c["intrinsics"], c["ii"], c["jj"],
                      fixedp=c["fixedp"])["S"]
    assert (torch.linalg.cholesky_ex(S)[1] != 0).tolist() == [False, False, True, False]


def test_near_plane_p20_covers_both_depth_branches_and_both_crossings():
    _assert_near_plane_bands(domain_cases()["near_plane_p20"])


def test_ba_system_returns_the_reduced_system_of_ba():
    """ba() is ba_system()'s poses / disps, and dx solves S dx = y"""
    c = domain_cases()["fixedp0"]
    args = (c["target"], c["weight"], c["eta"], oba.SE3(c["poses"]), c["disps"], c["intrinsics"], c["ii"], c["jj"])
    r = oba.ba_system(*args, fixedp=0, ep=1e-2, lm=1e-3)
    P, D = oba.ba(*args, fixedp=0, ep=1e-2, lm=1e-3)
    assert torch.equal(P.data, r["poses"].data) and torch.equal(D, r["disps"])
    assert float((r["S"] @ r["dx"][..., None] - r["y"][..., None]).abs().max()) < 1e-10 * float(r["y"].abs().max())
