"""Training's flow loss and upsample_disp on the device (csrc/geom.cu through droid_slam_b200.modules.flow_loss / upsample_disp): the
loss and every gradient against autograd through the fp64 oracle (oracle/flow_loss.py, oracle/upsample.py), bounded by twice the
oracle's own fp32 execution error on the same inputs with a floor; the metric counts; bit-reproducibility; host synchronisations; the
upsample forward bit-identical to cvx_upsample; the strict policy."""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from droid_slam_b200 import install, modules  # noqa: E402
from droid_slam_b200 import lietorch as lt  # noqa: E402
from flow_loss_cases import cases, make_case, upsample_case, upsample_cases  # noqa: E402
from oracle import upsample as oup  # noqa: E402
from test_flow_loss_cpu import oracle_flow  # noqa: E402
from util import host_syncs  # noqa: E402

pytestmark = pytest.mark.gpu

FLOOR = 2e-5          # relative to the largest magnitude of each compared tensor


def gpu_cases():
    out = dict(cases())
    out["b1_N7_n15_384x512"] = make_case(B=1, N=7, ht=384, wd=512, n=15, seed=21)
    out["b2_N15_n15_37x53"] = make_case(B=2, N=15, ht=37, wd=53, n=15, seed=22)       # 1961 pixels: not a multiple of 256
    out["b2_N2_n1_48x64"] = make_case(B=2, N=2, ht=48, wd=64, n=1, seed=23)
    nan = make_case(N=7, n=2, ht=24, wd=32, seed=24)
    nan["disps_est"][1][0, 3, 5, 7] = float("nan")
    out["nan_disparity"] = nan
    none = make_case(N=3, n=2, seed=25)
    none["disps"].zero_()                                        # val0 = 0 everywhere: no valid pixel
    out["no_valid_pixel"] = none
    return out


def run_native(c, dev="cuda"):
    f = lambda t: t.to(dev, torch.float32)  # noqa: E731
    pe = [f(p).requires_grad_(True) for p in c["poses_est"]]
    de = [f(d).requires_grad_(True) for d in c["disps_est"]]
    loss, metrics = modules.flow_loss(lt.SE3(f(c["Ps"])), f(c["disps"]), [lt.SE3(p) for p in pe], de, f(c["intrinsics"]), None)
    g = torch.autograd.grad(loss, de + pe)
    n = len(pe)
    return dict(loss=loss.detach(), metrics=metrics, grad_disps_est=list(g[:n]), grad_poses_est=list(g[n:]))


def rel(a, b):
    """max |a - b| / max |b| over b's finite entries; a must be NaN exactly where b is"""
    a, b = a.double(), b.double()
    nan = torch.isnan(b)
    assert torch.equal(torch.isnan(a), nan), "NaN in different places"
    if not bool((~nan).any()):
        return 0.0
    return float((a[~nan] - b[~nan]).abs().max()) / max(float(b[~nan].abs().max()), 1e-30)


def rel2(a, b):
    """|a - b| / |b| (2-norms) over b's finite entries; a must be NaN exactly where b is"""
    a, b = a.double(), b.double()
    nan = torch.isnan(b)
    assert torch.equal(torch.isnan(a), nan), "NaN in different places"
    return float((a[~nan] - b[~nan]).norm()) / max(float(b[~nan].norm()), 1e-30)


def check_against_oracle(c, what):
    """the loss and the pose gradients (sums over pixels) by their largest error; the disparity gradients as vectors, by the 2-norm:
    at a pixel where c1 is close to c0 the gradient's direction is (c1 - c0) / |c1 - c0|, which both fp32 executions round differently,
    so the largest single-pixel error of each is a different draw from the same tail"""
    nat = run_native(c)
    o64, o32 = oracle_flow(c, torch.float64, "cuda"), oracle_flow(c, torch.float32, "cuda")
    report = []
    pairs = [("loss", nat["loss"], o64["loss"], o32["loss"])]
    for k in ("grad_disps_est", "grad_poses_est"):
        pairs += [("%s[%d]" % (k, i), a, b, d) for i, (a, b, d) in enumerate(zip(nat[k], o64[k], o32[k]))]
    for label, a, b, d in pairs:
        err = rel2 if label.startswith("grad_disps_est") else rel
        e, e32 = err(a, b), err(d, b)
        report.append((label, e, e32))
        assert e <= max(2 * e32, FLOOR), (what, label, e, e32)
    print(what, ["%s %.2e (fp32 oracle %.2e)" % r for r in report[:4]])
    return nat, o64


@pytest.mark.parametrize("name", sorted(gpu_cases()))
def test_loss_and_gradients_against_oracle(name):
    check_against_oracle(gpu_cases()[name], name)


@pytest.mark.parametrize("name", ["train_n3", "b2_N15_n15_37x53", "b1_N7_n15_384x512", "no_valid_pixel", "thresholds"])
def test_metric_counts(name):
    """the count of v > 0.5 equal to fp64's (no case has a Z within fp32 rounding of 0.2); the count with epe < 1 equal up to the
    pixels whose fp64 epe is within 1e-3 of 1; f_error and 1px NaN exactly when no pixel is valid"""
    c = gpu_cases()[name]
    f = lambda t: t.cuda().float()  # noqa: E731
    s, count, below = install().flow_loss_forward(f(c["Ps"]), f(c["disps"]), [f(p) for p in c["poses_est"]],
                                                   [f(d) for d in c["disps_est"]], f(c["intrinsics"]), 0.9)[1].tolist()
    from oracle import ba_layer as oba, flow_loss as ofl
    d = lambda t: t.cuda().double()  # noqa: E731
    _, epe, v = ofl.flow_loss(oba.SE3(d(c["Ps"])), d(c["disps"]), [oba.SE3(d(p)) for p in c["poses_est"]], [d(x) for x in c["disps_est"]],
                              d(c["intrinsics"]))
    valid = v > 0.5
    assert count == int(valid.sum()), (count, int(valid.sum()))
    near = int((valid & ((epe - 1).abs() < 1e-3)).sum())
    assert abs(below - int((valid & (epe < 1)).sum())) <= near
    m = run_native(c)["metrics"]
    if count == 0:
        assert m["f_error"] != m["f_error"] and m["1px"] != m["1px"]
    else:
        assert abs(m["f_error"] - float(epe[valid].mean())) <= 1e-4 * max(1.0, float(epe[valid].mean()))


def test_reproducible_bits():
    c = gpu_cases()["b2_N15_n15_37x53"]
    a, b = run_native(c), run_native(c)
    assert torch.equal(a["loss"], b["loss"]) and a["metrics"] == b["metrics"]
    for k in ("grad_disps_est", "grad_poses_est"):
        for x, y in zip(a[k], b[k]):
            assert torch.equal(x, y), k


def test_one_host_read_forward_none_backward():
    c = make_case(B=1, N=7, ht=96, wd=128, n=15, seed=26)
    f = lambda t: t.cuda().float()  # noqa: E731
    pe = [f(p).requires_grad_(True) for p in c["poses_est"]]
    de = [f(x).requires_grad_(True) for x in c["disps_est"]]
    args = lambda: (lt.SE3(f(c["Ps"])), f(c["disps"]), [lt.SE3(p) for p in pe], de, f(c["intrinsics"]), None)  # noqa: E731
    loss, _ = modules.flow_loss(*args())                        # warm up: the extension and allocator
    torch.autograd.grad(loss, de + pe)
    a = args()
    n_fwd, (loss, _) = host_syncs(lambda: modules.flow_loss(*a))
    n_bwd, _ = host_syncs(lambda: torch.autograd.grad(loss, de + pe))
    assert (n_fwd, n_bwd) == (1, 0), (n_fwd, n_bwd)


# ---- upsample_disp ----------------------------------------------------------------------------------------------------------------

def up_native(c, dtype=torch.float32):
    disp = c["disp"].cuda().to(dtype).requires_grad_(True)
    mask = c["mask"].cuda().to(dtype).requires_grad_(True)
    out = modules.upsample_disp(disp, mask)
    gd, gm = torch.autograd.grad(out, [disp, mask], c["cot"].cuda().to(dtype))
    return out.detach(), gd, gm


def up_oracle(c, dtype):
    disp = c["disp"].cuda().to(dtype).requires_grad_(True)
    mask = c["mask"].cuda().to(dtype).requires_grad_(True)
    out = oup.upsample_disp(disp, mask)
    gd, gm = torch.autograd.grad(out, [disp, mask], c["cot"].cuda().to(dtype))
    return out.detach(), gd, gm


def up_cases():
    out = dict(upsample_cases())
    out["train_7x48x64"] = upsample_case(B=1, N=7, ht=48, wd=64, seed=31)
    out["odd_2x3x13x17"] = upsample_case(B=2, N=3, ht=13, wd=17, seed=32)
    return out


@pytest.mark.parametrize("name", sorted(up_cases()))
def test_upsample_disp_against_oracle(name):
    c = up_cases()[name]
    nat, o64, o32 = up_native(c), up_oracle(c, torch.float64), up_oracle(c, torch.float32)
    for label, a, b, d in zip(("out", "grad_disp", "grad_mask"), nat, o64, o32):
        e, e32 = rel(a, b), rel(d, b)
        assert e <= max(2 * e32, FLOOR), (name, label, e, e32)
    B, N, ht, wd = c["disp"].shape
    fwd = install().cvx_upsample(c["disp"].cuda().float().reshape(B * N, ht, wd), c["mask"].cuda().float().reshape(B * N, 576, ht, wd))
    assert torch.equal(nat[0], fwd.view(B, N, 8 * ht, 8 * wd))
    again = up_native(c)
    assert all(torch.equal(x, y) for x, y in zip(nat, again))


def test_upsample_masked_taps():
    """a -inf tap has weight 0 and gradient 0; an all -inf pixel gives NaN, as torch.softmax does"""
    c = upsample_case(ht=3, wd=4, seed=33)
    c["mask"].view(1, 1, 9, 64, 3, 4)[:, :, 2, :, 1, 1] = float("-inf")
    c["mask"].view(1, 1, 9, 64, 3, 4)[:, :, :, 5, 2, 3] = float("-inf")
    nat, o32 = up_native(c), up_oracle(c, torch.float32)
    for a, b in zip(nat, o32):
        assert torch.equal(torch.isnan(a), torch.isnan(b))
    assert bool((nat[2].view(1, 1, 9, 64, 3, 4)[:, :, 2, :, 1, 1] == 0).all())


def test_upmask_gradient_through_upsample_and_flow_loss():
    """the path by which the update operator's upmask learns: flow_loss(upsample_disp(disps, upmask)) per iterate, the mask and
    coarse-disparity gradients through both native functions against the fp64 oracle's, within twice the fp32 oracle's error"""
    B, N, h, w, n = 1, 4, 6, 8, 3
    c = make_case(B=B, N=N, ht=8 * h, wd=8 * w, n=n, seed=34)
    g = torch.Generator().manual_seed(35)
    coarse = [c["disps_est"][i][..., 3::8, 3::8].clone() for i in range(n)]
    masks = [torch.randn(B, N, 576, h, w, generator=g, dtype=torch.float64) for _ in range(n)]

    def run(dtype, native):
        to = lambda t: t.cuda().to(dtype)  # noqa: E731
        m = [to(x).requires_grad_(True) for x in masks]
        d = [to(x).requires_grad_(True) for x in coarse]
        up = modules.upsample_disp if native else oup.upsample_disp
        de = [up(di, mi) for di, mi in zip(d, m)]
        if native:
            loss, _ = modules.flow_loss(lt.SE3(to(c["Ps"])), to(c["disps"]), [lt.SE3(to(p)) for p in c["poses_est"]], de, to(c["intrinsics"]))
        else:
            from oracle import ba_layer as oba, flow_loss as ofl
            loss = ofl.flow_loss(oba.SE3(to(c["Ps"])), to(c["disps"]), [oba.SE3(to(p)) for p in c["poses_est"]], de, to(c["intrinsics"]))[0]
        return torch.autograd.grad(loss, m + d)

    nat, o64, o32 = run(torch.float32, True), run(torch.float64, False), run(torch.float32, False)
    for a, b, d in zip(nat, o64, o32):
        e, e32 = rel(a, b), rel(d, b)
        assert e <= max(2 * e32, FLOOR), (e, e32)


# ---- the strict policy ------------------------------------------------------------------------------------------------------------

def test_strict_policy_every_reason():
    c = make_case(N=3, n=2, seed=36)
    f = lambda t: t.cuda().float()  # noqa: E731
    good = dict(Ps=lt.SE3(f(c["Ps"])), disps=f(c["disps"]), poses_est=[lt.SE3(f(p)) for p in c["poses_est"]],
                disps_est=[f(d) for d in c["disps_est"]], intrinsics=f(c["intrinsics"]), graph=None)
    one = make_case(N=1, n=1, seed=37)
    bad = {
        "Ps must be an SE3": dict(Ps=f(c["Ps"])),
        "poses_est\\[1\\] must be an SE3": dict(poses_est=[good["poses_est"][0], f(c["poses_est"][1])]),
        "disps_est\\[0\\] must be a CUDA float32": dict(disps_est=[good["disps_est"][0].double(), good["disps_est"][1]]),
        "intrinsics must be a CUDA float32": dict(intrinsics=good["intrinsics"].cpu()),
        "disps_est\\[1\\] has shape": dict(disps_est=[good["disps_est"][0], good["disps_est"][1][..., :-1]]),
        "N = 1": dict(Ps=lt.SE3(f(one["Ps"])), disps=f(one["disps"]), poses_est=[lt.SE3(f(one["poses_est"][0]))],
                      disps_est=[f(one["disps_est"][0])], intrinsics=f(one["intrinsics"])),
        "0 pose and 0 disparity iterates": dict(poses_est=[], disps_est=[]),
        "disps requires grad": dict(disps=good["disps"].clone().requires_grad_(True)),
    }
    calls = []
    losses = types.ModuleType("losses")
    losses.flow_loss = lambda *a, **k: calls.append(1) or "reference"
    modules.install_flow_loss_hook(losses)
    for why, change in bad.items():
        with pytest.raises(RuntimeError, match="flow_loss has no kernel for this call: " + why):
            losses.flow_loss(**{**good, **change})
    for _ in range(2):
        modules.install_flow_loss_hook(losses, strict=False)
    for why, change in bad.items():
        assert losses.flow_loss(**{**good, **change}) == "reference", why
    assert len(calls) == len(bad)
    net = types.ModuleType("droid_net")
    net.upsample_disp = lambda *a, **k: "reference"
    modules.install_upsample_disp_hook(net)
    u = upsample_case(seed=38)
    disp, mask = u["disp"].cuda().float(), u["mask"].cuda()
    with pytest.raises(RuntimeError, match="upsample_disp has no kernel for this call: mask must be a CUDA float32"):
        net.upsample_disp(disp, mask.half())
    with pytest.raises(RuntimeError, match="upsample_disp has no kernel for this call: mask must be a CUDA float32"):
        net.upsample_disp(disp, mask.float()[:, :, :575])
    for _ in range(2):
        modules.install_upsample_disp_hook(net, strict=False)
    assert net.upsample_disp(disp, mask.half()) == "reference"
    assert modules.install_upsample_disp_hook(net).upsample_disp(disp, mask.float()).shape == (1, 1, 40, 48)
