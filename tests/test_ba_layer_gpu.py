"""The dense BA layer on the device (csrc/ba_layer.cu through droid_slam_b200.modules.ba_layer): outputs and every input gradient against
autograd through the fp64 oracle (oracle/ba_layer.py), bounded by twice the oracle's own fp32 execution error on the same inputs with a
floor; the Cholesky-failure semantics; bit-reproducibility and batch independence; host synchronisations; the status word."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from droid_slam_b200 import install, modules  # noqa: E402
from droid_slam_b200 import lietorch as lt  # noqa: E402
from oracle import ba_layer as oba  # noqa: E402
from ba_layer_cases import cases, loss_weights, make_inputs, radius_graph  # noqa: E402
from util import host_syncs  # noqa: E402

pytestmark = pytest.mark.gpu

FLOOR = 2e-5          # relative to the largest magnitude of each compared tensor
NAMES = ("target", "weight", "eta", "poses", "disps")


def run_native(c, dev="cuda"):
    """outputs (poses' of every call, disps' of every call) and the gradients of NAMES, fp32 on the device"""
    B, N, ht, wd = c["disps"].shape
    a, b = loss_weights(B, N, ht, wd)
    x = {k: c[k].to(dev, torch.float32).requires_grad_(k in NAMES) for k in NAMES + ("intrinsics",)}
    x["intrinsics"].requires_grad_(False)
    ii, jj = c["ii"].to(dev), c["jj"].to(dev)
    poses, disps, outs, loss = lt.SE3(x["poses"]), x["disps"], [], 0.0
    for _ in range(c["chain"]):
        poses, disps = modules.ba_layer(x["target"], x["weight"], x["eta"], poses, disps, x["intrinsics"], ii, jj, fixedp=c["fixedp"])
        outs.append((poses.data.detach(), disps.detach()))
        loss = loss + (a[..., :6].to(dev, torch.float32) * poses.log()).sum() + (b.to(dev, torch.float32) * disps).sum()
    grads = torch.autograd.grad(loss, [x[k] for k in NAMES])
    return outs, dict(zip(NAMES, grads))


def run_oracle(c, dtype, dev="cuda"):
    """the same through the oracle; the pose gradient as lietorch's left-tangent gradient (poses = Exp(eps) X, d/d eps)"""
    B, N, ht, wd = c["disps"].shape
    a, b = loss_weights(B, N, ht, wd)
    x = {k: c[k].to(dev, dtype).requires_grad_(k in NAMES and k != "poses") for k in NAMES + ("intrinsics",)}
    eps = torch.zeros(B, N, 6, dtype=dtype, device=dev, requires_grad=True)
    poses, disps, outs, loss = oba.SE3(oba.left_perturbed(x["poses"], eps)), x["disps"], [], 0.0
    ii, jj = c["ii"].to(dev), c["jj"].to(dev)
    for _ in range(c["chain"]):
        poses, disps = oba.ba(x["target"], x["weight"], x["eta"], poses, disps, x["intrinsics"], ii, jj, fixedp=c["fixedp"])
        outs.append((poses.data.detach(), disps.detach()))
        loss = loss + (a[..., :6].to(dev, dtype) * poses.log()).sum() + (b.to(dev, dtype) * disps).sum()
    grads = torch.autograd.grad(loss, [x[k] if k != "poses" else eps for k in NAMES])
    g = dict(zip(NAMES, grads))
    g["poses"] = torch.cat([g["poses"], torch.zeros_like(g["poses"][..., :1])], -1)
    return outs, g


def rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(float(b.double().abs().max()), 1e-30)


def check_against_oracle(c, what):
    nat_out, nat_g = run_native(c)
    o64_out, o64_g = run_oracle(c, torch.float64)
    o32_out, o32_g = run_oracle(c, torch.float32)
    report = []
    for k in range(c["chain"]):
        for t, label in ((0, "poses'"), (1, "disps'")):
            e, e32 = rel(nat_out[k][t], o64_out[k][t]), rel(o32_out[k][t], o64_out[k][t])
            report.append((label, k, e, e32))
            assert e <= max(2 * e32, FLOOR), (what, label, k, e, e32)
    for n in NAMES:
        e, e32 = rel(nat_g[n], o64_g[n]), rel(o32_g[n], o64_g[n])
        report.append(("grad " + n, e, e32))
        assert e <= max(2 * e32, FLOOR), (what, n, e, e32)
    print(what, ["%s %.2e (fp32 oracle %.2e)" % (r[0] + (" #%d" % r[1] if len(r) == 4 else ""), r[-2], r[-1]) for r in report])
    return report


@pytest.mark.parametrize("name", sorted(cases()))
def test_fixture_cases_against_oracle(name):
    check_against_oracle(cases()[name], name)


def test_training_shape_against_oracle():
    ii, jj = radius_graph(7)
    check_against_oracle(make_inputs(ii, jj, 7, ht=48, wd=64, seed=21), "48x64")


def test_cholesky_failure_zeroes_dx_for_the_batch():
    c = cases()["indefinite"]
    c2 = make_inputs(c["ii"], c["jj"], 7, B=2, seed=31)
    c2["weight"][0] = c2["weight"][0] - 0.9                # element 0 indefinite, element 1 not
    x = {k: c2[k].cuda().float() for k in NAMES + ("intrinsics",)}
    P, _ = modules.ba_layer(x["target"], x["weight"], x["eta"], lt.SE3(x["poses"]), x["disps"], x["intrinsics"], c2["ii"].cuda(),
                            c2["jj"].cuda(), fixedp=2)
    ref = lt.SE3.exp(torch.zeros(2, 7, 6, device="cuda")) * lt.SE3(x["poses"])
    assert torch.equal(P.data, ref.data), "a failed factor must leave every pose of the batch at Exp(0) X"
    # gradient only through dz = Q w: none reaches target / weight through dx, and the oracle agrees
    check_against_oracle(c2, "indefinite_batch")


def test_reproducible_and_batch_independent():
    c = cases()["batch2"]
    o1, g1 = run_native(c)
    o2, g2 = run_native(c)
    for k in range(2):
        assert torch.equal(o1[0][k], o2[0][k])
    for n in NAMES:
        assert torch.equal(g1[n], g2[n]), n
    x = {k: c[k].cuda().float() for k in NAMES + ("intrinsics",)}
    ii, jj = c["ii"].cuda(), c["jj"].cuda()
    full = modules.ba_layer(x["target"], x["weight"], x["eta"], lt.SE3(x["poses"]), x["disps"], x["intrinsics"], ii, jj, fixedp=2)
    for b in range(2):
        one = modules.ba_layer(*(x[k][b:b + 1] for k in ("target", "weight", "eta")), lt.SE3(x["poses"][b:b + 1]), x["disps"][b:b + 1],
                               x["intrinsics"][b:b + 1], ii, jj, fixedp=2)
        assert torch.equal(full[0].data[b:b + 1], one[0].data) and torch.equal(full[1][b:b + 1], one[1])
    # and so are its gradients, for the same upstream gradient
    g = torch.Generator().manual_seed(3)
    gp = torch.randn(2, 7, 7, generator=g).cuda()
    gp[..., 6] = 0
    gd = torch.randn(2, 7, 12, 16, generator=g).cuda()

    def grads(sl):
        xs = {k: x[k][sl].detach().clone().requires_grad_(k != "intrinsics") for k in x}
        P, D = modules.ba_layer(xs["target"], xs["weight"], xs["eta"], lt.SE3(xs["poses"]), xs["disps"], xs["intrinsics"], ii, jj, fixedp=2)
        return torch.autograd.grad([P.data, D], [xs[k] for k in NAMES], [gp[sl], gd[sl]])

    gfull = grads(slice(0, 2))
    for b in range(2):
        for n, u, v in zip(NAMES, gfull, grads(slice(b, b + 1))):
            assert torch.equal(u[b:b + 1], v), (n, b)


def test_no_host_syncs():
    c = cases()["train_graph"]
    x = {k: c[k].cuda().float().requires_grad_(k in NAMES) for k in NAMES + ("intrinsics",)}
    x["intrinsics"].requires_grad_(False)
    ii, jj = c["ii"].cuda(), c["jj"].cuda()
    args = lambda: (x["target"], x["weight"], x["eta"], lt.SE3(x["poses"]), x["disps"], x["intrinsics"], ii, jj)  # noqa: E731
    out = modules.ba_layer(*args(), fixedp=2)                       # warm up: the extension and allocator
    torch.autograd.grad(out[1].sum() + out[0].data.sum(), [x["disps"]])
    n_fwd, out = host_syncs(lambda: modules.ba_layer(*args(), fixedp=2))
    gd, gp = torch.ones_like(out[1]), torch.ones_like(out[0].data)
    n_bwd, _ = host_syncs(lambda: torch.autograd.grad([out[1], out[0].data], [x["disps"], x["weight"]], [gd, gp]))
    assert (n_fwd, n_bwd) == (0, 0), (n_fwd, n_bwd)


def test_status_word_raises_on_out_of_range_index():
    be = install()
    c = cases()["train_graph"]
    x = {k: c[k].cuda().float() for k in NAMES + ("intrinsics",)}
    keep = {k: v.clone() for k, v in x.items()}
    ii = c["ii"].cuda().clone()
    ii[3] = 9
    with pytest.raises(IndexError):
        be.ba_layer_forward(x["target"], x["weight"], x["eta"], x["poses"], x["disps"], x["intrinsics"], ii, c["jj"].cuda(), 2, 0.1, 1e-4, True)
    for k in x:
        assert torch.equal(x[k], keep[k]), k
