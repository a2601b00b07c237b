"""Training's flow loss and upsample_disp's backward (csrc/geom.cu) through the C ABI, element by element against fp64 under the running
error model of flow_loss_model, at the stage cases of flow_loss_cases (their corners and the model's fp64 values checked on the host
in tests/test_flow_loss_stages_cpu.py).

Buffers.  Every output lies in a NaN-filled fp32 buffer with GUARD floats of NaN on each side, the flow workspace is exactly
dba_flow_loss_workspace_bytes of 0xFF bytes and the tap partials exactly n 9 8 ht wd NaN floats, each between guards; the guards must
come back untouched, no NaN may remain where fp64 is finite, and the 7th entry of every pose gradient is +0.
Values.  kappa = |native - fp64| / bound <= 1 for the loss, the metric sum, every disparity-gradient pixel, every pose-gradient
component, every mask-gradient element and every coarse disparity gradient; where the bound is 0 the value must be exact, where fp64
is NaN or inf the native value must be the same.  The fp64 truth is computed on the card, iterate by iterate.  The metric counts are
exact up to the ambiguous decisions.  Up to 64x64 the native values are also held to the model's bound around autograd through the
fp64 oracles (oracle/flow_loss.py, oracle/upsample.py), a yardstick that does not share the model's closed form.
Hooks.  modules.flow_loss under an upstream gradient of 0.05 and modules.upsample_disp under a stride-0 and a misaligned grad_out give
the C ABI's bits; both give the same bits on a side stream.  upsample_disp -> flow_loss at training size is checked element by
element, the flow gradient's bound carried into the upsample backward as the cotangent's error.

Worst kappa per case and quantity on one NVIDIA H100 80GB HBM3 at a 700 W power limit (card and limit read in the same run); in
brackets the ambiguous decisions / all decisions of the case.  The whole file took 46 s there.
  case                       loss      metric_sum  grad_disps  grad_poses
  N2_B1_n1_1x1               0.00683   0.00454     0.00133     0.00139   [0 / 8]
  N3_B2_n3_1x300             0.000736  0.00469     0.0518      0.00402   [0 / 19200]
  N7_B4_n1_300x1             0.000546  0.000715    0.191       0.027     [0 / 57600]
  N33_B1_n3_hw255            0.000382  0.000362    0.0356      0.00772   [0 / 130560]
  N2_B2_n15_hw256            0.000958  0.00393     0.0419      0.00494   [0 / 32768]
  N3_B1_n3_hw257             0.000108  0.0024      0.0327      0.00231   [0 / 8224]
  N7_B1_n3_hw513             0.000374  0.00253     0.0675      0.00503   [0 / 49248]
  N7_B2_n3_37x53             0.00133   1.76e-06    0.0409      0.00496   [0 / 376512]
  N3_B4_n3_13x11             1.79e-05  0.00353     0.0463      0.00516   [0 / 18304]
  train_N7_B1_n15_384x512    0.00035   0.0035      0.0962      0.00734   [1894 / 75497472]
  placed_thresholds          0.00892   0.0257      0.0734      0.0108    [0 / 1152]
  exact_equal                0.00024   0.000151    0.0304      0.00317   [0 / 11520]
  zero_translation           0.000548  0.00249     0 (exact)   0.00219   [0 / 6912]
  no_valid_rows              0.00187   0.000943    0.0214      0.00788   [0 / 4608]
  nonfinite_iterate          NaN       0           0.0258      0.00369   [0 / 9216]
  nonfinite_ground_truth     NaN       0           0.0343      NaN       [0 / 6912]
  gamma0.5_grad0.05          0.00252   0.000408    0.0492      0.00848   [0 / 7488]
  gamma1_grad-2.5            0.000903  0.0013      0.0518      0.0119    [0 / 7488]
  gamma0_grad1               0.00193   0.00176     0.0362      0.00345   [0 / 7488]
  gamma0.9_grad0             0.00159   0.00305     0 (exact)   0 (exact) [0 / 7488]
  quaternions_scaled         0.0014    0.00184     0.0324      0.00459   [0 / 19712]
  upsample (grad_disps / grad_mask): up_1x1 0.0195 / 0.296, up_1x9 0.0231 / 0.357, up_7x1 0.0359 / 0.39, up_13x17 0.0417 / 0.406,
  up_43x70 0.0657 / 0.492, up_44x69 0.072 / 0.487, up_train_7x48x64 0.0761 / 0.486, up_sigma20 0.058 / 0.95, up_tied 0.0258 / 0.129,
  up_dominant 0.0204 / 0.549, up_neginf 0.0494 / 0.437, up_underflow 0.024 / 0.862, up_nan_inf 0.0306 / 0.343, up_nan_cot 0.0328 / 0.422
  upsample_disp -> flow_loss at 7 x 48x64 -> 384x512: grad_mask 0.0436, grad_coarse 0.00765
(NaN: the value is NaN where fp64's is, so no finite entry is left to measure.)  The flow bounds are first-order worst cases over
hundreds of roundings per pixel, so the flow kappas stay far below 1; the mask gradient's reach 0.95.

Single edits of geom.cu, each built on a scratch copy and run against tests/test_flow_loss_gpu.py and this file:
  edit                                                        test_flow_loss_gpu   this file
  no disparity gradient written for the last pixel of a frame fails                fails (NaN left in the output)
  second out-edge dropped from the disparity in the last chunk fails                fails
  gather's right-border test sx > wd                          fails                fails (up_1x1)
  no quaternion normalisation in flow_edges_kernel            passes               fails (quaternions_scaled)
  source-edge adjT applied with slot 0's Gij                  fails                fails
  upstream gradient read as 1                                 passes               fails (gamma0.5_grad0.05, kappa 3.5e5)
  gamma fixed at 0.9 in the backward                          passes               fails (gamma0.5_grad0.05, kappa 4.1e4)
  softmax weights below 1e-6 flushed to 0 in the backward     passes               fails (up_13x17, kappa 1.3e6)
  __expf instead of expf in the backward                      passes               fails (up_train_7x48x64, kappa 1.01)
The older file's 2-norm of the disparity gradients has a floor of 2e-5, so it did notice the first two edits at 384x512 (2.7e-3 for
the unwritten last pixels, which hold whatever the allocator left there, and 3.3e-2 for the dropped edge).  What it did not see are
arguments other than the defaults, non-unit quaternions and entries far below the largest of their tensor.  No edit read or wrote
outside its guarded allocations, and none faulted.
"""
import json
import os

import pytest
import torch

from droid_slam_b200 import c_api, modules
from droid_slam_b200 import lietorch as lt
import flow_loss_cases as fc
import flow_loss_model as fm
import geometry_model as gm
from test_geometry_stages_gpu import kappa as _kappa, same_bits
from test_tensor_core_fp64_gpu import Guarded
from util import ptr, stream

pytestmark = pytest.mark.gpu
dev = "cuda"
AMBIGUOUS_ALLOWANCE = 4
ORACLE_MAX_HW = 64 * 64
WS_GUARD = 256                       # bytes of 0xFF before and after the workspace


def kappa(got, r, what):
    """geometry's kappa with the fp64 truth brought to the host"""
    return _kappa(got, gm.R(r.v.cpu(), r.b.cpu()), what)


def _report(case, stats):
    print("FLOW_STAGES %s %s" % (case, json.dumps(stats)))
    out = os.environ.get("FLOW_STAGES_REPORT")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(dict(case=case, **stats)) + "\n")


def _ptrs(ts):
    return torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device=dev)


class Workspace:
    """exactly `nbytes` of 0xFF between WS_GUARD guard bytes of 0xFF"""

    def __init__(self, nbytes):
        self.buf = torch.full((nbytes + 2 * WS_GUARD,), 255, dtype=torch.uint8, device=dev)
        self.t = self.buf[WS_GUARD:WS_GUARD + nbytes]
        self.n = nbytes

    def check_guards(self, what):
        assert bool((self.buf[:WS_GUARD] == 255).all()) and bool((self.buf[WS_GUARD + self.n:] == 255).all()), "%s wrote outside its workspace" % what


def to_dev(c):
    f = lambda t: t.to(dev, torch.float32).contiguous()  # noqa: E731
    return dict(Ps=f(c["Ps"]), disps=f(c["disps"]), intr=f(c["intrinsics"]), poses_est=[f(p) for p in c["poses_est"]],
                disps_est=[f(x) for x in c["disps_est"]])


def c_forward(L, d, gamma):
    B, N, ht, wd = d["disps"].shape
    n = len(d["poses_est"])
    nbytes = L.dba_flow_loss_workspace_bytes(B, N, ht, wd, n)
    ws = Workspace(nbytes)
    loss, met = Guarded(1, dtype=torch.float32), Guarded(6, dtype=torch.float32)
    pp, dp = _ptrs(d["poses_est"]), _ptrs(d["disps_est"])
    c_api.check(L.dba_flow_loss_forward(ptr(d["Ps"]), ptr(d["disps"]), ptr(d["intr"]), ptr(pp), ptr(dp), n, ptr(loss.t), ptr(met.t), B, N, ht, wd,
                                        gamma, ptr(ws.t), nbytes, stream()), "flow_loss_forward")
    torch.cuda.synchronize()
    loss.check_guards("flow_loss_forward loss"); met.check_guards("flow_loss_forward metrics"); ws.check_guards("flow_loss_forward")
    return loss.t.clone(), met.t.view(torch.float64).clone()


def c_backward(L, d, gamma, grad):
    B, N, ht, wd = d["disps"].shape
    n = len(d["poses_est"])
    nbytes = L.dba_flow_loss_workspace_bytes(B, N, ht, wd, n)
    ws = Workspace(nbytes)
    g = torch.tensor(grad, dtype=torch.float32, device=dev)
    gp = [Guarded(B, N, 7, dtype=torch.float32) for _ in range(n)]
    gd = [Guarded(B, N, ht, wd, dtype=torch.float32) for _ in range(n)]
    pp, dp = _ptrs(d["poses_est"]), _ptrs(d["disps_est"])
    gpp, gdp = _ptrs([x.t for x in gp]), _ptrs([x.t for x in gd])
    c_api.check(L.dba_flow_loss_backward(ptr(g), ptr(d["Ps"]), ptr(d["disps"]), ptr(d["intr"]), ptr(pp), ptr(dp), n, ptr(gpp), ptr(gdp), B, N, ht,
                                         wd, gamma, ptr(ws.t), nbytes, stream()), "flow_loss_backward")
    torch.cuda.synchronize()
    ws.check_guards("flow_loss_backward")
    for s in range(n):
        gp[s].check_guards("grad_poses_est[%d]" % s); gd[s].check_guards("grad_disps_est[%d]" % s)
        assert bool((gp[s].t[..., 6].view(torch.int32) == 0).all()), "grad_poses_est[%d]: a 7th entry is not +0" % s
    return [x.t.clone() for x in gp], [x.t.clone() for x in gd]


def c_upsample_backward(L, disps, mask, gout):
    n, ht, wd = disps.shape
    gd, gm_, taps = Guarded(n, ht, wd, dtype=torch.float32), Guarded(n, 576, ht, wd, dtype=torch.float32), Guarded(n, 9, 8, ht, wd, dtype=torch.float32)
    c_api.check(L.dba_cvx_upsample_backward(ptr(disps), ptr(mask), ptr(gout), ptr(gd.t), ptr(gm_.t), ptr(taps.t), n, ht, wd, stream()),
                "cvx_upsample_backward")
    torch.cuda.synchronize()
    gd.check_guards("grad_disps"); gm_.check_guards("grad_mask"); taps.check_guards("tap partials")
    return gd.t.clone(), gm_.t.clone()


def _oracle_kappa(got, ref, r, what):
    """the native value against an autograd fp64 value, under the model r's bound plus 1e-12 of the largest value (the two fp64
    evaluations' own difference) plus the autograd value itself where the model has an exact 0 of an expf that surely underflows"""
    r = gm.R(r.v.cpu(), r.b.cpu())
    ref = ref.reshape(r.b.shape)
    fin = torch.isfinite(ref)
    scale = float(ref[fin].abs().max()) if bool(fin.any()) else 0.0
    under = (r.v == 0) & (r.b == 0) & fin
    return kappa(got, gm.R(ref, r.b + 1e-12 * scale + torch.where(under, ref.abs(), torch.zeros_like(ref))), what)


# ---- the flow loss -------------------------------------------------------------------------------------------------------------------
def check_flow(L, name):
    st = fc.stage(name)
    c, gamma, grad = st["case"], st["gamma"], st["grad"]
    d = to_dev(c)
    B, N, ht, wd = d["disps"].shape
    n = len(d["poses_est"])
    M = fm.Flow(c, gamma, grad, dev=dev)
    stats = {}
    loss, met = c_forward(L, d, gamma)
    stats["loss"] = kappa(loss.reshape(()), M.forward(), "loss")
    stats["metric_sum"] = kappa(met[0], M.metric_sum, "metric sum")
    count, below = int(met[1]), int(met[2])
    assert M.count_sure <= count <= M.count_sure + M.count_amb, (count, M.count_sure, M.count_amb)
    assert M.below - M.below_amb <= below <= M.below + M.below_amb, (below, M.below, M.below_amb)
    gp, gd = c_backward(L, d, gamma, grad)
    stats["grad_disps"] = stats["grad_poses"] = 0.0
    small = ht * wd <= ORACLE_MAX_HW
    if small:
        from test_flow_loss_stages_cpu import oracle
        _, od, op = oracle({k: (v.cuda() if torch.is_tensor(v) else [x.cuda() for x in v]) for k, v in c.items()}, gamma, grad)
    for s in range(n):
        mgd, mgp = M.backward_iterate(s)
        stats["grad_disps"] = max(stats["grad_disps"], kappa(gd[s].reshape(B, N, -1), mgd, "grad_disps_est[%d]" % s))
        stats["grad_poses"] = max(stats["grad_poses"], kappa(gp[s][..., :6], mgp, "grad_poses_est[%d]" % s))
        if small:
            _oracle_kappa(gd[s].reshape(B, N, -1), od[s].cpu(), mgd, "grad_disps_est[%d] vs autograd" % s)
            _oracle_kappa(gp[s][..., :6], op[s].cpu(), mgp, "grad_poses_est[%d] vs autograd" % s)
        del mgd, mgp
    amb = M.amb["v0"] + M.amb["v1"] + M.amb["1px"]
    decisions = 2 * B * len(M.edges) * ht * wd * (n + 1)
    stats.update(ambiguous=amb, decisions=decisions)
    _report(name, stats)
    assert amb <= AMBIGUOUS_ALLOWANCE + decisions // 1000, stats
    return stats, gp, gd


@pytest.mark.parametrize("name", list(fc.STAGES))
def test_flow_loss_against_fp64(capi, name):
    stats, gp, gd = check_flow(capi, name)
    if name == "placed_thresholds":
        assert stats["ambiguous"] == 0
    if name == "exact_equal":                    # c1 == c0 bit for bit on every third column of iterate 0: the gradient there is 0
        c = fc.stage(name)["case"]
        eq = (c["disps_est"][0].float() == c["disps"].float()).to(dev)
        assert bool((gd[0][eq] == 0).all())
    if name == "zero_translation":
        for x in gd:
            assert bool((x == 0).all()), "a disparity gradient without translation"
    if name == "no_valid_rows":
        for x in gd:
            assert bool((x[..., 2:5, :] == 0).all())


# ---- cvx_upsample_backward ---------------------------------------------------------------------------------------------------------
def check_upsample(L, name, c):
    B, N, ht, wd = c["disp"].shape
    n = B * N
    dd = c["disp"].reshape(n, ht, wd).to(dev).float().contiguous()
    mm = c["mask"].reshape(n, 576, ht, wd).to(dev).float().contiguous()
    go = c["cot"].reshape(n, 8 * ht, 8 * wd).to(dev).float().contiguous()
    gd, gmask = c_upsample_backward(L, dd, mm, go)
    md, mmask = fm.upsample_backward(dd, mm, go, dev=dev)
    stats = {"grad_disps": kappa(gd, md, "grad_disps"), "grad_mask": kappa(gmask, mmask, "grad_mask")}
    if ht * wd <= ORACLE_MAX_HW:
        dv, mv = dd.double().requires_grad_(True), mm.double().requires_grad_(True)
        from oracle import upsample as oup
        od, om = torch.autograd.grad(oup.cvx_upsample(dv[..., None], mv).squeeze(-1), [dv, mv], go.double())
        _oracle_kappa(gd, od.cpu(), md, "grad_disps vs autograd")
        _oracle_kappa(gmask, om.cpu(), mmask, "grad_mask vs autograd")
    _report(name, stats)
    return gd, gmask


@pytest.mark.parametrize("name", list(fc.UPSAMPLE_STAGES))
def test_upsample_backward_against_fp64(capi, name):
    c = fc.upsample_stage(name)
    gd, gmask = check_upsample(capi, name, c)
    if name == "up_nan_cot":
        want = torch.zeros(576, 5, 6, dtype=torch.bool)
        want.view(9, 64, 5, 6)[:, 3 * 8 + 5, 2, 4] = True
        assert torch.equal(torch.isnan(gmask[0]).cpu(), want)
        wdn = torch.zeros(5, 6, dtype=torch.bool)
        wdn[1:4, 3:6] = True
        assert torch.equal(torch.isnan(gd[0]).cpu(), wdn)
    if name == "up_underflow":
        _, mmask = fm.upsample_backward(c["disp"][0], c["mask"][0], c["cot"][0])
        z = (mmask.v == 0) & (mmask.b == 0)
        assert bool(z.any()) and bool((gmask.cpu()[z] == 0).all())


# ---- through the hooks ---------------------------------------------------------------------------------------------------------------
def _native_flow(c, scale):
    f = lambda t: t.to(dev, torch.float32).contiguous()  # noqa: E731
    pe = [f(p).requires_grad_(True) for p in c["poses_est"]]
    de = [f(x).requires_grad_(True) for x in c["disps_est"]]
    loss, _ = modules.flow_loss(lt.SE3(f(c["Ps"])), f(c["disps"]), [lt.SE3(p) for p in pe], de, f(c["intrinsics"]), None)
    g = torch.autograd.grad(loss * scale, pe + de)
    return loss.detach(), list(g)


def _native_upsample(c, how):
    disp = c["disp"].to(dev).float().requires_grad_(True)
    mask = c["mask"].to(dev).float().requires_grad_(True)
    out = modules.upsample_disp(disp, mask)
    if how == "sum":
        return torch.autograd.grad(out.sum(), [disp, mask])
    cot = torch.ones_like(out) if how == "ones" else c["cot"].to(dev).float()
    if how == "misaligned":
        buf = torch.empty(cot.numel() + 1, device=dev)
        buf[1:].copy_(cot.reshape(-1))
        cot = buf[1:].view(cot.shape)
        assert cot.data_ptr() % 16 == 4
    return torch.autograd.grad(out, [disp, mask], cot)


def test_hooks_give_the_c_abi_bits(capi):
    c = fc.stage("gamma0.5_grad0.05")["case"]
    d = to_dev(c)
    _, g = _native_flow(c, 0.05)
    n = len(c["poses_est"])
    gp, gd = c_backward(capi, d, 0.9, 0.05)
    for s in range(n):
        same_bits(g[s], gp[s], "hook grad_poses_est[%d]" % s)
        same_bits(g[n + s], gd[s], "hook grad_disps_est[%d]" % s)
    u = fc.upsample_stage("up_13x17")
    a, b = _native_upsample(u, "sum"), _native_upsample(u, "ones")
    for x, y, w in zip(a, b, ("grad_disp", "grad_mask")):
        same_bits(x, y, "stride-0 grad_out " + w)
    a, b = _native_upsample(u, "misaligned"), _native_upsample(u, "cot")
    for x, y, w in zip(a, b, ("grad_disp", "grad_mask")):
        same_bits(x, y, "misaligned grad_out " + w)
    B, N, ht, wd = u["disp"].shape
    gd2, gm2 = c_upsample_backward(capi, u["disp"].reshape(B * N, ht, wd).to(dev).float(), u["mask"].reshape(B * N, 576, ht, wd).to(dev).float(),
                                   u["cot"].reshape(B * N, 8 * ht, 8 * wd).to(dev).float().contiguous())
    same_bits(b[0].reshape(gd2.shape), gd2, "hook grad_disp vs C ABI")
    same_bits(b[1].reshape(gm2.shape), gm2, "hook grad_mask vs C ABI")


def test_side_stream_gives_the_same_bits():
    c = fc.stage("N7_B2_n3_37x53")["case"]
    u = fc.upsample_stage("up_13x17")
    base = _native_flow(c, 0.05), _native_upsample(u, "cot")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = _native_flow(c, 0.05), _native_upsample(u, "cot")
    torch.cuda.synchronize()
    same_bits(base[0][0], other[0][0], "loss on a side stream")
    for k, (x, y) in enumerate(zip(base[0][1], other[0][1])):
        same_bits(x, y, "flow gradient %d on a side stream" % k)
    for x, y in zip(base[1], other[1]):
        same_bits(x, y, "upsample gradient on a side stream")


def test_upsample_into_flow_loss_at_training_size(capi):
    """upsample_disp -> flow_loss: 7 x 48x64 coarse maps to 384x512, 3 iterates; the mask and coarse-disparity gradients element by
    element, the flow gradient's bound carried as the cotangent's error"""
    B, N, h, w, n = 1, 7, 48, 64, 3
    c = fc.make_case(B=B, N=N, ht=8 * h, wd=8 * w, n=n, seed=300)
    g = torch.Generator().manual_seed(301)
    coarse = [c["disps_est"][i][..., 3::8, 3::8].to(dev).float().contiguous().requires_grad_(True) for i in range(n)]
    masks = [torch.randn(B, N, 576, h, w, generator=g, dtype=torch.float64).to(dev).float().requires_grad_(True) for _ in range(n)]
    f = lambda t: t.to(dev, torch.float32).contiguous()  # noqa: E731
    de = [modules.upsample_disp(di, mi) for di, mi in zip(coarse, masks)]
    loss, _ = modules.flow_loss(lt.SE3(f(c["Ps"])), f(c["disps"]), [lt.SE3(f(p)) for p in c["poses_est"]], de, f(c["intrinsics"]))
    got = torch.autograd.grad(loss, masks + coarse)
    M = fm.Flow(dict(c, disps_est=[x.detach() for x in de]), dev=dev)
    worst = {"grad_mask": 0.0, "grad_coarse": 0.0}
    for s in range(n):
        gd, _ = M.backward_iterate(s)
        cot = gm.R(gd.v.reshape(B * N, 8 * h, 8 * w), gd.b.reshape(B * N, 8 * h, 8 * w))
        md, mm = fm.upsample_backward(coarse[s].detach().reshape(B * N, h, w), masks[s].detach().reshape(B * N, 576, h, w), cot, dev=dev)
        worst["grad_mask"] = max(worst["grad_mask"], kappa(got[s].reshape(B * N, 576, h, w), mm, "grad_mask[%d]" % s))
        worst["grad_coarse"] = max(worst["grad_coarse"], kappa(got[n + s].reshape(B * N, h, w), md, "grad_coarse[%d]" % s))
    _report("upsample_into_flow_loss", worst)


def test_card():
    p = torch.cuda.get_device_properties(0)
    try:
        import subprocess
        lim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        lim = "unknown"
    _report("card", {"name": p.name, "power_limit": lim})
