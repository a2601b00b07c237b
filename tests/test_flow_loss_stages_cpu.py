"""Host checks for tests/test_flow_loss_stages_gpu.py: the error model of flow_loss_model has the fp64 values of autograd through the
fp64 oracles (oracle/flow_loss.py, oracle/upsample.py) on every small stage case and of the reference's own functions on the fixture
(tests/golden/flow_loss.pt); the placed threshold pixels land where they are meant to and are sure decisions; the block-sum constant
follows from the kernels' reduction structure and bounds an fp32 restatement of it; the cases regenerate bit for bit from their seeds."""
import hashlib
import os

import pytest
import torch

import flow_loss_cases as fc
import flow_loss_model as fm
import geometry_model as gm
from oracle import ba_layer as oba, flow_loss as ofl, upsample as oup

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flow_loss.pt"), weights_only=False)
SMALL = [k for k in fc.STAGES if not k.startswith("train")]
SMALL_UP = [k for k in fc.UPSAMPLE_STAGES if k != "up_train_7x48x64"]


def oracle(c, gamma=0.9, grad=1.0, fp32_inputs=True):
    """loss and gradients (poses in lietorch's left tangent, 6 components) by autograd through oracle/flow_loss.py in fp64"""
    to = (lambda t: t.float().double()) if fp32_inputs else (lambda t: t.double())  # noqa: E731
    n = len(c["poses_est"])
    d = [to(x).requires_grad_(True) for x in c["disps_est"]]
    eps = [torch.zeros(*p.shape[:-1], 6, dtype=torch.float64, device=p.device, requires_grad=True) for p in c["poses_est"]]
    P = [oba.SE3(oba.left_perturbed(to(p), e)) for p, e in zip(c["poses_est"], eps)]
    loss = ofl.flow_loss(oba.SE3(to(c["Ps"])), to(c["disps"]), P, d, to(c["intrinsics"]), gamma)[0]
    if fp32_inputs:
        grad = float(torch.tensor(grad, dtype=torch.float32))        # the kernel reads the upstream gradient in fp32
    g = torch.autograd.grad(loss * grad, d + eps)
    return loss.detach(), list(g[:n]), list(g[n:])


def close(a, b, tol=1e-12):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    nan = torch.isnan(b)
    assert torch.equal(torch.isnan(a), nan), "NaN at %d places, the oracle at %d" % (int(torch.isnan(a).sum()), int(nan.sum()))
    if not bool((~nan).any()):
        return
    err = float((a[~nan] - b[~nan]).abs().max())
    assert err <= tol * max(1.0, float(b[~nan].abs().max())), err


def model(c, gamma, grad, fp32_inputs=True):
    M = fm.Flow(c, gamma, grad, fp32_inputs=fp32_inputs)
    loss = M.forward()
    gp, gd = M.backward()
    return M, loss, gp, gd


def assert_bounded(r, what):
    """a finite value has a finite bound"""
    bad = torch.isfinite(r.v) & ~torch.isfinite(r.b)
    assert not bool(bad.any()), "%s: %d finite values without a bound" % (what, int(bad.sum()))


@pytest.mark.parametrize("name", SMALL)
def test_model_values_are_the_oracles(name):
    st = fc.stage(name)
    c = st["case"]
    M, loss, gp, gd = model(c, st["gamma"], st["grad"])
    l64, gd64, gp64 = oracle(c, st["gamma"], st["grad"])
    close(loss.v, l64)
    B, N, ht, wd = c["disps"].shape
    for s in range(len(gd)):
        close(gd[s].v.reshape(B, N, ht, wd), gd64[s])
        close(gp[s].v, gp64[s])
        assert_bounded(gd[s], "grad_disps_est[%d]" % s)
        assert_bounded(gp[s], "grad_poses_est[%d]" % s)
    assert_bounded(loss, "loss")


@pytest.mark.parametrize("name", sorted(fc.cases()))
def test_model_values_are_the_reference_fixtures(name):
    want = GOLDEN["flow"][name]
    M, loss, gp, gd = model(fc.cases()[name], 0.9, 1.0, fp32_inputs=False)
    close(loss.v, want["loss"])
    for s in range(len(gd)):
        close(gd[s].v.reshape(want["grad_disps_est"][s].shape), want["grad_disps_est"][s])
        close(gp[s].v, want["grad_poses_est"][s][..., :6])


def _upsample_oracle(c, fp32_inputs=True):
    to = (lambda t: t.float().double()) if fp32_inputs else (lambda t: t.double())  # noqa: E731
    disp, mask = to(c["disp"]).requires_grad_(True), to(c["mask"]).requires_grad_(True)
    return torch.autograd.grad(oup.upsample_disp(disp, mask), [disp, mask], to(c["cot"]))


def _upsample_model(c, fp32_inputs=True):
    B, N, ht, wd = c["disp"].shape
    return fm.upsample_backward(c["disp"].reshape(B * N, ht, wd), c["mask"].reshape(B * N, 576, ht, wd),
                                c["cot"].reshape(B * N, 8 * ht, 8 * wd), fp32_inputs=fp32_inputs)


@pytest.mark.parametrize("name", SMALL_UP)
def test_upsample_model_values_are_the_oracles(name):
    c = fc.upsample_stage(name)
    gd, gmask = _upsample_model(c)
    od, om = _upsample_oracle(c)
    close(gd.v.reshape(od.shape), od)
    if name == "up_underflow":       # the model's exact zeros where expf underflows surely: the oracle's values there are below 1e-40
        z = (gmask.b == 0) & (gmask.v == 0)
        assert bool(z.any()) and float(om.reshape(gmask.v.shape)[z].abs().max()) < 1e-40
    close(gmask.v.reshape(om.shape), om)
    assert_bounded(gd, "grad_disps")
    assert_bounded(gmask, "grad_mask")


@pytest.mark.parametrize("name", sorted(fc.upsample_cases()))
def test_upsample_model_values_are_the_reference_fixtures(name):
    want = GOLDEN["upsample"][name]
    gd, gmask = _upsample_model(fc.upsample_cases()[name], fp32_inputs=False)
    close(gd.v.reshape(want["grad_disp"].shape), want["grad_disp"])
    close(gmask.v.reshape(want["grad_mask"].shape), want["grad_mask"])


def test_nan_cotangent_reaches_its_taps_and_nothing_else():
    c = fc.upsample_stage("up_nan_cot")
    gd, gmask = _upsample_model(c)
    y, x, i, j = 2, 4, 3, 5                                    # the NaN sub-pixel: coarse (2, 4), sub-row 3, column 5
    want = torch.zeros(576, 5, 6, dtype=torch.bool)
    want.view(9, 64, 5, 6)[:, i * 8 + j, y, x] = True
    assert torch.equal(torch.isnan(gmask.v[0]), want)
    wd_ = torch.zeros(5, 6, dtype=torch.bool)
    wd_[y - 1:y + 2, x - 1:x + 2] = True                       # the coarse pixels its 9 taps read
    assert torch.equal(torch.isnan(gd.v[0]), wd_)


def test_placed_thresholds_land_on_their_margins_and_are_sure():
    c = fc.stage("placed_thresholds")["case"]
    M = fm.Flow(c)
    G = fm.edge_transforms(M.Ps)
    X = [gm.R(torch.zeros(1)), gm.R(torch.zeros(1)), gm.R(torch.ones(1)), gm.R(M.disps[:, 0].reshape(1, 1, -1))]
    z0 = gm.act_se3(*G, X)[2][0, 0]                                                 # edge 0 -> 1
    z0 = gm.R(z0.v[None], z0.b[None])
    d0 = M.disps[0, 0].reshape(-1)
    placed = (d0 - float(torch.tensor(0.8, dtype=torch.float32))).abs() <= 64 * fc.GRID
    assert int(placed.sum()) == d0.numel() - 3
    assert bool((z0.b[0][placed] == 0).all()) and torch.equal(z0.v[0][placed], 1.0 - d0[placed]), "edge 0 -> 1 does not map d to 1 - d"
    thr = gm.REPROJ_VALID
    steps = torch.round((z0.v[0] - thr) / fc.GRID)
    assert bool((steps[placed] < 0).any() and (steps[placed] > 0).any())
    assert float((z0.v[0][placed] - thr).abs().min()) <= fc.GRID, "no pixel within one step of 0.2f"
    assert M.amb["v0"] == 0
    for s in range(M.n):
        it = M.iterate(s)
        assert bool(it["sure"].all()), "iterate %d: an ambiguous v" % s
        z1 = (1.0 - M.disps_est[s][0, 0].reshape(-1), 1.0 + M.disps_est[s][0, 1].reshape(-1))
        assert bool((((z1[0] - thr).abs() <= 2 * fc.GRID) | ((z1[1] - thr).abs() <= 2 * fc.GRID)).any())
        assert bool(((z1[0] < 0) | (z1[1] < 0)).any()), "no pixel behind the camera"
    d = M.disps[0].reshape(2, -1)[:, :3]
    assert d[0, 0] == 0 and torch.signbit(d[0, 1]) and d[0, 1] == 0 and d[0, 2] < 0


def _fp32_block_sum(x):
    """flow_block_sum in fp32 on the host: the xor-shuffle warp tree (every lane ends with the same sum; lane 0's order), then the
    8 warp partials added in order to 0"""
    w = x.float().view(8, 32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, torch.arange(32) ^ o]
    s = torch.zeros((), dtype=torch.float32)
    for k in range(8):
        s = s + w[k, 0]
    return s


def test_block_sum_constant_follows_the_reduction():
    threads, warp = 256, 32
    levels = (warp - 1).bit_length()
    assert fm.BLOCK_DEPTH == levels + threads // warp - 1 and fm.THREADS == threads
    g = torch.Generator().manual_seed(5)
    worst = 0.0
    for trial in range(200):
        x = torch.randn(256, generator=g, dtype=torch.float64) * torch.exp(4 * torch.randn(256, generator=g, dtype=torch.float64))
        if trial % 2:
            x = x.abs()
        x = x.float().double()
        err = abs(float(_fp32_block_sum(x)) - float(x.sum()))
        bound = fm.BLOCK_DEPTH * gm.U * float(x.abs().sum())
        assert err <= bound, (trial, err, bound)
        worst = max(worst, err / bound)
    assert worst > 1 / 64, "the bound is vacuous"


def _digest(obj):
    h = hashlib.sha256()
    def walk(o):
        if torch.is_tensor(o):
            h.update(o.contiguous().view(torch.uint8).numpy().tobytes())
        elif isinstance(o, dict):
            for k in sorted(o):
                h.update(str(k).encode()); walk(o[k])
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v)
        else:
            h.update(repr(o).encode())
    walk(obj)
    return h.hexdigest()[:16]


def test_cases_regenerate_bit_for_bit():
    for name in SMALL:
        assert _digest(fc.stage(name)) == _digest(fc.stage(name)), name
    for name in SMALL_UP:
        assert _digest(fc.upsample_stage(name)) == _digest(fc.upsample_stage(name)), name
    got = _digest([fc.stage(k) for k in SMALL] + [fc.upsample_stage(k) for k in SMALL_UP])
    assert got == DIGEST, got


DIGEST = "12d23b83bd429351"
