"""Host checks for tests/test_geometry_stages_gpu.py: every case of geometry_cases reaches the corner it names, and the error model of
geometry_model holds for the fp32 restatements (oracle/geom.py, oracle/upsample.py and the kernel-order cvx loop) against fp64 -- and is
not vacuous: somewhere the fp32 error reaches at least 1/64 of its bound."""
import math

import pytest
import torch

import oracle.geom as og
import geometry_cases as gc
import geometry_model as gm

_ALL = gc.cases()


def _case(name):
    return _ALL[name]


def _d64(c):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in c.items()}


def _kappa(got32, ref64, b):
    """max |got32 - ref64| / b over finite references with a finite bound; asserts the non-finite rule (same NaN, same inf)"""
    got = got32.double()
    fin = torch.isfinite(ref64)
    assert torch.equal(torch.isnan(got), torch.isnan(ref64)), "NaN where fp64 has none, or the reverse"
    assert torch.equal(got[torch.isinf(ref64)], ref64[torch.isinf(ref64)])
    err = (got - ref64).abs()
    ok = fin & torch.isfinite(b)
    assert bool((err[ok & (b == 0)] == 0).all()), "an exact value differs"
    k = torch.where(ok & (b > 0), err / b.clamp(min=1e-300), torch.zeros_like(err))
    return float(k.max()) if k.numel() else 0.0


def _same(a, b):
    return torch.allclose(a, b, rtol=0, atol=0, equal_nan=True)


# ---- corners ------------------------------------------------------------------------------------------------------------------
def test_shapes_reach_the_launch_tails():
    hw = {k: h * w for k, (h, w) in gc.SHAPES.items()}
    assert hw["hw255"] == 255 and hw["hw256"] == 256 and hw["hw257"] == 257 and hw["s1x1"] == 1
    assert gc.SHAPES["s1x7"][0] == 1 and gc.SHAPES["s7x1"][1] == 1
    assert any(v % 256 and v > 256 for v in hw.values()) and any(v < 256 for v in hw.values())
    for k in gc.SHAPES:
        c = _case(k)
        assert bool((c["ii"] == c["jj"]).any()), "no stereo edge"
        assert not torch.equal(c["intr_pf"][c["ii"]], c["intr_pf"][c["jj"]]), "Ki == Kj on every edge"
        qn = c["poses"][:, 3:].norm(dim=1)
        assert float((qn - 1).abs().max()) > 1e-3, "unit quaternions only"


def test_many_edges_exceed_grid_y_limit_on_a_2x3_map():
    c = gc.case("many_edges")
    assert c["disps"].shape == (70000, 2, 3) and len(c["ii"]) == 70000 > 65535 and len(c["df_ix"]) == 70000
    assert bool((c["ii"] == c["jj"]).any())


def test_thresholds_are_hit_exactly_and_straddled():
    c = _case("thresholds")
    m = gm.projmap(c["poses"], c["disps"], c["intr"], c["ii"][:1], c["jj"][:1])
    k = len(c["target_z"])
    Z = m["Z"][0, :k]
    assert torch.equal(Z.v, c["target_z"]) and bool((Z.b == 0).all()), "Z is not the placed fp32 value in both evaluations"
    fd = gm.frame_distance(c["poses"], c["disps"], c["intr"], c["ii"][:1], c["jj"][:1], 1.0)   # the translation-only Z is the same
    names = c["target_names"]
    for name, thr in gc.THRESHOLDS.items():
        z = c["target_z"][[i for i, n in enumerate(names) if n == name]]
        assert float((z - thr)[z <= thr].max()) > -2 * gc.GRID and float((z - thr)[z > thr].min()) < 2 * gc.GRID, name
        assert float((z - thr).abs().max()) > 1e-4 + 2 ** -24, name          # reaches past a 1e-4 shift of the constant
    assert bool((c["target_z"] == 0.25).any())


def test_three_quarters_is_exact():
    c = _case("fd_three_quarters")
    fd = gm.frame_distance(c["poses"], c["disps"], c["intr"], c["ii"], c["jj"], 1.0)
    assert float(fd["vv"].v[0]) == 192 and float(fd["t"].v[0]) == 256 and float(fd["vv"].b[0]) == 0
    assert float(fd["vv"].v[1]) == 193
    r = og.frame_distance(c["poses"].double(), c["disps"].double(), c["intr"].double(), c["ii"], c["jj"], 1.0)
    assert float(r[0]) == 1000.0 and float(r[1]) != 1000.0


def test_depth_filter_cells_reach_every_edge():
    c = _case("df_cells")
    wd = c["disps"].shape[2]
    ht = c["disps"].shape[1]
    t, q = gm.edge_transform(c["poses"], torch.tensor([0]), torch.tensor([3]), False)
    Xi = gm.backproject(c["disps"].double()[0].reshape(1, -1), gm._K(c["intr"]), ht, wd)
    Xj = gm.act_se3(t, q, Xi)
    uj = gm.R(1.0) * (Xj[0] / Xj[2]) + 0.0
    lo, hi, sure = gm.floor_cells(uj)
    assert bool(sure.all()), "a placed projection is not exact"
    u0 = lo.reshape(-1)
    for want in (3, 5, wd - 2, wd - 1, -1, 2 ** 31 - 1, -2 ** 31):
        assert bool((u0 == want).any()), want
    assert bool((uj.v.reshape(-1) == wd - 2).any()) and bool((uj.v.reshape(-1) == 3).any()), "no exact integer column"
    assert bool(((uj.v.reshape(-1) < 0) & (uj.v.reshape(-1) > -1)).any()), "nothing just below 0"
    th = c["df_thresh"]
    assert math.isinf(float(th[0])) and float(th[1]) == 0 and len(set(th.tolist())) == 3


def test_nan_projection_counts_in_cell_0():
    c = _case("df_nan")
    n, r, cc = c["nan_pixel"]
    K = c["intr"]
    assert float(K[2]) == cc and float(K[3]) == r and float(c["disps"][n, r, cc]) == 1.0
    t, q = gm.edge_transform(c["poses"], torch.tensor([n]), torch.tensor([n - 1]), False)
    Xi = gm.backproject(c["disps"].double()[n].reshape(1, -1), gm._K(K), *c["disps"].shape[1:])
    Xj = gm.act_se3(t, q, Xi)
    k = r * c["disps"].shape[2] + cc
    assert float(Xj[0].v[0, k]) == 0 and float(Xj[1].v[0, k]) == 0 and float(Xj[2].v[0, k]) == 0
    assert bool((c["disps"][n - 1, :2, :2] > 1 / c["df_thresh"][0]).all())
    cnt = og.depth_filter(c["poses"], c["disps"], K, c["df_ix"], c["df_thresh"])
    cnt64 = og.depth_filter(c["poses"].double(), c["disps"].double(), K.double(), c["df_ix"], c["df_thresh"])
    assert float(cnt[0, r, cc]) >= 1 and float(cnt64[0, r, cc]) >= 1


def test_neighbour_sets_are_clipped_at_both_ends():
    seen = set()
    for num in range(1, 8):
        c = _case("df_num%d" % num)
        assert c["disps"].shape[0] == num and torch.equal(c["df_ix"], torch.arange(num))
        for i in range(num):
            js = [i - k - 1 if k < 3 else i + k for k in range(6)]
            seen.add(sum(0 <= j < num for j in js))
        th = c["df_thresh"]
        assert math.isinf(float(th[0])) and (num == 1 or float(th[-1]) == 0)
    assert seen == {0, 1, 2, 3, 4}


def test_nonfinite_disparities_on_one_frame():
    c = _case("nonfinite")
    d = c["disps"]
    assert bool(torch.isnan(d[1]).any()) and bool((d[1] == math.inf).any()) and bool((d[1] == -math.inf).any())
    assert bool((d[1] == 0).any()) and bool((d[1] < 0).any())
    others = torch.cat([d[0], d[2], d[3]])
    assert bool(torch.isfinite(others).all()) and bool((others > 0).all())


def test_upsample_cases_reach_their_masks():
    d, m = gc.upsample_case("up_equal")
    mm = m.float().view(2, 9, 64, 5, 7)
    assert bool((mm == mm[:, :1]).all())
    d, m = gc.upsample_case("up_dominant")
    mm = m.float().view(2, 9, 64, 6, 5)
    assert bool(((mm == 65504).sum(1) == 1).all()) and bool(((mm == -65504).sum(1) == 8).all()) and m.dtype == torch.float16
    d, m = gc.upsample_case("up_neginf")
    mm = m.view(1, 9, 64, 6, 7)
    assert bool(torch.isneginf(mm[..., 0, :]).all()) and bool(torch.isneginf(mm).any(1)[..., 1:, :].any())
    d, m = gc.upsample_case("up_nan_inf")
    assert bool(torch.isnan(m).any()) and bool(torch.isposinf(m).any())
    assert gc.upsample_case("up_ht1")[0].shape[1] == 1 and gc.upsample_case("up_wd1")[0].shape[2] == 1


# ---- the model against the fp32 restatements ----------------------------------------------------------------------------------
_WORST = {}


def _note(kernel, k):
    _WORST[kernel] = max(_WORST.get(kernel, 0.0), k)
    assert k <= 1.0, (kernel, k)


@pytest.mark.parametrize("name", gc.CASES)
def test_model_bounds_the_fp32_restatement(name):
    c = _case(name)
    P, D, K, ii, jj = c["poses"], c["disps"], c["intr"], c["ii"], c["jj"]
    N, ht, wd = D.shape
    if ht * wd == 0:
        r = og.frame_distance(P, D, K, ii, jj, 0.3)
        assert bool((r == 1000).all())
        return
    c64 = _d64(c)
    # projmap
    m = gm.projmap(P, D, K, ii, jj)
    o32, v32 = og.projmap(P, D, K, ii, jj)
    o64, v64 = og.projmap(c64["poses"], c64["disps"], c64["intr"], ii, jj)
    take, sure = gm.decide(m["Z"], gm.PROJ_Z, ">")
    assert _same(m["cu"].v[take], o64[..., 0].reshape(len(ii), -1)[take]), "model value is not the oracle's fp64 value"
    br = take & sure & (o32[..., 0].reshape(len(ii), -1) != m["u"].expand_as(take)) | take & sure
    _note("projmap", _kappa(o32[..., 0].reshape(len(ii), -1)[br], o64[..., 0].reshape(len(ii), -1)[br], m["cu"].b[br]))
    _note("projmap", _kappa(o32[..., 1].reshape(len(ii), -1)[br], o64[..., 1].reshape(len(ii), -1)[br], m["cv"].b[br]))
    vd, vs = gm.decide(m["Z"], gm.MIN_DEPTH, ">")
    assert torch.equal((v32.reshape(len(ii), -1) > 0)[vs], vd[vs])
    # reproject
    m = gm.reproject(P, D, c["intr_pf"], ii, jj)
    r32, _ = og.reproject(P, D, c["intr_pf"], ii, jj)
    r64, _ = og.reproject(c64["poses"], c64["disps"], c64["intr_pf"], ii, jj)
    small, ssure = gm.decide(m["Z"], gm.REPROJ_SMALL, "<")
    keep = ~small & ssure
    for ch, key in ((0, "x"), (1, "y")):
        a32, a64 = r32[..., ch].reshape(len(ii), -1), r64[..., ch].reshape(len(ii), -1)
        assert _same(m[key].v[keep], a64[keep])
        _note("reproject", _kappa(a32[keep], a64[keep], m[key].b[keep]))
        _note("reproject", _kappa(a32[small & ssure], a64[small & ssure], m[key + "1"].b[small & ssure]))
    # iproj
    pts = gm.iproj(P, D, K)
    p32, p64 = og.iproj(P, D, K), og.iproj(c64["poses"], c64["disps"], c64["intr"])
    for k in range(3):
        _note("iproj", _kappa(p32[..., k].reshape(N, -1), p64[..., k].reshape(N, -1), pts[k].b))
    # frame_distance
    for beta in c["betas"]:
        fd = gm.frame_distance(P, D, K, ii, jj, beta)
        f32 = og.frame_distance(P, D, K, ii, jj, beta)
        f64 = og.frame_distance(c64["poses"], c64["disps"], c64["intr"], ii, jj, beta)
        far, fsure = gm.decide(fd["ratio"], gm.FRAC, "<")
        assert torch.equal((f32 == 1000)[fsure], far[fsure]) and torch.equal((f64 == 1000)[fsure], far[fsure])
        ok = fsure & ~far
        _note("frame_distance", _kappa(f32[ok], f64[ok], fd["dist"].b[ok]))
    # depth_filter
    s, p, _ = gm.depth_filter(P, D, K, c["df_ix"], c["df_thresh"])
    cnt32 = og.depth_filter(P, D, K, c["df_ix"], c["df_thresh"]).double()
    cnt64 = og.depth_filter(c64["poses"], c64["disps"], c64["intr"], c["df_ix"], c["df_thresh"])
    assert bool(((cnt32 >= s) & (cnt32 <= p)).all()) and bool(((cnt64 >= s) & (cnt64 <= p)).all())


@pytest.mark.parametrize("name", gc.UPSAMPLE)
def test_upsample_model_bounds_the_kernel_order_fp32_loop(name):
    d, m = gc.upsample_case(name)
    ref, b = gm.cvx_upsample(d, m)
    o64 = __import__("oracle.upsample", fromlist=["x"]).cvx_upsample(d.double()[..., None], m.double())[..., 0]
    fin = torch.isfinite(o64)
    assert torch.allclose(ref[fin], o64[fin], rtol=1e-13, atol=0) and torch.equal(torch.isnan(ref), torch.isnan(o64))
    got = gm.cvx_upsample_f32(d, m)
    _note("cvx_upsample", _kappa(got, ref, b))


def test_model_is_not_vacuous():
    """run after the model tests (pytest keeps file order): every kernel's fp32 error reaches 1/64 of its bound somewhere"""
    if len(_WORST) < 5:
        pytest.skip("needs the model tests of this module in the same session")
    for k, v in _WORST.items():
        assert v >= 1 / 64, (k, v)
