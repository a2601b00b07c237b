"""The geometry kernels (csrc/geom.cu) and cvx_upsample through the C ABI, element by element against fp64 under the running error
model of geometry_model, at the edges of geometry_cases (their corners checked in tests/test_geometry_stages_cpu.py, where the model's
fp64 values are also shown to be oracle/geom.py's on .double() inputs).

Every output lies in a NaN-filled fp32 buffer with GUARD floats of NaN on each side; the guards must come back untouched.

Values.  kappa = |got - ref64| / bound <= 1 for coords (projmap, reproject, motion_features), points (iproj), frame distances and
upsampled depths; where the bound is 0 the value must be exact.  Where the fp64 value is NaN the kernel's must be NaN, where it is
+-inf the same inf: the reference's device semantics, which the fixtures below pin for projmap, iproj and depth_filter.
Decisions.  Where the fp64 margin to a threshold exceeds the bound the kernel decides as fp64 does; inside the window either answer
passes, but the outputs must be those of the branch taken: (u, v) exactly on projmap's fallback, the Z := 1 values in reproject.  The
ambiguous decisions of a case may number at most the placed ones plus allowance(): the generator places every threshold pixel exactly,
so none of them is ambiguous, and random pixels rarely are.  A depth_filter count lies between its sure hits and its sure-plus-ambiguous hits.
Exact parts.  projmap's channel 2 is +0; coords and coords_t hold the same bits and motion_features' coords are reproject's, rows
gathered through edge_index; motn is the fp32 clamp(coords - grid, target - coords); graph_writeback and the damping gather are
bit-identical to the fp32 torch restatement (.2f d + ep, two roundings); rows that edge_index, n_inactive, src_frames or ba_frames do
not name stay untouched.  Every n-edge call equals n one-edge calls bit for bit.  Where all exps are exactly 0 or 1 (equal masks, ties
against -inf, one tap at 65504 against -65504) cvx_upsample equals the kernel-order fp32 loop bit for bit.
Reference build.  projmap, iproj and depth_filter are bit-identical to the unmodified reference build at every case (fixtures
`geometry_edges/...` of tests/golden/reference_build.pt); its frame distances (all pairs, or a seeded sample of 2048 at 70 000 pairs)
sum in another order and are held to the model's bound, with the margin rule for 1000.

Worst kappa per kernel and case on one H100 80GB HBM3 at a 700 W power limit; in brackets the ambiguous decisions over all calls of
the case (frame_distance: its four betas; depth_filter: counts whose sure and possible hits differ) / the pixels placed on thresholds:
  case                 projmap        reproject      iproj   frame_distance   depth_filter
  s1x1                 0.148  [0 / 0]  0.155  [0 / 0]  0.327    0.0493 [0 / 0]  [0 / 0]
  s1x7                 0.268  [0 / 0]  0.212  [0 / 0]  0.535    0.0631 [0 / 0]  [0 / 0]
  s7x1                 0.19   [0 / 0]  0.278  [0 / 0]  0.551    0.0621 [0 / 0]  [0 / 0]
  hw255                0.286  [0 / 0]  0.632  [0 / 0]  0.683    0.0668 [0 / 0]  [3 / 0]
  hw256                0.37   [0 / 0]  0.698  [0 / 0]  0.76     0.0535 [0 / 0]  [11 / 0]
  hw257                0.412  [0 / 0]  0.748  [0 / 0]  0.645    0.0494 [0 / 0]  [27 / 0]
  s43x70               0.42   [0 / 0]  0.754  [0 / 0]  0.748    0.0267 [0 / 0]  [135 / 0]
  s48x64               0.441  [0 / 0]  0.749  [0 / 0]  0.776    0.0389 [0 / 0]  [103 / 0]
  s60x80               0.413  [0 / 0]  0.721  [0 / 0]  0.785    0.0533 [0 / 0]  [80 / 0]
  thresholds           0.981  [0 / 60]  0.981  [0 / 60]  0.948    0.057  [0 / 60]  [0 / 60]
  fd_three_quarters    0.553  [0 / 0]  0.5    [0 / 0]  0.75     0.0567 [2 / 0]  [60 / 0]
  df_cells             0.248  [0 / 0]  0.248  [0 / 0]  0.959    0.0763 [0 / 0]  [0 / 0]
  df_nan               0.505  [0 / 0]  0.439  [0 / 0]  0.837    0.0759 [0 / 0]  [2 / 0]
  nonfinite            0.335  [0 / 0]  0.574  [0 / 0]  0.613    0.0281 [0 / 0]  [0 / 0]
  df_num1              0.0543 [0 / 0]  0.369  [0 / 0]  0.496    0      [0 / 0]  [0 / 0]
  df_num2              0.264  [0 / 0]  0.483  [0 / 0]  0.598    0.0437 [0 / 0]  [0 / 0]
  df_num3              0.33   [0 / 0]  0.339  [0 / 0]  0.602    0.0201 [0 / 0]  [0 / 0]
  df_num4              0.314  [0 / 0]  0.33   [0 / 0]  0.526    0.0409 [0 / 0]  [0 / 0]
  df_num5              0.279  [0 / 0]  0.398  [0 / 0]  0.528    0.0249 [0 / 0]  [0 / 0]
  df_num6              0.393  [0 / 0]  0.369  [0 / 0]  0.696    0.0189 [0 / 0]  [0 / 0]
  df_num7              0.392  [0 / 0]  0.533  [0 / 0]  0.685    0.0282 [0 / 0]  [0 / 0]
  many_edges           0.611  [1 / 0]  0.593  [1 / 0]  0.878    0.17   [0 / 0]  [774 / 0]
  cvx_upsample: up_equal 0.086, up_dominant 0, up_ties 0.0304, up_f16_extremes 0.348, up_neginf 0.258, up_nan_inf 0.237, up_ht1 0.233, up_wd1 0.215, up_random_48x64 0.373, up_random_43x70 0.42
No kappa exceeds 0.99: the placed threshold pixels reach 0.98 through their 1/Z.  Each of these edits to geom.cu, built on a scratch
copy, failed this file: projmap's valid threshold 0.25 -> 0.2499f, the stereo branch dropped from reproject, u0 / v0 by (int)
truncation, __expf one ulp up on every other tap, projmap's last grid.y chunk shifted back by one pixel, and coords[2] = 0 skipped.
"""
import json
import os
import sys

import pytest
import torch

from droid_slam_b200 import c_api
import geometry_cases as gc
import geometry_model as gm
from test_tensor_core_fp64_gpu import Guarded
from util import ptr, stream

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_reference_build_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"
AMBIGUOUS_ALLOWANCE = 4


def allowance(decisions, per=1000):
    """ambiguous decisions allowed beyond the placed ones: a few, plus one per thousand for the random scenes' near-singular pixels
    (Z near 0 makes the bounds of the projections large).  depth_filter gets one per 32 of its decisions: a pair of frames with
    equal poses projects every pixel onto its own integer column and row, within rounding, and both cells are then admissible."""
    return AMBIGUOUS_ALLOWANCE + decisions // per


def _report(kernel, name, stats):
    print("GEOM_STAGES %s %s %s" % (kernel, name, json.dumps(stats)))
    out = os.environ.get("GEOM_STAGES_REPORT")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(dict(kernel=kernel, case=name, **stats)) + "\n")


@pytest.fixture(scope="module")
def gold():
    return torch.load(mk.GOLD, weights_only=False)


def kappa(got, r, what):
    """worst kappa of fp32 `got` (any device) against the R `r`, after the non-finite and exact rules"""
    got = got.double().cpu().reshape(r.v.shape)
    ref, b = r.v, r.b
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), "%s: NaN at %d places, fp64 at %d" % (what, int(torch.isnan(got).sum()), int(nan.sum()))
    inf = torch.isinf(ref)
    assert torch.equal(got[inf], ref[inf]), "%s: an inf differs" % what
    ok = torch.isfinite(ref) & torch.isfinite(b)
    err = (got - ref).abs()
    bad0 = ok & (b == 0) & (err > 0)
    assert not bool(bad0.any()), "%s: %d exact values differ" % (what, int(bad0.sum()))
    k = torch.where(ok & (b > 0), err / b.clamp(min=1e-300), torch.zeros_like(err))
    worst = float(k.max()) if k.numel() else 0.0
    assert worst <= 1.0, "%s: kappa %.3g at %s" % (what, worst, tuple(int(i) for i in (k == k.max()).nonzero()[0]))
    return worst


def same_bits(a, b, what):
    a, b = a.contiguous().cpu(), b.contiguous().cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    d = a.view(torch.int32) != b.view(torch.int32)
    assert not bool(d.any()), "%s: %d of %d elements differ" % (what, int(d.sum()), a.numel())


def to_dev(c):
    return {k: (v.to(dev).contiguous() if torch.is_tensor(v) else v) for k, v in c.items()}


# ---- calls through the C ABI -------------------------------------------------------------------------------------------------
def c_projmap(L, d, ii, jj):
    N, ht, wd = d["disps"].shape
    E = len(ii)
    co, va = Guarded(E, ht, wd, 3, dtype=torch.float32), Guarded(E, ht, wd, dtype=torch.float32)
    c_api.check(L.dba_projmap(ptr(d["poses"]), ptr(d["disps"]), ptr(d["intr"]), ptr(ii), ptr(jj), ptr(co.t), ptr(va.t), E, ht, wd, stream()), "projmap")
    torch.cuda.synchronize()
    co.check_guards("projmap coords"); va.check_guards("projmap valid")
    return co.t, va.t


def c_reproject(L, d, ii, jj):
    N, ht, wd = d["disps"].shape
    E = len(ii)
    co, va = Guarded(E, ht, wd, 2, dtype=torch.float32), Guarded(E, ht, wd, dtype=torch.float32)
    c_api.check(L.dba_reproject(ptr(d["poses"]), ptr(d["disps"]), ptr(d["intr_pf"]), ptr(ii), ptr(jj), ptr(co.t), ptr(va.t), E, ht, wd, stream()),
                "reproject")
    torch.cuda.synchronize()
    co.check_guards("reproject coords"); va.check_guards("reproject valid")
    return co.t, va.t


def c_iproj(L, d, n=None):
    N, ht, wd = d["disps"].shape
    n = N if n is None else n
    pts = Guarded(n, ht, wd, 3, dtype=torch.float32)
    c_api.check(L.dba_iproj(ptr(d["poses"]), ptr(d["disps"]), ptr(d["intr"]), ptr(pts.t), n, ht, wd, stream()), "iproj")
    torch.cuda.synchronize()
    pts.check_guards("iproj")
    return pts.t


def c_frame_distance(L, d, ii, jj, beta):
    N, ht, wd = d["disps"].shape
    out = Guarded(len(ii), dtype=torch.float32)
    c_api.check(L.dba_frame_distance(ptr(d["poses"]), ptr(d["disps"]), ptr(d["intr"]), ptr(ii), ptr(jj), ptr(out.t), len(ii), ht, wd, beta, stream()),
                "frame_distance")
    torch.cuda.synchronize()
    out.check_guards("frame_distance")
    return out.t


def c_depth_filter(L, d, ix, th):
    N, ht, wd = d["disps"].shape
    out = Guarded(len(ix), ht, wd, dtype=torch.float32)
    c_api.check(L.dba_depth_filter(ptr(d["poses"]), ptr(d["disps"]), ptr(d["intr"]), ptr(ix), ptr(th), ptr(out.t), len(ix), N, ht, wd, stream()),
                "depth_filter")
    torch.cuda.synchronize()
    out.check_guards("depth_filter")
    return out.t


# ---- checks -------------------------------------------------------------------------------------------------------------------
def check_projmap(c, co, va):
    E = len(c["ii"])
    m = gm.projmap(c["poses"], c["disps"], c["intr"], c["ii"], c["jj"])
    co = co.cpu().reshape(E, -1, 3)
    assert bool((co[..., 2].view(torch.int32) == 0).all()), "projmap channel 2 is not +0"
    u, v = m["u"].expand(E, -1), m["v"].expand(E, -1)
    fell_back = (co[..., 0].double() == u) & (co[..., 1].double() == v)
    take, sure = gm.decide(m["Z"], gm.PROJ_Z, ">")
    assert bool(fell_back[sure & ~take].all()), "projmap: a sure fallback pixel is not (u, v)"
    proj = sure & take | ~sure & ~fell_back
    w = max(kappa(co[..., 0][proj], m["cu"][proj], "projmap u"), kappa(co[..., 1][proj], m["cv"][proj], "projmap v"))
    vd, vs = gm.decide(m["Z"], gm.MIN_DEPTH, ">")
    va = va.cpu().reshape(E, -1)
    assert bool(((va == 0) | (va == 1)).all())
    assert torch.equal((va > 0)[vs], vd[vs]), "projmap valid: %d sure decisions differ" % int(((va > 0) != vd)[vs].sum())
    return w, int((~sure).sum() + (~vs).sum())


def check_reproject(c, co, va):
    E = len(c["ii"])
    m = gm.reproject(c["poses"], c["disps"], c["intr_pf"], c["ii"], c["jj"])
    co = co.cpu().reshape(E, -1, 2)
    small, ss = gm.decide(m["Z"], gm.REPROJ_SMALL, "<")
    w = 0.0
    for ch, key in ((0, "x"), (1, "y")):
        g = co[..., ch]
        w = max(w, kappa(g[ss & ~small], m[key][ss & ~small], "reproject %s" % key), kappa(g[ss & small], m[key + "1"][ss & small], "reproject %s (Z := 1)" % key))
        amb = ~ss
        if bool(amb.any()):
            gd = g[amb].double()
            e0 = (gd - m[key].v[amb]).abs() <= m[key].b[amb]
            e1 = (gd - m[key + "1"].v[amb]).abs() <= m[key + "1"].b[amb]
            assert bool((e0 | e1).all()), "reproject: an ambiguous pixel matches neither branch"
    vd, vs = gm.decide(m["Z"], gm.REPROJ_VALID, ">")
    va = va.cpu().reshape(E, -1)
    assert bool(((va == 0) | (va == 1)).all())
    assert torch.equal((va > 0)[vs], vd[vs]), "reproject valid: %d sure decisions differ" % int(((va > 0) != vd)[vs].sum())
    return w, int((~ss).sum() + (~vs).sum())


def check_frame_distance(c, got, beta, what, sel=None):
    """`got` holds the distances of all pairs, or of the pairs `sel` when it is given"""
    fd = gm.frame_distance(c["poses"], c["disps"], c["intr"], c["ii"], c["jj"], beta)
    if sel is not None:
        fd = dict(ratio=fd["ratio"][sel], dist=fd["dist"][sel], amb=fd["amb"][sel])
    got = got.cpu().double()
    far, fs = gm.decide(fd["ratio"], gm.FRAC, "<")
    assert bool((got[fs & far] == 1000).all()), "%s: a sure 1000 is not" % what
    near = fs & ~far
    w = kappa(got[near], fd["dist"][near], what)
    amb = ~fs
    if bool(amb.any()):
        d = fd["dist"][amb]
        assert bool(((got[amb] == 1000) | ((got[amb] - d.v).abs() <= d.b)).all()), what
    return w, int(amb.sum() + fd["amb"].sum())


def check_depth_filter(c, got):
    s, p, amb = gm.depth_filter(c["poses"], c["disps"], c["intr"], c["df_ix"], c["df_thresh"])
    got = got.cpu().double()
    assert bool((got == torch.round(got)).all())
    bad = (got < s) | (got > p)
    assert not bool(bad.any()), "depth_filter: %d counts outside [sure, sure + ambiguous]" % int(bad.sum())
    return 0.0, int((p - s).sum())


def _placed(c):
    return len(c["target_z"]) if "target_z" in c else 0


@pytest.mark.parametrize("name", gc.CASES + ["many_edges"])
def test_geometry_kernels_against_fp64(capi, name):
    c = gc.case(name)
    d = to_dev(c)
    N, ht, wd = c["disps"].shape
    stats = {}
    co, va = c_projmap(capi, d, d["ii"], d["jj"])
    rc, rv = c_reproject(capi, d, d["ii"], d["jj"])
    pts = c_iproj(capi, d)
    cnt = c_depth_filter(capi, d, d["df_ix"], d["df_thresh"])
    dists = {b: c_frame_distance(capi, d, d["ii"], d["jj"], b) for b in c["betas"]}
    if ht * wd == 0:
        for t in (co, va, rc, rv, pts, cnt):
            assert t.numel() == 0
        for b, t in dists.items():
            assert bool((t == 1000).all()), "frame_distance at hw = 0 must be 1000"
        return
    stats["projmap"] = check_projmap(c, co, va)
    stats["reproject"] = check_reproject(c, rc, rv)
    P = gm.iproj(c["poses"], c["disps"], c["intr"])
    pc = pts.cpu().reshape(N, -1, 3)
    stats["iproj"] = (max(kappa(pc[..., k], P[k], "iproj %d" % k) for k in range(3)), 0)
    w, a = 0.0, 0
    for b, t in dists.items():
        wb, ab = check_frame_distance(c, t, b, "frame_distance beta=%g" % b)
        w, a = max(w, wb), a + ab
    stats["frame_distance"] = (w, a)
    stats["depth_filter"] = check_depth_filter(c, cnt)
    placed = _placed(c)
    E, B, hw = len(c["ii"]), len(c["df_ix"]), ht * wd
    decisions = {"projmap": 2 * E * hw, "reproject": 2 * E * hw, "iproj": 0, "frame_distance": 2 * E * hw * len(c["betas"]),
                 "depth_filter": 6 * B * hw}
    for k, (w, amb) in stats.items():
        _report(k, name, dict(kappa=w, ambiguous=amb, placed=placed, decisions=decisions[k]))
        assert amb <= placed + allowance(decisions[k], 32 if k == "depth_filter" else 1000), (k, amb, placed, decisions[k])


@pytest.mark.parametrize("name", ["s43x70", "hw257", "thresholds", "df_num7", "nonfinite"])
def test_n_edge_call_equals_one_edge_calls(capi, name):
    d = to_dev(gc.case(name))
    E = len(d["ii"])
    co, va = c_projmap(capi, d, d["ii"], d["jj"])
    rc, rv = c_reproject(capi, d, d["ii"], d["jj"])
    cnt = c_depth_filter(capi, d, d["df_ix"], d["df_thresh"])
    fd = c_frame_distance(capi, d, d["ii"], d["jj"], 0.3)
    for e in range(E):
        a, b = c_projmap(capi, d, d["ii"][e:e + 1], d["jj"][e:e + 1])
        same_bits(a[0], co[e], "projmap coords edge %d" % e); same_bits(b[0], va[e], "projmap valid edge %d" % e)
        a, b = c_reproject(capi, d, d["ii"][e:e + 1], d["jj"][e:e + 1])
        same_bits(a[0], rc[e], "reproject coords edge %d" % e); same_bits(b[0], rv[e], "reproject valid edge %d" % e)
        same_bits(c_frame_distance(capi, d, d["ii"][e:e + 1], d["jj"][e:e + 1], 0.3), fd[e:e + 1], "frame_distance pair %d" % e)
    for r in range(len(d["df_ix"])):
        same_bits(c_depth_filter(capi, d, d["df_ix"][r:r + 1], d["df_thresh"][r:r + 1])[0], cnt[r], "depth_filter row %d" % r)
    pts = c_iproj(capi, d)
    one = c_iproj(capi, d, n=1)
    same_bits(one[0], pts[0], "iproj frame 0")


# ---- motion features and write-back ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["s43x70", "hw257", "s7x1", "thresholds", "nonfinite"])
@pytest.mark.parametrize("rows", ["identity", "perm", "repeat"])
def test_motion_features_are_reproject_gathered(capi, name, rows):
    c = gc.case(name)
    d = to_dev(c)
    N, ht, wd = c["disps"].shape
    E, hw = len(c["ii"]), ht * wd
    g = torch.Generator().manual_seed(7)
    if rows == "identity":
        ei, idx = None, torch.arange(E)
    elif rows == "perm":
        idx = torch.randperm(E, generator=g)[:max(1, E - 1)]
        ei = idx.to(dev)
    else:
        idx = torch.randint(0, E, (E + 2,), generator=g)
        idx[1] = idx[0]
        ei = idx.to(dev)
    R = len(idx)
    target = (wd * torch.rand(E, ht, wd, 2, generator=g)).float().to(dev)
    target.view(-1)[:3] = torch.tensor([float("nan"), 1e6, -1e6])
    co, cot, mo = Guarded(R, ht, wd, 2, dtype=torch.float32), Guarded(R, 2, ht, wd, dtype=torch.float32), Guarded(R, 4, ht, wd, dtype=torch.float32)
    c_api.check(capi.dba_motion_features(ptr(d["poses"]), ptr(d["disps"]), ptr(d["intr_pf"]), ptr(d["ii"]), ptr(d["jj"]), ptr(ei), ptr(target),
                                         ptr(co.t), ptr(cot.t), ptr(mo.t), R, ht, wd, stream()), "motion_features")
    torch.cuda.synchronize()
    for b, w in ((co, "coords"), (cot, "coords_t"), (mo, "motn")):
        b.check_guards("motion_features " + w)
    rc, _ = c_reproject(capi, d, d["ii"], d["jj"])
    same_bits(co.t, rc[idx.to(dev)], "motion_features coords vs reproject")
    same_bits(cot.t, co.t.permute(0, 3, 1, 2), "coords_t vs coords")
    i, j = torch.meshgrid(torch.arange(ht, dtype=torch.float32, device=dev), torch.arange(wd, dtype=torch.float32, device=dev), indexing="ij")
    grid = torch.stack([j, i], -1)
    want = torch.cat([co.t - grid, target[idx.to(dev)] - co.t], -1).clamp(-64, 64).permute(0, 3, 1, 2)
    same_bits(mo.t, want, "motn")


def _wb_call(L, w, d, out, ep):
    ht, wd = w["ht"], w["wd"]
    n = w["delta"].shape[0]
    c_api.check(L.dba_graph_writeback(ptr(d["delta"]), ptr(d["weight"]), ptr(d["coords"]), ptr(d.get("edge_index")), n,
                                      ptr(out["target"].t), ptr(out["weight"].t), ptr(out["ba_target"].t), ptr(out["ba_weight"].t), w["n_inactive"],
                                      ptr(d["eta"]), ptr(d["src_frames"]), len(w["src_frames"]), ptr(out["damping"].t),
                                      ptr(d["ba_frames"]), len(w["ba_frames"]), ptr(out["ba_damping"].t), ep, ht, wd, stream()), "graph_writeback")
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", list(gc.WRITEBACK))
def test_graph_writeback_is_the_fp32_restatement(capi, name):
    w = gc.writeback(name)
    ht, wd, G, ni, F = w["ht"], w["wd"], w["n_graph"], w["n_inactive"], w["n_frames"]
    hw = ht * wd
    d = to_dev({k: v for k, v in w.items() if v is not None})
    out = {"target": Guarded(G, ht, wd, 2, dtype=torch.float32), "weight": Guarded(G, ht, wd, 2, dtype=torch.float32),
           "ba_target": Guarded(ni + G, 2, ht, wd, dtype=torch.float32), "ba_weight": Guarded(ni + G, 2, ht, wd, dtype=torch.float32),
           "damping": Guarded(F, ht, wd, dtype=torch.float32), "ba_damping": Guarded(len(w["ba_frames"]), ht, wd, dtype=torch.float32)}
    damp0 = torch.rand(F, ht, wd, generator=torch.Generator().manual_seed(3)).to(dev)
    out["damping"].t.copy_(damp0)                                   # frames src_frames does not name keep these
    before = {k: o.t.clone() for k, o in out.items()}
    ep = torch.tensor(w["ep"], dtype=torch.float32).item()
    _wb_call(capi, w, d, out, ep)
    for k, o in out.items():
        o.check_guards("graph_writeback " + k)
    n = w["delta"].shape[0]
    e = w["edge_index"] if w["edge_index"] is not None else torch.arange(n)
    e = e.to(dev)
    t = d["coords"] + d["delta"]
    named = torch.zeros(G, dtype=torch.bool, device=dev); named[e] = True
    same_bits(out["target"].t[e], t, "target"); same_bits(out["weight"].t[e], d["weight"], "weight")
    same_bits(out["ba_target"].t[ni + e], t.permute(0, 3, 1, 2), "ba_target"); same_bits(out["ba_weight"].t[ni + e], d["weight"].permute(0, 3, 1, 2), "ba_weight")
    for k, rows in (("target", ~named), ("weight", ~named)):
        same_bits(out[k].t[rows], before[k][rows], k + " rows not named")
    rest = torch.ones(ni + G, dtype=torch.bool, device=dev); rest[ni + e] = False
    for k in ("ba_target", "ba_weight"):
        same_bits(out[k].t[rest], before[k][rest], k + " rows not named")
    damp = damp0.clone()
    if len(w["src_frames"]):
        damp[d["src_frames"]] = d["eta"]
    same_bits(out["damping"].t, damp, "damping")
    if len(w["ba_frames"]):
        same_bits(out["ba_damping"].t, damp[d["ba_frames"]] * torch.tensor(0.2, dtype=torch.float32) + ep, "ba damping gather")
    else:
        same_bits(out["ba_damping"].t, before["ba_damping"], "ba damping untouched")


# ---- cvx_upsample -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", gc.UPSAMPLE)
def test_cvx_upsample_against_fp64(capi, name):
    dsp, m = gc.upsample_case(name)
    n, ht, wd = dsp.shape
    out = Guarded(n, 8 * ht, 8 * wd, dtype=torch.float32)
    dt = c_api.DBA_F16 if m.dtype == torch.float16 else c_api.DBA_F32
    dd, md = dsp.to(dev), m.to(dev)
    c_api.check(capi.dba_cvx_upsample(ptr(dd), ptr(md), ptr(out.t), n, ht, wd, dt, stream()), "cvx_upsample")
    torch.cuda.synchronize()
    out.check_guards("cvx_upsample")
    ref, b = gm.cvx_upsample(dsp, m)
    w = kappa(out.t, gm.R(ref, b), "cvx_upsample " + name)
    if name in ("up_equal", "up_ties", "up_dominant"):
        same_bits(out.t, gm.cvx_upsample_f32(dsp, m), "cvx_upsample " + name + " (exps exactly 0 or 1)")
    _report("cvx_upsample", name, dict(kappa=w, ambiguous=0, placed=0))


# ---- the reference build at these edges -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", mk.GEOMETRY_EDGE_CASES)
def test_reference_build_at_the_edges(backends, gold, name):
    out = mk.geometry_edges_case(backends, dev, name)
    c = gc.case(name)
    for k, v in out.items():
        key = "geometry_edges/%s/%s" % (name, k)
        rec = gold[key]
        if k.startswith("frame_distance"):
            beta = float(k.split("=")[1])
            assert rec["n"] == v.numel(), (key, rec["n"], v.numel())
            sel = mk.fd_sample_index(rec["n"])
            check_frame_distance(c, rec["val"], beta, "reference frame_distance beta=%g" % beta, sel)
            check_frame_distance(c, v, beta, "frame_distance beta=%g" % beta)
        else:
            assert tuple(v.shape) == rec["shape"], (key, tuple(v.shape), rec["shape"])
            assert mk.digest(v) == rec["sha256"], "%s: not bit-identical to the reference build" % key
