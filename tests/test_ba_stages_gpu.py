"""Every stage of the native bundle adjustment against fp64, on every Schur route, pixels-per-thread variant and window edge
(case builders and references: tests/test_ba_stages_cpu.py).

The C entry points run one stage at a time: `dba_ba_prepare` once, then per Gauss-Newton iteration `dba_ba_build` (the reduced
system is read from the workspace), `dba_ba_solve`, and `dx_out`, `dz_out`, poses and inverse depths are read.  Each stage is compared
with fp64 computed from the native state at the start of its iteration, so errors do not compound.

Bounds, each a normalised error:
  system  entry (i, j) of the lower triangle over sqrt(A_ii A_jj), A the fp64 pose blocks before the Schur complement (by
          Cauchy-Schwarz this bounds the summed magnitude of every A and S term); b_i over sqrt(A_ii chi2), chi2 the fp64 weighted
          cost including the RGB-D prior; <= 1e-5.  A pose with no edges is exactly 0.  A motion-only build of the same state gives
          A alone, held to the same bound.
  solve   dx against an fp64 solve of the native system (lower triangle, damped with the fp32 lm / ep): <= 1e-6 max|x|.
  backsub dz against fp64 Q (w - E^T dx_native) over Q (w_mag + sum |E_c dx_c|) per pixel: <= 1e-5, w_mag the magnitude of the
          operands of w (its terms in absolute value, each residual counted as |r| + |target|, the prior's d - d_sens as
          |d| + |d_sens|).  |w| itself is not a scale for the fp32 error: the terms of w cancel, and measured against Q (|w| + ...)
          the error reaches 1.1e-2 of it (empty_window), and 1.7e3 where the RGB-D prior's d - d_sens cancels (window_stereo_rgbd).
          The inverse depths of depth frames become exactly disps + dz, every other frame is untouched.
  retract window poses against the fp64 retraction of dx_native: <= 1e-6 (1 + |t|); poses outside [t0, t1) are untouched.

Worst observed on one H100 80GB HBM3 at a 400 W power limit (system / motion-only A / solve / backsub / retract), per case, with
the Schur routes and the pixels per thread (ppt) of the build that the case takes; boundary_48x64 and degree_254_8x12 (* below) were
taken again on one H100 80GB HBM3 at a 700 W power limit once their frames above 100 rows ran in pair mode:
  boundary_48x64 *           5.8e-07 / 5.5e-07 / 3.0e-08 / 3.1e-06 / 1.0e-07  (packed, single, pair up to 255 rows; ppt 2)
  mixed_47x63_nan_ws         5.2e-07 / 6.0e-07 / 5.2e-08 / 3.6e-06 / 6.2e-08  (packed, single, pair; ppt 2)
  mixed_7x9                  1.6e-07 / 1.7e-07 / 3.0e-08 / 1.1e-06 / 7.4e-08  (packed, single, pair; ppt 1)
  mixed_3x5                  1.7e-07 / 1.7e-07 / 3.7e-08 / 6.7e-07 / 5.0e-08  (packed, single, pair; ppt 1)
  mixed_72x96                3.4e-07 / 4.3e-07 / 4.0e-08 / 5.2e-06 / 6.3e-08  (packed, single, pair; ppt 4)
  mixed_96x128               4.8e-07 / 5.2e-07 / 4.7e-08 / 2.2e-06 / 5.2e-08  (packed, single, pair; ppt 4)
  window_stereo_rgbd         9.0e-08 / 9.1e-08 / 5.4e-08 / 1.6e-06 / 4.0e-08  (packed; ppt 1)
  t0_zero_eta_one            1.6e-07 / 1.2e-07 / 3.6e-08 / 1.1e-06 / 6.8e-08  (packed; ppt 1)
  eta_by_frame_zero_weight   1.1e-07 / 1.1e-07 / 3.5e-08 / 9.0e-07 / 5.4e-08  (packed; ppt 1)
  empty_window               0 / 0 / 0 / 2.1e-06 / 0                       (no pose system; ppt 1)
  metric                     2.1e-07 / 6.7e-07 / 4.4e-08 / 6.6e-07 / 8.0e-08  (packed; ppt 4)
  c3_global                  9.7e-07 / 3.9e-06 / 3.0e-08 / 3.4e-06 / 1.2e-07  (packed; ppt 4)
  degree_254_8x12 *          1.1e-07 / 1.9e-07 / 3.7e-08 / 3.5e-07 / 6.3e-08  (packed, pair (255 rows); ppt 1)
"""
import ctypes
import json
import os

import pytest
import torch

from droid_slam_b200 import c_api
from test_ba_stages_cpu import (CASES, make_case, eta_for_kx, ref_system, ref_solve, ref_backsub, ref_retract, degree_graph)
from droid_slam_b200 import synth

pytestmark = pytest.mark.gpu
dev = "cuda"

BOUND = dict(system=1e-5, motion_only=1e-5, solve=1e-6, backsub=1e-5, retract=1e-6)


class StageDriver:
    """one native BA call driven stage by stage through the C ABI"""

    def __init__(self, L, s):
        self.L, self.s = L, s
        g = lambda k: s[k].to(dev).contiguous()
        self.poses, self.disps = g("poses"), g("disps")
        self.intr, self.ds, self.tg, self.wt, self.eta = g("intrinsics"), g("disps_sens"), g("targets"), g("weights"), g("eta")
        self.ii, self.jj = g("ii"), g("jj")
        N, ht, wd = self.disps.shape
        E = self.ii.shape[0]
        self.t0, self.t1 = s["t0"], s["t1"]
        self.P, self.n = self.t1 - self.t0, 6 * (self.t1 - self.t0)
        self.M = int(s["kx"].numel())
        ws_bytes = L.dba_ba_workspace_bytes(N, E, ht, wd, self.t0, self.t1)
        self.ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        if s["ws_fill"] is not None:
            self.ws.fill_(s["ws_fill"])
        self.off = L.dba_ba_system_offset(N, E, ht, wd, self.t0, self.t1)
        self.dx = torch.full((max(self.P, 1), 6), float("nan"), device=dev)
        self.dz = torch.full((self.M, ht * wd), float("nan"), device=dev)
        self.a = c_api.ba_args(self.poses, self.disps, self.intr, self.ds, self.tg, self.wt, self.eta, self.ii, self.jj, self.t0, self.t1,
                               s["lm"], s["ep"], self.dx, self.dz, self.ws, torch.cuda.current_stream().cuda_stream,
                               eta_by_frame=s["eta_by_frame"])

    def call(self, fn):
        c_api.check(getattr(self.L, fn)(ctypes.byref(self.a)), fn)

    def system(self):
        buf = self.ws[self.off:self.off + 8 * (self.n * self.n + self.n)].view(torch.float64).clone()
        return buf[:self.n * self.n].reshape(self.n, self.n), buf[self.n * self.n:]

    def build(self, motion_only=False):
        self.a.motion_only = int(motion_only)
        self.call("dba_ba_build")
        self.a.motion_only = 0
        return self.system()

    def status(self):
        m, st = ctypes.c_int(0), ctypes.c_int(0)
        c_api.check(self.L.dba_ba_read_info(ctypes.byref(self.a), ctypes.byref(m), ctypes.byref(st)), "dba_ba_read_info")
        return m.value, st.value


def _lower_err(Hn, Href, scale):
    """max over the lower triangle of |Hn - Href| / scale; entries with scale 0 must match exactly (inf otherwise)"""
    low = torch.tril(torch.ones_like(Href, dtype=torch.bool))
    d = (Hn - Href).abs()
    nz = low & (scale > 0)
    assert bool((d[low & (scale == 0)] == 0).all()), "entries of a pose without edges are not exactly 0"
    return float((d[nz] / scale[nz]).max()) if bool(nz.any()) else 0.0


def run_stages(L, s):
    """all stage checks of one case; returns the worst normalised error per stage"""
    drv = StageDriver(L, s)
    t0, t1, P = drv.t0, drv.t1, drv.P
    worst = dict(system=0.0, motion_only=0.0, solve=0.0, backsub=0.0, retract=0.0, backsub_over_abs_w=0.0)
    drv.call("dba_ba_prepare")
    eta = eta_for_kx(dict(s, eta=drv.eta))
    kx = s["kx"].to(dev)
    other = torch.ones(drv.disps.shape[0], dtype=torch.bool, device=dev)
    other[kx] = False
    with torch.device(dev):
        for it in range(s["itrs"]):
            p0, d0 = drv.poses.clone(), drv.disps.clone()
            ref = ref_system(p0, d0, drv.intr, drv.ds, drv.tg, drv.wt, eta, drv.ii, drv.jj, t0, t1)
            if P > 0:
                A_n, bA_n = drv.build(motion_only=True)
            H_n, b_n = drv.build()
            drv.call("dba_ba_solve")
            torch.cuda.synchronize()
            if P > 0:
                dA = ref["A"].diagonal().clamp(min=0)
                scale = torch.sqrt(dA[:, None] * dA[None, :])
                bscale = torch.sqrt(dA * ref["chi2"])
                assert bool((b_n[bscale == 0] == 0).all()) and bool((bA_n[bscale == 0] == 0).all())
                nzb = bscale > 0
                e_sys = max(_lower_err(H_n, ref["H"], scale), float(((b_n - ref["b"]).abs()[nzb] / bscale[nzb]).max()))
                e_mo = max(_lower_err(A_n, ref["A"], scale), float(((bA_n - ref["bA"]).abs()[nzb] / bscale[nzb]).max()))
                x = ref_solve(H_n, b_n, s["lm"], s["ep"])
                dx_n = drv.dx[:P].double().reshape(-1)
                e_solve = float((dx_n - x).abs().max()) / max(float(x.abs().max()), 1e-30)
                pref = ref_retract(drv.dx[:P], p0[t0:t1])
                tol = 1.0 + pref[:, :3].norm(dim=1, keepdim=True)
                e_retr = float(((drv.poses[t0:t1].double() - pref).abs() / tol).max())
            else:
                e_sys = e_mo = e_solve = e_retr = 0.0
                dx_n = torch.zeros(0, dtype=torch.float64)
            dz_ref, dz_scale = ref_backsub(ref["aux"], dx_n, P, w_mag=ref["w_mag"])
            d = (drv.dz.double() - dz_ref).abs()
            assert bool((d[dz_scale == 0] == 0).all()), "dz is not 0 at a pixel whose Q is 0"
            e_bs = float((d[dz_scale > 0] / dz_scale[dz_scale > 0]).max())
            _, abs_w_scale = ref_backsub(ref["aux"], dx_n, P)       # Q (|w| + ...): not a bound where the terms of w cancel; reported only
            worst["backsub_over_abs_w"] = max(worst["backsub_over_abs_w"], float((d[abs_w_scale > 0] / abs_w_scale[abs_w_scale > 0]).max()))
            got = dict(system=e_sys, motion_only=e_mo, solve=e_solve, backsub=e_bs, retract=e_retr)
            for k, v in got.items():
                assert v <= BOUND[k], ("iteration", it, k, v, got)
                worst[k] = max(worst[k], v)
            # inverse depths: disps + dz on depth frames, bit for bit; nothing else moves
            assert torch.equal(drv.disps[kx], (d0[kx].reshape(drv.M, -1) + drv.dz).reshape(drv.M, *d0.shape[1:])), "disps != disps + dz"
            assert torch.equal(drv.disps[other], d0[other])
            assert torch.equal(drv.poses[:t0], p0[:t0]) and torch.equal(drv.poses[t1:], p0[t1:])
    m, st = drv.status()
    assert m == drv.M and st == 0, (m, st)
    return worst


def _report(name, worst):
    print("BA_STAGES %s %s" % (name, json.dumps({k: float("%.3g" % v) for k, v in worst.items()})))
    out = os.environ.get("BA_STAGES_REPORT")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(dict(case=name, **worst)) + "\n")


@pytest.mark.parametrize("name", list(CASES))
def test_ba_stages_match_fp64(capi, name):
    s = make_case(name)
    _report(name, run_stages(capi, s))


def test_ba_empty_window_updates_inverse_depths(backends):
    """t0 == t1 with depths: no pose moves, the inverse depths still take dz = Q w, like the reference"""
    s = make_case("empty_window")
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    dx, dz = backends.ba(P, D, *args, s["t0"], s["t1"], 1, s["lm"], s["ep"], False)
    assert dx.shape == (0, 6) and dz.shape == (s["M"], 24 * 32) and bool(torch.isfinite(dz).all())
    assert torch.equal(P.cpu(), s["poses"])
    assert torch.equal(D.cpu(), s["disps"] + dz.cpu().reshape(D.shape)) and float(dz.abs().max()) > 0.1


def _degree_scene(deg):
    ii, jj = degree_graph(deg=deg)
    return synth.make_scene(dict(E=len(ii), N=30, ht=8, wd=12, stereo=False, itrs=1, lm=1e-4, ep=0.1, graph=(ii, jj)), seed=9)


def test_ba_more_than_254_out_edges_raises_before_modifying(backends):
    s = _degree_scene(255)
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    with pytest.raises(RuntimeError, match="254 out-edges"):
        backends.ba(P, D, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    torch.cuda.synchronize()
    assert torch.equal(P.cpu(), s["poses"]) and torch.equal(D.cpu(), s["disps"])
    # motion-only runs no Schur complement and has no degree limit
    dx, _ = backends.ba(P, D, *args, s["t0"], s["t1"], 1, s["lm"], s["ep"], True)
    assert bool(torch.isfinite(dx).all()) and not torch.equal(P.cpu(), s["poses"]) and torch.equal(D.cpu(), s["disps"])


def test_ba_254_out_edges_passes_every_stage(capi):
    s = _degree_scene(254)
    s.update(itrs=1, eta_by_frame=False, ws_fill=None, kx=torch.unique(torch.cat([torch.arange(s["t0"], s["t1"]), s["ii"]])))
    _report("degree_254_8x12", run_stages(capi, s))
