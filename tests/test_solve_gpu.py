"""The damped fp64 pose solve (`dba_solve_spd`) through the C ABI on every route, against fp64 LAPACK (case builders, references and
criteria: tests/test_solve_cpu.py).

Every solve of the case table must give fail == 0 (4 would be a hand-over that timed out) and meet the factor criterion on the factor
the kernel leaves at the start of its workspace (row-major, leading dimension 32 nt, lower triangle), the residual criterion, and the
forward criterion where kappa is known.  The route each case took is checked on the device: the resident kernel leaves the upper tiles
of that factor unwritten (the cluster kernel zeroes them), and the cluster kernel leaves its envelope `first[]` after the factor (the
numpy restatement with the envelope on, all zeros with it off).

Every route is then solved under changed conditions -- dirty, NaN-filled and reused workspaces, a NaN or different upper triangle,
a replayed CUDA graph -- and must give the same bits; and the failure cases (non-positive, indefinite, zero, NaN and infinite pivots,
on a resident size and a cluster size each) must give fail == 1 and x = +0.0.  No input holds the resident kernel's sentinel bit
pattern.

Worst observed on one H100 80GB HBM3 at a 700 W power limit, per route (e_L / gamma, residual ratio, forward ratio, where each bound
is 1; the number of cases in brackets).  The forward ratio is bounded below 0.5 only by the rounding of x to fp32:
  resident, cluster 1      0.021 / 0.25 / 0.42   (10)
  resident, cluster 2      0.016 / 0.14 / 0.46   (4)
  resident, cluster 4      0.015 / 0.28 / 0.47   (6)
  resident, cluster 8      0.020 / 0.10 / 0.48   (10)
  resident, cluster 16     0.015 / 0.38 / 0.49   (17)
  envelope                 0.011 / 0.41 / 0.50   (21)
  dense                    0.00065 / 0.36 / 0.49 (3)
The whole file takes about a minute there.
"""
import json
import os

import numpy as np
import pytest
import torch

from droid_slam_b200 import c_api
from test_solve_cpu import (CASES, EPS32, OLD_RANDOM_N, T, cdiv, f32, factor_error, forward_ratio, lapack_solve, make_case,
                            old_random, residual_ratio, route, spectrum)
from util import ptr, stream

pytestmark = pytest.mark.gpu
dev = "cuda"
SENTINEL = np.int64(np.uint64(0xFFF7DEADBEEF5A5A).astype(np.int64))   # the resident kernel's "not written yet" bit pattern


class Solve:
    """one workspace, fail flag and output for systems of up to nmax unknowns"""

    def __init__(self, L, nmax, fill=0):
        self.L = L
        self.bytes = L.dba_solve_workspace_bytes(nmax)
        self.ws = torch.full((self.bytes,), fill, dtype=torch.uint8, device=dev)
        self.fail = torch.full((1,), 7, dtype=torch.int32, device=dev)
        self.x = torch.full((nmax,), float("nan"), device=dev)

    def launch(self, H, b, lm, ep):
        n = b.shape[0]
        c_api.check(self.L.dba_solve_spd(ptr(H), ptr(b), n, lm, ep, ptr(self.x), ptr(self.fail), ptr(self.ws), self.bytes, stream()),
                    "dba_solve_spd")

    def __call__(self, H, b, lm, ep):
        """(x [n] fp32 on the host, fail)"""
        assert not bool((H.view(torch.int64) == int(SENTINEL)).any()) and not bool((b.view(torch.int64) == int(SENTINEL)).any())
        n = b.shape[0]
        self.x.fill_(float("nan"))
        self.fail.fill_(7)
        self.launch(H, b, lm, ep)
        torch.cuda.synchronize()
        return self.x[:n].cpu().clone(), int(self.fail)

    def factor(self, n):
        """(L-hat [n, n] lower triangle valid, first[] [nt], upper tile (0, 1) still holds the workspace's fill)"""
        nt = cdiv(n, T)
        ld = nt * T
        lb = (nt + 1) * T * ld * 8
        Lw = self.ws[:lb].view(torch.float64).view((nt + 1) * T, ld)
        off = lb + (nt * T * T + nt * T) * 8
        first = self.ws[off:off + 4 * nt].view(torch.int32).cpu().numpy()
        upper = self.ws[:lb].view((nt + 1) * T, ld * 8)[:T, T * 8:2 * T * 8] if nt > 1 else None
        return Lw[:n, :n].cpu().numpy(), first, upper


def _dev(c):
    return torch.from_numpy(c["H"]).to(dev), torch.from_numpy(c["b"]).to(dev)


def _report(name, **kw):
    print("SOLVE %s %s" % (name, json.dumps({k: (float("%.3g" % v) if isinstance(v, float) else v) for k, v in kw.items()})))
    out = os.environ.get("SOLVE_REPORT")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(dict(case=name, **kw)) + "\n")


def _all_plus_zero(x):
    return torch.equal(x.view(torch.int32), torch.zeros_like(x, dtype=torch.int32))


# ---- every case meets every criterion -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_solve_meets_criteria(capi, name):
    c = make_case(name)
    n, Hd, b = c["n"], c["Hd"], c["b"]
    nt = cdiv(n, T)
    r, cs = route(n)
    H_, b_ = _dev(c)
    s = Solve(capi, n, fill=255)
    x, fail = s(H_, b_, c["lm"], c["ep"])
    del H_
    assert fail == 0, (name, fail)
    Lhat, first, upper = s.factor(n)
    # the route the device took
    if upper is not None:
        assert bool((upper == 255).all()) == (r == "resident"), (name, r)
        if r != "resident":
            assert not bool(upper.any())
    assert list(first) == (list(c["first"]) if r == "envelope" else [0] * nt), (name, r)
    del s
    xn = x.double().numpy()
    e_l = factor_error(Lhat, Hd, c["first"])
    del Lhat
    res = residual_ratio(Hd, xn, b)
    fwd = forward_ratio(xn, lapack_solve(Hd, b), c["kappa"]) if c["kappa"] is not None else None
    _report(name, route=r, cluster=cs, nt=nt, n=n, e_L=e_l, residual=res, forward=fwd)
    assert e_l <= 1 and res <= 1 and (fwd is None or fwd <= 1), (name, e_l, res, fwd)
    p = c["free_pose"]
    if p is not None:                              # a pose without edges: x = b / ep32 there
        want = b[6 * p:6 * p + 6] / f32(c["ep"])
        assert np.all(np.abs(xn[6 * p:6 * p + 6] - want) <= EPS32 * np.abs(want))


# ---- the same bits under every condition ----------------------------------------------------------------------------------------------
# one size per resident cluster size (1, 2, 4, 8, 16 CTAs), the envelope route on the arrow pattern, the dense route
BITS = ["size_32", "size_63", "size_127", "size_223", "size_426", "pattern_arrow", "size_8192"]


def _other_matrix(n, seed):
    H, b = spectrum(n, 1e2, seed)
    return torch.from_numpy(H).to(dev), torch.from_numpy(b).to(dev)


@pytest.mark.parametrize("name", BITS)
def test_solve_same_bits_under_every_condition(capi, name):
    c = make_case(name)
    n, lm, ep = c["n"], c["lm"], c["ep"]
    r, _ = route(n)
    H, b = _dev(c)
    other_n = 1000 if r == "resident" else 426                  # the other kernel
    nmax = max(n, other_n)
    x0, f0 = Solve(capi, nmax)(H, b, lm, ep)                    # clean (zeroed) workspace
    assert f0 == 0
    same = lambda got, what: (torch.equal(got[0].view(torch.int32), x0.view(torch.int32)) and got[1] == f0) or pytest.fail(what)
    s = Solve(capi, nmax)
    for k in range(3):
        same(s(H, b, lm, ep), "repeat %d" % k)
    same(Solve(capi, nmax, fill=255)(H, b, lm, ep), "workspace of 0xFF")
    Ho, bo = _other_matrix(other_n, 5)
    s = Solve(capi, nmax)
    s(Ho, bo, 1e-4, 0.1)
    same(s(H, b, lm, ep), "workspace just used with n = %d" % other_n)
    H2, b2 = 1.5 * H, b.flip(0).contiguous()                    # a different system of the same size
    s(H2, b2, lm, ep)
    same(s(H, b, lm, ep), "workspace just used by another system of the same n")
    upper = torch.triu(torch.ones(n, n, dtype=torch.bool, device=dev), 1)
    same(s(torch.where(upper, float("nan"), H), b, lm, ep), "upper triangle NaN")
    g = torch.Generator(device=dev).manual_seed(3)
    same(s(torch.where(upper, torch.randn(n, n, generator=g, device=dev, dtype=torch.float64), H), b, lm, ep), "different upper triangle")
    del upper
    # a captured graph, replayed after H and b are rewritten in place
    xe2, fe2 = Solve(capi, nmax)(H2, b2, lm, ep)
    Hg, bg = H.clone(), b.clone()
    sg = Solve(capi, nmax)
    sg(Hg, bg, lm, ep)                                          # eager first (one-time kernel attributes are set outside the capture)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sg.launch(Hg, bg, lm, ep)
    Hg.copy_(H2); bg.copy_(b2); sg.fail.fill_(7); sg.x.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(sg.x[:n].cpu().view(torch.int32), xe2.view(torch.int32)) and int(sg.fail) == fe2, "graph replay, new contents"
    Hg.copy_(H); bg.copy_(b); sg.fail.fill_(7)
    graph.replay()
    torch.cuda.synchronize()
    same((sg.x[:n].cpu(), int(sg.fail)), "graph replay, original contents")


# ---- failures and edges ---------------------------------------------------------------------------------------------------------------
FAIL_N = [320, 300, 640, 631]            # resident (nt = 10) and cluster (nt = 20) kernel, a multiple of 32 and not


def _spd(n):
    H, b = spectrum(n, 1e2, seed=1000 + n)
    return torch.from_numpy(H).to(dev), torch.from_numpy(b).to(dev)


def _expect_failure(capi, H, b, lm=0.0, ep=0.0, what=""):
    x, fail = Solve(capi, b.shape[0], fill=255)(H, b, lm, ep)
    assert fail == 1 and _all_plus_zero(x), (what, fail, x[:8])


@pytest.mark.parametrize("n", FAIL_N)
@pytest.mark.parametrize("row", ["first", "31", "32", "half", "last"])
def test_negative_pivot_fails(capi, n, row):
    """row 0 is the unrolled warp_potrf of the cluster kernel's tile 0; rows 31 / 32 are either side of a tile edge; the last row is
    followed by the padding rows when n % 32 != 0"""
    H, b = _spd(n)
    i = dict(first=0, half=n // 2, last=n - 1).get(row) if not row.isdigit() else int(row)
    H[i, i] = -1.0
    _expect_failure(capi, H, b, what=(n, i))


@pytest.mark.parametrize("n", FAIL_N)
def test_indefinite_block_with_positive_diagonal_fails(capi, n):
    H = torch.eye(n, dtype=torch.float64, device=dev)
    H[31, 32] = H[32, 31] = 2.0                                 # [[1, 2], [2, 1]] across the tile edge
    b = torch.ones(n, dtype=torch.float64, device=dev)
    _expect_failure(capi, H, b)


@pytest.mark.parametrize("n", FAIL_N)
def test_zero_row(capi, n):
    """a pose without edges: fails undamped, solves with ep > 0 (x_z = b_z / ep32 there)"""
    H, b = _spd(n)
    z = n // 2 + 3
    H[z, :] = 0.0; H[:, z] = 0.0
    _expect_failure(capi, H, b, what="zero row, lm = ep = 0")
    lm, ep = 1e-4, 0.1
    x, fail = Solve(capi, n)(H, b, lm, ep)
    assert fail == 0
    Hn, bn = H.cpu().numpy(), b.cpu().numpy()
    Hd = Hn.copy(); Hd[np.diag_indices(n)] += f32(ep) + f32(lm) * np.diagonal(Hn)
    xn = x.double().numpy()
    want = bn[z] / f32(ep)
    assert abs(xn[z] - want) <= EPS32 * abs(want)
    assert residual_ratio(Hd, xn, bn) <= 1


@pytest.mark.parametrize("n", FAIL_N)
@pytest.mark.parametrize("where", ["diagonal", "off_diagonal"])
def test_nan_in_lower_triangle_fails(capi, n, where):
    H, b = _spd(n)
    if where == "diagonal":
        H[n // 2, n // 2] = float("nan")
    else:
        H[n - 1, 1] = float("nan")
    _expect_failure(capi, H, b, what=where)


@pytest.mark.parametrize("n", FAIL_N)
def test_zero_rhs_gives_zero(capi, n):
    H, _ = _spd(n)
    x, fail = Solve(capi, n, fill=255)(H, torch.zeros(n, dtype=torch.float64, device=dev), 1e-4, 0.1)
    assert fail == 0 and bool((x == 0).all())


@pytest.mark.parametrize("n", [320, 640])
@pytest.mark.parametrize("lm,ep", [(0.0, 0.0), (1e-4, 0.1)])
def test_infinite_last_pivot_fails(capi, n, lm, ep):
    """+Inf passes a `d > 0` pivot test, and its reciprocal square root is NaN: without a finiteness test the NaN spreads into x, which
    comes out zero with fail == 0 -- a zero step that does not report the failure.  Undamped, the damping's 0 * Inf makes the pivot
    NaN instead; `ba` always damps with lm > 0, which keeps it +Inf."""
    H, b = _spd(n)
    H[n - 1, n - 1] = float("inf")
    _expect_failure(capi, H, b, lm, ep)


@pytest.mark.parametrize("n", OLD_RANDOM_N)
def test_negative_pivot_at_half_of_the_first_test_matrices(capi, n):
    """the solver's first failure check, kept on its matrices: A A^T + 1e-3 I with H[n/2, n/2] = -5, undamped"""
    H, b = old_random(n)
    H[n // 2, n // 2] = -5.0
    _expect_failure(capi, torch.from_numpy(H).to(dev), torch.from_numpy(b).to(dev))
