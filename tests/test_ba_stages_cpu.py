"""Bundle adjustment stage by stage: the case builders and fp64 stage references that tests/test_ba_stages_gpu.py checks the native
kernels with, and the CPU tests that pin them.

Each Gauss-Newton iteration of the native `ba` is four stages: build the reduced pose system (pose blocks A minus the Schur complement S
of the inverse-depth blocks), solve it, back-substitute the inverse-depth updates, retract the poses.  The references below evaluate
each stage in fp64 from the native state at the start of that iteration, so a failing check names its stage.

The Schur complement of a depth frame runs on one of three 3xTF32 tensor-core routes, chosen by its row count (its own pose if it is
in [t0, t1), plus one row per out-edge whose target is in [t0, t1)): packed tiles up to 10 rows, one tile up to 21, pairs of 10-row
tiles above that, up to 255 rows (45 CTAs per frame, each running every 45th pair: one pair per CTA up to 100 rows, several above).
The build kernel runs at 1, 2 or 4 pixels per thread (`ppt` below)."""
import torch

import oracle
from droid_slam_b200 import synth

SMS_H100 = 132            # streaming multiprocessors of an H100 SXM
BUILD_THREADS = 256       # threads per CTA of ba_build_kernel
ALPHA = float(torch.tensor(0.05, dtype=torch.float32))      # weight of the RGB-D prior, a C float in the reference


def rows_per_frame(ii, jj, N, t0, t1):
    """Schur rows of every frame: its own pose if the frame is in [t0, t1), plus one per out-edge whose target is in [t0, t1)"""
    rows = torch.zeros(N, dtype=torch.long)
    rows[t0:t1] += 1
    keep = (jj >= t0) & (jj < t1)
    rows.index_add_(0, ii[keep], torch.ones(int(keep.sum()), dtype=torch.long))
    return rows


def route(rows, deg):
    """Schur kernel of a depth frame with `rows` rows and `deg` out-edges (dba_ba_build's routing table); None: nothing to subtract"""
    if deg == 0 or rows == 0:
        return None
    return "packed" if rows <= 10 else "single" if rows <= 21 else "pair"


def ppt(N, HW, sms=SMS_H100):
    """pixels per thread of ba_build_kernel: 4 when N frames x ceil(HW / (4 * 256)) pixel chunks reach one CTA per SM, else 2 when
    N x ceil(HW / (2 * 256)) do, else 1 (N is the frame count of the call, not the depth-frame count)"""
    cdiv = lambda a, b: (a + b - 1) // b
    return 4 if N * cdiv(HW, 4 * BUILD_THREADS) >= sms else 2 if N * cdiv(HW, 2 * BUILD_THREADS) >= sms else 1


# ---- graphs ---------------------------------------------------------------------------------------------------------------------------
def _sliding(N, skip=()):
    return [(i, j) for i in range(N) if i not in skip for j in (i - 2, i - 1, i + 1, i + 2) if 0 <= j < N]


def _targets(f, n, lo, hi):
    """n out-edge targets of frame f within 12 frames and inside [lo, hi): the first target twice at the start (a repeat inside one
    row tile) and once more at the end (a repeat in another tile), the rest cycling through the neighbourhood"""
    nb = [j for j in range(max(lo, f - 12), min(hi, f + 13)) if j != f]
    if n < 2:
        return nb[:n]
    return [nb[0]] + [nb[k % len(nb)] for k in range(n - 2)] + [nb[0]]


def boundary_graph(N=40):
    """frames whose row count sits on each side of every route switch, t0 = 1, and on each side of the pair kernel's one pair per CTA.
    Frames 12 and 20 have out-edges into frame 0, which is outside the window, so their degree exceeds their row count - 1: frame 12
    has 21 rows but 22 out-edges (it is in the pair kernel's frame list and is left to the single-tile kernel), frame 20 has 100 rows
    and 100 out-edges (45 tile pairs, one per CTA).  Frame 24 has 101 rows (55 pairs: a second pair for 10 CTAs), frame 32 has 136 rows
    (14 tiles, 91 pairs = 2 x 45 + 1: a partial last round), frame 28 has 254 out-edges: 255 rows, the most a frame may have
    (325 pairs, up to 8 per CTA)."""
    want = {5: 10, 8: 11, 12: 21, 16: 22, 20: 100, 24: 101, 28: 255, 32: 136}
    extra_out = {12: 2, 20: 1}
    e = _sliding(N, skip=want)
    for f, r in want.items():
        e += [(f, j) for j in _targets(f, r - 1, 1, N)] + [(f, 0)] * extra_out.get(f, 0)
    return [a for a, _ in e], [b for _, b in e], want


def mixed_graph(N=34):
    """frames with 3-5 rows (packed), 16 rows (single tile) and 25 rows (tile pairs), plus a duplicated edge"""
    e = _sliding(N)
    e += [(17, j) for j in range(5, 30) if abs(j - 17) > 2]
    e += [(26, j) for j in range(18, 34) if abs(j - 26) > 2]
    e += [(9, 10)]
    return [a for a, _ in e], [b for _, b in e]


def window_graph(N=20):
    """t0 = 5, t1 = 14: fixed frames with edges into the window and window frames with edges to fixed frames, frames >= t1 with edges
    among themselves and into the window, window frame 9 without out-edges, window frame 11 in no edge at all, stereo edges (i, i)"""
    e = [(i, j) for i, j in _sliding(N) if i != 9 and 11 not in (i, j)]
    e += [(2, 7), (7, 2), (12, 3), (16, 12), (12, 17), (15, 18), (18, 15)]
    e += [(i, i) for i in (3, 6, 10, 15)]
    return [a for a, _ in e], [b for _, b in e]


def degree_graph(N=30, f=10, deg=255):
    """frame f with `deg` out-edges, all inside the window"""
    e = _sliding(N, skip=(f,)) + [(f, j) for j in _targets(f, deg, 1, N)]
    return [a for a, _ in e], [b for _, b in e]


# name -> scene parameters.  eta: "rows" (one row per depth frame), "one" (one broadcast row) or "frame" (one row per frame, eta_by_frame);
# zero_frame: a frame whose out-edges carry no weight and whose eta row is 0 (C = 0: Q = 0 and dz = 0 there); itrs: Gauss-Newton iterations
CASES = {
    "boundary_48x64": dict(graph=boundary_graph, N=40, ht=48, wd=64, itrs=2, seed=3),
    "mixed_47x63_nan_ws": dict(graph=mixed_graph, N=34, ht=47, wd=63, ws_fill=255, seed=1),
    "mixed_7x9": dict(graph=mixed_graph, N=34, ht=7, wd=9, seed=1),
    "mixed_3x5": dict(graph=mixed_graph, N=34, ht=3, wd=5, seed=1),
    "mixed_72x96": dict(graph=mixed_graph, N=34, ht=72, wd=96, itrs=2, seed=1),
    "mixed_96x128": dict(graph=mixed_graph, N=34, ht=96, wd=128, itrs=2, seed=1),
    "window_stereo_rgbd": dict(graph=window_graph, N=20, ht=24, wd=32, t0=5, t1=14, rgbd=True, seed=4),
    "t0_zero_eta_one": dict(graph=lambda: _list(_sliding(14)), N=14, ht=24, wd=32, t0=0, eta="one", seed=5),
    "eta_by_frame_zero_weight": dict(graph=lambda: _list(_sliding(16)), N=16, ht=24, wd=32, t0=2, eta="frame", zero_frame=6, seed=6),
    "empty_window": dict(graph=lambda: _list(_sliding(5)), N=5, ht=24, wd=32, t0=3, t1=3, seed=0),
    "metric": dict(config="metric", itrs=1),
    "c3_global": dict(config="c3_global", itrs=1),
}


def _list(e):
    return [a for a, _ in e], [b for _, b in e]


def case_graph(name):
    """(ii, jj, N, ht, wd, t0, t1) of a case without generating its pixels"""
    c = CASES[name]
    if "config" in c:
        cfg = synth.CONFIGS[c["config"]]
        ii, jj = synth.make_graph(cfg["E"], cfg["N"], stereo=cfg["stereo"])
        return ii, jj, cfg["N"], cfg["ht"], cfg["wd"], 1, cfg["N"]
    g = c["graph"]()
    ii, jj = torch.tensor(g[0]), torch.tensor(g[1])
    return ii, jj, c["N"], c["ht"], c["wd"], c.get("t0", 1), c.get("t1", c["N"])


def make_case(name):
    """the scene of a case (synth.make_scene) with its eta layout and zero-weight frame applied; adds eta_by_frame and ws_fill"""
    c = CASES[name]
    if "config" in c:
        s = synth.make_scene(c["config"])
    else:
        ii, jj, N, ht, wd, t0, t1 = case_graph(name)
        s = synth.make_scene(dict(E=len(ii), N=N, ht=ht, wd=wd, stereo=False, itrs=c.get("itrs", 3), lm=1e-4, ep=0.1,
                                  graph=(ii, jj), t0=t0, t1=t1), seed=c.get("seed", 0), rgbd=c.get("rgbd", False))
    s["itrs"] = c.get("itrs", 3)
    N, ht, wd = s["disps"].shape
    kx = torch.unique(torch.cat([torch.arange(s["t0"], s["t1"]), s["ii"]]))
    eta_mode = c.get("eta", "rows")
    g = torch.Generator().manual_seed(77)
    if eta_mode == "one":
        s["eta"] = s["eta"][:1].contiguous()
    elif eta_mode == "frame":
        s["eta"] = (0.002 * torch.rand(N, ht, wd, generator=g) + 1e-7).contiguous()
    s["eta_by_frame"] = eta_mode == "frame"
    zf = c.get("zero_frame")
    if zf is not None:
        assert s["eta_by_frame"] and not bool((s["disps_sens"][zf] > 0).any())
        s["weights"][s["ii"] == zf] = 0.0
        s["eta"][zf] = 0.0
    s["kx"] = kx
    s["ws_fill"] = c.get("ws_fill")
    return s


def eta_for_kx(s):
    """eta as the reference lays it out: one row per depth frame (or one broadcast row)"""
    return s["eta"][s["kx"].to(s["eta"].device)] if s["eta_by_frame"] else s["eta"]


# ---- fp64 stage references ------------------------------------------------------------------------------------------------------------
def ref_system(poses, disps, intr, disps_sens, targets, weights, eta, ii, jj, t0, t1):
    """fp64 reduced system of the state (poses, disps).  Returns dict: H, b (after the Schur complement), A, bA (pose blocks alone,
    what a motion-only build gives), chi2 (weighted cost including the RGB-D prior term), w_mag (the
    magnitude of the operands of w [M, HW]: its terms in absolute value, each residual counted as |r| + |target| and the prior's
    d - d_sens as |d| + |d_sens|) and aux (C, w, Q, E rows, ... of
    oracle.ba_system).  Pixels with C <= 0 get Q = 0 (INTEGRATION.md section 5); the reference divides by zero there."""
    d64 = lambda x: x.double()
    p, d, ds = d64(poses), d64(disps), d64(disps_sens)
    T = oracle.ba_edge_terms(p, d, d64(intr), d64(targets), d64(weights), ii, jj)
    A, bA, _ = oracle.ba_system(T, d, ds, eta, ii, jj, t0, t1, True, torch.float64)
    H, b, aux = oracle.ba_system(T, d, ds, eta, ii, jj, t0, t1, False, torch.float64, drop_nonpositive_c=True)
    kx = aux["kx"]
    m = (ds[kx] > 0).double()
    chi2 = float(T["r2"].sum()) + float((m * ALPHA * (d[kx] - ds[kx]) ** 2).sum())
    k_of = torch.searchsorted(kx, ii)
    w_mag = torch.zeros_like(aux["w"]).index_add_(0, k_of, T["bz_mag"]) + (m * ALPHA * (d[kx].abs() + ds[kx].abs())).reshape(aux["w"].shape)
    return dict(H=H, b=b, A=A, bA=bA, chi2=chi2, w_mag=w_mag, aux=aux)


def symmetric_from_lower(H):
    return torch.tril(H) + torch.tril(H, -1).transpose(0, 1)


def ref_solve(H_lower, b, lm, ep):
    """fp64 solution of the damped system (diag += ep + lm * diag, lm and ep rounded to fp32 like the C ABI's floats), built from
    the lower triangle of H"""
    lm32 = float(torch.tensor(lm, dtype=torch.float32)); ep32 = float(torch.tensor(ep, dtype=torch.float32))
    S = symmetric_from_lower(H_lower.double())
    dg = torch.diagonal(S)
    dg += ep32 + lm32 * dg.clone()
    return torch.linalg.solve(S, b.double()[:, None])[:, 0]


def ref_backsub(aux, dx, P, w_mag=None):
    """fp64 dz = Q (w - sum of E dx) per depth frame, with quirk Q9 (rows of pose index 0 are skipped) and Q = 0 where C <= 0.
    Returns (dz [M, HW], scale [M, HW]): scale = Q (|w| + sum of |E_c dx_c|), or, given w_mag, Q (w_mag + sum of |E_c dx_c|):
    the magnitude the fp32 sums work against."""
    kx, Q, w, Er, pose = aux["kx"], aux["Q"], aux["w"], aux["Erows"], aux["pose"]
    valid = (pose > 0) & (pose < P)
    k_of = torch.searchsorted(kx, aux["ii_exp"])
    prod = Er[valid] * dx.double().reshape(-1, 6)[pose[valid]][:, :, None]           # [rows, 6, HW]
    dw = torch.zeros_like(w).index_add_(0, k_of[valid], prod.sum(1))
    mag = torch.zeros_like(w).index_add_(0, k_of[valid], prod.abs().sum(1))
    return Q * (w - dw), Q * ((w.abs() if w_mag is None else w_mag) + mag)


def ref_retract(dx, poses_window):
    """fp64 left-multiplicative retraction of the window poses [P, 7]"""
    p = poses_window.double()
    t, q = oracle.retr_se3(dx.double().reshape(-1, 6), p[:, :3], p[:, 3:])
    return torch.cat([t, q], dim=-1)


# ---- CPU tests ------------------------------------------------------------------------------------------------------------------------
def _routes_and_rows(name):
    ii, jj, N, ht, wd, t0, t1 = case_graph(name)
    rows = rows_per_frame(ii, jj, N, t0, t1)
    deg = torch.bincount(ii, minlength=N)
    routes = {route(int(rows[f]), int(deg[f])) for f in range(N)} - {None}
    return rows, deg, routes, ppt(N, ht * wd)


def test_boundary_case_has_every_row_count_switch():
    rows, deg, routes, p = _routes_and_rows("boundary_48x64")
    _, _, want = boundary_graph()
    assert {f: int(rows[f]) for f in want} == want
    assert int(deg[12]) == 22 and int(deg[20]) == 100 and int(deg[28]) == 254       # degree + 1 != rows where targets leave the window
    assert [route(int(rows[f]), int(deg[f])) for f in sorted(want)] == ["packed", "single", "single", "pair", "pair", "pair", "pair", "pair"]
    assert routes == {"packed", "single", "pair"} and p == 2
    tiles = {f: (r + 9) // 10 for f, r in want.items() if r > 21}
    assert {f: t * (t - 1) // 2 for f, t in tiles.items()} == {16: 3, 20: 45, 24: 55, 28: 325, 32: 91}
    ii, jj, *_ = case_graph("boundary_48x64")
    for f in (8, 16, 24, 28, 32):   # a target repeated inside the frame's first row tile and again in a later position
        t = jj[ii == f].tolist()
        assert t[0] == t[1] == t[-1]


def test_cases_cover_pixels_per_thread_and_routes():
    got = {name: _routes_and_rows(name)[2:] for name in CASES}
    assert got["mixed_47x63_nan_ws"] == ({"packed", "single", "pair"}, 2)
    assert got["mixed_7x9"] == ({"packed", "single", "pair"}, 1)
    assert got["mixed_3x5"] == ({"packed", "single", "pair"}, 1)
    assert got["mixed_72x96"] == ({"packed", "single", "pair"}, 4)
    assert got["mixed_96x128"] == ({"packed", "single", "pair"}, 4)
    assert got["metric"][1] == 4 and got["c3_global"][1] == 4
    assert {p for _, p in got.values()} == {1, 2, 4}
    ht, wd = CASES["mixed_3x5"]["ht"], CASES["mixed_3x5"]["wd"]
    assert ht * wd < BUILD_THREADS and (47 * 63) % 4 != 0


def test_window_cases_have_their_edges():
    ii, jj, N, _, _, t0, t1 = case_graph("window_stereo_rgbd")
    e = set(zip(ii.tolist(), jj.tolist()))
    assert any(i < t0 <= j < t1 for i, j in e) and any(j < t0 <= i < t1 for i, j in e)        # into and out of fixed frames
    assert any(i >= t1 and j >= t1 for i, j in e) and any(i >= t1 and t0 <= j < t1 for i, j in e)
    assert 9 not in ii.tolist() and 11 not in ii.tolist() + jj.tolist()                     # no out-edges / no edges at all
    assert any(i == j for i, j in e)
    assert case_graph("t0_zero_eta_one")[5] == 0
    g = case_graph("empty_window")
    assert g[5] == g[6] == 3


def test_degree_graph_has_the_limit():
    ii, jj = (torch.tensor(x) for x in degree_graph(deg=255))
    assert int(torch.bincount(ii)[10]) == 255 and int(rows_per_frame(ii, jj, 30, 1, 30)[10]) == 256


def _chain(s, iterations):
    """the stage references chained into whole Gauss-Newton iterations"""
    poses, disps = s["poses"].double().clone(), s["disps"].double().clone()
    t0, t1 = s["t0"], s["t1"]
    P = t1 - t0
    dx = dz = None
    for _ in range(iterations):
        r = ref_system(poses, disps, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], eta_for_kx(s), s["ii"], s["jj"], t0, t1)
        dx = ref_solve(r["H"], r["b"], s["lm"], s["ep"]) if P > 0 else torch.zeros(0, dtype=torch.float64)
        dz, _ = ref_backsub(r["aux"], dx, P)
        disps[r["aux"]["kx"]] += dz.reshape(-1, *disps.shape[1:])
        poses[t0:t1] = ref_retract(dx, poses[t0:t1])
    return poses, disps, dx, dz


def _oracle(s, iterations):
    P64, D64 = s["poses"].double(), s["disps"].double()
    dx, dz = oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], eta_for_kx(s), s["ii"], s["jj"], s["t0"],
                       s["t1"], iterations, s["lm"], s["ep"], False, dtype=torch.float64)
    return P64, D64, dx, dz


def test_stage_references_chain_to_oracle_ba():
    """stereo edges, an RGB-D prior, fixed frames on both sides of the window and a pose with no edges, at 6x8"""
    c = dict(CASES["window_stereo_rgbd"], ht=6, wd=8)
    CASES["_small"] = c
    try:
        s = make_case("_small")
    finally:
        del CASES["_small"]
    P, D, dx, dz = _chain(s, 2)
    P0, D0, dx0, dz0 = _oracle(s, 2)
    assert float((P - P0).abs().max()) < 1e-12 and float((D - D0).abs().max()) < 1e-12
    assert float((dx.reshape(-1, 6) - dx0).abs().max()) < 1e-12 and float((dz - dz0).abs().max()) < 1e-12


def test_stage_references_chain_to_oracle_ba_on_an_empty_window():
    """t0 == t1: no pose moves, the inverse depths still take dz = Q w"""
    s = make_case("empty_window")
    P, D, _, dz = _chain(s, 2)
    P0, D0, _, dz0 = _oracle(s, 2)
    assert torch.equal(P, s["poses"].double()) and torch.equal(P0, P)
    assert float((D - D0).abs().max()) < 1e-12 and float((D - s["disps"].double()).abs().max()) > 0.1


def test_reduced_system_drops_pixels_without_a_depth_block():
    """a frame whose out-edges carry no weight, with eta = 0: C = 0 at every pixel, so Q = 0 and those pixels add nothing"""
    s = make_case("eta_by_frame_zero_weight")
    r = ref_system(s["poses"], s["disps"], s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], eta_for_kx(s), s["ii"], s["jj"],
                   s["t0"], s["t1"])
    aux = r["aux"]
    k = int((aux["kx"] == 6).nonzero())
    assert bool((aux["C"][k] == 0).all()) and bool((aux["Q"][k] == 0).all())
    assert bool(torch.isfinite(r["H"]).all()) and bool(torch.isfinite(r["b"]).all())
    dz, scale = ref_backsub(aux, torch.zeros(6 * (s["t1"] - s["t0"]), dtype=torch.float64), s["t1"] - s["t0"])
    assert bool((dz[k] == 0).all()) and bool((scale[k] == 0).all())
