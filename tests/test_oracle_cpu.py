"""CPU tests (no GPU): the oracle against independent derivations, the synthetic generator, the C-ABI exports."""
import ctypes
import subprocess
import math
import os
import re

import pytest
import torch

import oracle
from droid_slam_b200 import c_api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- corr_index oracle vs a direct transcription of the kernel loops (reference src/correlation_kernels.cu:20-71) ----
def _corr_index_loops(volume, coords, r):
    N, h1, w1, h2, w2 = volume.shape
    rd = 2 * r + 1
    out = torch.zeros(N, rd, rd, h1, w1, dtype=torch.float64)
    for n in range(N):
        for y in range(h1):
            for x in range(w1):
                x0 = float(coords[n, 0, y, x]); y0 = float(coords[n, 1, y, x])
                dx = x0 - math.floor(x0); dy = y0 - math.floor(y0)
                for i in range(rd + 1):
                    for j in range(rd + 1):
                        x1 = math.floor(x0) - r + i; y1 = math.floor(y0) - r + j
                        if 0 <= y1 < h2 and 0 <= x1 < w2:
                            s = float(volume[n, y, x, y1, x1])
                            if i > 0 and j > 0: out[n, i - 1, j - 1, y, x] += s * dx * dy
                            if i > 0 and j < rd: out[n, i - 1, j, y, x] += s * dx * (1 - dy)
                            if i < rd and j > 0: out[n, i, j - 1, y, x] += s * (1 - dx) * dy
                            if i < rd and j < rd: out[n, i, j, y, x] += s * (1 - dx) * (1 - dy)
    return out


def test_corr_index_oracle_matches_kernel_loops():
    g = torch.Generator().manual_seed(0)
    vol = torch.randn(2, 3, 4, 5, 6, generator=g)
    co = torch.rand(2, 2, 3, 4, generator=g) * 9 - 2
    for r in (1, 3):
        ref = _corr_index_loops(vol, co, r)
        got, = oracle.corr_index_forward(vol.double(), co, r)
        assert torch.allclose(got, ref, atol=1e-12)
        got32, = oracle.corr_index_forward(vol, co, r)
        assert torch.allclose(got32.double(), ref, atol=1e-5)
        got16, = oracle.corr_index_forward(vol.half(), co, r)
        assert torch.allclose(got16.double(), ref, atol=2e-2)


def test_corr_index_backward_is_transpose_of_forward():
    g = torch.Generator().manual_seed(1)
    vol = torch.randn(2, 3, 4, 5, 6, generator=g, dtype=torch.float64)
    co = torch.rand(2, 2, 3, 4, generator=g) * 9 - 2
    gout = torch.randn(2, 7, 7, 3, 4, generator=g, dtype=torch.float64)
    fwd, = oracle.corr_index_forward(vol, co, 3)
    bwd, = oracle.corr_index_backward(vol, co, gout, 3)
    assert abs(float((fwd * gout).sum()) - float((vol * bwd).sum())) < 1e-9   # <A v, g> == <v, A^T g>


def test_altcorr_equals_corr_volume_lookup():
    """SURVEY.md section 4, cross-check 1: CorrBlock + corr_index == AltCorrBlock + altcorr (pooling is linear)."""
    g = torch.Generator().manual_seed(2)
    B, N, C, H, W = 1, 3, 8, 8, 8
    fmaps = torch.randn(B, N, C, H, W, generator=g, dtype=torch.float64)
    ii = torch.tensor([0, 1, 2, 0]); jj = torch.tensor([1, 2, 0, 2])
    coords = torch.rand(B, 4, H, W, 2, generator=g) * 10 - 1
    pyr = oracle.corr_pyramid(fmaps[:, ii], fmaps[:, jj], num_levels=3)
    a = oracle.corr_block_lookup(pyr, coords, radius=2)
    b = oracle.altcorr_block_lookup(oracle.fmap_pyramid(fmaps, 3), coords, ii, jj, radius=2)
    assert a.shape == b.shape
    assert torch.allclose(a, b, atol=1e-6)   # bilinear weights are fp32 products in one path, fp64 in the other


def test_altcorr_backward_matches_autograd():
    g = torch.Generator().manual_seed(3)
    B, N, C, H, W = 1, 2, 3, 4, 5
    f1 = torch.randn(B, N, C, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    f2 = torch.randn(B, N, C, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    ii = torch.tensor([0, 1]); jj = torch.tensor([1, 1])
    coords = (torch.rand(B, 2, 2, H, W, generator=g) * 6 - 1)
    out, = oracle.altcorr_forward(f1, f2, coords, ii, jj, 1)
    gout = torch.randn(out.shape, generator=g, dtype=torch.float64)
    (out * gout).sum().backward()
    # the kernel drops the two /4 scalings in the backward pass (src/altcorr_kernel.cu:121-122): gradients are 16x larger
    g1, g2 = oracle.altcorr_backward(f1.detach(), f2.detach(), coords, gout.float(), ii, jj, 1)
    assert torch.allclose(g1 / 16, f1.grad, atol=1e-6)
    assert torch.allclose(g2 / 16, f2.grad, atol=1e-6)


# ---- SE3 identities (thirdparty/lietorch/lietorch/run_tests.py:16-52) on the kernel-faithful helpers ----
def test_se3_helpers():
    g = torch.Generator().manual_seed(4)
    xi = 0.3 * torch.randn(5, 6, generator=g, dtype=torch.float64)
    t, q = oracle.exp_se3(xi)
    assert torch.allclose(q.norm(dim=-1), torch.ones(5, dtype=torch.float64), atol=1e-12)
    t2, q2 = oracle.exp_se3(-xi)
    # Exp(xi) * Exp(-xi) = identity
    tt, qq = oracle.retr_se3(xi, t2, q2)
    assert torch.allclose(tt, torch.zeros_like(tt), atol=1e-12)
    assert torch.allclose(qq.abs(), torch.tensor([0, 0, 0, 1.0], dtype=torch.float64).expand(5, 4), atol=1e-12)
    # rel_se3(Ti, Tj) maps points like Tj * Ti^-1
    ti, qi = oracle.exp_se3(torch.randn(5, 6, generator=g, dtype=torch.float64) * 0.2)
    tj, qj = oracle.exp_se3(torch.randn(5, 6, generator=g, dtype=torch.float64) * 0.2)
    tij, qij = oracle.rel_se3(ti, qi, tj, qj)
    X = torch.randn(5, 3, generator=g, dtype=torch.float64)
    Xw = oracle.act_so3(torch.cat([-qi[:, :3], qi[:, 3:]], -1), X - ti)     # Ti^-1 X
    assert torch.allclose(oracle.act_so3(qij, X) + tij, oracle.act_so3(qj, Xw) + tj, atol=1e-12)
    # small-angle branch is continuous
    small = torch.tensor([[1e-5, 0, 0, 2e-5, 1e-5, 0]], dtype=torch.float64)
    ts, qs = oracle.exp_se3(small)
    assert abs(float(qs[0, 3]) - 1.0) < 1e-9


# ---- BA oracle: Jacobians of K1 against autograd through the same projection model ----
def _project(pose_i, pose_j, disp, intr, ht, wd, stereo=False):
    fx, fy, cx, cy = intr
    u, v = oracle.pixel_grid(ht, wd, torch.float64)
    if stereo:
        tij = torch.tensor([-0.1, 0, 0], dtype=torch.float64); qij = torch.tensor([0, 0, 0, 1.0], dtype=torch.float64)
    else:
        tij, qij = oracle.rel_se3(pose_i[:3], pose_i[3:], pose_j[:3], pose_j[3:])
    X = torch.stack([(u - cx) / fx, (v - cy) / fy, torch.ones_like(u), disp], -1)
    Y = oracle.act_se3(tij, qij, X)
    return torch.stack([fx * Y[:, 0] / Y[:, 2] + cx, fy * Y[:, 1] / Y[:, 2] + cy], -1)     # [HW,2]


def test_ba_edge_terms_match_autograd_jacobians():
    g = torch.Generator().manual_seed(5)
    ht, wd = 3, 4
    HW = ht * wd
    intr = torch.tensor([6.0, 6.5, 1.5, 1.0], dtype=torch.float64)
    pi = torch.cat(oracle.exp_se3(0.2 * torch.randn(6, generator=g, dtype=torch.float64)))
    pj = torch.cat(oracle.exp_se3(0.2 * torch.randn(6, generator=g, dtype=torch.float64)))
    disp = 0.5 + torch.rand(HW, generator=g, dtype=torch.float64)
    target = torch.randn(2, ht, wd, generator=g, dtype=torch.float64) * 3
    weight = torch.rand(2, ht, wd, generator=g, dtype=torch.float64)

    def retr1(xi, t, q):
        # first-order left retraction Exp(xi)*T (autograd-safe at xi = 0, where sqrt(theta^2) has no gradient)
        dq = torch.cat([0.5 * xi[3:], torch.ones(1, dtype=torch.float64)])
        q1 = torch.stack([dq[3] * q[0] + dq[0] * q[3] + dq[1] * q[2] - dq[2] * q[1],
                          dq[3] * q[1] + dq[1] * q[3] + dq[2] * q[0] - dq[0] * q[2],
                          dq[3] * q[2] + dq[2] * q[3] + dq[0] * q[1] - dq[1] * q[0],
                          dq[3] * q[3] - dq[0] * q[0] - dq[1] * q[1] - dq[2] * q[2]])
        return oracle.act_so3(dq, t) + xi[:3], q1

    def f(xi_i, xi_j, dd):
        ti, qi = retr1(xi_i, pi[:3], pi[3:]); tj, qj = retr1(xi_j, pj[:3], pj[3:])
        return _project(torch.cat([ti, qi]), torch.cat([tj, qj]), disp + dd, intr, ht, wd)

    z6 = torch.zeros(6, dtype=torch.float64); zd = torch.zeros(HW, dtype=torch.float64)
    Ji, Jj, Jd = torch.autograd.functional.jacobian(f, (z6, z6, zd))      # [HW,2,6],[HW,2,6],[HW,2,HW]
    Jz = torch.stack([Jd[p, :, p] for p in range(HW)])                      # [HW,2]
    r = target.reshape(2, HW).t() - f(z6, z6, zd)                           # [HW,2]
    w = 0.001 * weight.reshape(2, HW).t()
    J = torch.cat([Ji, Jj], -1)                                             # [HW,2,12]
    H = torch.einsum("pk,pkn,pkm->nm", w, J, J)
    v = torch.einsum("pk,pkn->n", w * r, J)
    Eii = torch.einsum("pk,pkn->np", w * Jz, Ji); Eij = torch.einsum("pk,pkn->np", w * Jz, Jj)
    C = (w * Jz * Jz).sum(-1); bz = (w * r * Jz).sum(-1)

    poses = torch.stack([pi, pj]); disps = torch.stack([disp.reshape(ht, wd), torch.ones(ht, wd, dtype=torch.float64)])
    T = oracle.ba_edge_terms(poses, disps, intr, target[None], weight[None], torch.tensor([0]), torch.tensor([1]))
    Hs = T["Hs"]
    Href = torch.cat([torch.cat([Hs[0, 0], Hs[1, 0]], 1), torch.cat([Hs[2, 0], Hs[3, 0]], 1)], 0)
    assert torch.allclose(Href, H, atol=1e-9)
    assert torch.allclose(torch.cat([T["vs"][0, 0], T["vs"][1, 0]]), v, atol=1e-9)
    assert torch.allclose(T["Eii"][0], Eii, atol=1e-9) and torch.allclose(T["Eij"][0], Eij, atol=1e-9)
    assert torch.allclose(T["Cii"][0], C, atol=1e-9) and torch.allclose(T["bz"][0], bz, atol=1e-9)


def test_ba_schur_step_equals_full_normal_equations():
    """the reduced system of ba_system + back-substitution solves the full damped normal equations
    [[H+D, E],[E^T, C]] [dx;dz] = [v;w]   (SURVEY.md section 4, cross-check 2; Q9 disabled by looking at dx only)."""
    s = synth.make_scene(dict(E=10, N=4, ht=4, wd=6, stereo=False, itrs=1, lm=1e-4, ep=0.1), seed=3)
    p, d = s["poses"].double(), s["disps"].double()
    ii, jj, t0, t1 = s["ii"], s["jj"], s["t0"], s["t1"]
    T = oracle.ba_edge_terms(p, d, s["intrinsics"].double(), s["targets"].double(), s["weights"].double(), ii, jj)
    A, b, aux = oracle.ba_system(T, d, s["disps_sens"].double(), s["eta"].double(), ii, jj, t0, t1, False, torch.float64)
    P, HW = t1 - t0, 24
    kx = aux["kx"]; M = kx.shape[0]
    n = 6 * P
    # full system assembled independently
    Hfull = torch.zeros(n + M * HW, n + M * HW, dtype=torch.float64); rhs = torch.zeros(n + M * HW, dtype=torch.float64)
    Hs, vs = T["Hs"], T["vs"]
    k_of = {int(k): m for m, k in enumerate(kx.tolist())}
    for e in range(ii.shape[0]):
        i, j = int(ii[e]) - t0, int(jj[e]) - t0
        m = k_of[int(ii[e])]
        for (a, c, blk) in ((i, i, 0), (i, j, 1), (j, i, 2), (j, j, 3)):
            if a >= 0 and c >= 0: Hfull[6 * a:6 * a + 6, 6 * c:6 * c + 6] += Hs[blk, e]
        if i >= 0: rhs[6 * i:6 * i + 6] += vs[0, e]
        if j >= 0: rhs[6 * j:6 * j + 6] += vs[1, e]
        for pidx in range(HW):
            col = n + m * HW + pidx
            if i >= 0: Hfull[6 * i:6 * i + 6, col] += T["Eii"][e, :, pidx]; Hfull[col, 6 * i:6 * i + 6] += T["Eii"][e, :, pidx]
            if j >= 0: Hfull[6 * j:6 * j + 6, col] += T["Eij"][e, :, pidx]; Hfull[col, 6 * j:6 * j + 6] += T["Eij"][e, :, pidx]
    Hfull[n:, n:] = torch.diag(aux["C"].reshape(-1)); rhs[n:] = aux["w"].reshape(-1)
    dg = torch.diagonal(Hfull)[:n]
    lm = float(torch.tensor(s["lm"], dtype=torch.float32)); ep = float(torch.tensor(s["ep"], dtype=torch.float32))
    # damping is applied to the REDUCED system's diagonal in the reference (A-S), reproduce: solve reduced system directly
    Sred = Hfull[:n, :n] - Hfull[:n, n:] @ torch.diag(1 / torch.diagonal(Hfull[n:, n:])) @ Hfull[n:, :n]
    bred = rhs[:n] - Hfull[:n, n:] @ (rhs[n:] / torch.diagonal(Hfull[n:, n:]))
    assert torch.allclose(Sred, A, atol=1e-8) and torch.allclose(bred, b, atol=1e-8)
    Sd = Sred.clone(); Sd.diagonal().add_(ep + lm * Sred.diagonal())
    dx_ref = torch.linalg.solve(Sd, bred).reshape(P, 6)
    po, do = p.clone(), d.clone()
    (dx, dz) = oracle.ba(po, do, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], ii, jj, t0, t1, 1, s["lm"], s["ep"], False, dtype=torch.float64)
    assert torch.allclose(dx, dx_ref, atol=1e-9)
    # dz with Q9: pose t0's dx is ignored in the back substitution
    dxq = dx_ref.clone(); dxq[0] = 0
    dz_ref = (rhs[n:] - Hfull[n:, :n] @ dxq.reshape(-1)) / torch.diagonal(Hfull[n:, n:])
    assert torch.allclose(dz.reshape(-1), dz_ref, atol=1e-9)


def test_ba_fp32_restatement_close_to_fp64():
    s = synth.make_scene("c1_plumbing")
    p32, d32 = s["poses"].clone(), s["disps"].clone()
    p64, d64 = s["poses"].double(), s["disps"].double()
    args = (s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 3, s["lm"], s["ep"], False)
    oracle.ba(p32, d32, *args)
    oracle.ba(p64, d64, *args, dtype=torch.float64)
    assert (p32.double() - p64).abs().max() < 1e-4
    assert ((d32.double() - d64).abs() / d64.abs().clamp(min=1)).max() < 1e-3


def test_motion_only_and_stereo_paths_run():
    s = synth.make_scene(dict(E=20, N=6, ht=6, wd=8, stereo=True, itrs=2, lm=1e-4, ep=0.1), seed=1)
    p, d = s["poses"].clone(), s["disps"].clone()
    dx, dz = oracle.ba(p, d, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2, 1e-4, 0.1, True)
    assert dz is None and torch.isfinite(dx).all() and torch.equal(d, s["disps"])
    dx, dz = oracle.ba(p, d, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2, 1e-4, 0.1, False)
    assert torch.isfinite(dz).all()


def test_geometry_oracles_consistency():
    """SURVEY.md section 4, cross-checks 3 and 4: projmap == reprojection; a static scene is self-consistent for
    depth_filter (count = number of in-range neighbours)."""
    s = synth.make_scene(dict(E=12, N=8, ht=12, wd=16, stereo=False, itrs=1, lm=1e-4, ep=0.1), seed=2)
    coords, valid = oracle.projmap(s["poses_gt"], s["disps_gt"], s["intrinsics"], s["ii"], s["jj"])
    assert torch.allclose(coords[..., :2], s["coords_gt"], atol=2e-3)
    assert float(valid.mean()) > 0.9
    # planar fronto-parallel static scene, pure x-translation: every neighbour that exists must agree
    N, ht, wd = 8, 12, 16
    poses = torch.zeros(N, 7); poses[:, 6] = 1; poses[:, 0] = -0.01 * torch.arange(N)
    disps = torch.full((N, ht, wd), 0.5)
    ix = torch.arange(N)
    cnt = oracle.depth_filter(poses, disps, s["intrinsics"], ix, torch.full((N,), 0.05))
    inner = cnt[:, 2:-2, 2:-2]
    expect = torch.tensor([sum(1 for k in range(6) if 0 <= (i - k - 1 if k < 3 else i + k) < N) for i in range(N)], dtype=torch.float32)
    assert torch.equal(inner.amax(dim=(1, 2)), expect) and torch.equal(inner.amin(dim=(1, 2)), expect)
    pts = oracle.iproj(poses, disps, s["intrinsics"])
    assert torch.allclose(pts[..., 2], torch.full((N, ht, wd), 2.0), atol=1e-5)
    d = oracle.frame_distance(poses, disps, s["intrinsics"], torch.tensor([0, 0]), torch.tensor([1, 4]), 0.3)
    fx = float(s["intrinsics"][0])
    assert torch.allclose(d, torch.tensor([fx * 0.01 * 0.5, fx * 0.04 * 0.5]), rtol=1e-4)


# ---- the C-ABI library exports every symbol the header declares (no compute calls without a GPU) ----
def test_capi_exports_match_header():
    hdr = open(os.path.join(ROOT, "include", "droid_b200.h")).read()
    declared = set(re.findall(r"\b(dba_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"dba_stream_t"}
    assert declared == set(c_api.SYMBOLS), (declared ^ set(c_api.SYMBOLS))
    L = ctypes.CDLL(c_api.lib_path())
    for name in sorted(declared):
        assert hasattr(L, name), name
    assert c_api.load().dba_version() >= 100


# ---- the Python view of the C ABI (droid_slam_b200/c_api.py) against the header: a struct that grows or is reordered, or a parameter
# whose type changes, fails here by name instead of handing the kernels misplaced or truncated arguments ----
HEADER = os.path.join(ROOT, "include", "droid_b200.h")
MIRRORS = {"dba_ba_args": c_api.BAArgs, "dba_update_weights": c_api.UpdateWeights, "dba_update_args": c_api.UpdateArgs,
           "dba_encoder_weights": c_api.EncoderWeights, "dba_encoder_args": c_api.EncoderArgs, "dba_frame_format": c_api.FrameFormat}


def _header_probe(tmp_path, lines):
    """compile and run a C program that includes the header and prints `key value` lines -> {key: int}"""
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text("\n".join(['#include <stdio.h>', '#include <stddef.h>', '#include "droid_b200.h"', 'int main(void) {'] + lines
                             + ['  return 0; }']))
    subprocess.run(["gcc", "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    return {k: int(v) for k, v in (line.split() for line in out if line)}


def _header_fields(struct):
    """the member names of `typedef struct { ... } struct;` in the header, in order"""
    hdr = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\}\s*%s;" % struct, hdr).group(1)
    return [re.search(r"(\w+)\s*(\[\w+\])?$", d.strip()).group(1) for s in body.split(";") if s.strip() for d in s.split(",")]


def test_capi_args_struct_layout_matches_header(tmp_path):
    """every ctypes mirror has the header's members in the header's order, its size, and each member's offset and size (arrays
    included)"""
    for struct, cls in MIRRORS.items():
        assert [f for f, _ in cls._fields_] == _header_fields(struct), struct
    lines, want = [], {}
    for struct, cls in MIRRORS.items():
        lines.append('  printf("%s %%zu\\n", sizeof(%s));' % (struct, struct))
        want[struct] = ctypes.sizeof(cls)
        for f, _ in cls._fields_:
            key = "%s.%s" % (struct, f)
            lines.append('  printf("%s@offset %%zu\\n%s@size %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));'
                         % (key, key, struct, f, struct, f))
            want[key + "@offset"], want[key + "@size"] = getattr(cls, f).offset, getattr(cls, f).size
    got = _header_probe(tmp_path, lines)
    bad = ["%s: header %d, c_api %d" % (k, got[k], v) for k, v in want.items() if got[k] != v]
    assert not bad, bad


def _c_kind(t):
    t = " ".join(t.replace("*", " * ").split())
    if t == "const char *":
        return "const char*"
    m = re.fullmatch(r"(const )?(\w+) \*", t)
    if m and m.group(2) in MIRRORS:
        return "pointer to " + m.group(2)
    if t.endswith("*") or t == "dba_stream_t":
        return "pointer"
    return {"int": "int", "float": "float", "double": "double", "size_t": "size_t", "long long int": "int64", "int64_t": "int64"}[t]


def _py_kind(t):
    for struct, cls in MIRRORS.items():
        if t is ctypes.POINTER(cls):
            return "pointer to " + struct
    return {ctypes.c_void_p: "pointer", ctypes.c_char_p: "const char*", ctypes.c_int: "int", ctypes.c_float: "float",
            ctypes.c_double: "double", ctypes.c_size_t: "size_t", ctypes.c_longlong: "int64"}[t]


def test_capi_prototypes_match_header(tmp_path):
    """every function of the header has a prototype in c_api with the header's return kind and per-parameter kinds: pointer
    (dba_stream_t included; a pointer to a mirrored struct must be typed as a pointer to its mirror), int, float, double, size_t, 64-bit
    integer, const char*.  gcc's -aux-info prints each prototype of the header on one normalised line."""
    src, aux = tmp_path / "protos.c", tmp_path / "protos.txt"
    src.write_text('#include "droid_b200.h"\n')
    subprocess.run(["gcc", "-fsyntax-only", "-I", os.path.dirname(HEADER), "-aux-info", str(aux), str(src)], check=True)
    header = {}
    for line in aux.read_text().splitlines():
        m = re.search(r"droid_b200\.h:\d+:\w+ \*/ extern (.*?)\s*\b(dba_\w+) \((.*)\);$", line)
        if m:
            header[m.group(2)] = (m.group(1), [] if m.group(3) == "void" else m.group(3).split(", "))
    assert len(header) == 57 and set(header) == set(c_api.PROTOTYPES), set(header) ^ set(c_api.PROTOTYPES)
    bad = []
    for name, (ret, params) in header.items():
        restype, argtypes = c_api.PROTOTYPES[name]
        if _c_kind(ret) != _py_kind(restype):
            bad.append("%s returns %s (%s), c_api %s" % (name, _c_kind(ret), ret, _py_kind(restype)))
        if len(params) != len(argtypes):
            bad.append("%s takes %d parameters, c_api %d" % (name, len(params), len(argtypes)))
        for i, (p, a) in enumerate(zip(params, argtypes)):
            if _c_kind(p) != _py_kind(a):
                bad.append("%s parameter %d: header %s (%s), c_api %s" % (name, i, _c_kind(p), p, _py_kind(a)))
    assert not bad, bad


def test_capi_constants_match_header(tmp_path):
    names = ("DBA_F32", "DBA_F16", "DBA_F64", "DBA_BF16", "DBA_ENCODER_CONVS")
    got = _header_probe(tmp_path, ['  printf("%s %%d\\n", %s);' % (n, n) for n in names])
    assert got == {n: getattr(c_api, n) for n in names}


def test_update_weights_mirror_follows_packed_order():
    """the binding stores the k-th packed weight in the k-th pointer of dba_update_weights, so PACKED_ORDER must be its member order"""
    from droid_slam_b200.update import PACKED_ORDER
    assert tuple(f for f, _ in c_api.UpdateWeights._fields_) == PACKED_ORDER


def test_capi_argument_validation_without_gpu():
    L = c_api.load()
    assert L.dba_corr_index_forward(None, None, None, -1, 1, 1, 1, 1, 3, 0, None) == 1
    assert b"invalid" in L.dba_last_error()
    assert L.dba_corr_index_forward(None, None, None, 0, 4, 4, 4, 4, 3, 0, None) == 0      # empty batch: no launch
    assert L.dba_corr_index_forward(None, None, None, 1, 4, 4, 4, 4, 3, 7, None) == 1      # unknown dtype
    assert L.dba_iproj(None, None, None, None, 0, 4, 4, None) == 0
    assert L.dba_ba_workspace_bytes(8, 24, 48, 64, 1, 8) > 24 * 6 * 48 * 64 * 4
    assert L.dba_ba_system_bytes(1, 8) == 8 * (42 * 42 + 42)


def test_binding_imports_and_rejects_cpu_tensors(backends):
    names = ["ba", "frame_distance", "projmap", "depth_filter", "iproj", "altcorr_forward", "altcorr_backward",
             "corr_index_forward", "corr_index_backward"]                # reference src/droid.cpp:248-258
    for n in names:
        assert callable(getattr(backends, n))
    with pytest.raises(RuntimeError):
        backends.corr_index_forward(torch.zeros(1, 2, 2, 2, 2), torch.zeros(1, 2, 2, 2), 3)
    with pytest.raises(RuntimeError):
        backends.iproj(torch.zeros(2, 7), torch.zeros(2, 4, 4), torch.zeros(4))


def test_synthetic_graph_properties():
    for name in ("c1_plumbing", "c2_frontend", "c4_stereo"):
        c = synth.CONFIGS[name]
        ii, jj = synth.make_graph(c["E"], c["N"], stereo=c["stereo"], seed=0)
        assert ii.shape[0] == c["E"] and int(ii.max()) < c["N"] and int(jj.max()) < c["N"]
        assert set(range(1, c["N"])) <= set(ii.tolist())          # every optimised frame has an out edge (eta row alignment)
        assert len(set(zip(ii.tolist(), jj.tolist()))) == c["E"]  # no duplicate edges
        ii2, jj2 = synth.make_graph(c["E"], c["N"], stereo=c["stereo"], seed=0)
        assert torch.equal(ii, ii2) and torch.equal(jj, jj2)      # deterministic

