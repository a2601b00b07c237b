"""GPU tests at BASELINE.json's full sizes.  The CPU oracle is too slow for whole-problem comparisons there, so these
use (a) the oracle on a sub-sample of the same tensors and (b) size-independent properties: linearity / exact scaling,
chunk invariance, adjointness, Gauss-Newton descent, sharded == unsharded."""
import pytest
import torch

import oracle
from droid_slam_b200 import synth
from util import c_ba, rel_err

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def metric_scene():
    return synth.make_scene("metric")            # 512 edges, 72 keyframes, 48x64


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_corr_index_full_size_properties(backends, metric_scene, dtype):
    s = metric_scene
    E = 160                                          # 160 edges x 18.9 MB (f16) level-0 planes: > L2, > 2^31 elements with f32 strides exercised
    sub = dict(s); sub["ii"] = s["ii"][:E]; sub["jj"] = s["jj"][:E]; sub["coords_gt"] = s["coords_gt"][:E]; sub["cfg"] = dict(s["cfg"], E=E)
    pyr, coords, _ = synth.make_corr_inputs(sub, dtype=dtype, device=dev)
    for lvl, vol in enumerate(pyr):
        c = (coords / 2 ** lvl).contiguous()
        out, = backends.corr_index_forward(vol, c, 3)
        assert out.shape == (E, 7, 7, 48, 64) and torch.isfinite(out.float()).all()
        # (a) oracle on a sub-sample of edges (first, middle, last)
        for e in (0, E // 2, E - 1):
            ref, = oracle.corr_index_forward(vol[e:e + 1].cpu(), c[e:e + 1].cpu(), 3)
            assert torch.equal(out[e:e + 1].cpu(), ref)
        # (b) exact scaling by a power of two (every rounding step commutes with it) and chunk invariance
        out2, = backends.corr_index_forward(vol * 4, c, 3)
        if dtype == torch.float32:
            assert torch.equal(out2, out * 4)
        else:       # f16: a subnormal intermediate may flip a later tie, and cancellation can amplify that ulp
            d = (out2.float() - 4 * out.float()).abs()
            assert float((d == 0).float().mean()) > 0.999
            assert float(d.max()) <= 2e-3 * float(out2.float().abs().max())
        outc = torch.cat([backends.corr_index_forward(vol[a:a + 64], c[a:a + 64].contiguous(), 3)[0] for a in range(0, E, 64)])
        assert torch.equal(outc, out)
    # (c) adjointness of forward/backward at level 2 (f32 only: sums are exact enough).  <fwd, g> and <vol, bwd> are the same sum in
    # exact arithmetic; what separates them is the fp32 rounding of each fwd and bwd element, which cancels at random.  So the bound is
    # a fraction of u times the size of the terms, not of |<fwd, g>|: that sum has random sign and is near zero for some g (on an H100,
    # |a - b| stays below 1e-3 u sum |fwd g| over 12 seeds).  g has its own generator, so the result does not depend on test order.
    if dtype == torch.float32:
        vol = pyr[2]; c = (coords / 4).contiguous()
        g = torch.randn(E, 7, 7, 48, 64, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        fwd, = backends.corr_index_forward(vol, c, 3)
        bwd, = backends.corr_index_backward(vol, c, g, 3)
        a = float((fwd.double() * g.double()).sum()); b = float((vol.double() * bwd.double()).sum())
        terms = float((fwd.double() * g.double()).abs().sum())
        assert abs(a - b) <= 0.01 * 2.0 ** -24 * terms, (a, b, terms)


def test_ba_full_size_matches_oracle_and_descends(backends, metric_scene):
    s = metric_scene
    torch.set_num_threads(min(16, torch.get_num_threads()))
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    dx, dz = backends.ba(P, D, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    assert dx.shape == (71, 6) and dz.shape == (s["M"], 48 * 64)
    P64, D64 = s["poses"].double(), s["disps"].double()
    oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2,
              s["lm"], s["ep"], False, dtype=torch.float64)
    assert rel_err(P, P64, floor=1.0) < 1e-4 and rel_err(D, D64, floor=1.0) < 1e-4
    # Gauss-Newton descent towards the ground truth used to synthesise the targets
    assert float((P.cpu() - s["poses_gt"]).abs().max()) < float((s["poses"] - s["poses_gt"]).abs().max())


def test_global_ba_config3_runs_and_descends(backends):
    """BASELINE config 3: 2048 edges / 400 keyframes, backend damping (lm=1e-5, ep=1e-2); 6P = 2394 exercises the
    75-tile cluster Cholesky.  Property: the weighted reprojection cost decreases and stays finite."""
    s = synth.make_scene("c3_global")
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]

    def cost(Pc, Dc):
        c, _ = backends.projmap(Pc, Dc, args[0], args[5], args[6])
        r = (s["targets"].to(dev).permute(0, 2, 3, 1) - c[..., :2])
        return float((s["weights"].to(dev).permute(0, 2, 3, 1) * r * r).sum())

    c0 = cost(P, D)
    dx, dz = backends.ba(P, D, *args, s["t0"], s["t1"], 3, s["lm"], s["ep"], False)
    torch.cuda.synchronize()
    assert torch.isfinite(P).all() and torch.isfinite(D).all() and float(dx.abs().max()) > 0
    c1 = cost(P, D)
    assert c1 < 0.7 * c0
    assert float((P.cpu() - s["poses_gt"]).abs().max()) < float((s["poses"] - s["poses_gt"]).abs().max())


def test_stereo_config4_matches_oracle(backends):
    s = synth.make_scene("c4_stereo")
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    backends.ba(P, D, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    P64, D64 = s["poses"].double(), s["disps"].double()
    oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2,
              s["lm"], s["ep"], False, dtype=torch.float64)
    assert rel_err(P, P64, floor=1.0) < 1e-4 and rel_err(D, D64, floor=1.0) < 1e-4


def test_stress_shape_72x96_bf16_and_ba(backends):
    """BASELINE config 5 shapes (72x96 feature maps, bf16 volumes) at a reduced edge count: exercises wd = 96 (pyramid level 3 has
    12-wide rows -> generic lookup path), HW = 6912 (not a multiple of the BA pixel chunk) and the bf16 extension."""
    s = synth.make_scene(dict(E=40, N=10, ht=72, wd=96, stereo=False, itrs=2, lm=1e-4, ep=0.1), seed=8)
    pyr, coords, _ = synth.make_corr_inputs(s, dtype=torch.bfloat16, device=dev, channels=32, edge_chunk=8)
    for lvl, vol in enumerate(pyr):
        c = (coords / 2 ** lvl).contiguous()
        out, = backends.corr_index_forward(vol, c, 3)
        ref, = oracle.corr_index_forward(vol[:2].float().cpu(), c[:2].cpu(), 3)          # bf16: fp32 math on bf16-rounded inputs
        assert rel_err(out[:2].float(), ref, floor=float(ref.abs().max())) < 1e-2
        f16, = backends.corr_index_forward(vol.half(), c, 3)
        r16, = oracle.corr_index_forward(vol[:2].half().cpu(), c[:2].cpu(), 3)
        assert torch.equal(f16[:2].cpu(), r16)
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    backends.ba(P, D, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    P64, D64 = s["poses"].double(), s["disps"].double()
    oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2,
              s["lm"], s["ep"], False, dtype=torch.float64)
    assert rel_err(P, P64, floor=1.0) < 1e-4 and rel_err(D, D64, floor=1.0) < 1e-4


def _mixed_degree_graph(N=34):
    """frames with 3-5 rows (packed tensor-core tiles), 16 rows (one tile per 32 pixels) and 25 rows (tensor-core tile pairs),
    plus a duplicated edge: every tensor-core Schur mode and the duplicate-pose rule (both (r,c) and (c,r) land on one diagonal
    block), at every image size.  The extra edges stay within 12 frames so that the problem is as well conditioned as a covisibility
    graph."""
    e = []
    for i in range(N):
        for j in (i - 2, i - 1, i + 1, i + 2):
            if 0 <= j < N:
                e.append((i, j))
    e += [(17, j) for j in range(5, 30) if abs(j - 17) > 2]           # frame 17: 24 out-edges -> 25 rows
    e += [(26, j) for j in range(18, 34) if abs(j - 26) > 2]          # frame 26: 15 out-edges -> 16 rows
    e += [(9, 10)]                                                     # duplicate of an existing edge
    return [a for a, _ in e], [b for _, b in e]


def _mixed_degree_ba_matches_oracle(backends, ht, wd):
    ii, jj = _mixed_degree_graph()
    s = synth.make_scene(dict(E=len(ii), N=34, ht=ht, wd=wd, stereo=False, itrs=2, lm=1e-4, ep=0.1, graph=(ii, jj)), seed=1)
    deg = torch.bincount(s["ii"], minlength=34)
    assert int(deg[17]) == 24 and int(deg[26]) == 15 and int(deg.min()) >= 2
    torch.set_num_threads(min(16, torch.get_num_threads()))
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    backends.ba(P, D, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    P64, D64 = s["poses"].double(), s["disps"].double()
    oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2,
              s["lm"], s["ep"], False, dtype=torch.float64)
    assert rel_err(P, P64, floor=1.0) < 1e-4 and rel_err(D, D64, floor=1.0) < 1e-4


def test_ba_every_schur_kernel_matches_oracle(backends):
    _mixed_degree_ba_matches_oracle(backends, 48, 64)


def test_ba_every_schur_kernel_on_padded_rows_matches_oracle(backends):
    """47x63: HW % 4 != 0, so the workspace pixel rows end in pad pixels, and the tensor-core kernels read them with the last 16-byte
    piece of each row"""
    _mixed_degree_ba_matches_oracle(backends, 47, 63)


def _high_degree_graph():
    """_mixed_degree_graph plus frame 12 with its 24 targets within 12 frames repeated 5 times: 124 out-edges -> 125 rows (120 after
    dropping the 5 rows of frame 0, which is outside the window).  That frame takes the tensor-core pair mode with more than 100 rows
    (12 tiles, 66 tile pairs: a second pair for some CTAs), where repeated targets put rows with one pose into different tiles (the
    duplicate-pose rule)."""
    ii, jj = _mixed_degree_graph()
    extra = [j for _ in range(5) for j in range(0, 25) if j != 12]
    return ii + [12] * len(extra), jj + extra


@pytest.mark.parametrize("ht,wd", [(48, 64), (47, 63)])
def test_ba_schur_pair_frame_over_100_rows_matches_oracle(capi, ht, wd):
    """every Schur kernel in one graph, with a workspace that starts as NaN: a pad pixel that the Schur kernels read but nothing
    zeroed would turn the result into NaN"""
    ii, jj = _high_degree_graph()
    s = synth.make_scene(dict(E=len(ii), N=34, ht=ht, wd=wd, stereo=False, itrs=2, lm=1e-4, ep=0.1, graph=(ii, jj)), seed=7)
    deg = torch.bincount(s["ii"], minlength=34)
    assert int(deg[12]) == 124 and int(deg[17]) == 24 and int(deg[26]) == 15
    torch.set_num_threads(min(16, torch.get_num_threads()))
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    _, _, M, st, _ = c_ba(capi, P, D, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False, s["M"], ws_fill=255)
    assert M == s["M"] and st == 0
    P64, D64 = s["poses"].double(), s["disps"].double()
    oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2,
              s["lm"], s["ep"], False, dtype=torch.float64)
    assert rel_err(P, P64, floor=1.0) < 1e-4 and rel_err(D, D64, floor=1.0) < 1e-4, (rel_err(P, P64, floor=1.0), rel_err(D, D64, floor=1.0))


@pytest.mark.parametrize("N,res", [(40, (24, 32)), (30, (48, 64))])
def test_ba_dense_graph_pair_mode_matches_oracle(backends, N, res):
    """complete directed graphs (every frame has N-1 out-edges -> N rows per depth frame, 3-4 row tiles): every frame takes the tensor-core
    PAIR mode of the Schur kernel -- the shape an edge-sharded rank of the 8-GPU run sees.  Includes duplicated edges whose two rows
    fall into different tiles (the doubled-entry rule)."""
    ii = [i for i in range(N) for j in range(N) if i != j]
    jj = [j for i in range(N) for j in range(N) if i != j]
    ii += [3, 3, 7]; jj += [N - 1, N - 2, N - 1]                       # duplicates: same (source, target) as rows of the first and the last tile
    ht, wd = res
    s = synth.make_scene(dict(E=len(ii), N=N, ht=ht, wd=wd, stereo=False, itrs=2, lm=1e-4, ep=0.1, graph=(ii, jj)), seed=2)
    torch.set_num_threads(min(16, torch.get_num_threads()))
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    backends.ba(P, D, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    P64, D64 = s["poses"].double(), s["disps"].double()
    oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], 2,
              s["lm"], s["ep"], False, dtype=torch.float64)
    assert rel_err(P, P64, floor=1.0) < 1e-4 and rel_err(D, D64, floor=1.0) < 1e-4, (rel_err(P, P64, floor=1.0), rel_err(D, D64, floor=1.0))
