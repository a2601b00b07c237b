"""GPU parity tests: the hand-written sm_90a kernels, called through the C ABI (ctypes) and through the
`droid_backends` pybind surface, against the CPU oracle on the same seeded inputs.

Tolerances (BASELINE.json north_star): fp32 outputs within 1e-4 relative (with an absolute floor of 1e-4*scale),
index/count outputs bit-exact.  corr_index f16/f32 are expected bit-identical to the oracle's restatement of the
reference rounding order; the tests assert >= 99.9 % identical elements and the tolerance for the rest.
"""
import pytest
import torch

import oracle
from droid_slam_b200 import synth
from util import (DT, assert_bit_identical, c_ba, c_corr_index_backward, c_corr_index_forward, frac_equal, rel_err)

pytestmark = pytest.mark.gpu
dev = "cuda"


def _corr_case(n, h1, w1, h2, w2, dtype, seed, spread=1.0):
    g = torch.Generator().manual_seed(seed)
    vol = torch.randn(n, h1, w1, h2, w2, generator=g).to(dtype)
    cx = torch.rand(n, 1, h1, w1, generator=g) * (w2 + 8 * spread) - 4 * spread
    cy = torch.rand(n, 1, h1, w1, generator=g) * (h2 + 8 * spread) - 4 * spread
    return vol, torch.cat([cx, cy], 1).contiguous()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32, torch.float64, torch.bfloat16])
@pytest.mark.parametrize("shape", [(2, 6, 8, 6, 8), (3, 5, 7, 12, 16), (2, 4, 6, 24, 32), (1, 3, 5, 9, 11), (2, 2, 3, 6, 12)])
def test_corr_index_forward_matches_oracle(capi, dtype, shape):
    vol, coords = _corr_case(*shape, dtype, seed=sum(shape))
    # a few special coordinates: integers, far outside, exactly on the border
    coords[0, :, 0, 0] = torch.tensor([3.0, 2.0]); coords[0, :, 0, 1] = torch.tensor([-100.0, 5.0])
    coords[0, :, 1, 0] = torch.tensor([1e9, -1e9]); coords[0, :, 1, 1] = torch.tensor([-0.5, shape[3] - 0.5])
    got = c_corr_index_forward(capi, vol.to(dev), coords.to(dev), 3)
    if dtype == torch.bfloat16:      # not dispatched by the reference: oracle = fp32 math on bf16-rounded inputs
        ref, = oracle.corr_index_forward(vol.float(), coords, 3)
        assert rel_err(got.float(), ref, floor=1.0) < 1e-2
        return
    ref, = oracle.corr_index_forward(vol, coords, 3)
    assert torch.isfinite(got.float()).all()
    assert_bit_identical(got, ref, "corr_index_forward %s" % dtype)        # the oracle restates the reference's rounding order (pinned bit-exactly)


def test_corr_index_forward_bf16_fast_path_equals_generic_path(backends):
    """bf16 volumes (BASELINE config 5; not dispatched by the reference): the vector-load kernel computes the same function as the
    generic one -- checked bit for bit by pushing the same volume through the generic path via a 2-byte misaligned view"""
    vol, coords = _corr_case(3, 6, 8, 24, 32, torch.bfloat16, seed=77)
    coords[0, :, 0, 0] = torch.tensor([float("nan"), 2.0])
    fast = backends.corr_index_forward(vol.to(dev), coords.to(dev), 3)[0]
    buf = torch.zeros(vol.numel() + 1, dtype=torch.bfloat16, device=dev)
    v = buf[1:].view(vol.shape); v.copy_(vol)
    slow = backends.corr_index_forward(v, coords.to(dev), 3)[0]
    assert_bit_identical(fast, slow, "bf16 fast vs generic path")
    ref, = oracle.corr_index_forward(vol.float(), coords, 3)
    ok = torch.isfinite(ref)
    assert rel_err(fast.float().cpu()[ok], ref[ok], floor=1.0) < 1e-2


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("radius", [0, 1, 2, 4])
def test_corr_index_forward_other_radii(capi, dtype, radius):
    vol, coords = _corr_case(2, 4, 5, 8, 8, dtype, seed=radius)
    got = c_corr_index_forward(capi, vol.to(dev), coords.to(dev), radius)
    ref, = oracle.corr_index_forward(vol, coords, radius)
    assert_bit_identical(got, ref, "corr_index_forward radius %d %s" % (radius, dtype))


def test_corr_index_forward_nonfinite_coords(capi):
    vol, coords = _corr_case(1, 4, 8, 8, 8, torch.float32, seed=11)
    coords[0, 0, 0, 0] = float("inf"); coords[0, 1, 0, 1] = float("-inf")
    got = c_corr_index_forward(capi, vol.to(dev), coords.to(dev), 3).cpu()
    assert (got[0, :, :, 0, 0] == 0).all() and (got[0, :, :, 0, 1] == 0).all()     # nothing in bounds -> zeros, like the reference
    ref, = oracle.corr_index_forward(vol, coords, 3)
    assert torch.equal(got[0, :, :, 1:], ref[0, :, :, 1:])


def test_corr_index_forward_empty_and_unaligned(capi, backends):
    e = backends.corr_index_forward(torch.zeros(0, 4, 4, 4, 8, device=dev), torch.zeros(0, 2, 4, 4, device=dev), 3)[0]
    assert e.shape == (0, 7, 7, 4, 4)
    # a volume view whose base pointer is not 16-byte aligned must take the generic path and still be right
    vol, coords = _corr_case(2, 4, 4, 8, 8, torch.float16, seed=5)
    buf = torch.zeros(vol.numel() + 1, dtype=torch.float16, device=dev)
    v = buf[1:].view(vol.shape); v.copy_(vol)
    got = backends.corr_index_forward(v, coords.to(dev), 3)[0]
    ref, = oracle.corr_index_forward(vol, coords, 3)
    assert torch.equal(got.cpu(), ref)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32, torch.float64])
def test_corr_index_backward_matches_oracle(capi, dtype):
    vol, coords = _corr_case(2, 5, 6, 12, 16, dtype, seed=7)
    g = torch.Generator().manual_seed(8)
    grad = torch.randn(2, 7, 7, 5, 6, generator=g).to(dtype)
    got = c_corr_index_backward(capi, vol.to(dev), coords.to(dev), grad.to(dev), 3)
    ref, = oracle.corr_index_backward(vol, coords, grad, 3)
    assert_bit_identical(got, ref, "corr_index_backward %s" % dtype)


def test_corr_pyramid_lookup_like_corrblock(backends):
    """CorrBlock.__call__ call pattern (reference modules/corr.py:40-50) on fp16 volumes, 4 levels."""
    s = synth.make_scene(dict(E=6, N=4, ht=16, wd=24, stereo=False, itrs=1, lm=1e-4, ep=0.1), seed=4)
    pyr, coords, _ = synth.make_corr_inputs(s, dtype=torch.float16, channels=16, levels=3)
    outs = []
    for i, vol in enumerate(pyr):
        c, = backends.corr_index_forward(vol.to(dev), (coords / 2 ** i).to(dev), 3)
        outs.append(c.view(1, 6, -1, 16, 24))
    got = torch.cat(outs, dim=2).cpu()
    ref = oracle.corr_block_lookup(pyr, coords.permute(0, 2, 3, 1)[None], 3)
    assert got.shape == ref.shape == (1, 6, 3 * 49, 16, 24)
    assert_bit_identical(got, ref, "CorrBlock lookup")


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32, torch.float64])
def test_altcorr_forward_matches_oracle(backends, dtype):
    g = torch.Generator().manual_seed(21)
    B, N, C, H, W = 1, 4, 32, 12, 16
    fmaps = torch.randn(B, N, C, H, W, generator=g).to(dtype)
    pyr = oracle.fmap_pyramid(fmaps, 3)
    ii = torch.tensor([0, 1, 2, 3, 0]); jj = torch.tensor([1, 2, 3, 3, 3])
    coords = torch.rand(B, 5, 2, H, W, generator=g) * torch.tensor([W + 6.0, H + 6.0]).view(1, 1, 2, 1, 1) - 3
    for lvl in range(3):
        c = (coords / 2 ** lvl).contiguous()
        got, = backends.altcorr_forward(pyr[0].to(dev), pyr[lvl].contiguous().to(dev), c.to(dev), ii.to(dev), jj.to(dev), 3)
        ref, = oracle.altcorr_forward(pyr[0], pyr[lvl], c, ii, jj, 3)
        assert got.shape == ref.shape and got.stride() == ref.stride()      # same permuted view as the reference (:171)
        tol = {torch.float16: 2e-2, torch.float32: 1e-4, torch.float64: 1e-6}[dtype]   # channel summation order differs
        assert rel_err(got, ref, floor=1.0) < tol


def test_altcorr_backward_matches_oracle(backends):
    g = torch.Generator().manual_seed(22)
    B, N, C, H, W = 1, 3, 8, 6, 8
    f1 = torch.randn(B, N, C, H, W, generator=g); f2 = torch.randn(B, N, C, H, W, generator=g)
    ii = torch.tensor([0, 1, 2]); jj = torch.tensor([1, 2, 2])
    coords = torch.rand(B, 3, 2, H, W, generator=g) * 8 - 1
    grad = torch.randn(B, 3, 7, 7, H, W, generator=g)
    g1, g2 = backends.altcorr_backward(f1.to(dev), f2.to(dev), coords.to(dev), grad.to(dev), ii.to(dev), jj.to(dev), 3)
    r1, r2 = oracle.altcorr_backward(f1, f2, coords, grad, ii, jj, 3)
    assert rel_err(g1, r1) < 1e-4 and rel_err(g2, r2) < 1e-4


# ---------------------------------------------------------------------------------------------------
def _scene(E=40, N=10, ht=24, wd=32, stereo=False, seed=0, **kw):
    return synth.make_scene(dict(E=E, N=N, ht=ht, wd=wd, stereo=stereo, itrs=2, lm=1e-4, ep=0.1), seed=seed, **kw)


def test_projmap_iproj_frame_distance_depth_filter(backends):
    s = _scene(seed=3)
    P, D, K = s["poses"], s["disps"], s["intrinsics"]
    ii, jj = s["ii"], s["jj"]
    c, v = backends.projmap(P.to(dev), D.to(dev), K.to(dev), ii.to(dev), jj.to(dev))
    rc, rv = oracle.projmap(P, D, K, ii, jj)
    assert c.shape == (40, 24, 32, 3) and v.shape == (40, 24, 32, 1)
    assert rel_err(c, rc, floor=1.0) < 1e-4 and frac_equal(v, rv) > 0.9999
    pts = backends.iproj(P.to(dev), D.to(dev), K.to(dev))
    assert rel_err(pts, oracle.iproj(P, D, K), floor=1.0) < 1e-4
    fd = backends.frame_distance(P.to(dev), D.to(dev), K.to(dev), ii.to(dev), jj.to(dev), 0.3)
    assert rel_err(fd, oracle.frame_distance(P, D, K, ii, jj, 0.3), floor=1.0) < 1e-4
    # DepthVideo.distance pattern (reference depth_video.py:181-211): bidirectional, all pairs
    n = 6
    a, b = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    a = a.reshape(-1); b = b.reshape(-1)
    d1 = backends.frame_distance(P[:n].clone().to(dev), D.to(dev), K.to(dev), a.to(dev), b.to(dev), 0.3)
    d2 = backends.frame_distance(P[:n].clone().to(dev), D.to(dev), K.to(dev), b.to(dev), a.to(dev), 0.3)
    ref = .5 * (oracle.frame_distance(P, D, K, a, b, 0.3) + oracle.frame_distance(P, D, K, b, a, 0.3))
    assert rel_err(.5 * (d1 + d2), ref, floor=1.0) < 1e-4
    ix = torch.arange(10)
    th = torch.full((10,), 0.05)
    cnt = backends.depth_filter(P.to(dev), D.to(dev), K.to(dev), ix.to(dev), th.to(dev))
    rcnt = oracle.depth_filter(P, D, K, ix, th)
    assert cnt.shape == rcnt.shape
    assert frac_equal(cnt, rcnt) > 0.999            # integer counts; a threshold flip needs |err - t| < 1e-7
    assert float(rcnt.max()) >= 1


def test_frame_distance_invalid_pairs_return_1000(backends):
    s = _scene(seed=4)
    P = s["poses"].clone(); P[5, 2] = -50.0          # frame 5 far behind: almost nothing valid
    fd = backends.frame_distance(P.to(dev), s["disps"].to(dev), s["intrinsics"].to(dev), torch.tensor([0], device=dev), torch.tensor([5], device=dev), 0.3)
    ref = oracle.frame_distance(P, s["disps"], s["intrinsics"], torch.tensor([0]), torch.tensor([5]), 0.3)
    assert float(ref) == 1000.0 and float(fd) == 1000.0


# ---------------------------------------------------------------------------------------------------
def _run_ba(capi, s, itrs, motion_only=False, lm=None, ep=None):
    lm = s["lm"] if lm is None else lm; ep = s["ep"] if ep is None else ep
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    dx, dz, M, st, _ = c_ba(capi, P, D, s["intrinsics"].to(dev), s["disps_sens"].to(dev), s["targets"].to(dev), s["weights"].to(dev),
                            s["eta"].to(dev), s["ii"].to(dev), s["jj"].to(dev), s["t0"], s["t1"], itrs, lm, ep, motion_only, s["M"])
    P64, D64 = s["poses"].double(), s["disps"].double()
    (rdx, rdz), ok = oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"],
                               s["t0"], s["t1"], itrs, lm, ep, motion_only, dtype=torch.float64, return_info=True)
    return dict(P=P.cpu(), D=D.cpu(), dx=dx.cpu(), dz=dz.cpu(), M=M, st=st, P64=P64, D64=D64, rdx=rdx, rdz=rdz, ok=ok)


@pytest.mark.parametrize("cfg", [dict(E=24, N=8, ht=48, wd=64), dict(E=40, N=10, ht=24, wd=32), dict(E=60, N=12, ht=20, wd=28, rgbd=True),
                                 dict(E=30, N=9, ht=16, wd=24, stereo=True)])
@pytest.mark.parametrize("itrs", [1, 3])
def test_ba_matches_fp64_oracle(capi, cfg, itrs):
    rgbd = cfg.pop("rgbd", False) if "rgbd" in cfg else False
    cfg = dict(cfg)
    s = _scene(seed=itrs, rgbd=rgbd, **cfg)
    r = _run_ba(capi, s, itrs)
    assert r["M"] == s["M"] and r["st"] == 0 and r["ok"]
    assert rel_err(r["P"], r["P64"], floor=1.0) < 1e-4            # updated poses
    assert rel_err(r["D"], r["D64"], floor=1.0) < 1e-4            # updated inverse depths
    assert rel_err(r["dx"], r["rdx"], floor=1e-2) < 1e-3          # last step itself (small numbers: looser relative floor)
    assert rel_err(r["dz"], r["rdz"], floor=1.0) < 1e-4


def test_ba_motion_only(capi):
    s = _scene(seed=9)
    r = _run_ba(capi, s, 2, motion_only=True)
    assert r["st"] == 0
    assert rel_err(r["P"], r["P64"], floor=1.0) < 1e-4
    assert torch.equal(r["D"], s["disps"])                        # depths untouched
    assert torch.isnan(r["dz"]).all()                             # dz_out untouched when motion_only


def test_ba_backend_settings_and_fixed_window(capi):
    """global-BA settings of update_lowmem (lm=1e-5, ep=1e-2, reference factor_graph.py:327-328) and a window whose
    first frames are fixed (t0 > 1) with edges reaching into the fixed part."""
    s = _scene(E=60, N=14, ht=16, wd=24, seed=10)
    s["t0"] = 4
    kx = torch.unique(torch.cat([torch.arange(s["t0"], s["t1"]), s["ii"]])); s["M"] = kx.shape[0]
    r = _run_ba(capi, s, 2, lm=1e-5, ep=1e-2)
    assert r["st"] == 0 and r["M"] == s["M"]
    assert rel_err(r["P"], r["P64"], floor=1.0) < 1e-4 and rel_err(r["D"], r["D64"], floor=1.0) < 1e-4
    assert torch.equal(r["P"][:4], s["poses"][:4])                # poses before t0 are not touched


def test_ba_pybind_matches_capi_and_mutates_in_place(capi, backends):
    s = _scene(seed=12)
    r = _run_ba(capi, s, 2)
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    out = backends.ba(P, D, s["intrinsics"].to(dev), s["disps_sens"].to(dev), s["targets"].to(dev), s["weights"].to(dev),
                      s["eta"].to(dev), s["ii"].to(dev), s["jj"].to(dev), s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    assert len(out) == 2 and out[0].shape == (s["t1"] - s["t0"], 6) and out[1].shape == (s["M"], 24 * 32)
    assert rel_err(P.cpu(), r["P"], floor=1.0) < 1e-6 and rel_err(D.cpu(), r["D"], floor=1.0) < 1e-6
    with pytest.raises(RuntimeError):
        backends.ba(P, D, s["intrinsics"].to(dev), s["disps_sens"].to(dev), s["targets"].to(dev).permute(0, 1, 3, 2), s["weights"].to(dev),
                    s["eta"].to(dev), s["ii"].to(dev), s["jj"].to(dev), s["t0"], s["t1"], 2, s["lm"], s["ep"], False)   # non-contiguous (src/droid.cpp:110)


def test_ba_cholesky_failure_gives_zero_update(capi):
    """non-SPD reduced system -> dx = 0 like the reference (src/droid_kernels.cu:1216-1219); forced with ep << 0"""
    s = _scene(seed=13)
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    dx, dz, M, st, _ = c_ba(capi, P, D, s["intrinsics"].to(dev), s["disps_sens"].to(dev), s["targets"].to(dev), s["weights"].to(dev),
                            s["eta"].to(dev), s["ii"].to(dev), s["jj"].to(dev), s["t0"], s["t1"], 1, 0.0, -1e9, True, s["M"])
    assert st & 4
    assert float(dx.abs().max()) == 0.0 and torch.equal(P.cpu(), s["poses"])


# ---------------------------------------------------------------------------------------------------
def test_corr_volume_pyramid_tcgen05_matches_reference_formula(backends):
    """CorrBlock.__init__ (reference modules/corr.py:24-38,63-71) in one wgmma/TMA kernel vs matmul + avg_pool2d"""
    g = torch.Generator().manual_seed(31)
    N, C, ht, wd = 5, 128, 16, 64
    fmaps = torch.randn(N, C, ht, wd, generator=g).half()
    ii = torch.tensor([0, 1, 2, 4, 3, 0]); jj = torch.tensor([1, 0, 4, 2, 3, 4])
    got = backends.corr_volume_pyramid(fmaps.to(dev), fmaps.to(dev), ii.to(dev), jj.to(dev))
    ref = oracle.corr_pyramid(fmaps[None, ii].float(), fmaps[None, jj].float(), num_levels=4)      # fp32 math on the fp16 inputs
    assert len(got) == 4
    for l in range(4):
        assert got[l].shape == (6, ht, wd, ht >> l, wd >> l)
        r = ref[l]
        err = (got[l].float().cpu() - r).abs().max()
        assert float(err) < 2e-2 + 2e-3 * float(r.abs().max()), (l, float(err))      # fp16 rounding of each level (values ~ +-30)
    # against the same pipeline on the GPU in fp16 (what the live system computes with cuBLAS + avg_pool2d)
    f = fmaps.to(dev)
    corr = torch.matmul((f[ii].reshape(6, C, -1) / 4.0).transpose(1, 2), f[jj].reshape(6, C, -1) / 4.0).reshape(6 * ht * wd, 1, ht, wd)
    for l in range(4):
        assert float((got[l].reshape(-1).float() - corr.reshape(-1).float()).abs().max()) < 6e-2
        corr = torch.nn.functional.avg_pool2d(corr, 2, stride=2)


def test_tensor_core_volume_plus_lookup_matches_oracle_corrblock(backends):
    """CorrBlock end to end the way the reference's class runs it on this module (constructor through the corr-volume hook,
    droid_slam_b200/modules.py; lookups through corr_index_forward / altcorr_forward) vs the oracle's CorrBlock restatement, and
    CorrBlock == AltCorrBlock (SURVEY section 4)"""
    g = torch.Generator().manual_seed(41)
    N, C, ht, wd = 4, 128, 16, 64
    fmaps = torch.randn(N, C, ht, wd, generator=g).half()
    ii = torch.tensor([0, 1, 2, 3, 0]); jj = torch.tensor([1, 2, 3, 0, 2])
    coords = torch.stack([torch.rand(1, 5, ht, wd, generator=g) * (wd + 4) - 2, torch.rand(1, 5, ht, wd, generator=g) * (ht + 4) - 2], dim=-1)
    f = fmaps.to(dev)
    pyr = backends.corr_volume_pyramid(f, f, ii.to(dev), jj.to(dev))
    c = coords.permute(0, 1, 4, 2, 3).contiguous().view(5, 2, ht, wd).to(dev)
    got = torch.cat([backends.corr_index_forward(pyr[l], (c / 2 ** l).contiguous(), 3)[0].view(1, 5, -1, ht, wd) for l in range(4)], dim=2)
    ref = oracle.corr_block_lookup(oracle.corr_pyramid(fmaps[None, ii].float(), fmaps[None, jj].float(), 4), coords, 3)
    assert got.shape == ref.shape == (1, 5, 196, ht, wd)
    assert float((got.float().cpu() - ref).abs().max()) < 0.1 and rel_err(got.float(), ref, floor=float(ref.abs().max())) < 5e-3
    lv = []
    fl = f
    c5 = coords.permute(0, 1, 4, 2, 3).contiguous().to(dev)
    for l in range(4):
        o, = backends.altcorr_forward(f[None].contiguous(), fl[None].contiguous(), (c5 / 2 ** l).contiguous(), ii.to(dev), jj.to(dev), 3)
        lv.append(o.flatten(2, 3))
        fl = torch.nn.functional.avg_pool2d(fl, 2, stride=2)
    alt = torch.stack(lv, dim=2).flatten(2, 3)
    assert alt.shape == got.shape
    assert rel_err(alt.float(), got.float(), floor=float(ref.abs().max())) < 1e-2      # two fp16 pipelines with different rounding points


@pytest.mark.parametrize("ht", [16, 48])
def test_fused_pyramid_lookup_and_tiled_volumes_are_bit_identical(backends, ht):
    """corr_lookup_pyramid (one launch, [E,196,H,W]) == cat of the four corr_index_forward results, for the reference layout and for
    the tiled private layout written by corr_volume_pyramid(tiled=True); the tiled planes are a pure re-ordering of the same values"""
    g = torch.Generator().manual_seed(51 + ht)
    N, C, wd, E = 5, 128, 64, 7
    fmaps = torch.randn(N, C, ht, wd, generator=g).half().to(dev)
    ii = torch.randint(0, N, (E,), generator=g).to(dev); jj = torch.randint(0, N, (E,), generator=g).to(dev)
    coords = torch.stack([torch.rand(E, ht, wd, generator=g) * (wd + 10) - 5, torch.rand(E, ht, wd, generator=g) * (ht + 10) - 5], dim=1)
    coords[0, :, 0, 0] = torch.tensor([float("inf"), 3.0]); coords[0, :, 0, 1] = torch.tensor([2.0, float("nan")]); coords[1, :, 1, 1] = torch.tensor([-50.0, 1e6])
    coords = coords.contiguous().to(dev)
    pyr = backends.corr_volume_pyramid(fmaps, fmaps, ii, jj)
    per_level = torch.cat([backends.corr_index_forward(pyr[l], (coords / 2 ** l).contiguous(), 3)[0].view(E, 49, ht, wd) for l in range(4)], dim=1)
    fused = backends.corr_lookup_pyramid(pyr, coords)
    assert fused.shape == (E, 196, ht, wd)
    assert_bit_identical(fused, per_level, "fused lookup, reference layout")
    tpyr = backends.corr_volume_pyramid(fmaps, fmaps, ii, jj, True)
    assert torch.equal(tpyr[2], pyr[2]) and torch.equal(tpyr[3], pyr[3])
    for l in (0, 1):                                   # [h2/4][w2/8][4][8] tiles -> [h2][w2]
        h2, w2 = ht >> l, wd >> l
        untiled = tpyr[l].view(E, ht, wd, h2 // 4, w2 // 8, 4, 8).permute(0, 1, 2, 3, 5, 4, 6).reshape(E, ht, wd, h2, w2)
        assert_bit_identical(untiled, pyr[l], "tiled level %d" % l)
    assert_bit_identical(backends.corr_lookup_pyramid(tpyr, coords, True), per_level, "fused lookup, tiled layout")


def test_fused_reproject_matches_projective_transform_restatement(backends):
    """A5: DepthVideo.reproject / pops.projective_transform(jacobian=False) in one kernel, incl. per-frame intrinsics, stereo edges
    and the MIN_DEPTH = 0.2 / Z < 0.1 -> 1 quirk (Q3)"""
    from droid_slam_b200.modules import reproject
    s = _scene(E=30, N=9, ht=16, wd=24, stereo=True, seed=6)
    K = s["intrinsics"][None].repeat(9, 1) * (1 + 0.01 * torch.arange(9)[:, None])      # per-frame intrinsics
    P = s["poses"].clone(); P[4, 2] += 1.2                                               # push some points behind / close to a camera
    c, v = reproject(P.to(dev), s["disps"].to(dev), K.to(dev), s["ii"], s["jj"])
    rc, rv = oracle.reproject(P, s["disps"], K, s["ii"], s["jj"])
    assert c.shape == (1, 30, 16, 24, 2) and v.shape == (1, 30, 16, 24, 1)
    assert rel_err(c[0], rc, floor=1.0) < 1e-4 and frac_equal(v[0], rv) > 0.999
    assert 0.05 < float(rv.mean()) < 1.0 and bool((s["ii"] == s["jj"]).any())


def _fused_p2p_two_virtual_ranks(backends, s):
    """The cross-GPU reduction fused into the Cholesky kernel (DESIGN.md section 6), exercised on ONE device: two edge shards
    ("ranks") build their partial pose systems into two buffers that play the role of peer memory, publish their epochs, and each
    rank's solve sums both copies itself.  Result must match the unsharded BA and be identical on both ranks."""
    from droid_slam_b200 import sharded

    class VirtualPeer:                       # what sharded.P2PSystem provides, without symmetric memory
        def __init__(self, nd, ptrs, rank):
            self.nd, self.ptrs, self.world, self.rank, self.epoch = nd, ptrs, len(ptrs), rank, 0
            self.epoch_dev = torch.zeros(1, dtype=torch.int64, device=dev)

    N, ht, wd = s["disps"].shape
    n = 6 * (s["t1"] - s["t0"]); nd = n * n + n
    bufs = [torch.zeros(2 * nd + 8, dtype=torch.float64, device=dev) for _ in range(2)]
    ptrs = [b.data_ptr() for b in bufs]
    bounds = sharded.partition_frames(s["ii"], N, 2)
    kx = torch.unique(torch.cat([torch.arange(s["t0"], s["t1"]), s["ii"]]))
    eta_f = torch.zeros(N, ht, wd); eta_f[kx] = s["eta"]
    common = [s[k].to(dev) for k in ("intrinsics", "disps_sens")]
    ranks = []
    for r in range(2):
        idx = sharded.shard_edges(s["ii"], *bounds[r])
        st = dict(P=s["poses"].to(dev), D=s["disps"].to(dev), tg=s["targets"][idx].contiguous().to(dev), wt=s["weights"][idx].contiguous().to(dev),
                  ii=s["ii"][idx].contiguous().to(dev), jj=s["jj"][idx].contiguous().to(dev), eta=eta_f.to(dev))
        eng = sharded.CApiEngine(dev)
        eng.setup(st["P"], st["D"], common[0], common[1], st["tg"], st["wt"], st["eta"], st["ii"], st["jj"], s["t0"], s["t1"], s["lm"], s["ep"],
                  bounds[r], p2p=VirtualPeer(nd, ptrs, r))
        ranks.append((eng, st))
    for _ in range(2):
        for eng, _ in ranks: eng.build()
        for eng, _ in ranks: eng.publish()
        for eng, _ in ranks: eng.solve()
    torch.cuda.synchronize()
    (e0, s0), (e1, s1) = ranks
    assert torch.equal(s0["P"], s1["P"]) and torch.equal(e0.dx, e1.dx)                 # replicated solve: bit-identical on both ranks
    D = torch.cat([s0["D"][:bounds[0][1]], s1["D"][bounds[1][0]:]])
    P1, D1 = s["poses"].to(dev), s["disps"].to(dev)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    backends.ba(P1, D1, *args, s["t0"], s["t1"], 2, s["lm"], s["ep"], False)
    assert float((s0["P"] - P1).abs().max()) < 2e-5 and float((D - D1).abs().max()) < 5e-5


def test_fused_p2p_reduction_two_virtual_ranks_on_one_gpu(backends):
    """the fused reduction on a frontend window (n = 144): resident Cholesky kernel"""
    _fused_p2p_two_virtual_ranks(backends, synth.make_scene("c2_frontend"))


def test_fused_p2p_reduction_cluster_kernel_two_virtual_ranks(backends):
    """the fused reduction on a 100-frame window at 24x32 (n = 594 > 448): the cluster Cholesky kernel's peer loader"""
    s = synth.make_scene(dict(E=400, N=100, ht=24, wd=32, stereo=False, itrs=2, lm=1e-4, ep=0.1))
    assert 448 < 6 * (s["t1"] - s["t0"]) <= 1024
    _fused_p2p_two_virtual_ranks(backends, s)
