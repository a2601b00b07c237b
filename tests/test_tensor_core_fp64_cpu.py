"""The fp16-against-fp64 checker (`util.assert_faithful_f16`) on constructed values, and the case tables of
tests/test_tensor_core_fp64_gpu.py: the correlation volumes and the convolution route matrix, whose tiling is read back from
`dba_conv_nhwc_plan` so that a retune of the tiling rule cannot silently drop a route from the suite."""
import ctypes
import warnings

import numpy as np
import pytest
import torch

from droid_slam_b200 import c_api
from util import F16_OVERFLOW, assert_faithful_f16, faithful_f16

H100_SMS = 132          # SMs of an H100 SXM: more CTA tiles than this makes the persistent conv kernel loop


# ---- the checker -------------------------------------------------------------------------------------------------------------
def _f16(*vals):
    return np.array(vals, dtype=np.float64).astype(np.float16)


def _rn(x):
    """round-to-nearest-even fp16 of fp64 values, straight from fp64 (numpy rounds once)"""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.asarray(x, dtype=np.float64).astype(np.float16)


def _truth(h, exact, beta):
    """h is a rounding of some v in [exact - beta, exact + beta] iff RN(exact - beta) <= h <= RN(exact + beta): RN is monotone and
    every fp16 value between two roundings is itself the rounding of a value in between (exact - beta, exact + beta exact in fp64)"""
    lo, hi = _rn(exact - beta).astype(np.float64), _rn(exact + beta).astype(np.float64)
    hv = h.astype(np.float64)
    return ~np.isnan(hv) & (lo <= hv) & (hv <= hi)


def _grid():
    """fp16 values at every edge of the format, and exact values at, around and between them"""
    base = [0.0, 2.0 ** -24, 2 * 2.0 ** -24, 3 * 2.0 ** -24, 1023 * 2.0 ** -24, 2.0 ** -14, 2.0 ** -14 + 2.0 ** -24, 2.0 ** -13,
            2.0 ** -13 + 2.0 ** -23, 0.5, 1.0, 1.0 + 2.0 ** -10, 1.0 - 2.0 ** -11, 2.0, 3.0, 1000.5, 2048.0, 65472.0, 65504.0]
    hs = np.concatenate([_f16(*base), -_f16(*base[1:]), _f16(np.inf, -np.inf, np.nan)])
    ex = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for v in _f16(*base):
            for s in (1.0, -1.0):
                v64 = s * float(v)
                dn = float(np.nextafter(np.float16(v64), np.float16(-np.inf)))
                up = float(np.nextafter(np.float16(v64), np.float16(np.inf)))
                for n in (dn, up):
                    if np.isfinite(n):
                        for f in (0.0, 0.25, 0.5, 0.75):
                            ex.append(v64 + f * (n - v64))
                            ex.append(v64 + f * (n - v64) + 2.0 ** -40 * abs(n - v64))
                            ex.append(v64 + f * (n - v64) - 2.0 ** -40 * abs(n - v64))
    ex += [F16_OVERFLOW, -F16_OVERFLOW, F16_OVERFLOW - 2.0 ** -20, 65536.0, 1e6, -1e6]
    return hs, np.unique(np.array(ex, dtype=np.float64))


BETAS = [0.0, 2.0 ** -27, 2.0 ** -26, 2.0 ** -25, 2.0 ** -24, 2.0 ** -13, 2.0 ** -12, 2.0 ** -11, 2.0 ** -10, 0.25, 8.0, 16.0, 17.0]


def test_checker_accepts_exactly_the_roundings_of_the_beta_interval():
    hs, ex = _grid()
    H, X, B = np.meshgrid(hs, ex, np.array(BETAS), indexing="ij")
    want = _truth(H, X, B)
    ok, dist = faithful_f16(torch.from_numpy(H.copy()), torch.from_numpy(X.copy()), torch.from_numpy(B.copy()))
    got = ok.numpy()
    bad = np.argwhere(got != want)
    assert bad.size == 0, ["h %r exact %r beta %r: checker %s" % (H[tuple(i)], X[tuple(i)], B[tuple(i)], got[tuple(i)]) for i in bad[:8]]
    assert want.any() and not want.all()
    # the distance to the rounding interval is what beta must reach (some distances are a few fp64 ulps of `exact`, hence 1.5 and 0.5)
    d = dist.numpy()
    fin = np.isfinite(d) & (d > 0)
    ok2, _ = faithful_f16(torch.from_numpy(H[fin]), torch.from_numpy(X[fin]), torch.from_numpy(d[fin] * 1.5))
    assert bool(ok2.all())
    ok3, _ = faithful_f16(torch.from_numpy(H[fin]), torch.from_numpy(X[fin]), torch.from_numpy(d[fin] * 0.5))
    assert not bool(ok3.any())


@pytest.mark.parametrize("h, exact, beta, accepted", [
    (1.0, 1.0 + 2.0 ** -11, 0.0, True),                        # tie between 1 (even) and 1 + 2^-10 (odd): rounds to 1
    (1.0 + 2.0 ** -10, 1.0 + 2.0 ** -11, 0.0, False),
    (1.0 + 2.0 ** -10, 1.0 + 2.0 ** -11, 2.0 ** -40, True),    # any beta > 0 reaches past the tie
    (2.0, 2.0 - 2.0 ** -11, 0.0, True),                        # below a power of two the spacing halves: tie at 2 - 2^-11, 2 is even
    (2.0 - 2.0 ** -10, 2.0 - 2.0 ** -11, 0.0, False),
    (2.0, 2.0 - 2.0 ** -10, 2.0 ** -11 - 2.0 ** -30, False),
    (2.0, 2.0 + 2.0 ** -10, 0.0, True),                        # above it the tie is at 2 + 2^-10
    (2.0, 2.0 + 2.0 ** -10 + 2.0 ** -30, 0.0, False),
    (2.0 ** -24, 2.0 ** -25, 0.0, False),                      # smallest subnormal: the tie with 0 goes to 0
    (0.0, 2.0 ** -25, 0.0, True),
    (2.0 ** -24, 1.5 * 2.0 ** -24, 0.0, False),                # 1.5 ulp ties to 2 * 2^-24 (even), not to 2^-24 (odd)
    (2.0 ** -24, 1.5 * 2.0 ** -24, 2.0 ** -30, True),
    (2 * 2.0 ** -24, 1.5 * 2.0 ** -24, 0.0, True),
    (1023 * 2.0 ** -24, 2.0 ** -14 - 2.0 ** -25, 0.0, False),  # largest subnormal (odd) / smallest normal: the tie goes up
    (2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 0.0, True),
    (-(2.0 ** -14), -(2.0 ** -14) - 2.0 ** -25 + 2.0 ** -30, 0.0, True),
    (65504.0, 65519.0, 0.0, True),
    (65504.0, F16_OVERFLOW, 0.0, False),                       # 65520 rounds to inf
    (np.inf, F16_OVERFLOW, 0.0, True),
    (np.inf, 65519.0, 0.0, False),
    (np.inf, 65519.0, 1.0, True),
    (-np.inf, -65500.0, 19.0, False),
    (-np.inf, -65500.0, 20.0, True),
    (np.nan, 1.0, 1e9, False),                                 # NaN is never a rounding of a finite value
    (-0.0, -(2.0 ** -26), 0.0, True),
    (0.0, -(2.0 ** -26), 0.0, True),
])
def test_checker_on_named_edges(h, exact, beta, accepted):
    got = torch.tensor([h], dtype=torch.float64).half()
    ok, _ = faithful_f16(got, torch.tensor([exact], dtype=torch.float64), torch.tensor([beta], dtype=torch.float64))
    assert bool(ok[0]) == accepted
    assert bool(_truth(got.numpy(), np.array([exact]), np.array([beta]))[0]) == accepted


def test_assert_faithful_reports_rounding_fraction_and_kappa():
    exact = torch.tensor([1.0, 1.0 + 2.0 ** -12, 3.0, 100.0], dtype=torch.float64)
    got = torch.tensor([1.0, 1.0, 3.0, 100.0 + 2.0 ** -4], dtype=torch.float16)      # the last one is one ulp (2^-4) off
    unit = torch.full_like(exact, 2.0 ** -10)
    frac, kappa = assert_faithful_f16(got, exact, 64 * unit, "demo", unit=unit)
    assert frac == 0.75
    assert kappa == 32.0                                        # 2^-5 past the half-ulp midpoint = 32 units of 2^-10
    with pytest.raises(AssertionError, match="1 of 4"):
        assert_faithful_f16(got, exact, 31 * unit, "demo", unit=unit)
    with pytest.raises(AssertionError):
        assert_faithful_f16(torch.tensor([float("nan")]).half(), torch.tensor([0.0], dtype=torch.float64), 1e30)


# ---- correlation volume cases ------------------------------------------------------------------------------------------------
# (name, ht, wd, n_frames1, n_frames2, ii, jj, tiled, feature scale).  The wd = 64, ht % 8 == 0 shapes take the whole-chunk tiling
# (optionally writing levels 0-1 in the tiled layout); every other shape the row tiling, staged through rows padded to 8 pixels when
# wd % 8 != 0.  Row chunks are 4 target rows: odd and even chunk counts pair level-2 rows into level-3 rows differently.
def _edges(n1, n2, E, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, n1, (E,), generator=g).tolist(), torch.randint(0, n2, (E,), generator=g).tolist()


CORR_CASES = [
    ("wd64_16x64", 16, 64, 3, 3, [0, 1, 2], [1, 2, 0], False, 1.0),
    ("wd64_16x64_tiled", 16, 64, 3, 3, [0, 1, 2], [1, 2, 0], True, 1.0),
    ("wd64_48x64", 48, 64, 2, 2, [0, 1], [1, 0], False, 1.0),
    ("wd64_48x64_tiled", 48, 64, 2, 2, [0, 1], [1, 0], True, 1.0),
    ("rows_8x8", 8, 8, 3, 3, [0, 1, 2], [2, 0, 1], False, 1.0),
    ("rows_30x40", 30, 40, 3, 3, [0, 2, 1], [1, 1, 2], False, 1.0),
    ("rows_72x96", 72, 96, 2, 2, [1], [0], False, 1.0),
    ("rows_24x128", 24, 128, 2, 2, [0, 1], [1, 0], False, 1.0),              # two full 64-column tiles
    ("staged_9x13", 9, 13, 3, 3, [0, 1, 2, 0], [1, 2, 0, 0], False, 1.0),
    ("staged_43x70", 43, 70, 2, 2, [0, 1], [1, 0], False, 1.0),              # 11 row chunks, trailing row dropped
    ("staged_44x69", 44, 69, 2, 2, [1], [0], False, 1.0),                    # trailing column dropped
    ("staged_41x73", 41, 73, 2, 2, [0], [1], False, 1.0),                    # both dropped, two column tiles
    ("staged_10x19", 10, 19, 3, 3, [0, 1], [2, 2], False, 1.0),
    ("staged_11x30", 11, 30, 3, 3, [2, 0], [0, 1], False, 1.0),
    ("staged_14x27", 14, 27, 3, 3, [0, 1], [1, 2], False, 1.0),              # an even chunk count on the staged route
    ("frames_staged_43x70", 43, 70, 3, 5, [2, 0, 2, 1], [4, 4, 0, 3], False, 1.0),
    ("frames_wd64_16x64", 16, 64, 5, 2, [4, 1, 4, 0], [1, 1, 0, 1], False, 1.0),
    ("frames_wd64_16x64_tiled", 16, 64, 5, 2, [4, 1, 4, 0], [1, 1, 0, 1], True, 1.0),
    ("many_edges_8x8", 8, 8, 8, 6) + _edges(8, 6, 300, 11) + (False, 1.0),
    ("subnormal_30x40", 30, 40, 3, 3, [0, 1, 2], [1, 2, 0], False, 2.0 ** -5),   # level 0 partly in fp16's subnormal range
]


def corr_features(case, seed=0):
    name, ht, wd, n1, n2 = case[:5]
    scale = case[8]
    g = torch.Generator().manual_seed(1000 * ht + wd + seed)
    f1 = (torch.randn(n1, 128, ht, wd, generator=g) * scale).half()
    f2 = (torch.randn(n2, 128, ht, wd, generator=g) * scale).half()
    return f1, f2


def test_corr_cases_cover_both_tilings_and_staging():
    routes = set()
    for name, ht, wd, n1, n2, ii, jj, tiled, _ in CORR_CASES:
        assert len(ii) == len(jj) and max(ii) < n1 and max(jj) < n2 and ht >= 8 and wd >= 8
        assert not tiled or (wd == 64 and ht % 8 == 0)
        route = "wd64" if (wd == 64 and ht % 8 == 0) else ("rows" if wd % 8 == 0 else "staged")
        routes.add((route, tiled, n1 != n2, ((ht + 3) // 4) % 2))
    assert {("wd64", False, False, 0), ("wd64", True, False, 0), ("wd64", False, True, 0), ("rows", False, False, 0),
            ("staged", False, False, 1), ("staged", False, False, 0), ("staged", False, True, 1)} <= routes


# ---- convolution route matrix ------------------------------------------------------------------------------------------------
# (name, E, ht, wd, c0, stride0, c1, stride1, ksize, n_out, relu, out_stride, value scale).  The first 18 rows are the cases of the
# earlier torch-conv comparisons; the rest add the routes those never took.
CONV_CASES = [
    ("tw64_mt2", 3, 16, 64, 128, 128, 0, 0, 3, 128, True, 128, 1.0),
    ("tw64_two_src_n256", 2, 16, 64, 128, 128, 320, 320, 3, 256, False, 256, 1.0),
    ("tw64_n384", 2, 8, 64, 128, 128, 0, 0, 3, 384, True, 384, 1.0),
    ("tw32_1x1_c196_pitch200", 3, 16, 32, 196, 200, 0, 0, 1, 128, True, 128, 1.0),
    ("tw32_n64", 2, 24, 96, 128, 128, 0, 0, 3, 64, True, 64, 1.0),
    ("tw32_partial_n32", 2, 10, 40, 64, 64, 0, 0, 3, 32, False, 32, 1.0),
    ("tw64_300_tiles", 150, 8, 64, 64, 64, 0, 0, 3, 128, True, 128, 1.0),
    ("flat_43x70_156_tiles", 12, 43, 70, 128, 128, 0, 0, 3, 128, True, 128, 1.0),
    ("flat_two_src_n256", 12, 44, 69, 128, 128, 320, 320, 3, 256, False, 256, 1.0),
    ("flat_n384", 6, 41, 73, 128, 128, 0, 0, 3, 384, True, 384, 1.0),
    ("flat_1x1_c196_pitch200", 12, 44, 69, 196, 200, 0, 0, 1, 128, True, 128, 1.0),
    ("flat_n64", 12, 43, 70, 128, 128, 0, 0, 3, 64, True, 64, 1.0),
    ("flat_n32", 12, 41, 73, 64, 64, 0, 0, 3, 32, False, 32, 1.0),
    ("flat_eta_head", 24, 41, 73, 256, 256, 0, 0, 1, 32, False, 32, 1.0),
    ("flat_9x13", 3, 9, 13, 128, 128, 0, 0, 3, 128, True, 128, 1.0),
    ("flat_9x13_1x1", 3, 9, 13, 64, 64, 0, 0, 1, 32, True, 32, 1.0),
    ("rect_pitch160_smem", 2, 12, 157, 128, 128, 0, 0, 3, 128, True, 128, 1.0),
    ("rect_pitch264", 2, 6, 261, 64, 64, 0, 0, 3, 64, True, 64, 1.0),
    ("tw32_n96_out_stride", 2, 20, 48, 128, 128, 0, 0, 3, 96, True, 104, 1.0),
    ("flat_n160", 2, 17, 37, 128, 128, 0, 0, 3, 160, False, 160, 1.0),
    ("tw64_1x1_n192_out_stride", 2, 12, 64, 64, 64, 0, 0, 1, 192, True, 256, 1.0),
    ("flat_n224_c96", 2, 11, 30, 96, 96, 0, 0, 3, 224, True, 224, 1.0),
    ("tw64_mt4", 2, 16, 64, 256, 256, 0, 0, 3, 64, True, 64, 1.0),
    ("tw32_mt4_c1_136", 2, 16, 32, 128, 128, 136, 136, 3, 32, False, 32, 1.0),
    ("flat_mt4", 2, 21, 45, 256, 256, 0, 0, 3, 64, True, 64, 1.0),
    ("flat_mt4_c1_100", 2, 13, 50, 128, 128, 100, 104, 3, 32, True, 40, 1.0),
    ("flat_c0_40", 2, 9, 20, 40, 40, 0, 0, 3, 128, True, 128, 1.0),
    ("tw32_c0_48", 2, 9, 24, 48, 48, 0, 0, 3, 64, False, 64, 1.0),
    ("tiny_1x1", 2, 1, 1, 64, 64, 0, 0, 3, 32, True, 32, 1.0),
    ("tiny_1x9", 2, 1, 9, 128, 128, 0, 0, 3, 64, False, 64, 1.0),
    ("tiny_2x3", 3, 2, 3, 72, 72, 0, 0, 3, 96, True, 96, 1.0),
    ("subnormal_out", 2, 12, 40, 128, 128, 0, 0, 3, 128, False, 128, 2.0 ** -14),
]
CONV_IDS = [c[0] for c in CONV_CASES]


def conv_plan(L, ht, wd, c0, c1, ks, n):
    plan = (ctypes.c_int * 8)()
    c_api.check(L.dba_conv_nhwc_plan(ht, wd, c0, c1, ks, n, ctypes.cast(plan, ctypes.c_void_p)), "conv_nhwc_plan")
    return dict(zip(("flat", "TW", "MT", "N", "n_ntiles", "tiles", "a_stages", "b_stages"), list(plan)))


def route(plan, wd):
    if plan["flat"]:
        return "flat"
    if plan["TW"] == 64:
        return "tw64"
    return "tw32" if wd % 8 == 0 else ("tw32_fallback_pitch" if (wd + 7) // 8 * 8 > 256 else "tw32_fallback_smem")


def test_conv_plan_matches_the_tiling_rule():
    L = c_api.load()
    p = conv_plan(L, 16, 64, 128, 0, 3, 128)
    assert p == dict(flat=0, TW=64, MT=2, N=128, n_ntiles=1, tiles=4, a_stages=3, b_stages=5)   # 6-row halo boxes of 48 KB
    p = conv_plan(L, 41, 73, 128, 0, 3, 384)
    assert (p["flat"], p["TW"], p["MT"], p["N"], p["n_ntiles"]) == (1, 80, 1, 192, 2) and p["tiles"] == (41 * 80 + 127) // 128
    plan = (ctypes.c_int * 8)()
    for bad in ((0, 8, 64, 0, 3, 64), (8, 8, 64, 0, 5, 64), (8, 8, 64, 0, 3, 288), (8, 8, 100, 64, 3, 64), (8, 8, 0, 0, 3, 64)):
        assert L.dba_conv_nhwc_plan(*bad, ctypes.cast(plan, ctypes.c_void_p)) == 1


def test_conv_matrix_covers_every_route():
    L = c_api.load()
    seen = dict(route=set(), mt=set(), n=set(), ks=set())
    flags = set()
    for name, E, ht, wd, c0, s0, c1, s1, ks, n, relu, ostride, scale in CONV_CASES:
        p = conv_plan(L, ht, wd, c0, c1, ks, n)
        r = route(p, wd)
        seen["route"].add(r)
        seen["mt"].add((p["flat"], p["MT"]))
        seen["n"].add(n)
        seen["ks"].add(ks)
        if p["n_ntiles"] * E * p["tiles"] > H100_SMS:
            flags.add("more_tiles_than_sms")
        if c0 < 64:
            flags.add("c0_below_64")
        if s0 > c0:
            flags.add("c0_on_longer_pitch")
        if c1 and c1 % 64:
            flags.add("c1_remainder")
        if ostride > n:
            flags.add("out_stride")
        if scale < 2.0 ** -10:
            flags.add("subnormal")
        if (ht, wd) in ((1, 1), (1, 9), (2, 3)):
            flags.add((ht, wd))
    assert seen["route"] == {"flat", "tw64", "tw32", "tw32_fallback_pitch", "tw32_fallback_smem"}
    assert seen["mt"] == {(f, m) for f in (0, 1) for m in (1, 2, 4)}         # MT 1, 2, 4 on the rectangular and the flattened tiles
    assert seen["n"] == {32, 64, 96, 128, 160, 192, 224, 256, 384}
    assert seen["ks"] == {1, 3}
    assert flags == {"more_tiles_than_sms", "c0_below_64", "c0_on_longer_pitch", "c1_remainder", "out_stride", "subnormal", (1, 1), (1, 9), (2, 3)}
