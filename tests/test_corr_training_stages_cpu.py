"""The stage checks of the training CorrBlock (tests/test_corr_training_stages_gpu.py) without a GPU: that every case of
corr_training_cases.STAGES reaches the corner it is named for, and that the committed bounds sit below the worst-case error model.

Worst-case error model, in units of u A (u = 2^-24, A the summed magnitude of an output's K terms), first order in u:
  * 3xTF32 product.  x = hi + lo + d with hi = tf32(x), lo = tf32(x - hi); x - hi is exact in fp32 and below 2^-11 |x|, so rounding it
    to tf32 leaves |d| <= 2^-22 |x|.  Of (a_hi + a_lo)(b_hi + b_lo) the products hi.hi, hi.lo, lo.hi are exact in the fp32 accumulator
    (11 x 11 significant bits); the dropped lo.lo (<= 2^-22 |ab|) and the two lo roundings (<= 2^-22 |ab| each) cost 3 2^-22 = 12 per
    product, so 12 in all.
  * Tensor-core chunk sums.  Each 32-deep chunk is 4 k-steps of 3 MMAs accumulating from zero; each MMA is taken to round once, by
    truncation (2u), relative to at most the chunk's magnitude: 12 x 2 = 24 in all over the chunks.
  * fp32 adds of the chunk partials into the running sum: ceil(K / 32) adds, each <= u A: K / 32.
  * The volume's epilogue pools with two fp32 adds per level (the x 0.25 is exact), each bounded by the pooled magnitude: 2 l at level l.
  * The adjoint's pooled copy of f2 sums the 4^l pixels of a block in sequence, (4^l - 1) u P_l(|f2|) at most: 63 at level 3.
  * g_f2's spread adds the four levels' columns with three fp32 adds: 3.
So kappa <= 40 + 2 l for the volume (K = 128), 99 + ceil(Q / 32) for g_f1 (K = Q), 39 + ceil(HW / 32) for g_f2 (K = HW).  The
committed bounds c sqrt(K) (corr_training_cases.KAPPA_PER_SQRT_K) sit this far below the model, over the cases:
  volume  c = 0.6   K = 128          bound 6.8       model 40-46     5.9x below
  g_f1    c = 0.6   K = Q = 85-6370  bound 5.5-47.9  model 102-299   5.9-18x below
  g_f2    c = 1.25  K = HW = 64-4800 bound 10-87     model 41-189    1.8-4.1x below
The model is a worst case: rounding errors that all push one way, each at its bound.  The H100's worst kappa (tabled in the GPU test)
is 5.0 for the volume and 5.0 / 10.1 for g_f1 / g_f2, nearly flat in K: the chunked accumulation keeps long sums at a few units, and
the largest values come from sparse sums (few non-zero gradient terms, so nothing averages) at the smallest K.
"""
import math

import pytest
import torch

from corr_training_cases import KAPPA_PER_SQRT_K, NONFINITE, STAGES, special_coords, stage_cases, stage_inputs, stage_K


def kappa_model(stage, ht, wd, level=3):
    K = stage_K(stage, ht, wd)
    base = 12 + 24 + math.ceil(K / 32)
    return base + {"volume": 2 * level, "g_f1": 4 ** 3 - 1, "g_f2": 3}[stage]


def levels(ht, wd):
    return [(ht >> l, wd >> l) for l in range(4)]


def test_stage_cases_regenerate_from_seeds():
    assert [c[0] for c in stage_cases()] == list(STAGES)
    a, b = stage_inputs("odd_23x31"), stage_inputs("odd_23x31")
    for x, y in zip(a[:2], b[:2]):
        assert torch.equal(x, y)
    for x, y in zip(a[2] + a[3], b[2] + b[3]):
        assert torch.equal(torch.nan_to_num(x), torch.nan_to_num(y)) and torch.equal(torch.isnan(x), torch.isnan(y))


def test_each_case_reaches_its_corner():
    S = STAGES
    # 8x8: one 64-pixel source tile, one 8x8 target block, level 3 is 1x1
    n, ht, wd, _ = S["8x8"]
    assert ht * wd == 64 and (ht + 7) // 8 == (wd + 7) // 8 == 1 and levels(ht, wd)[3] == (1, 1)
    # odd_23x31: the floor rule drops a row and a column at every level, partial 8x8 blocks both ways, HW % 64 = 9
    n, ht, wd, _ = S["odd_23x31"]
    assert (ht * wd) % 64 == 9 and ht % 8 and wd % 8
    assert all((ht >> l) % 2 == 1 and (wd >> l) % 2 == 1 for l in range(3))
    assert [h for h, _ in levels(ht, wd)] == [23, 11, 5, 2] and [w for _, w in levels(ht, wd)] == [31, 15, 7, 3]
    # portrait: more block rows than block columns; every level width takes the generic lookup
    n, ht, wd, _ = S["portrait_70x43"]
    assert (ht + 7) // 8 > (wd + 7) // 8
    assert [wd >> l for l in range(4)] == [43, 21, 10, 5] and all((wd >> l) % 4 for l in range(4))
    # 8 rows / 8 columns with a long other side: level 3 is one row (column); 136 takes the chunked lookup at levels 0-1
    for name, one, long in (("rows8_8x136", 0, 1), ("cols8_136x8", 1, 0)):
        n, ht, wd, _ = S[name]
        l3 = levels(ht, wd)[3]
        assert l3[one] == 1 and l3[long] == 17
        assert [(wd >> l) % 4 == 0 for l in range(4)] == [True, True, False, False]
    # many edges: grid.z = n
    assert S["many_edges_9x13"][0] == 300
    assert S["train_24x48x64"] == (24, 48, 64, 15)
    # the adjoint's longest sums: longer than the training shape's K = Q = 4080 and K = HW = 3072
    n, ht, wd, _ = S["large_60x80"]
    assert stage_K("g_f1", ht, wd) == 6370 and stage_K("g_f2", ht, wd) == 4800
    assert stage_K("g_f1", 48, 64) == 4080 and stage_K("g_f2", 48, 64) == 3072
    assert all(stage_K("volume", ht, wd) == 128 for _, _, ht, wd, _ in stage_cases())
    assert max(stage_K("g_f1", ht, wd) for _, _, ht, wd, _ in stage_cases()) == 6370


def _windows(coords, ht, wd):
    """per call and level: [n, HW] whether pixel p's 8x8 footprint (the floor of coords / 2^l, -3 .. +4) meets level l, as
    corr_grad_accumulate decides it (NaN floors to 0; the floor saturates); and whether it lies partly outside"""
    meets, partly = [], []
    for c in coords:
        for l, (h, w) in enumerate(levels(ht, wd)):
            x, y = c[:, 0].reshape(c.shape[0], -1) / 2 ** l, c[:, 1].reshape(c.shape[0], -1) / 2 ** l
            fx = torch.nan_to_num(torch.floor(x), nan=0.0).clamp(-2 ** 30, 2 ** 30)
            fy = torch.nan_to_num(torch.floor(y), nan=0.0).clamp(-2 ** 30, 2 ** 30)
            mx, my = (fx + 4 >= 0) & (fx - 3 < w), (fy + 4 >= 0) & (fy - 3 < h)
            meets.append(mx & my)
            partly.append(mx & my & ((fx - 3 < 0) | (fx + 4 >= w) | (fy - 3 < 0) | (fy + 4 >= h)))
    return torch.stack(meets), torch.stack(partly)


@pytest.mark.parametrize("name", list(STAGES))
def test_coordinates_reach_every_category(name):
    n, ht, wd, calls = STAGES[name]
    _, _, coords, grads, pix, cats = stage_inputs(name)
    assert len(coords) == len(grads) == calls and coords[0].shape == (n, 2, ht, wd) and grads[0].shape == (n, 196, ht, wd)
    assert set(cats) >= {"half", "last0", "last1", "last2", "last3", "huge"} | set(NONFINITE)
    for c in coords:
        flat = c.view(n, 2, -1)
        for cat, (x, y), p in zip(cats, [s[1:] for s in special_coords(ht, wd)], pix.tolist()):
            edges = [0] if cat in NONFINITE else range(n)
            for e in edges:
                got, want = flat[e, :, p], torch.tensor([x, y], dtype=torch.float32)
                assert torch.equal(got.isnan(), want.isnan()) and torch.equal(got.nan_to_num(), want.nan_to_num()), (name, cat, e, got)
            if cat in NONFINITE and n > 1:
                assert bool(torch.isfinite(flat[1:, :, p]).all())
        # half-integers and each level's last row and column, scaled as the kernel scales them
        for l, (h, w) in enumerate(levels(ht, wd)):
            assert bool((flat[:, 0] / 2 ** l == w - 1).any()) and bool((flat[:, 1] / 2 ** l == h - 1).any())
        assert bool((torch.frac(flat) == 0.5).any()) and bool((flat.abs() == 1e30).any())
    meets, partly = _windows(coords, ht, wd)
    zero_rows = ~meets.any(0)                                   # [n, HW]: gradient rows that stay all zero
    assert bool(zero_rows[0].any()) and bool(zero_rows[1:].any())
    assert all(bool(partly[l::4].any()) for l in range(4)), name          # windows partly outside at every level (meets: call-major)
    if min(ht, wd) > 8:                                                   # and wholly inside level 0 (8 wide: only at floor 3)
        assert bool((meets & ~partly)[0::4].any()), name


@pytest.mark.parametrize("name", list(STAGES))
def test_committed_bounds_sit_below_the_error_model(name):
    _, ht, wd, _ = STAGES[name]
    for stage, c in KAPPA_PER_SQRT_K.items():
        bound = c * math.sqrt(stage_K(stage, ht, wd))
        worst = kappa_model(stage, ht, wd, level=0)
        assert bound < worst, (name, stage, bound, worst)


def test_error_model_terms():
    assert kappa_model("volume", 48, 64, 0) == 40 and kappa_model("volume", 48, 64, 3) == 46
    assert kappa_model("g_f1", 48, 64) == 36 + 128 + 63 and kappa_model("g_f2", 48, 64) == 36 + 96 + 3
    assert kappa_model("g_f1", 60, 80) == 36 + 200 + 63 and kappa_model("g_f2", 60, 80) == 36 + 150 + 3
