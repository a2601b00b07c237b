"""The training CorrBlock's kernels (csrc/corr_train.cu) stage by stage through the C ABI, against fp64 formulas evaluated on the card,
element by element (cases: corr_training_cases.STAGES, their corners checked in tests/test_corr_training_stages_cpu.py).

Every output lies in a NaN-filled fp32 buffer with GUARD floats of NaN on each side (test_tensor_core_fp64_gpu.Guarded): the guards must
come back untouched, and no NaN may remain where the fp64 value is finite.  The adjoint's workspace is exactly
dba_corr_adjoint_workspace_bytes of 0xFF bytes (NaN floats) between two guards, so a read of a part the kernels never wrote shows up as
a NaN in an output.

With u = 2^-24 and A the summed magnitude of an output's terms, kappa = |native - exact| / (u A):
  volume  exact_0 = sum_c f1 f2 / 16 in fp64 from the fp32 maps, A_0 = sum_c |f1 f2| / 16; levels 1-3 the fp64 avg_pool2d (floor) of
          exact_0 and A_0.  K = 128.
  g_f1    (1/16) sum_l sum_q P_l(f2)[c,q] G_l[p,q], P_l the 2^l x 2^l block mean; A with |.| on every factor.  K = Q.
  g_f2    (1/16) sum_l [(y>>l, x>>l) inside level l's floor grid] 4^-l sum_p f1[c,p] G_l[p,(y>>l, x>>l)]; A likewise.  K = HW.
Where A = 0 the output must be exactly 0 (a gradient row that is all zero gives an exactly zero g_f1 column).  Where the fp64 value is
not finite the native one must not be finite either; NaN is accepted where fp64 has +-inf, because 3xTF32 splits an infinite x into
hi = inf and lo = inf - inf = NaN.  The adjoint runs on the gradient pyramid the case's lookups produce (with all-zero rows and, on
edge 0, NaN from NaN coordinates) and on a dense N(0,1) pyramid with every column non-zero.  The bounds are kappa <= c sqrt(K), one c
per stage (corr_training_cases.KAPPA_PER_SQRT_K); the worst-case model they sit under is derived in the CPU test.

The gradient pyramid after 1, 2 and all of a case's calls to dba_corr_grad_accumulate must equal, bit for bit and NaN for NaN, the
call-order fp32 sum of dba_corr_index_backward on each level at coords / 2^l.  Every stage's n-edge call equals n one-edge calls bit
for bit.

Worst kappa on one H100 80GB HBM3 at a 700 W power limit.  Volume levels 0 / 1 / 2 / 3 (K = 128, bound 6.8); g_f1 (K = Q) and g_f2
(K = HW) on the lookups' pyramid / the dense one, with the bound 0.6 sqrt(Q) / 1.25 sqrt(HW):
  case              volume                    Q     g_f1          bound   HW    g_f2          bound
  8x8               3.13 1.35  0.543 0.249      85  3.73  3.66     5.5     64  4.0   2.9     10.0
  odd_23x31         3.98 1.71  0.802 0.344     919  2.86  1.34    18.2    713  4.83  1.38    33.4
  portrait_70x43    3.85 1.89  0.785 0.425    3955  2.0   1.03    37.7   3010  4.14  1.11    68.6
  rows8_8x136       3.75 1.68  0.788 0.398    1445  2.06  1.56    22.8   1088  2.4   1.1     41.2
  cols8_136x8       3.75 1.71  0.724 0.342    1445  3.06  1.2     22.8   1088  2.11  1.03    41.2
  many_edges_9x13   3.35 1.57  0.767 0.346     148  4.99  3.29     7.3    117  10.1  3.4     13.5
  train_24x48x64    5.04 2.1   0.974 0.501    4080  2.14  1.76    38.3   3072  1.67  1.25    69.3
  large_60x80       4.26 2.02  0.939 0.404    6370  2.73  1.23    47.9   4800  2.33  0.978   86.6
kappa hardly grows with K; the c of g_f1 and g_f2 are set by many_edges_9x13, whose 300 edges give the most sparse sums at the
smallest K.  Accumulating all of K inside the MMAs (the adjoint GEMM carrying its sum through the tensor cores, built once on a
scratch copy) gave g_f1 kappa 8.2-80 and fails the g_f1 bound in every case, on the dense pyramid at least.  The sqrt(K) bounds do
not separate it in g_f1 on the lookups' pyramid at portrait_70x43, rows8_8x136, cols8_136x8 and large_60x80 (18.8-37.1), and in
g_f2 they separate it only at many_edges_9x13 and on odd_23x31's lookups pyramid (elsewhere g_f2 reached 5.8-68.4 under it).
"""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from droid_slam_b200 import c_api
from corr_training_cases import KAPPA_PER_SQRT_K, STAGES, stage_inputs, stage_K
from test_tensor_core_fp64_gpu import GUARD, UNIT, Guarded
from util import ptr, stream

pytestmark = pytest.mark.gpu
dev = "cuda"
C = 128
WS_GUARD = 4 * GUARD            # bytes of 0xFF before and after the adjoint's workspace
CHUNK = 1 << 26                 # fp64 elements per truth slice: edges are taken a few at a time
_CACHE = {}


def _report(stage, name, stats):
    print("CORR_STAGES %s %s %s" % (stage, name, json.dumps(stats)))
    out = os.environ.get("CORR_STAGES_REPORT")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(dict(stage=stage, case=name, **stats)) + "\n")


def inputs(name):
    if name not in _CACHE:
        _CACHE.clear()
        _CACHE[name] = stage_inputs(name, dev=dev)
    return _CACHE[name]


def sizes(ht, wd):
    hw = [(ht >> l, wd >> l) for l in range(4)]
    return hw, sum(h * w for h, w in hw)


def edge_slices(n, per_edge):
    step = max(1, CHUNK // per_edge)
    return [slice(e, min(n, e + step)) for e in range(0, n, step)]


def kappa(got, exact, mag, what):
    """worst kappa of `got` (fp32) against `exact` with magnitudes `mag` (fp64), after the non-finite and zero rules of the module
    docstring"""
    fin = torch.isfinite(exact)
    assert bool(torch.isfinite(got[fin]).all()), "%s: %d non-finite outputs where fp64 is finite" % (what, int((~torch.isfinite(got) & fin).sum()))
    assert not bool(torch.isfinite(got[~fin]).any()), "%s: finite outputs where fp64 is not" % what
    assert bool((torch.isnan(got) | ~torch.isnan(exact)).all()), "%s: a number where fp64 is NaN" % what
    zero = fin & (mag == 0)
    assert bool((got[zero] == 0).all()), "%s: non-zero outputs whose terms are all zero" % what
    err = torch.where(fin, (got.double() - exact).abs(), torch.zeros_like(exact))
    k = torch.where(fin & (mag > 0), err / (UNIT * mag), torch.zeros_like(exact))
    return float(k.max()) if k.numel() else 0.0


def same_bits(got, want, what):
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), "%s: NaN at %d places, expected %d" % (what, int(gn.sum()), int(wn.sum()))
    diff = (got.view(torch.int32) != want.view(torch.int32)) & ~gn
    assert not bool(diff.any()), "%s: %d of %d elements differ" % (what, int(diff.sum()), got.numel())


# ---- calls through the C ABI -------------------------------------------------------------------------------------------------
def c_volume(L, f1, f2):
    n, _, ht, wd = f1.shape
    hw, _ = sizes(ht, wd)
    outs = [Guarded(n, ht, wd, h, w, dtype=torch.float32) for h, w in hw]
    c_api.check(L.dba_corr_volume_pyramid_f32(ptr(f1), ptr(f2), *[ptr(o.t) for o in outs], n, C, ht, wd, stream()), "corr_volume_pyramid_f32")
    torch.cuda.synchronize()
    for l, o in enumerate(outs):
        o.check_guards("corr_volume_pyramid_f32 level %d" % l)
    return [o.t for o in outs]


def c_accumulate(L, coords, grads, gpyr):
    """one dba_corr_grad_accumulate call per (coords, grad) pair, in order"""
    for c, g in zip(coords, grads):
        n, _, ht, wd = c.shape
        c_api.check(L.dba_corr_grad_accumulate(ptr(c), ptr(g), ptr(gpyr), n, ht, wd, stream()), "corr_grad_accumulate")


def grad_pyramid(L, coords, grads, ht, wd):
    """the native gradient pyramid [n, HW, Q] of all calls, in a zeroed guarded buffer"""
    n = coords[0].shape[0]
    g = Guarded(n, ht * wd, sizes(ht, wd)[1], dtype=torch.float32)
    g.t.zero_()
    c_accumulate(L, coords, grads, g.t)
    torch.cuda.synchronize()
    g.check_guards("corr_grad_accumulate")
    return g.t


def c_adjoint(L, f1, f2, gpyr):
    n, _, ht, wd = f1.shape
    need = L.dba_corr_adjoint_workspace_bytes(n, C, ht, wd)
    ws = torch.full((need + 2 * WS_GUARD,), 255, dtype=torch.uint8, device=dev)
    g1, g2 = Guarded(n, C, ht, wd, dtype=torch.float32), Guarded(n, C, ht, wd, dtype=torch.float32)
    c_api.check(L.dba_corr_adjoint(ptr(f1), ptr(f2), ptr(gpyr), ptr(g1.t), ptr(g2.t), n, C, ht, wd, ptr(ws[WS_GUARD:]), need, stream()),
                "corr_adjoint")
    torch.cuda.synchronize()
    g1.check_guards("corr_adjoint g_f1")
    g2.check_guards("corr_adjoint g_f2")
    assert bool((ws[:WS_GUARD] == 255).all() and (ws[-WS_GUARD:] == 255).all()), "corr_adjoint wrote outside its workspace"
    return g1.t, g2.t


def index_backward_pyramid(L, coords, grad, ht, wd):
    """[n, HW, Q]: dba_corr_index_backward of each level at coords / 2^l, levels concatenated along the row"""
    n = coords.shape[0]
    hw, _ = sizes(ht, wd)
    parts = []
    for l, (h, w) in enumerate(hw):
        out = torch.full((n, ht, wd, h, w), float("nan"), device=dev)
        cl, gl = (coords / 2 ** l).contiguous(), grad[:, 49 * l:49 * (l + 1)].contiguous()
        c_api.check(L.dba_corr_index_backward(ptr(cl), ptr(gl), ptr(out), n, ht, wd, h, w, 3, c_api.DBA_F32, stream()), "corr_index_backward")
        parts.append(out.view(n, ht * wd, h * w))
    return torch.cat(parts, 2)


# ---- fp64 truths ---------------------------------------------------------------------------------------------------------------
def volume_truth(f1, f2):
    """levels 0-3 [m, ht, wd, h_l, w_l] of exact and of A, fp64"""
    m, _, ht, wd = f1.shape
    a, b = f1.reshape(m, C, -1).double(), f2.reshape(m, C, -1).double()
    ex = (a.transpose(1, 2) @ b / 16).view(-1, 1, ht, wd)
    mag = (a.abs().transpose(1, 2) @ b.abs() / 16).view(-1, 1, ht, wd)
    out = []
    for l in range(4):
        if l:
            ex, mag = F.avg_pool2d(ex, 2, stride=2), F.avg_pool2d(mag, 2, stride=2)
        out.append((ex.view(m, ht, wd, ht >> l, wd >> l), mag.view(m, ht, wd, ht >> l, wd >> l)))
    return out


def pooled(f):
    """[m, C, Q]: P_l(f) of every level, concatenated"""
    return torch.cat([(F.avg_pool2d(f, 2 ** l) if l else f).flatten(2) for l in range(4)], 2)


def spread(H, ht, wd):
    """g_f2 [m, C, ht, wd] from H [m, C, Q]: level l's element (y >> l, x >> l) / 4^l on every pixel of its block"""
    m = H.shape[0]
    out = H[..., :ht * wd].reshape(m, C, ht, wd).clone()
    off = ht * wd
    for l in range(1, 4):
        h, w, b = ht >> l, wd >> l, 1 << l
        blk = H[..., off:off + h * w].reshape(m, C, h, w) / 4 ** l
        out[..., :h * b, :w * b] += blk.repeat_interleave(b, 2).repeat_interleave(b, 3)
        off += h * w
    return out


def adjoint_truth(f1, f2, G):
    """(g_f1, A), (g_f2, A) in fp64, [m, C, ht, wd]"""
    m, _, ht, wd = f1.shape
    a, b, g = f1.double(), f2.double(), G.double()
    g1 = (pooled(b) @ g.transpose(1, 2) / 16).view(m, C, ht, wd)
    a1 = (pooled(b.abs()) @ g.abs().transpose(1, 2) / 16).view(m, C, ht, wd)
    g2 = spread(a.reshape(m, C, -1) @ g / 16, ht, wd)
    a2 = spread(a.abs().reshape(m, C, -1) @ g.abs() / 16, ht, wd)
    return (g1, a1), (g2, a2)


# ---- tests ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(STAGES))
def test_volume_and_levels_match_fp64(capi, name):
    n, ht, wd, _ = STAGES[name]
    f1, f2 = inputs(name)[:2]
    got = c_volume(capi, f1, f2)
    for l, v in enumerate(got):
        assert not bool(torch.isnan(v).any()), "%s level %d: an element was never written" % (name, l)
    bound = KAPPA_PER_SQRT_K["volume"] * stage_K("volume", ht, wd) ** 0.5
    worst = [0.0] * 4
    for s in edge_slices(n, 2 * (ht * wd) ** 2):
        for l, (ex, mag) in enumerate(volume_truth(f1[s], f2[s])):
            worst[l] = max(worst[l], kappa(got[l][s], ex, mag, "%s level %d" % (name, l)))
    _report("volume", name, dict(kappa=[float("%.3g" % k) for k in worst], per_sqrt_K=float("%.3g" % (max(worst) / 128 ** 0.5))))
    assert max(worst) <= bound, (name, worst, bound)


@pytest.mark.parametrize("name", list(STAGES))
def test_gradient_pyramid_is_the_call_order_sum_of_corr_index_backward(capi, name):
    n, ht, wd, calls = STAGES[name]
    _, _, coords, grads = inputs(name)[:4]
    g = Guarded(n, ht * wd, sizes(ht, wd)[1], dtype=torch.float32)
    g.t.zero_()
    want = torch.zeros_like(g.t)
    for k in range(calls):
        c_accumulate(capi, coords[k:k + 1], grads[k:k + 1], g.t)
        want += index_backward_pyramid(capi, coords[k], grads[k], ht, wd)
        if k in (0, 1, calls - 1):
            torch.cuda.synchronize()
            g.check_guards("corr_grad_accumulate")
            same_bits(g.t, want, "%s after %d calls" % (name, k + 1))
    zero_rows = int((want == 0).all(2).sum())
    nan_rows = int(torch.isnan(want).any(2).sum())
    assert zero_rows > 0 and nan_rows > 0, (name, zero_rows, nan_rows)
    _report("gpyr", name, dict(zero_rows=zero_rows, nan_rows=nan_rows))


@pytest.mark.parametrize("dense", [False, True], ids=["lookups", "dense"])
@pytest.mark.parametrize("name", list(STAGES))
def test_adjoint_matches_fp64(capi, name, dense):
    n, ht, wd, _ = STAGES[name]
    f1, f2, coords, grads = inputs(name)[:4]
    _, Q = sizes(ht, wd)
    if dense:
        G = torch.randn(n, ht * wd, Q, device=dev, generator=torch.Generator(device=dev).manual_seed(n * 1000 + ht + wd))
    else:
        G = grad_pyramid(capi, coords, grads, ht, wd)
        assert bool((G == 0).all(2).any()), "%s: no all-zero gradient row" % name
    g1, g2 = c_adjoint(capi, f1, f2, G)
    b1 = KAPPA_PER_SQRT_K["g_f1"] * stage_K("g_f1", ht, wd) ** 0.5
    b2 = KAPPA_PER_SQRT_K["g_f2"] * stage_K("g_f2", ht, wd) ** 0.5
    k1 = k2 = 0.0
    zero_cols = 0
    for s in edge_slices(n, 4 * ht * wd * Q):
        (t1, a1), (t2, a2) = adjoint_truth(f1[s], f2[s], G[s])
        k1 = max(k1, kappa(g1[s], t1, a1, "%s g_f1" % name))
        k2 = max(k2, kappa(g2[s], t2, a2, "%s g_f2" % name))
        zero = (G[s] == 0).all(2).view(-1, 1, ht, wd).expand_as(g1[s])
        assert bool((g1[s][zero] == 0).all()), "%s: a zero gradient row gave a non-zero g_f1 column" % name
        zero_cols += int(zero[:, 0].sum())
    assert dense == (zero_cols == 0), (name, zero_cols)
    _report("adjoint_" + ("dense" if dense else "lookups"), name,
            dict(g_f1=float("%.3g" % k1), g_f2=float("%.3g" % k2), g_f1_per_sqrt_K=float("%.3g" % (k1 / Q ** 0.5)),
                 g_f2_per_sqrt_K=float("%.3g" % (k2 / (ht * wd) ** 0.5)), zero_cols=zero_cols))
    assert k1 <= b1 and k2 <= b2, (name, k1, b1, k2, b2)


@pytest.mark.parametrize("name", list(STAGES))
def test_each_stage_gives_the_same_bits_one_edge_at_a_time(capi, name):
    n, ht, wd, calls = STAGES[name]
    f1, f2, coords, grads = inputs(name)[:4]
    vol = c_volume(capi, f1, f2)
    G = grad_pyramid(capi, coords, grads, ht, wd)
    g1, g2 = c_adjoint(capi, f1, f2, G)
    for e in range(n):
        one = slice(e, e + 1)
        for l, v in enumerate(c_volume(capi, f1[one], f2[one])):
            same_bits(v, vol[l][one], "%s volume level %d edge %d" % (name, l, e))
        Ge = grad_pyramid(capi, [c[one] for c in coords], [g[one] for g in grads], ht, wd)
        same_bits(Ge, G[one], "%s gradient pyramid edge %d" % (name, e))
        a, b = c_adjoint(capi, f1[one], f2[one], Ge)
        same_bits(a, g1[one], "%s g_f1 edge %d" % (name, e))
        same_bits(b, g2[one], "%s g_f2 edge %d" % (name, e))
