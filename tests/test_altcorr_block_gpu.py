"""AltCorrBlock on the private channels-last pyramid (droid_backends.altcorr_pyramid / altcorr_lookup_pyramid, install_alt_corr_hook)
against the reference's own call sequence (modules/corr.py:89-117: avg_pool2d chain, then altcorr_forward per level + flatten + stack),
bit for bit, and against the stored outputs of the unmodified reference build."""
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

from util import assert_bit_identical

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_reference_build_golden as mkb  # noqa: E402
import make_reference_python_golden as mkp  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"


def _ref_pyramid(fmaps, levels):
    """AltCorrBlock.__init__ (modules/corr.py:90-101), without its extra pooling pass after the last level (which makes the reference
    class itself fail below 2^levels pixels; the kernels need only 2^(levels-1))"""
    B, N, C, H, W = fmaps.shape
    f = fmaps.view(B * N, C, H, W)
    out = [f.view(B, N, C, H, W)]
    for l in range(1, levels):
        f = F.avg_pool2d(f, 2, stride=2)
        out.append(f.view(B, N, C, H >> l, W >> l))
    return out


def _ref_lookup(be, fmaps, coords, ii, jj, levels):
    """AltCorrBlock.__call__ (modules/corr.py:104-117) on the drop-in altcorr_forward; coords [B,M,2,H,W]"""
    pyr = _ref_pyramid(fmaps, levels)
    outs = [be.altcorr_forward(pyr[0], pyr[l], coords / 2 ** l, ii, jj, 3)[0].flatten(2, 3) for l in range(levels)]
    return torch.stack(outs, dim=2).flatten(2, 3)


def _fmaps(B, N, C, H, W, dtype, seed=0, specials=False):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(B, N, C, H, W, generator=g)
    if specials:   # subnormal results of /4 and of the pooling, large values
        f.view(-1)[::97] *= 1e-6
        f.view(-1)[::101] *= 3e4 if dtype == torch.float16 else 1e30
    return f.to(dtype).to(dev)


def _coords(B, M, H, W, seed=1, specials=False):
    """[B,M,2,H,W]: a smooth field around identity plus a spread that crosses every border"""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    base = torch.stack([xs, ys])[None, None].expand(B, M, 2, H, W)
    c = base + 6 * torch.randn(B, M, 2, H, W, generator=g) + torch.randn(B, M, 2, 1, 1, generator=g) * torch.tensor([W / 4.0, H / 4.0]).view(1, 1, 2, 1, 1)
    if specials:
        flat = c.view(-1)
        for k, v in enumerate([float("nan"), float("inf"), -float("inf"), 1e30, -1e30, -0.0, W - 0.5, -3.5]):
            flat[k::53] = v
    return c.contiguous().to(dev)


def _edges(N, M, seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, N, (M,), generator=g).to(dev), torch.randint(0, N, (M,), generator=g).to(dev)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("hw", [(48, 64), (30, 40), (36, 60), (72, 96), (8, 16)])
@pytest.mark.parametrize("C", [16, 128])
def test_pyramid_is_the_quartered_avg_pool_chain(backends, dtype, hw, C):
    H, W = hw
    f = _fmaps(2, 3, C, H, W, dtype, seed=C + H, specials=True)
    got = backends.altcorr_pyramid(f, 4)
    ref = _ref_pyramid(f, 4)
    assert len(got) == 4
    for l in range(4):
        assert got[l].shape == (2, 3, H >> l, W >> l, C)
        assert_bit_identical(got[l], (ref[l] / 4).permute(0, 1, 3, 4, 2), "level %d" % l)


def test_pyramid_with_fewer_levels(backends):
    f = _fmaps(1, 2, 32, 13, 21, torch.float16, seed=4)
    ref = _ref_pyramid(f, 3)
    for L in (1, 2, 3):
        got = backends.altcorr_pyramid(f, L)
        assert len(got) == L
        for l in range(L):
            assert_bit_identical(got[l], (ref[l] / 4).permute(0, 1, 3, 4, 2), "L=%d level %d" % (L, l))


LOOKUP_CASES = {  # name: (B, N, C, H, W, M, dtype, levels, specials)
    "f16_48x64_C128_64e": (1, 16, 128, 48, 64, 64, torch.float16, 4, False),
    "f16_48x64_C128_512e": (1, 40, 128, 48, 64, 512, torch.float16, 4, False),
    "f32_48x64_C128": (1, 8, 128, 48, 64, 24, torch.float32, 4, False),
    "f32_30x40_C64_L3": (1, 6, 64, 30, 40, 16, torch.float32, 3, True),
    "f16_30x40_C128_L3": (1, 6, 128, 30, 40, 32, torch.float16, 3, False),
    "f16_72x96_C128": (1, 12, 128, 72, 96, 48, torch.float16, 4, False),
    "f16_36x60_C24_B2": (2, 5, 24, 36, 60, 20, torch.float16, 4, True),
    "f16_48x64_C128_specials": (1, 8, 128, 48, 64, 24, torch.float16, 4, True),
}


@pytest.mark.parametrize("case", list(LOOKUP_CASES))
def test_lookup_matches_the_drop_in_call_sequence(backends, case):
    B, N, C, H, W, M, dtype, L, specials = LOOKUP_CASES[case]
    f = _fmaps(B, N, C, H, W, dtype, seed=M)
    coords = _coords(B, M, H, W, seed=M + 1, specials=specials)
    ii, jj = _edges(N, M, seed=M + 2)
    got = backends.altcorr_lookup_pyramid(backends.altcorr_pyramid(f, L), coords, ii, jj, 3)
    assert got.shape == (B, M, L * 49, H, W) and got.dtype == dtype
    assert_bit_identical(got, _ref_lookup(backends, f, coords, ii, jj, L), case)


def test_lookup_with_rig_2_indices(backends):
    """update_lowmem on a stereo video: fmaps viewed as [1, 2N, ...], ii = 2i, jj = 2j + (i == j)"""
    N, M, C, H, W = 6, 30, 128, 48, 64
    f = _fmaps(1, 2 * N, C, H, W, torch.float16, seed=9)
    i, j = _edges(N, M, seed=10)
    i[:N], j[:N] = torch.arange(N, device=dev), torch.arange(N, device=dev)
    ii, jj = 2 * i, 2 * j + (i == j).long()
    coords = _coords(1, M, H, W, seed=11)
    got = backends.altcorr_lookup_pyramid(backends.altcorr_pyramid(f, 4), coords, ii, jj, 3)
    assert_bit_identical(got, _ref_lookup(backends, f, coords, ii, jj, 4), "rig 2")


class _Capture:
    """stands in for droid_backends in make_reference_build_golden.altcorr: keeps the inputs of its first altcorr_forward call"""

    def __init__(self, be):
        self.be, self.args = be, None

    def altcorr_forward(self, f1, f2, c, ii, jj, r):
        if self.args is None:
            self.args = (f1, c, ii, jj)
        return self.be.altcorr_forward(f1, f2, c, ii, jj, r)


def test_fused_path_matches_the_unmodified_reference_build(backends):
    gold = torch.load(mkb.GOLD, weights_only=False)
    cap = _Capture(backends)
    mkb.altcorr(cap, dev)
    fmaps, coords, ii, jj = cap.args
    out = backends.altcorr_lookup_pyramid(backends.altcorr_pyramid(fmaps, 4), coords, ii, jj, 3)
    B, M, _, H, W = out.shape
    for l in range(4):
        t = out[:, :, 49 * l:49 * (l + 1)].reshape(B, M, 7, 7, H, W)
        rec = gold["altcorr_l%d" % l]
        assert tuple(t.shape) == rec["shape"] and str(t.dtype) == rec["dtype"]
        assert mkb.digest(t) == rec["sha256"], "level %d: not bit-identical to the reference build" % l


class _RefShapedAltCorrBlock:
    def __init__(self, fmaps, num_levels=4, radius=3):
        raise AssertionError("the hook must replace the constructor")

    def __call__(self, coords, ii, jj):
        raise AssertionError("the hook must replace __call__")


def _hooked():
    from droid_slam_b200.modules import install_alt_corr_hook
    return install_alt_corr_hook(types.SimpleNamespace(AltCorrBlock=type("AltCorrBlock", (_RefShapedAltCorrBlock,), {})))


def test_hook_matches_the_reference_call_sequence(backends):
    mod = _hooked()
    N, M, C, H, W = 10, 40, 128, 48, 64
    f = _fmaps(1, N, C, H, W, torch.float16, seed=21)
    ii, jj = _edges(N, M, seed=22)
    c = _coords(1, M, H, W, seed=23)
    blk = mod.AltCorrBlock(f)
    got = blk(c.permute(0, 1, 3, 4, 2), ii, jj)            # the hook takes [B,M,H,W,2] like the reference
    assert got.shape == (1, M, 196, H, W)
    assert_bit_identical(got, _ref_lookup(backends, f, c, ii, jj, 4), "hook")


def test_hook_matches_the_reference_python_vector():
    """reference_python.pt["altcorrblock_lookup"]: AltCorrBlock(num_levels=3) of the reference's modules/corr.py over a CPU oracle,
    f32, 16 channels (summation order of the CPU run differs: 1e-5)"""
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "reference_python.pt"))
    _, (fm, ca, ii, jj) = mkp.corr_cases()
    blk = _hooked().AltCorrBlock(fm.to(dev), num_levels=3, radius=3)
    got = blk(ca.to(dev), ii.to(dev), jj.to(dev)).cpu()
    want = gold["altcorrblock_lookup"]
    assert got.shape == want.shape and torch.allclose(got, want, rtol=1e-5, atol=1e-5)


def test_hook_is_strict():
    mod = _hooked()
    f = _fmaps(1, 2, 16, 8, 16, torch.float32)
    for bad in (f.cpu(), f.double(), f[:, :, :12].contiguous(), f[..., :4, :]):
        with pytest.raises(RuntimeError, match="no kernel"):
            mod.AltCorrBlock(bad)
    with pytest.raises(RuntimeError, match="no kernel"):
        mod.AltCorrBlock(f, radius=2)
    with pytest.raises(RuntimeError, match="no kernel"):
        mod.AltCorrBlock(f, num_levels=5)
    blk = mod.AltCorrBlock(f)
    ii = torch.tensor([0, 1], device=dev)
    c = torch.zeros(1, 2, 8, 16, 2, device=dev)
    with pytest.raises(RuntimeError, match="forward only"):
        blk(c.clone().requires_grad_(), ii, ii)
    with pytest.raises(RuntimeError, match="forward only"):
        mod.AltCorrBlock(f.clone().requires_grad_())
    with torch.no_grad():
        assert blk(c.clone().requires_grad_(), ii, ii).shape == (1, 2, 196, 8, 16)
    with pytest.raises(RuntimeError):
        blk(c.cpu(), ii, ii)


def test_hook_call_replays_in_a_cuda_graph():
    """captured without a host synchronisation; replays read the current coordinates"""
    mod = _hooked()
    N, M, C, H, W = 8, 24, 128, 48, 64
    f = _fmaps(1, N, C, H, W, torch.float16, seed=31)
    ii, jj = _edges(N, M, seed=32)
    c = _coords(1, M, H, W, seed=33).permute(0, 1, 3, 4, 2).contiguous()
    blk = mod.AltCorrBlock(f)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        blk(c, ii, jj)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = blk(c, ii, jj)
    for seed in (33, 34):
        c.copy_(_coords(1, M, H, W, seed=seed).permute(0, 1, 3, 4, 2))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, blk(c, ii, jj)), seed
