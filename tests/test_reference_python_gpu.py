"""GPU side of the reference-Python pinning: the native kernels against vectors produced by the reference's own Python files
(tests/golden/make_reference_python_golden.py imports geom/projective_ops.py and modules/corr.py unmodified; /root/reference does
not exist on the GPU box, so the stored vectors are what is compared here)."""
import os
import sys

import pytest
import torch

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_reference_python_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_python.pt"))


@pytest.mark.parametrize("case", [c[0] for c in mk.reproject_cases()])
def test_reproject_kernel_matches_reference_projective_transform(backends, gold, case):
    """row A5: dba_reproject vs pops.projective_transform(jacobian=False) as DepthVideo.reproject calls it"""
    name, poses, disps, intr, ii, jj = [c for c in mk.reproject_cases() if c[0] == case][0]
    coords, valid = backends.reproject(poses.to(dev), disps.to(dev), intr.to(dev), ii.to(dev), jj.to(dev))
    gc, gv = gold["reproject_%s_coords" % name][0], gold["reproject_%s_valid" % name][0]
    assert torch.equal(valid.cpu(), gv)
    rel = ((coords.cpu() - gc).abs() / gc.abs().clamp(min=1.0)).max()
    assert float(rel) < 1e-4, float(rel)
    from droid_slam_b200.modules import reproject
    c2, v2 = reproject(poses.to(dev), disps.to(dev), intr.to(dev), ii, jj)
    assert c2.shape == gold["reproject_%s_coords" % name].shape and v2.shape == gold["reproject_%s_valid" % name].shape


class _RefShapedCorrBlock:
    """the call pattern of the reference's CorrBlock.__call__ (modules/corr.py:40-50) for the hook test"""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        raise AssertionError("the hook must replace the constructor")

    def __call__(self, coords):
        import droid_backends
        out = []
        batch, num, ht, wd, _ = coords.shape
        coords = coords.permute(0, 1, 4, 2, 3).contiguous().view(batch * num, 2, ht, wd)
        for i in range(self.num_levels):
            corr, = droid_backends.corr_index_forward(self.corr_pyramid[i], coords / 2 ** i, self.radius)
            out.append(corr.view(batch, num, -1, ht, wd))
        return torch.cat(out, dim=2)


def test_corrblock_lookups_match_reference_classes(backends, gold):
    """CorrBlock / AltCorrBlock results of the reference classes (oracle-backed on CPU) vs the native ops called the same way"""
    (f1, f2, coords), (fm, ca, ii, jj) = mk.corr_cases()
    pyr = [v.to(dev) for v in oracle.corr_pyramid(f1, f2, 3)]          # bit-identical to the reference's (test_reference_python_cpu.py)
    c = coords.permute(0, 1, 4, 2, 3).contiguous().view(5, 2, 8, 16).to(dev)
    outs = [backends.corr_index_forward(pyr[l], (c / 2 ** l).contiguous(), 3)[0].view(1, 5, -1, 8, 16) for l in range(3)]
    assert torch.equal(torch.cat(outs, 2).cpu(), gold["corrblock_lookup"])
    fmd = fm.to(dev)
    ca_d = ca.permute(0, 1, 4, 2, 3).contiguous().to(dev)
    lv = []
    f = fmd[0]
    for l in range(3):
        o, = backends.altcorr_forward(fmd, f[None].contiguous(), (ca_d / 2 ** l).contiguous(), ii.to(dev), jj.to(dev), 3)
        lv.append(o.flatten(2, 3))
        f = torch.nn.functional.avg_pool2d(f, 2, stride=2)
    got = torch.stack(lv, dim=2).flatten(2, 3).cpu()                   # f32 dot products over 16 channels: summation order differs from the CPU run
    assert got.shape == gold["altcorrblock_lookup"].shape and torch.allclose(got, gold["altcorrblock_lookup"], rtol=1e-5, atol=1e-5)


def test_corr_volume_hook_replaces_the_constructor_only(backends):
    from droid_slam_b200.modules import install_corr_volume_hook
    import types
    mod = types.SimpleNamespace(CorrBlock=type("CorrBlock", (_RefShapedCorrBlock,), {}))
    install_corr_volume_hook(mod)
    g = torch.Generator().manual_seed(1)
    f1 = torch.randn(1, 3, 128, 16, 64, generator=g).half().to(dev)
    f2 = torch.randn(1, 3, 128, 16, 64, generator=g).half().to(dev)
    blk = mod.CorrBlock(f1, f2)
    assert len(blk.corr_pyramid) == 4 and blk.corr_pyramid[0].shape == (3, 16, 64, 16, 64) and blk.corr_pyramid[3].shape == (3, 16, 64, 2, 8)
    import oracle
    ref = oracle.corr_pyramid(f1.float().cpu(), f2.float().cpu(), 4)
    for l in range(4):
        assert float((blk.corr_pyramid[l].float().cpu() - ref[l]).abs().max()) < 2e-2        # f16 volume vs fp32 formula
    coords = torch.rand(1, 3, 16, 64, 2, generator=g) * torch.tensor([64.0, 16.0])
    out = blk(coords.to(dev))
    assert out.shape == (1, 3, 4 * 49, 16, 64)
    with pytest.raises(RuntimeError):
        mod.CorrBlock(f1.float(), f2.float())                  # no silent library fallback for shapes / dtypes without a kernel
    # fused mode: tiled volumes + one-launch lookup give the same bits as the reference-layout path
    mod2 = types.SimpleNamespace(CorrBlock=type("CorrBlock", (_RefShapedCorrBlock,), {}))
    install_corr_volume_hook(mod2, fused_lookup=True)
    out2 = mod2.CorrBlock(f1, f2)(coords.to(dev))
    assert torch.equal(out2, out)
