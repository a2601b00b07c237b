"""Correlation pyramid build (corr_volume_pyramid) and fused lookup (corr_lookup_pyramid) at the image sizes the reference's scripts
produce, not only 512-wide inputs: 1/8-resolution feature maps of TUM (30x40), ETH3D (43x70), raw EuRoC (44x69), 16:9 video (41x73),
the c5 bench config (72x96) and the smallest legal ones (8x8, 9x13), plus 16x64 on the wd = 64 kernel."""
import pytest
import torch

from util import assert_bit_identical

pytestmark = pytest.mark.gpu
dev = "cuda"

SIZES = [(8, 8), (9, 13), (30, 40), (43, 70), (44, 69), (41, 73), (72, 96), (16, 64)]


def _edges(ht, wd):
    return 2 if ht * wd > 4000 else 5


def _fmaps(ht, wd, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 128, ht, wd, generator=g).half()


def _cublas_pyramid(f1, f2):
    """the f16 cuBLAS + avg_pool2d pipeline of the reference's CorrBlock.__init__, on the GPU (without its pooling after the last level)"""
    E, C, ht, wd = f1.shape
    corr = torch.matmul((f1.reshape(E, C, -1) / 4.0).transpose(1, 2), f2.reshape(E, C, -1) / 4.0).reshape(E * ht * wd, 1, ht, wd)
    pyr = [corr.view(E, ht, wd, ht, wd)]
    for l in range(1, 4):
        corr = torch.nn.functional.avg_pool2d(corr, 2, stride=2)
        pyr.append(corr.view(E, ht, wd, ht >> l, wd >> l))
    return pyr


def _coords(E, ht, wd, seed):
    g = torch.Generator().manual_seed(seed)
    c = torch.stack([torch.rand(E, ht, wd, generator=g) * (wd + 10) - 5, torch.rand(E, ht, wd, generator=g) * (ht + 10) - 5], dim=1)
    c[0, :, 0, 0] = torch.tensor([float("inf"), 3.0])
    c[0, :, 0, 1] = torch.tensor([2.0, float("nan")])
    c[-1, :, 1, 1] = torch.tensor([-50.0, 1e6])
    c[-1, :, ht - 1, wd - 1] = torch.tensor([float("-inf"), float("-inf")])
    c[0, :, ht - 1, 0] = torch.tensor([wd - 0.5, ht - 0.25])          # window across the right / bottom edge of every level
    return c.contiguous()


@pytest.mark.parametrize("ht, wd", SIZES)
def test_volume_matches_oracle_and_cublas_pipeline(backends, ht, wd):
    """the binding's volume against the reference's f16 cuBLAS + avg_pool2d pipeline, which rounds every level to fp16 before pooling
    the next (the values themselves are held to fp64 in tests/test_tensor_core_fp64_gpu.py)"""
    N, E = 4, _edges(ht, wd)
    fm = _fmaps(ht, wd, N, 100 + ht * wd)
    g = torch.Generator().manual_seed(ht + wd)
    ii, jj = torch.randint(0, N, (E,), generator=g), torch.randint(0, N, (E,), generator=g)
    f = fm.to(dev)
    got = backends.corr_volume_pyramid(f, f, ii.to(dev), jj.to(dev))
    lib = _cublas_pyramid(f[ii.to(dev)], f[jj.to(dev)])
    for l in range(4):
        assert got[l].shape == (E, ht, wd, ht >> l, wd >> l) == lib[l].shape
        assert float((got[l].float() - lib[l].float()).abs().max()) < 6e-2, l


@pytest.mark.parametrize("ht, wd", SIZES)
def test_fused_lookup_is_bit_identical_to_per_level_lookups(backends, ht, wd):
    """levels placed as slices of a NaN-filled buffer: a tap read from outside its plane would turn an output into NaN or change it"""
    N, E = 3, _edges(ht, wd)
    f = _fmaps(ht, wd, N, 7 + ht).to(dev)
    idx = torch.arange(E, device=dev) % N
    pyr = backends.corr_volume_pyramid(f, f, idx, (idx + 1) % N)
    sizes = [v.numel() for v in pyr]
    buf = torch.full((sum(sizes) + 4 * 64,), float("nan"), dtype=torch.float16, device=dev)
    placed, off = [], 24                                                 # 48 bytes in: 16-byte aligned, NaN before and after each level
    for v, n in zip(pyr, sizes):
        placed.append(buf[off:off + n].view(v.shape))
        placed[-1].copy_(v)
        off += (n + 7) // 8 * 8 + 32
    coords = _coords(E, ht, wd, 5 + wd).to(dev)
    per_level = torch.cat([backends.corr_index_forward(pyr[l], (coords / 2 ** l).contiguous(), 3)[0].view(E, 49, ht, wd) for l in range(4)], dim=1)
    fused = backends.corr_lookup_pyramid(placed, coords)
    assert fused.shape == (E, 196, ht, wd)
    assert_bit_identical(fused, per_level, "fused lookup %dx%d" % (ht, wd))
    assert not bool(torch.isnan(fused[:, :, 1:, 2:]).any())            # NaN only where the coordinates are NaN / inf


class _RefCorrBlock:
    """the reference CorrBlock's algorithm (modules/corr.py): cuBLAS volume + avg_pool2d, per-level corr_index_forward + cat"""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        batch, num, dim, ht, wd = fmap1.shape
        self.num_levels, self.radius = num_levels, radius
        self.corr_pyramid = _cublas_pyramid(fmap1.reshape(batch * num, dim, ht, wd), fmap2.reshape(batch * num, dim, ht, wd))

    def __call__(self, coords):
        import droid_backends
        batch, num, ht, wd, _ = coords.shape
        c = coords.permute(0, 1, 4, 2, 3).contiguous().view(batch * num, 2, ht, wd)
        out = [droid_backends.corr_index_forward(self.corr_pyramid[i], c / 2 ** i, self.radius)[0].view(batch, num, -1, ht, wd)
               for i in range(self.num_levels)]
        return torch.cat(out, dim=2)


def _hooked(fused):
    import types
    from droid_slam_b200.modules import install_corr_volume_hook
    mod = types.SimpleNamespace(CorrBlock=type("CorrBlock", (_RefCorrBlock,), {}))
    return install_corr_volume_hook(mod, fused_lookup=fused).CorrBlock


@pytest.mark.parametrize("ht, wd", [(30, 40), (43, 70), (41, 73), (16, 64)])
def test_hooked_corrblock_matches_reference_class(backends, ht, wd):
    E = 3
    g = torch.Generator().manual_seed(ht * wd)
    f1 = torch.randn(1, E, 128, ht, wd, generator=g).half().to(dev)
    f2 = torch.randn(1, E, 128, ht, wd, generator=g).half().to(dev)
    coords = (torch.rand(1, E, ht, wd, 2, generator=g) * torch.tensor([wd + 4.0, ht + 4.0]) - 2).to(dev)
    ref_blk = _RefCorrBlock(f1, f2)
    blk, blk_f = _hooked(False)(f1, f2), _hooked(True)(f1, f2)
    assert blk_f._b200_tiled == (wd == 64 and ht % 8 == 0)
    for l in range(4):
        assert blk.corr_pyramid[l].shape == ref_blk.corr_pyramid[l].shape
        assert float((blk.corr_pyramid[l].float() - ref_blk.corr_pyramid[l].float()).abs().max()) < 6e-2
    out, out_f, want = blk(coords), blk_f(coords), ref_blk(coords)
    assert out.shape == want.shape == (1, E, 196, ht, wd)
    assert float((out.float() - want.float()).abs().max()) < 6e-2
    assert torch.equal(out, out_f)


def test_hook_build_and_lookup_replay_in_a_cuda_graph(backends):
    ht, wd, E = 41, 73, 3
    g = torch.Generator().manual_seed(9)
    f1 = torch.randn(1, E, 128, ht, wd, generator=g).half().to(dev)
    f2 = torch.randn(1, E, 128, ht, wd, generator=g).half().to(dev)
    coords = (torch.rand(1, E, ht, wd, 2, generator=g) * torch.tensor([wd + 4.0, ht + 4.0]) - 2).to(dev)
    cls = _hooked(True)

    def step():
        return cls(f1, f2)(coords)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
