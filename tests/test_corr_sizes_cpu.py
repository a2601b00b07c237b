"""Correlation pyramid at every image size, without a GPU: which shapes the C ABI accepts (dba_corr_volume_supported with and
without the tiled layout, dba_corr_volume_workspace_bytes), the argument checks that run before any launch, and the
native / fallback / raise selection of install_corr_volume_hook on a stub backend."""
import ctypes
import types

import pytest
import torch

from droid_slam_b200 import c_api

F16, F32, BF16 = c_api.DBA_F16, c_api.DBA_F32, c_api.DBA_BF16
INVALID = 1
P = ctypes.c_void_p(1 << 20)            # a non-null, 16-byte aligned address: the calls below must return before touching it


def test_single_entry_point_symbols_are_exported(capi):
    for name in ("dba_corr_volume_pyramid", "dba_corr_volume_workspace_bytes", "dba_corr_volume_supported"):
        assert name in c_api.SYMBOLS and hasattr(capi, name)


@pytest.mark.parametrize("channels, ht, wd, dtype, want", [
    (128, 48, 64, F16, 1), (128, 16, 64, F16, 1), (128, 30, 40, F16, 1), (128, 43, 70, F16, 1), (128, 44, 69, F16, 1),
    (128, 41, 73, F16, 1), (128, 72, 96, F16, 1), (128, 8, 8, F16, 1), (128, 9, 13, F16, 1),
    (128, 7, 64, F16, 0), (128, 48, 7, F16, 0), (128, 0, 0, F16, 0), (64, 48, 64, F16, 0), (256, 30, 40, F16, 0),
    (128, 48, 64, F32, 0), (128, 48, 64, BF16, 0),
])
def test_volume_supported_truth_table_with_tiled_flag(capi, channels, ht, wd, dtype, want):
    assert capi.dba_corr_volume_supported(channels, ht, wd, dtype, 0) == want
    tiled = want and wd == 64 and ht % 8 == 0
    assert capi.dba_corr_volume_supported(channels, ht, wd, dtype, 1) == int(tiled)


def test_workspace_bytes(capi):
    for ht, wd in ((48, 64), (30, 40), (72, 96), (8, 8)):
        assert capi.dba_corr_volume_workspace_bytes(5, 5, 128, ht, wd) == 0
    for ht, wd in ((43, 70), (44, 69), (41, 73), (9, 13)):
        wp = (wd + 7) // 8 * 8
        one = lambda n: (n * 128 * ht * wp * 2 + 255) // 256 * 256
        assert capi.dba_corr_volume_workspace_bytes(3, 5, 128, ht, wd) == one(3) + one(5)


def _build(L, ht, wd, E=2, ws=None, ws_bytes=0, tiled=0, ptr=P):
    return L.dba_corr_volume_pyramid(*[ptr] * 8, E, 4, 4, 128, ht, wd, F16, tiled, ws, ws_bytes, None)


@pytest.mark.parametrize("ht, wd", [(7, 64), (48, 7), (5, 5)])
def test_single_entry_rejects_levels_without_a_pixel(capi, ht, wd):
    for tiled in (0, 1):
        for ws, ws_bytes in ((None, 0), (P, 1 << 30)):
            assert _build(capi, ht, wd, ws=ws, ws_bytes=ws_bytes, tiled=tiled) == INVALID
            assert "at least 8" in capi.dba_last_error().decode()


@pytest.mark.parametrize("ht, wd", [(30, 40), (43, 70), (72, 96), (44, 64)])
def test_tiled_flag_is_limited_to_wd64_shapes(capi, ht, wd):
    assert _build(capi, ht, wd, tiled=1) == INVALID
    assert "wd = 64" in capi.dba_last_error().decode()


def test_single_entry_checks_workspace_before_any_launch(capi):
    need = capi.dba_corr_volume_workspace_bytes(4, 4, 128, 43, 70)
    assert need > 0
    assert _build(capi, 43, 70, ws=None, ws_bytes=need) == INVALID and "workspace" in capi.dba_last_error().decode()
    assert _build(capi, 43, 70, ws=P, ws_bytes=need - 1) == INVALID and "workspace" in capi.dba_last_error().decode()
    assert _build(capi, 43, 70, ws=None, ws_bytes=0) == INVALID and "workspace" in capi.dba_last_error().decode()
    assert _build(capi, 43, 70, ws=ctypes.c_void_p((1 << 20) + 8), ws_bytes=need) == INVALID
    assert "16-byte aligned" in capi.dba_last_error().decode()


def test_single_entry_checks_edges_pointers_alignment(capi):
    assert _build(capi, 30, 40, E=65536) == INVALID and "65535" in capi.dba_last_error().decode()
    assert _build(capi, 30, 40, ptr=None) == INVALID and "null pointer" in capi.dba_last_error().decode()
    assert _build(capi, 30, 40, ptr=ctypes.c_void_p((1 << 20) + 2)) == INVALID and "16-byte aligned" in capi.dba_last_error().decode()
    assert _build(capi, 43, 70, E=0, ptr=None) == 0                     # nothing to do: no pointer, no workspace needed


@pytest.mark.parametrize("h1, w1, tiled, msg", [(7, 64, 0, "at least 8"), (48, 7, 0, "at least 8"), (30, 40, 3, "tiled_mask"),
                                                (48, 64, 1, "tiled_mask")])
def test_lookup_rejects(capi, h1, w1, tiled, msg):
    assert capi.dba_corr_lookup_pyramid(P, P, P, P, P, P, 2, h1, w1, tiled, F16, None) == INVALID
    assert msg in capi.dba_last_error().decode()


def test_lookup_accepts_every_size_at_zero_edges(capi):
    for h1, w1 in ((8, 8), (9, 13), (43, 70), (41, 73)):
        assert capi.dba_corr_lookup_pyramid(None, None, None, None, None, None, 0, h1, w1, 0, F16, None) == 0


# ---- install_corr_volume_hook on a stub backend ----------------------------------------------------------------------------
class _FakeCudaFmap:
    """shape / dtype / device flags of a [B,N,C,H,W] CUDA feature map; the stub backend never reads data"""

    def __init__(self, shape, dtype=torch.float16, is_cuda=True):
        self.shape, self.dtype, self.is_cuda, self.device = tuple(shape), dtype, is_cuda, "cpu"

    def dim(self):
        return len(self.shape)

    def reshape(self, *shape):
        return self

    def contiguous(self):
        return self


class _StubBackend:
    def __init__(self, capi):
        self.capi, self.calls = capi, []

    def corr_volume_supported(self, dim, ht, wd, tiled=False):
        return self.capi.dba_corr_volume_supported(dim, ht, wd, F16, int(tiled)) != 0

    def corr_volume_pyramid(self, f1, f2, ii, jj, tiled):
        self.calls.append(("build", tiled))
        return [torch.zeros(1)] * 4

    def corr_lookup_pyramid(self, pyramid, coords, tiled):
        self.calls.append(("lookup", tiled))
        return torch.zeros(coords.shape[0], 196, coords.shape[2], coords.shape[3])


class _StubCorrBlock:
    def __init__(self, fmap1, fmap2, num_levels=4, radius=3):
        self.calls = ["init"]

    def __call__(self, coords):
        self.calls.append("call")
        return "reference"


@pytest.fixture
def stub(capi, monkeypatch):
    import droid_slam_b200.modules as m
    be = _StubBackend(capi)
    monkeypatch.setattr(m, "install", lambda: be)
    return be


def _cls(**kw):
    from droid_slam_b200.modules import install_corr_volume_hook
    return install_corr_volume_hook(types.SimpleNamespace(CorrBlock=type("CorrBlock", (_StubCorrBlock,), {})), **kw).CorrBlock


@pytest.mark.parametrize("ht, wd, tiled", [(48, 64, True), (16, 64, True), (30, 40, False), (43, 70, False), (41, 73, False), (8, 8, False)])
def test_hook_builds_natively_at_every_supported_shape(stub, ht, wd, tiled):
    f = _FakeCudaFmap((1, 3, 128, ht, wd))
    blk = _cls()(f, f)
    assert stub.calls == [("build", False)] and not hasattr(blk, "calls")
    blk = _cls(fused_lookup=True)(f, f)
    assert stub.calls[-1] == ("build", tiled) and blk._b200_tiled == tiled
    out = blk(torch.zeros(1, 3, ht, wd, 2))
    assert stub.calls[-1] == ("lookup", tiled) and out.shape == (1, 3, 196, ht, wd)


@pytest.mark.parametrize("kw, why", [
    (dict(shape=(1, 3, 128, 7, 64)), "at least 8"),
    (dict(shape=(1, 3, 128, 48, 5)), "at least 8"),
    (dict(shape=(1, 3, 64, 48, 64)), "64 channels"),
    (dict(dtype=torch.float32), "float32"),
    (dict(dtype=torch.bfloat16), "bfloat16"),
    (dict(is_cuda=False), "CUDA device"),
    (dict(levels=3), "3 levels"),
])
def test_hook_raises_or_falls_back_naming_the_reason(stub, kw, why):
    levels = kw.pop("levels", 4)
    kw.setdefault("shape", (1, 3, 128, 43, 70))
    f = _FakeCudaFmap(**kw)
    with pytest.raises(RuntimeError, match=why):
        _cls()(f, f, num_levels=levels)
    for fused in (False, True):
        blk = _cls(strict=False, fused_lookup=fused)(f, f, num_levels=levels)
        assert blk.calls == ["init"]
        assert blk(torch.zeros(1, 3, 4, 4, 2)) == "reference" and blk.calls == ["init", "call"]
    assert stub.calls == []
