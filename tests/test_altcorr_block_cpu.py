"""AltCorrBlock on the private channels-last pyramid, without a GPU: argument checks of the C ABI
(dba_altcorr_pyramid / dba_altcorr_lookup_pyramid, include/droid_b200.h) and the dispatch of install_alt_corr_hook."""
import types

import pytest
import torch

from droid_slam_b200 import c_api

F16, F32, F64 = c_api.DBA_F16, c_api.DBA_F32, c_api.DBA_F64


def _pyramid(L, B=1, N=4, C=128, H=48, W=64, levels=4, dtype=F16):
    return L.dba_altcorr_pyramid(None, None, None, None, None, B, N, C, H, W, levels, dtype, None)


def _lookup(L, B=1, N=4, C=128, H=48, W=64, M=8, levels=4, radius=3, dtype=F16):
    return L.dba_altcorr_lookup_pyramid(None, None, None, None, None, None, None, None, B, N, C, H, W, M, levels, radius, dtype, None)


@pytest.mark.parametrize("kw, msg", [
    (dict(H=-1), "negative extent"),
    (dict(M=-3), "negative extent"),
    (dict(dtype=7), "unsupported dtype"),
    (dict(dtype=F64), "float16 or float32"),
    (dict(radius=2), "radius 3"),
    (dict(levels=5), "1..4 levels"),
    (dict(levels=0), "1..4 levels"),
    (dict(C=12), "multiple of 8"),
    (dict(H=4, levels=4), "at least 2^(levels-1)"),
])
def test_lookup_rejects_bad_arguments(capi, kw, msg):
    assert _lookup(capi, **kw) == 1
    assert msg in capi.dba_last_error().decode()


@pytest.mark.parametrize("kw, msg", [
    (dict(N=-1), "negative extent"),
    (dict(dtype=7), "unsupported dtype"),
    (dict(levels=5), "1..4 levels"),
    (dict(C=4), "multiple of 8"),
    (dict(W=7, levels=4), "at least 2^(levels-1)"),
])
def test_pyramid_rejects_bad_arguments(capi, kw, msg):
    assert _pyramid(capi, **kw) == 1
    assert msg in capi.dba_last_error().decode()


def test_empty_batches_return_without_a_launch(capi):
    # null pointers everywhere: a launch or a pointer check would fail
    assert _pyramid(capi, B=0) == 0 and _pyramid(capi, N=0) == 0 and _pyramid(capi, dtype=F32, N=0) == 0
    assert _lookup(capi, M=0) == 0 and _lookup(capi, B=0) == 0 and _lookup(capi, dtype=F32, M=0, levels=1) == 0


def test_null_pointers_are_rejected(capi):
    assert _pyramid(capi) == 1 and "null pointer" in capi.dba_last_error().decode()
    assert _lookup(capi) == 1 and "null pointer" in capi.dba_last_error().decode()


class _StubAltCorrBlock:
    """records which of the reference's methods ran"""

    def __init__(self, fmaps, num_levels=4, radius=3):
        self.calls = ["init"]
        self.num_levels, self.radius = num_levels, radius

    def __call__(self, coords, ii, jj):
        self.calls.append("call")
        return "reference"


def _stub_module():
    return types.SimpleNamespace(AltCorrBlock=type("AltCorrBlock", (_StubAltCorrBlock,), {}))


def test_hook_is_strict_about_cpu_tensors_and_unsupported_arguments():
    from droid_slam_b200.modules import install_alt_corr_hook
    mod = install_alt_corr_hook(_stub_module())
    with pytest.raises(RuntimeError, match="not on a CUDA device"):
        mod.AltCorrBlock(torch.zeros(1, 2, 16, 8, 8))
    with pytest.raises(RuntimeError, match="forward only"):
        mod.AltCorrBlock(torch.zeros(1, 2, 16, 8, 8, requires_grad=True))


def test_hook_falls_back_to_the_reference_methods_when_not_strict():
    from droid_slam_b200.modules import install_alt_corr_hook
    mod = install_alt_corr_hook(_stub_module(), strict=False)
    blk = mod.AltCorrBlock(torch.zeros(1, 2, 16, 8, 8), num_levels=3)
    assert blk(torch.zeros(1, 2, 8, 8, 2), torch.tensor([0, 1]), torch.tensor([1, 0])) == "reference"
    assert blk.calls == ["init", "call"] and blk.num_levels == 3
