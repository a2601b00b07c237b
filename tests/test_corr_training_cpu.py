"""The training CorrBlock without a GPU: the C ABI's symbols and the argument checks that run before any launch, install_corr_training_hook's
native / fallback / raise selection on a stub backend, and its hook-registry entry."""
import ctypes
import types

import pytest
import torch

from droid_slam_b200 import c_api

F16, F32 = c_api.DBA_F16, c_api.DBA_F32
INVALID = 1
P = ctypes.c_void_p(1 << 20)            # a non-null, 16-byte aligned address: the calls below must return before touching it


def test_symbols_are_exported(capi):
    for name in ("dba_corr_volume_pyramid_f32", "dba_corr_grad_accumulate", "dba_corr_adjoint_workspace_bytes", "dba_corr_adjoint"):
        assert name in c_api.SYMBOLS and hasattr(capi, name)


@pytest.mark.parametrize("C, ht, wd, msg", [(64, 48, 64, "128 feature channels"), (128, 7, 64, "at least 8"), (128, 48, 5, "at least 8")])
def test_build_and_adjoint_reject_shapes_without_a_kernel(capi, C, ht, wd, msg):
    assert capi.dba_corr_volume_pyramid_f32(*[P] * 6, 2, C, ht, wd, None) == INVALID and msg in capi.dba_last_error().decode()
    assert capi.dba_corr_adjoint(*[P] * 5, 2, C, ht, wd, P, 1 << 40, None) == INVALID and msg in capi.dba_last_error().decode()


def test_null_pointers_edges_and_workspace_are_checked(capi):
    assert capi.dba_corr_volume_pyramid_f32(*[None] * 6, 2, 128, 16, 24, None) == INVALID and "null pointer" in capi.dba_last_error().decode()
    assert capi.dba_corr_volume_pyramid_f32(*[P] * 6, 65536, 128, 16, 24, None) == INVALID and "65535" in capi.dba_last_error().decode()
    assert capi.dba_corr_volume_pyramid_f32(*[None] * 6, 0, 128, 16, 24, None) == 0
    assert capi.dba_corr_grad_accumulate(None, None, None, 2, 16, 24, None) == INVALID and "null pointer" in capi.dba_last_error().decode()
    assert capi.dba_corr_grad_accumulate(None, None, None, 0, 16, 24, None) == 0
    need = capi.dba_corr_adjoint_workspace_bytes(2, 128, 17, 23)
    q = sum((17 >> l) * (23 >> l) for l in range(4))
    assert need == 2 * ((2 * 128 * q * 4 + 255) // 256 * 256)
    assert capi.dba_corr_adjoint(*[P] * 5, 2, 128, 17, 23, P, need - 1, None) == INVALID and "workspace" in capi.dba_last_error().decode()
    assert capi.dba_corr_adjoint(*[P] * 5, 2, 128, 17, 23, ctypes.c_void_p((1 << 20) + 8), need, None) == INVALID
    assert "16-byte aligned" in capi.dba_last_error().decode()


def test_lookup_takes_f32_volumes_in_the_reference_layout_only(capi):
    assert capi.dba_corr_lookup_pyramid(P, P, P, P, P, P, 2, 48, 64, 3, F32, None) == INVALID
    assert "tiled_mask 0" in capi.dba_last_error().decode()
    assert capi.dba_corr_lookup_pyramid(None, None, None, None, None, None, 0, 17, 23, 0, F32, None) == 0


class _Fmap:
    """shape / dtype / device flags of a [B,N,C,H,W] feature map; the stub backend never reads data"""

    def __init__(self, shape=(1, 3, 128, 43, 70), dtype=torch.float32, is_cuda=True, requires_grad=False):
        self.shape, self.dtype, self.is_cuda, self.requires_grad = tuple(shape), dtype, is_cuda, requires_grad

    def dim(self):
        return len(self.shape)

    def reshape(self, *shape):
        return self

    def contiguous(self):
        return self

    def detach(self):
        return self


class _StubBackend:
    def __init__(self):
        self.calls = []

    def corr_volume_pyramid_f32(self, f1, f2):
        self.calls.append("build")
        return [torch.zeros(1)] * 4


@pytest.fixture
def stub(monkeypatch):
    import droid_slam_b200.modules as m
    be = _StubBackend()
    monkeypatch.setattr(m, "install", lambda: be)
    return be


def _net(**kw):
    from droid_slam_b200.modules import install_corr_training_hook
    return install_corr_training_hook(types.SimpleNamespace(CorrBlock=lambda *a, **k: ("reference", a, k)), **kw)


@pytest.mark.parametrize("shape", [(1, 24, 128, 48, 64), (2, 3, 128, 17, 23), (1, 2, 128, 8, 8), (1, 2, 128, 43, 70)])
def test_hook_builds_natively(stub, shape):
    f = _Fmap(shape)
    blk = _net().CorrBlock(f, f, num_levels=4, radius=3)
    assert stub.calls == ["build"] and blk._token is None


@pytest.mark.parametrize("kw, why", [
    (dict(dtype=torch.float16, requires_grad=True), "float16"),
    (dict(dtype=torch.bfloat16), "bfloat16"),
    (dict(is_cuda=False), "CUDA device"),
    (dict(shape=(1, 3, 64, 48, 64)), "64 channels"),
    (dict(shape=(1, 3, 128, 7, 64)), "at least 8"),
    (dict(levels=3), "3 levels"),
    (dict(radius=4), "radius 4"),
])
def test_hook_raises_or_falls_back_naming_the_reason(stub, kw, why):
    levels, radius = kw.pop("levels", 4), kw.pop("radius", 3)
    f = _Fmap(**kw)
    with pytest.raises(RuntimeError, match="CorrBlock has no kernel for this call: .*" + why):
        _net().CorrBlock(f, f, num_levels=levels, radius=radius)
    out = _net(strict=False).CorrBlock(f, f, num_levels=levels, radius=radius)
    assert out[0] == "reference" and out[2] == dict(num_levels=levels, radius=radius)
    assert stub.calls == []


def test_registry_entry_and_reference_kept_across_installs():
    from droid_slam_b200 import modules
    net = types.SimpleNamespace(CorrBlock="the reference class")
    modules.install_corr_training_hook(net, strict=False)
    modules.install_corr_training_hook(net)
    assert net._b200_reference_CorrBlock == "the reference class" and callable(net.CorrBlock)
    entries = [e for e in modules.hook_registry() if e["installer"] == "install_corr_training_hook"]
    assert entries and entries[-1]["kwargs"] == {"strict": True}
    assert "install_corr_training_hook" in modules.__all__


def test_oracle_restatement_matches_the_reference_fixture():
    """oracle/corr.py's CorrBlock restatement (corr_pyramid + corr_block_lookup, plain PyTorch, so autograd differentiates it) against
    the unmodified reference's forward and backward in fp64 (tests/golden/make_corr_training_golden.py)"""
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tests"))
    import oracle
    from corr_training_cases import FIXTURE, fixture_record, make_inputs
    G = torch.load(os.path.join(root, "tests", "golden", "corr_training.pt"))
    assert set(G) == set(FIXTURE)
    for name, (B, N, C, ht, wd, calls, used) in FIXTURE.items():
        f1, f2, coords, weights = make_inputs(B, N, ht, wd, calls, seed=11, C=C)
        a, b = f1.double().requires_grad_(True), f2.double().requires_grad_(True)
        pyr = oracle.corr_pyramid(a, b)
        outs = [oracle.corr_block_lookup(pyr, c) for c in coords]
        loss = sum((weights[k].double() * outs[k]).sum() for k in (used if used is not None else range(calls)))
        g1, g2 = torch.autograd.grad(loss, [a, b])
        rec = fixture_record([p.detach() for p in pyr], [o.detach() for o in outs], g1, g2)
        assert set(rec) == set(G[name])
        for k, want in G[name].items():
            assert rec[k].dtype == torch.float64 and rec[k].shape == want.shape, (name, k)
            assert float((rec[k] - want).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max())), (name, k)
