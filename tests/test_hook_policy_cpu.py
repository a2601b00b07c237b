"""The strict policy of the hooks, without a GPU: a hook installed again with strict=False after strict=True falls back to the reference's
own function -- for a method of a reference class (AltCorrBlock.__init__) and for a global of a reference module (droid_net.BA) -- and
not to the wrapper the first install put there."""
import types

import pytest
import torch

from droid_slam_b200 import modules


@pytest.fixture(autouse=True)
def registry(monkeypatch):
    monkeypatch.setattr(modules, "_HOOKS", [])      # the stubs' registry entries stay out of the process's registry


class _StubAltCorrBlock:
    """records which of the reference's methods ran"""

    def __init__(self, fmaps, num_levels=4, radius=3):
        self.calls = ["init"]

    def __call__(self, coords, ii, jj):
        self.calls.append("call")
        return "reference"


def test_class_method_hook_installed_again_falls_back_to_the_reference():
    mod = types.SimpleNamespace(AltCorrBlock=type("AltCorrBlock", (_StubAltCorrBlock,), {}))
    modules.install_alt_corr_hook(mod)
    modules.install_alt_corr_hook(mod, strict=False)
    blk = mod.AltCorrBlock(torch.zeros(1, 2, 16, 8, 8))                 # CPU maps: no native path
    assert blk(torch.zeros(1, 2, 8, 8, 2), torch.tensor([0, 1]), torch.tensor([1, 0])) == "reference"
    assert blk.calls == ["init", "call"]


def test_module_global_hook_installed_again_falls_back_to_the_reference():
    m = types.ModuleType("stub_droid_net")
    calls = []
    m.BA = lambda *a, **k: calls.append((a, k)) or "reference"
    modules.install_ba_layer_hook(m)
    modules.install_ba_layer_hook(m, strict=False)
    t = torch.zeros(1)
    assert m.BA(t, t, t, t, t, t, t, t, fixedp=2) == "reference"       # poses not SE3: no native path
    assert len(calls) == 1 and calls[0][1] == {"fixedp": 2}
