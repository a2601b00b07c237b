"""DroidAsync's backend without a GPU: the hand-over restatement (oracle/async_backend.py) against what the unmodified align.py and
backend_process computed (tests/golden/async_backend.pt), the hook registry, its re-installation in a spawned process, and the strict
policy of install_async_hook."""
import contextlib
import ctypes
import multiprocessing
import os
import pickle
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import async_backend as oab  # noqa: E402
from droid_slam_b200 import c_api, modules  # noqa: E402
import async_stubs  # noqa: E402

CASES = ("mono", "rgbd", "stereo", "t0_zero")


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "async_backend.pt"))


@contextlib.contextmanager
def isolated_registry():
    """an empty hook registry for the block (other test modules install hooks on objects that are not importable by name)"""
    saved = list(modules._HOOKS)
    modules._HOOKS.clear()
    try:
        yield
    finally:
        modules._HOOKS[:] = saved


@pytest.mark.parametrize("name", CASES[:3])
def test_alignment_is_bit_exact_against_the_reference(gold, name):
    g = gold[name]
    t0 = g["case"][1]
    for dt, tag in ((torch.float32, "fp32"), (torch.float64, "fp64")):
        dG, s = oab.align_pose_fragments(g["front"]["poses"][t0 - 10:t0 - 1].to(dt), g["back"]["poses"][t0 - 10:t0 - 1].to(dt))
        assert torch.equal(dG.data, g["align_" + tag][0]) and torch.equal(s, g["align_" + tag][1]), tag


@pytest.mark.parametrize("name", CASES)
def test_handover_matches_the_unmodified_backend_process(gold, name):
    g = gold[name]
    _, t0, stereo, rgbd, _ = g["case"]
    out, s, dG, align_scale = oab.handover(g["front"], g["back"], t0, g["t1"], stereo)
    assert align_scale == (name in ("mono", "t0_zero"))
    differ = [k for k in oab.BUFFERS if not torch.equal(out[k], g["after"][k])]
    assert not differ, differ
    assert g["record"] == {"steps": 12, "normalize": False, "counter2": g["t1"], "net": ("net", "droid.pth", "cpu")}


def test_the_scale_is_discarded_but_dg_keeps_it(gold):
    """rgbd / stereo: s = 1 is applied, dG is the one align.py computed from the s-scaled poses"""
    for name in ("rgbd", "stereo"):
        g = gold[name]
        _, s, dG, _ = oab.handover(g["front"], g["back"], g["case"][1], g["t1"], g["case"][2])
        assert s == 1.0 and torch.equal(dG, g["align_fp32"][0]) and float(g["align_fp32"][1]) != 1.0


def test_registry_records_every_hook_and_pickles():
    with isolated_registry():
        async_stubs.install_backend_hooks()
        modules.install_corr_volume_hook(async_stubs, fused_lookup=True)
        reg = modules.hook_registry()
        assert [e["installer"] for e in reg] == ["install_update_module_hook", "install_alt_corr_hook", "install_factor_graph_hook",
                                                "install_proximity_hook", "install_depth_video_hook", "install_corr_volume_hook"]
        assert all(e["transferable"] for e in reg)
        assert reg[2]["module"] == "async_stubs" and reg[2]["qualname"] == "FactorGraph" and reg[2]["kwargs"] == {"strict": True}
        assert reg[5]["kwargs"] == {"strict": True, "fused_lookup": True}
        assert pickle.loads(pickle.dumps(reg)) == reg
        modules.install_alt_corr_hook(async_stubs, strict=False)       # installing again on the same target replaces the entry
        assert [e["kwargs"] for e in modules.hook_registry() if e["installer"] == "install_alt_corr_hook"] == [{"strict": False}]
        ns = types.SimpleNamespace(CorrBlock=async_stubs.CorrBlock)
        modules.install_proximity_hook(type("Local", (), {}))
        modules.install_corr_volume_hook(ns)
        assert [e["transferable"] for e in modules.hook_registry()[-2:]] == [False, False]


def test_a_spawned_process_reinstalls_the_recorded_hooks():
    ctx = multiprocessing.get_context("spawn")
    with isolated_registry():
        async_stubs.install_backend_hooks()
        backend = async_stubs.backend_process
        assert isinstance(backend, modules.BackendProcess)
        q = ctx.Queue()
        proc = ctx.Process(target=async_stubs.report_hooks, args=(backend, q))
        try:
            proc.start()
            before, after, ext = q.get(timeout=300)
            proc.join(timeout=60)
        finally:
            if proc.is_alive():
                proc.terminate()
            proc.join(timeout=30)
    assert proc.exitcode == 0
    assert set(before.values()) <= {"async_stubs", None}, before
    assert after == {"UpdateModule": "droid_slam_b200.update", "AltCorrBlock.__init__": "droid_slam_b200.modules",
                     "FactorGraph.update_lowmem": "droid_slam_b200.modules", "FactorGraph.add_proximity_factors": "droid_slam_b200.modules",
                     "DepthVideo.reproject": "droid_slam_b200.modules"}, after
    assert ext == "droid_backends"


def test_strict_raises_on_a_missing_or_untransferable_hook():
    with isolated_registry():
        modules.install_async_hook(async_stubs)
        with pytest.raises(RuntimeError, match="backend_process has no kernel for this call: the native backend needs install_update_module_hook"):
            pickle.dumps(async_stubs.backend_process)
        with pytest.raises(RuntimeError, match="has no kernel for this call"):
            async_stubs.backend_process(None, None, None)
        async_stubs.install_backend_hooks()
        assert pickle.loads(pickle.dumps(async_stubs.backend_process)).native is True
        modules.install_corr_volume_hook(types.SimpleNamespace(CorrBlock=async_stubs.CorrBlock))
        with pytest.raises(RuntimeError, match="cannot import by name: install_corr_volume_hook on namespace"):
            pickle.dumps(async_stubs.backend_process)


def test_non_strict_keeps_the_reference_loop():
    with isolated_registry():
        modules.install_async_hook(async_stubs, strict=False)
        bp = async_stubs.backend_process
        assert isinstance(bp, modules.BackendProcess)
        del async_stubs.REFERENCE_CALLS[:]
        bp(None, None, None, "cuda:1")                                   # in this process: the reference's function
        assert async_stubs.REFERENCE_CALLS == ["cuda:1"]
        child = pickle.loads(pickle.dumps(bp))                           # in a spawned one: its module's own backend_process
        assert child.native is False and child.hooks == []
        modules.install_async_hook(async_stubs, strict=True)             # re-installing keeps the reference's function underneath
        assert async_stubs.backend_process.reference is bp.reference
    async_stubs.backend_process = bp.reference


def test_update_module_hook_sets_the_native_operator():
    from droid_slam_b200.update import UpdateModule
    ns = types.ModuleType("droid_net_standin")
    ns.UpdateModule = object
    with isolated_registry():
        assert modules.install_update_module_hook(ns).UpdateModule is UpdateModule
        assert modules.hook_registry()[0]["transferable"] is False       # not in sys.modules under its name


def test_c_abi_rejects_bad_arguments_before_any_launch():
    L = c_api.load()
    f = L.dba_fragment_handover
    assert L.dba_fragment_handover and hasattr(L, "dba_last_error")
    p = ctypes.c_void_p(64)
    for t0 in (1, 5, 9, -1):                              # the reference's negative slices are not reproduced
        assert f(p, p, p, p, 0, t0, 20, 12, 0, p, None, None) != 0
    assert f(p, p, p, p, 0, 0, 20, 0, 0, p, None, None) != 0          # hw = 0
    assert f(None, p, p, p, 0, 10, 20, 12, 0, p, None, None) != 0     # t0 > 0 needs the frontend's fragment
    assert f(p, p, p, p, 0, 0, 20, 12, 0, None, None, None) != 0      # no workspace
    assert f(p, p, p, p, 0, 0, 20, 12, 0, ctypes.c_void_p(68), None, None) != 0   # misaligned workspace
