"""DroidAsync's backend on the GPU: droid_backends.fragment_handover against the fp64 restatement (oracle/async_backend.py) at the
reference's image sizes and buffer lengths, the one host sync of a round, and a spawned backend process on the stand-in modules of
tests/async_stubs.py under strict=True."""
import contextlib
import os
import sys
import types
import warnings

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import async_backend as oab  # noqa: E402
from droid_slam_b200 import modules  # noqa: E402
import async_stubs  # noqa: E402

pytestmark = pytest.mark.gpu
TWO_GPUS = torch.cuda.is_available() and torch.cuda.device_count() > 1


@contextlib.contextmanager
def isolated_registry():
    saved = list(modules._HOOKS)
    modules._HOOKS.clear()
    try:
        yield
    finally:
        modules._HOOKS[:] = saved


def _cpu(video):
    return {k: getattr(video, k).cpu() for k in oab.BUFFERS}


def _ulps(a, b):
    """distance in fp32 ulps of a to b"""
    ai, bi = a.view(torch.int32).long(), b.view(torch.int32).long()
    ai = torch.where(ai < 0, -(ai & 0x7FFFFFFF), ai)
    bi = torch.where(bi < 0, -(bi & 0x7FFFFFFF), bi)
    return (ai - bi).abs()


def check_round(v1, v2, t0, t1, stereo):
    """one handover_round against the oracle on the same inputs"""
    front, back = _cpu(v1), _cpu(v2)
    diag = modules.handover_round(v1, v2, t0, t1, diagnostics=True).cpu()
    want, s_ref, dG_ref, align_scale = oab.handover(front, back, t0, t1, stereo, align_dtype=torch.float64)
    s_ref = float(s_ref)
    assert bool(diag[8]) == align_scale
    assert abs(float(diag[0]) - s_ref) <= 1e-6 * abs(s_ref)
    dG_ref = dG_ref.reshape(-1).double()
    assert (diag[1:8] - dG_ref).abs().max() <= 1e-6 * max(1.0, float(dG_ref[:3].abs().max())), (diag[1:8], dG_ref)
    got = _cpu(v2)
    n = max(t1 - t0, 0)
    poses = oab.reanchor(front["poses"][t0:t0 + n], float(diag[0]), diag[1:8])
    assert n == 0 or int(_ulps(got["poses"][t0:t0 + n], poses).max()) <= 2
    s_f = torch.tensor(float(diag[0]), dtype=torch.float32)
    assert torch.equal(got["disps"][t0:t0 + n], front["disps"][t0:t0 + n] / s_f)
    for k in oab.BUFFERS[2:]:
        assert torch.equal(got[k][t0:t0 + n], front[k][t0:t0 + n]), k
    outside = torch.ones(got["poses"].shape[0], dtype=torch.bool)
    outside[t0:t0 + n] = False
    for k in oab.BUFFERS:
        assert torch.equal(got[k][outside], back[k][outside]), ("written outside [t0,t1)", k)
    return diag


# (513, 47, 69): disps_sens has an odd element count, so the any() scan takes its scalar path
SHAPES = [(512, 48, 64), (1024, 44, 69), (513, 47, 69)]
# rgbd_last: the one nonzero sensor depth lies in the last slice of the any() scan, outside [t0, t1)
MODES = [("mono", 300), ("rgbd", 300), ("rgbd_last", 300), ("stereo", 300), ("mono", 0)]


@pytest.mark.parametrize("buffer,ht,wd", SHAPES)
@pytest.mark.parametrize("mode,t0", MODES)
def test_fragment_handover_matches_the_oracle(buffer, ht, wd, mode, t0):
    t1 = t0 + 64 if t0 else 40
    v1, v2 = async_stubs.make_videos(buffer, ht, wd, mode, t0, t1, seed=buffer + t0)
    diag = check_round(v1, v2, t0, t1, mode == "stereo")
    if mode == "mono" and t0:
        assert float(diag[0]) != 1.0
    assert bool(diag[8]) == (mode == "mono")


@pytest.mark.skipif(not TWO_GPUS, reason="needs two GPUs")
@pytest.mark.parametrize("mode", ["mono", "rgbd"])
def test_fragment_handover_across_devices(mode):
    v1, v2 = async_stubs.make_videos(512, 48, 64, mode, 300, 364, "cuda:0", "cuda:1", seed=7)
    check_round(v1, v2, 300, 364, False)


def test_empty_round_and_rejected_t0(backends):
    v1, v2 = async_stubs.make_videos(64, 16, 24, "mono", 30, 40, seed=3)
    back = _cpu(v2)
    diag = modules.handover_round(v1, v2, 30, 28, diagnostics=True).cpu()   # t1 < t0: nothing re-anchored, the alignment still runs
    _, s_ref, _, _ = oab.handover(_cpu(v1), back, 30, 31, False, align_dtype=torch.float64)
    assert abs(float(diag[0]) - float(s_ref)) <= 1e-6 * abs(float(s_ref))
    assert all(torch.equal(t, back[k]) for k, t in _cpu(v2).items())
    with pytest.raises(RuntimeError, match="t0 must be 0 or at least 10"):
        modules.handover_round(v1, v2, 5, 20)


def test_one_host_sync_per_round():
    v1, v2 = async_stubs.make_videos(512, 48, 64, "rgbd", 300, 364, seed=5)
    modules.handover_round(v1, v2, 300, 364)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            modules.handover_round(v1, v2, 300, 364)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert sum(str(w.message).startswith("called a synchronizing") for w in caught) == 1, [str(w.message) for w in caught]


@pytest.mark.parametrize("devices", [("cuda", "cuda"), ("cuda:0", "cuda:1")])
def test_spawned_backend_process_runs_the_final_round(tmp_path, devices):
    if devices[1] == "cuda:1" and not TWO_GPUS:
        pytest.skip("needs two GPUs")
    ctx = torch.multiprocessing.get_context("spawn")
    weights = str(tmp_path / "droid.pth")
    async_stubs.write_checkpoint(weights)
    t0, t1 = 28, 60
    v1, v2 = async_stubs.make_videos(128, 48, 64, "mono", t0, t1, devices[0], devices[1], seed=11)
    v2.ready.value = 1                                   # the last round: the loop runs once and returns
    front, back = _cpu(v1), _cpu(v2)
    proc = None
    with isolated_registry():
        async_stubs.install_backend_hooks(strict=True)
        try:
            proc = ctx.Process(target=async_stubs.backend_process, args=(types.SimpleNamespace(weights=weights), v1, v2, devices[1]))
            proc.start()
            proc.join(timeout=600)
        finally:
            if proc is not None and proc.is_alive():
                proc.terminate()
                proc.join(timeout=30)
    assert proc.exitcode == 0
    torch.cuda.synchronize()
    got = _cpu(v2)
    want, s_ref, dG_ref, _ = oab.handover(front, back, t0, t1, False, align_dtype=torch.float64)
    assert v2.counter.value == t1
    assert bool(v2.dirty[:t1].all()) and not bool(v2.dirty[t1:].any())
    assert torch.isfinite(got["poses"]).all()
    assert v2.record.tolist() == [8 if devices[1] == "cuda" else 12, 1]   # iterations; the network built the native update operator
    poses = oab.reanchor(front["poses"][t0:t1], float(s_ref), dG_ref.reshape(-1).double())
    assert (got["poses"][t0:t1] - poses).abs().max() <= 1e-5
    assert torch.allclose(got["disps"][t0:t1], front["disps"][t0:t1] / float(s_ref), rtol=2e-6, atol=0)
    for k in oab.BUFFERS[2:]:
        assert torch.equal(got[k][t0:t1], front[k][t0:t1]), k
