"""FactorGraph.update / update_lowmem hooks (droid_slam_b200.modules) on the GPU against oracle.factor_graph -- the reference's control flow
-- running the same native operators on an identical stub graph (tests/factor_graph_stubs.py): every piece of graph and video state
torch.equal.  BA's own result is not bit-reproducible between calls on large graphs (fp64 atomics), so the second path replays the
first one's BA results after checking its BA inputs bit for bit (factor_graph_stubs.compare).  Also: chunk composition does not change a
bit, host synchronisations per call, strict mode."""
import os
import sys
import warnings

import pytest
import torch

import oracle.factor_graph as ofg
from droid_slam_b200 import modules

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import factor_graph_stubs as fs  # noqa: E402

pytestmark = pytest.mark.gpu


def _frontend():
    """about 48 edges at 48x64, inactive edges behind the window"""
    v = fs.Video(16, 1, 48, 64, seed=1)
    edges = fs.neighbourhood(8, 16, 3, closures=[(8, 15), (15, 8), (9, 14), (14, 9), (10, 15), (15, 10),
                                                          (8, 12), (12, 8), (9, 13), (13, 9), (11, 15), (15, 11)])
    inac = fs.neighbourhood(2, 10, 2)
    return fs.Graph(v, edges, inac, upsample=True, seed=1)


def _filler():
    v = fs.Video(10, 1, 44, 69, seed=2)
    return fs.Graph(v, fs.neighbourhood(0, 10, 2), [], seed=2)


def _backend(upsample=False):
    """about 900 edges over 100 keyframes at 48x64, with loop closures and a quirk edge set beyond the reference's last chunk"""
    v = fs.Video(100, 1, 48, 64, seed=3)
    g = torch.Generator().manual_seed(3)
    closures = [(int(i), int((i + d) % 100)) for i, d in zip(torch.randint(0, 100, (120,), generator=g),
                                                              torch.randint(10, 90, (120,), generator=g))]
    edges = fs.neighbourhood(0, 100, 4) + sorted(set(closures) - set(fs.neighbourhood(0, 100, 4)))
    return fs.Graph(v, edges, fs.neighbourhood(0, 100, 6)[::7], upsample=upsample, seed=3, volume=False)


def _stereo():
    v = fs.Video(24, 2, 43, 70, seed=4)
    return fs.Graph(v, fs.neighbourhood(0, 24, 2, stereo=True), fs.neighbourhood(0, 12, 3)[::3], seed=4, volume=False)


CASES = {
    "frontend_update": (_frontend, "update", dict(t0=None, use_inactive=True)),
    "filler_motion_only_44x69": (_filler, "update", dict(t0=1, t1=10, motion_only=True)),
    "backend_lowmem_48x64": (_backend, "update_lowmem", dict(steps=2, use_inactive=True)),
    "stereo_lowmem_inactive_43x70": (_stereo, "update_lowmem", dict(steps=2, use_inactive=True)),
}


def _run_hook(graph, method, kw):
    with torch.no_grad():
        getattr(modules, method)(graph, **kw)
    torch.cuda.synchronize()
    return fs.state(graph)


def _run_oracle(graph, method, kw):
    with torch.no_grad():
        if method == "update":
            ofg.update(graph, **kw)
        else:
            ofg.update_lowmem(graph, alt_corr_block=fs.AltCorrBlock, **kw)
    torch.cuda.synchronize()
    return fs.state(graph)


@pytest.mark.parametrize("name", list(CASES))
def test_hook_equals_the_reference_control_flow(name):
    make, method, kw = CASES[name]
    want, got = fs.compare(lambda g: _run_oracle(g, method, kw), make, lambda g: _run_hook(g, method, kw), make)
    assert bool(torch.isfinite(want["poses"]).all()) and bool(torch.isfinite(want["disps"]).all())
    assert fs.differing(got, want) == []


def test_upsampling_in_update_lowmem():
    kw = dict(steps=1, use_inactive=False)
    make = lambda: _backend(upsample=True)                                  # noqa: E731
    want, got = fs.compare(lambda g: _run_oracle(g, "update_lowmem", kw), make, lambda g: _run_hook(g, "update_lowmem", kw), make)
    assert fs.differing(got, want) == []
    assert bool((got["disps_up"][:99] != 0).any(dim=(1, 2)).all())


def test_lowmem_bits_do_not_depend_on_chunk_composition(monkeypatch):
    kw = dict(steps=2, use_inactive=True)
    budgets = (37, 400)
    graph = _backend()
    n_chunks = [len(modules.plan_lowmem_chunks(graph.ii.cpu(), graph.jj.cpu(), b)[1]) for b in budgets]
    assert n_chunks[0] > n_chunks[1] > 1

    def run(budget):
        def f(g):
            monkeypatch.setattr(modules, "_lowmem_edge_budget", lambda *a: budget)
            return _run_hook(g, "update_lowmem", kw)
        return f
    small, large = fs.compare(run(budgets[0]), _backend, run(budgets[1]), _backend)
    assert fs.differing(small, large) == []


def _count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in caught)


@pytest.mark.parametrize("make,method,kw", [(_frontend, "update", dict(use_inactive=True)),
                                            (_stereo, "update_lowmem", dict(steps=3, use_inactive=True))])
def test_at_most_one_host_sync_per_call(make, method, kw, monkeypatch):
    monkeypatch.setattr(modules, "_lowmem_edge_budget", lambda *a: 20)      # several chunks per step
    graph = make()
    with torch.no_grad():
        getattr(modules, method)(graph, **kw)                              # warm-up: packs the operator's weights once
        n = _count_syncs(lambda: getattr(modules, method)(graph, **kw))
    assert n <= 1, n


class _FactorGraph:
    """stand-in for the reference class: its methods record that they ran"""

    def update(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, motion_only=False):
        self.ran = "reference update"

    def update_lowmem(self, t0=None, t1=None, itrs=2, use_inactive=False, EP=1e-7, steps=8):
        self.ran = "reference update_lowmem"


def test_strict_mode():
    strict = type("StrictFG", (_FactorGraph,), {})
    lenient = type("LenientFG", (_FactorGraph,), {})
    modules.install_factor_graph_hook(strict, strict=True)
    modules.install_factor_graph_hook(lenient, strict=False)
    src = _filler()
    foreign_op = lambda *a: None                                           # noqa: E731  (not droid_slam_b200's UpdateModule)
    for cls in (strict, lenient):
        g = cls()
        g.__dict__.update(src.__dict__)
        g.update_op = foreign_op
        if cls is strict:
            with pytest.raises(RuntimeError, match="UpdateModule"):
                g.update()
            with pytest.raises(RuntimeError, match="UpdateModule"):
                g.update_lowmem()
        else:
            g.update()
            assert g.ran == "reference update"
            g.update_lowmem()
            assert g.ran == "reference update_lowmem"
    g = lenient()
    g.__dict__.update(_filler().__dict__)
    g.update(t0=1, t1=10, motion_only=True)                                 # native: the reference method does not run
    assert not hasattr(g, "ran")
