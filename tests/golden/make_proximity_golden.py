"""Golden vectors for row F1 (proximity edge selection) from the reference's own method, run UNMODIFIED in this container:

    python tests/golden/make_proximity_golden.py        -> tests/golden/proximity.pt

`FactorGraph.add_proximity_factors` (droid_slam/factor_graph.py:346-412) is called as an unbound function on a stub object that has
exactly the attributes the method reads (video.counter.value, video.distance, video.stereo, the six edge lists, max_factors, device)
and records what it passes to `add_factors`.  Substituted for the import only: lietorch (oracle/shims), matplotlib (an empty module:
factor_graph.py imports pyplot and never uses it on this path), droid_backends (not called by this method).  Inputs are regenerated
from seeds by `cases()`; only the emitted edge lists are stored.
"""
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from reference import reference_modules  # noqa: E402


def distance_matrix(t0, t1, t, seed, spread=6.0, far=0.05, nan=0):
    """a plausible `video.distance` result over the (i in [t0,t), j in [t1,t)) grid: mean flow magnitude growing with |i-j|, a few
    revisits (small distance far from the diagonal), a fraction of far pairs > 100, all values distinct (argsort order unambiguous)"""
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(t0, t, dtype=torch.float32)[:, None]
    j = torch.arange(t1, t, dtype=torch.float32)[None, :]
    d = spread * (i - j).abs() * (0.6 + 0.8 * torch.rand(t - t0, t - t1, generator=g)) + 0.01 * torch.rand(t - t0, t - t1, generator=g)
    revisit = torch.rand(t - t0, t - t1, generator=g) < 0.08
    d = torch.where(revisit, 2.0 + 12.0 * torch.rand(t - t0, t - t1, generator=g), d)
    d = torch.where(torch.rand(t - t0, t - t1, generator=g) < far, d + 150.0, d)
    d = d.reshape(-1)
    # make every value distinct without changing the order of distinct ones
    d = d + 1e-4 * torch.argsort(torch.argsort(torch.rand(d.numel(), generator=g))).float() / d.numel()
    if nan:
        idx = torch.randperm(d.numel(), generator=g)[:nan]
        d[idx] = float("nan")
    return d.float()


def existing_edges(t, n, seed):
    g = torch.Generator().manual_seed(seed)
    if n == 0 or t < 2:
        return [torch.zeros(0, dtype=torch.long)] * 6
    out = []
    for k in range(3):
        m = n if k == 0 else n // 3
        ii = torch.randint(0, t, (m,), generator=g)
        jj = (ii + torch.randint(-6, 7, (m,), generator=g)).clamp(0, t - 1)
        out += [ii, jj]
    return out


def cases():
    """(name, kwargs of the method, t, stereo, max_factors, distance seed, existing-edge count, nan count)"""
    return [
        ("init_12",      dict(t0=0, t1=0, rad=2, nms=2, thresh=16.0, remove=False), 12, False, -1, 1, 0, 0),
        ("frontend_30",  dict(t0=25, t1=5, rad=2, nms=1, thresh=16.0, beta=0.3, remove=True), 30, False, -1, 2, 40, 0),
        ("frontend_8",   dict(t0=3, t1=0, rad=2, nms=1, thresh=16.0, beta=0.3, remove=True), 8, False, -1, 3, 10, 0),
        ("backend_90",   dict(t0=0, t1=0, rad=2, nms=2, thresh=22.0, beta=0.2), 90, False, 700, 4, 60, 0),
        ("backend_cap",  dict(t0=0, t1=0, rad=2, nms=2, thresh=22.0, beta=0.2), 60, False, 380, 5, 0, 0),
        ("stereo_20",    dict(t0=0, t1=0, rad=1, nms=2, thresh=12.0), 20, True, -1, 6, 12, 0),
        ("rad3_nms0",    dict(t0=2, t1=1, rad=3, nms=0, thresh=30.0), 26, False, -1, 7, 20, 0),
        ("with_nan",     dict(t0=0, t1=0, rad=2, nms=2, thresh=16.0), 24, False, -1, 8, 8, 5),
        ("wrap_t1_gt_j", dict(t0=4, t1=3, rad=2, nms=2, thresh=16.0), 16, False, -1, 9, 6, 0),     # j = i-rad-1 < t1 on the first rows: unchecked index
    ]


def import_reference_factor_graph():
    """the reference's factor_graph module, imported unmodified"""
    stubs = {"droid_backends": types.ModuleType("droid_backends")}
    if importlib.util.find_spec("matplotlib") is None:
        stubs["matplotlib"] = types.ModuleType("matplotlib")
        stubs["matplotlib.pyplot"] = stubs["matplotlib"].pyplot = types.ModuleType("matplotlib.pyplot")
    with reference_modules("factor_graph", stubs=stubs) as (fg,):
        return fg


class _Counter:
    def __init__(self, v):
        self.value = v


class _Video:
    def __init__(self, t, stereo, d):
        self.counter = _Counter(t)
        self.stereo = stereo
        self._d = d

    def distance(self, ii, jj, beta=0.3):
        assert ii.numel() == self._d.numel()
        return self._d.clone()


class _Graph:
    def __init__(self, video, edges, max_factors):
        self.video = video
        self.ii, self.jj, self.ii_bad, self.jj_bad, self.ii_inac, self.jj_inac = edges
        self.max_factors = max_factors
        self.device = "cpu"
        self.calls = []

    def add_factors(self, ii, jj, remove=False):
        self.calls.append((ii.clone(), jj.clone(), remove))


def run_reference(fg, case):
    name, kw, t, stereo, max_factors, seed, n_exist, nan = case
    d = distance_matrix(kw["t0"], kw["t1"], t, seed, nan=nan)
    graph = _Graph(_Video(t, stereo, d), existing_edges(t, n_exist, seed + 100), max_factors)
    fg.FactorGraph.add_proximity_factors(graph, **kw)
    (ii, jj, remove), = graph.calls
    return torch.stack([ii, jj], 1).long(), bool(remove)


def main(out=None):
    fg = import_reference_factor_graph()
    gold = {}
    for case in cases():
        es, remove = run_reference(fg, case)
        gold[case[0] + "_es"] = es
        gold[case[0] + "_remove"] = torch.tensor(remove)
    out = out or os.path.join(ROOT, "tests", "golden", "proximity.pt")
    torch.save(gold, out)
    for k, v in gold.items():
        if k.endswith("_es"):
            print("%-22s %4d edges" % (k, v.shape[0]))


if __name__ == "__main__":
    main()
