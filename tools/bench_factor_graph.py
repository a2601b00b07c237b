"""Time the native FactorGraph.update / update_lowmem (droid_slam_b200.modules) against oracle.factor_graph -- the reference's control flow
-- running the same native operators, on stub graphs built from seeds (tests/factor_graph_stubs.py):

  frontend   update(use_inactive=True), about 48 edges at 48x64
  filler     update(motion_only=True) at 44x69 (the trajectory filler's call)
  c3         one update_lowmem step on the 2048-edge / 400-keyframe global-BA graph at 48x64 (synth "c3_global")
  rig2       one update_lowmem step with use_inactive at 43x70, rig 2 (stereo)

Each call timed on its own, the two paths alternating, median over --reps rounds after --warmup calls of each.  BA's own status reads
are left out of the host-sync count (the stub video's ba).

    python tools/bench_factor_graph.py [--reps 15] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle.factor_graph as ofg  # noqa: E402
from droid_slam_b200 import modules, synth  # noqa: E402
import factor_graph_stubs as fs  # noqa: E402
from util import card, host_syncs, timed  # noqa: E402


def frontend():
    v = fs.Video(16, 1, 48, 64, seed=1)
    edges = fs.neighbourhood(8, 16, 3, closures=[(8, 15), (15, 8), (9, 14), (14, 9), (10, 15), (15, 10),
                                                          (8, 12), (12, 8), (9, 13), (13, 9), (11, 15), (15, 11)])
    return fs.Graph(v, edges, fs.neighbourhood(2, 10, 2), upsample=True, seed=1)


def filler():
    v = fs.Video(40, 1, 44, 69, seed=2)
    # 16 new frames, each tied to the two keyframes around it (trajectory_filler.py)
    edges = [(k, 16 + i) for i in range(16) for k in (i // 8, i // 8 + 1)] + [(16 + i, k) for i in range(16) for k in (i // 8, i // 8 + 1)]
    return fs.Graph(v, edges, [], seed=2)


def c3():
    c = synth.CONFIGS["c3_global"]
    v = fs.Video(c["N"], 1, c["ht"], c["wd"], seed=3)
    ii, jj = synth.make_graph(c["E"], c["N"], seed=3)
    return fs.Graph(v, list(zip(ii.tolist(), jj.tolist())), [], seed=3, volume=False)


def rig2():
    v = fs.Video(64, 2, 43, 70, seed=4)
    return fs.Graph(v, fs.neighbourhood(0, 64, 2, stereo=True), fs.neighbourhood(0, 32, 3)[::3], seed=4, volume=False)


SHAPES = [
    ("frontend update 48x64", frontend, "update", dict(use_inactive=True)),
    ("filler update(motion_only) 44x69", filler, "update", dict(t0=1, t1=40, motion_only=True)),
    ("c3 update_lowmem step 48x64", c3, "update_lowmem", dict(steps=1, use_inactive=False)),
    ("rig2 update_lowmem step 43x70", rig2, "update_lowmem", dict(steps=1, use_inactive=True)),
]


def native(graph, method, kw):
    getattr(modules, method)(graph, **kw)


def reference_flow(graph, method, kw):
    if method == "update":
        ofg.update(graph, **kw)
    else:
        ofg.update_lowmem(graph, alt_corr_block=fs.AltCorrBlock, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_factor_graph needs a CUDA device")
    rows = []
    with torch.no_grad():
        for name, make, method, kw in SHAPES:
            g_nat, g_ref = make(), make()
            paths = [("native", native, g_nat), ("reference flow", reference_flow, g_ref)]
            for _, fn, g in paths:
                for _ in range(args.warmup):
                    fn(g, method, kw)
            times = {p: [] for p, _, _ in paths}
            for r in range(args.reps):
                for p, fn, g in (paths if r % 2 == 0 else paths[::-1]):
                    times[p].append(timed(lambda: fn(g, method, kw))[0])
            n_sync = {p: host_syncs(lambda: fn(g, method, kw))[0] for p, fn, g in paths}
            row = dict(shape=name, edges=int(g_nat.ii.numel()),
                       native_ms=statistics.median(times["native"]), reference_flow_ms=statistics.median(times["reference flow"]),
                       native_syncs=n_sync["native"], reference_flow_syncs=n_sync["reference flow"])
            row["speedup"] = row["reference_flow_ms"] / row["native_ms"]
            rows.append(row)
            print("%-34s %5d edges  native %8.3f ms (%d syncs)  reference flow %8.3f ms (%d syncs)  %.2fx" % (
                name, row["edges"], row["native_ms"], row["native_syncs"], row["reference_flow_ms"], row["reference_flow_syncs"], row["speedup"]),
                flush=True)
            del g_nat, g_ref
            torch.cuda.empty_cache()
    info = card()
    print("card: %s" % ", ".join("%s=%s" % kv for kv in info.items()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=info, rows=rows, reps=args.reps, warmup=args.warmup), f, indent=1)


if __name__ == "__main__":
    main()
