"""Time the training CorrBlock (droid_slam_b200.modules.CorrBlock, csrc/corr_train.cu) against the reference's CorrBlock restated on this
package's drop-in ops (fp32 torch.matmul without tf32, 3x avg_pool2d, CorrSampler on corr_index_forward / corr_index_backward), both on
the same GPU, the two alternating, with the card's name, power limit and clocks read in the same run.

    python tools/bench_corr_training.py --rounds 5 [--json out.json]

Shapes: train.py's 24 edges of 48 x 64 feature maps (384 x 512 crops), and 24 edges of 72 x 96.  One step = build the block, look it up
15 times (--iters 15), backward of a loss on every lookup.  CUDA events split the step into build, lookups and backward; each figure is the
median over the rounds.  Peak memory is torch.cuda.max_memory_allocated over the step above what was allocated before it; host
synchronisations of one step are counted with tests/util.host_syncs."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from droid_slam_b200 import modules  # noqa: E402
from corr_training_cases import RefCorrBlock, make_inputs  # noqa: E402
from util import card, host_syncs  # noqa: E402

CALLS = 15


def reference(a, b):
    return RefCorrBlock(a, b)


def native(a, b):
    return modules.CorrBlock(a, b)


def step(make, f1, f2, coords, w, events=None):
    a, b = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)
    ev = events or [None] * 4
    ev[0] and ev[0].record()
    call = make(a, b)
    ev[1] and ev[1].record()
    loss = sum((w * call(c)).sum() for c in coords)
    ev[2] and ev[2].record()
    loss.backward()
    ev[3] and ev[3].record()
    return a.grad, b.grad


def measure(make, f1, f2, coords, w):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    step(make, f1, f2, coords, w, ev)
    torch.cuda.synchronize()
    t = [ev[k].elapsed_time(ev[k + 1]) for k in range(3)]
    return dict(build_ms=t[0], lookups_ms=t[1], backward_ms=t[2], total_ms=sum(t),
                peak_mb=(torch.cuda.max_memory_allocated() - base) / 2 ** 20)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    out = dict(card=card(), shapes=[])
    print(out["card"])
    for ht, wd in ((48, 64), (72, 96)):
        f1, f2, coords, _ = make_inputs(1, 24, ht, wd, CALLS, seed=0, dev="cuda")
        w = torch.randn(1, 24, 196, ht, wd, device="cuda")
        impls = dict(reference=reference, native=native)
        for make in impls.values():                       # warm-up
            step(make, f1, f2, coords, w)
        rows = {k: [] for k in impls}
        for _ in range(args.rounds):
            for name, make in impls.items():
                rows[name].append(measure(make, f1, f2, coords, w))
        res = dict(shape="24 edges, %dx%d, %d lookups" % (ht, wd, CALLS))
        for name, make in impls.items():
            med = {k: statistics.median(r[k] for r in rows[name]) for k in rows[name][0]}
            med["host_syncs"] = host_syncs(lambda: step(make, f1, f2, coords, w))[0]
            res[name] = med
        res["speedup_total"] = res["reference"]["total_ms"] / res["native"]["total_ms"]
        out["shapes"].append(res)
        print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
