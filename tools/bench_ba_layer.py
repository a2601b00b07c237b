"""Time the native dense BA layer (droid_slam_b200.modules.ba_layer, csrc/ba_layer.cu) against the reference's flow restated on the
stand-ins (oracle/ba_layer.py: geom/ba.py + chol.py + projective_ops.py on PyTorch ops), both fp32 on the same GPU, the two alternating,
with the card's name, power limit and clocks printed beside the numbers.

    python tools/bench_ba_layer.py --reps 10 --warmup 3 [--json out.json]

Shapes (12 x 16 is the fixture's; these are DroidNet's 1/8 maps of train.py's 384 x 512 crops): B = 1, N = 7, 48 x 64 with 22 edges (the
radius-2 training graph) and 24 edges (plus 0 <-> 3); N = 15 with 60 edges (radius 2 plus six long edges); B = 4 at the N = 7 graph.
fixedp = 2.  `fwd` is one BA call under no_grad; `fwd+bwd` one call and autograd's backward of a loss on both outputs.  CUDA events
around `--reps` calls after `--warmup`, the median of 5 such windows; the host synchronisations of one call are counted with
tests/util.host_syncs.  The reference's own lietorch / torch_scatter cannot be built here, so its exact launches are not measured: the
oracle's flow is the same sequence of PyTorch operations on the stand-ins."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from droid_slam_b200 import lietorch as lt  # noqa: E402
from droid_slam_b200 import modules  # noqa: E402
from oracle import ba_layer as oba  # noqa: E402
from ba_layer_cases import make_inputs, radius_graph  # noqa: E402
from util import card, host_syncs, timed  # noqa: E402


def shapes():
    ii, jj = radius_graph(7)
    ii24, jj24 = torch.cat([ii, torch.tensor([0, 3])]), torch.cat([jj, torch.tensor([3, 0])])
    i15, j15 = radius_graph(15)
    extra_i, extra_j = torch.tensor([0, 5, 10, 14, 7, 3]), torch.tensor([5, 10, 14, 9, 12, 8])
    i15, j15 = torch.cat([i15, extra_i]), torch.cat([j15, extra_j])
    return [("B1 N7 E22", make_inputs(ii, jj, 7, ht=48, wd=64, seed=1)),
            ("B1 N7 E24", make_inputs(ii24, jj24, 7, ht=48, wd=64, seed=2)),
            ("B1 N15 E60", make_inputs(i15, j15, 15, ht=48, wd=64, seed=3)),
            ("B4 N7 E22", make_inputs(ii, jj, 7, ht=48, wd=64, B=4, seed=4))]


def calls(c, native):
    dev = "cuda"
    x = {k: c[k].to(dev, torch.float32) for k in ("target", "weight", "eta", "poses", "disps", "intrinsics")}
    for k in ("target", "weight", "eta", "poses", "disps"):
        x[k].requires_grad_(True)
    ii, jj = c["ii"].to(dev), c["jj"].to(dev)
    layer, SE3 = (modules.ba_layer, lt.SE3) if native else (oba.ba, oba.SE3)

    def fwd():
        with torch.no_grad():
            return layer(x["target"], x["weight"], x["eta"], SE3(x["poses"]), x["disps"], x["intrinsics"], ii, jj, fixedp=2)

    def fwd_bwd():
        P, D = layer(x["target"], x["weight"], x["eta"], SE3(x["poses"]), x["disps"], x["intrinsics"], ii, jj, fixedp=2)
        return torch.autograd.grad(P.data.sum() + D.sum(), [x[k] for k in ("target", "weight", "eta", "poses", "disps")])

    return fwd, fwd_bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    info = card()
    print("card: %s, power limit %s, SM clock %s (max %s)" % (info["name"], info["power_limit"], info["sm_clock"], info["max_sm_clock"]))
    rows = []
    for name, c in shapes():
        paths = {p: calls(c, p == "native") for p in ("native", "oracle")}
        res = {}
        for p, (f, fb) in paths.items():
            res[p] = {"fwd syncs": host_syncs(f)[0], "fwd+bwd syncs": host_syncs(fb)[0], "fwd": [], "fwd+bwd": []}
        for _ in range(5):                                  # alternate the two paths window by window
            for p, (f, fb) in paths.items():
                res[p]["fwd"].append(timed(f, args.reps, args.warmup)[0])
                res[p]["fwd+bwd"].append(timed(fb, args.reps, args.warmup)[0])
        row = {"shape": name}
        for p in paths:
            for k in ("fwd", "fwd+bwd"):
                row["%s %s ms" % (p, k)] = statistics.median(res[p][k])
            row["%s syncs fwd/fwd+bwd" % p] = "%d/%d" % (res[p]["fwd syncs"], res[p]["fwd+bwd syncs"])
        rows.append(row)
        print("%-11s native fwd %.3f ms  fwd+bwd %.3f ms  syncs %s | oracle flow fwd %.3f ms  fwd+bwd %.3f ms  syncs %s | speed-up %.1fx / %.1fx" % (
            name, row["native fwd ms"], row["native fwd+bwd ms"], row["native syncs fwd/fwd+bwd"], row["oracle fwd ms"],
            row["oracle fwd+bwd ms"], row["oracle syncs fwd/fwd+bwd"], row["oracle fwd ms"] / row["native fwd ms"],
            row["oracle fwd+bwd ms"] / row["native fwd+bwd ms"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
