"""Time training's flow loss and upsample_disp (droid_slam_b200.modules.flow_loss / upsample_disp, csrc/geom.cu) against the reference's
flow restated by the oracle (oracle/flow_loss.py, oracle/upsample.py: the same torch ops as geom/losses.py and droid_net.py), both on the
same GPU, the two alternating, with the card's name, power limit and clocks read in the same run.

    python tools/bench_flow_loss.py --rounds 5 [--json out.json]

Shapes: train.py's defaults -- B = 1, N = 7 frames of 384 x 512 (12 chain edges), 15 iterates; upsample_disp of 7 frames of 48 x 64 with
their 576-channel masks, 15 calls.  Legs: the flow loss forward (under grad mode, as training calls it), the flow loss forward + backward,
and 15 upsample_disp forward + backward (a loss on every output).  Each figure is the CUDA-event median over the rounds; peak memory is
torch.cuda.max_memory_allocated over one call above what was allocated before it; host synchronisations of one call are counted with
tests/util.host_syncs.  The oracle's reprojection also forms the Jacobians the loss does not use, so its time and memory overstate the
reference's flow loss (not its upsample_disp)."""
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
from droid_slam_b200 import lietorch as lt  # noqa: E402
from flow_loss_cases import make_case, upsample_case  # noqa: E402
from oracle import ba_layer as oba, flow_loss as ofl, upsample as oup  # noqa: E402
from util import card, host_syncs  # noqa: E402

ITERS = 15


def flow_inputs():
    c = make_case(B=1, N=7, ht=384, wd=512, n=ITERS, seed=5)
    f = lambda t: t.cuda().float()  # noqa: E731
    return dict(Ps=f(c["Ps"]), disps=f(c["disps"]), intr=f(c["intrinsics"]), poses=[f(p).requires_grad_(True) for p in c["poses_est"]],
                d=[f(x).requires_grad_(True) for x in c["disps_est"]])


def flow(x, native, backward):
    if native:
        loss, metrics = modules.flow_loss(lt.SE3(x["Ps"]), x["disps"], [lt.SE3(p) for p in x["poses"]], x["d"], x["intr"], None)
    else:
        loss, epe, v = ofl.flow_loss(oba.SE3(x["Ps"]), x["disps"], [oba.SE3(p) for p in x["poses"]], x["d"], x["intr"])
        metrics = ofl.metrics(epe.detach(), v)
    if backward:
        torch.autograd.grad(loss, x["d"] + x["poses"])
    return metrics


def up_inputs():
    cs = [upsample_case(B=1, N=7, ht=48, wd=64, seed=40 + i) for i in range(ITERS)]
    return [(c["disp"].cuda().float().requires_grad_(True), c["mask"].cuda().float().requires_grad_(True), c["cot"].cuda().float()) for c in cs]


def upsample(xs, native):
    up = modules.upsample_disp if native else oup.upsample_disp
    outs = [up(d, m) for d, m, _ in xs]
    loss = sum((o * cot).sum() for o, (_, _, cot) in zip(outs, xs))
    torch.autograd.grad(loss, [t for d, m, _ in xs for t in (d, m)])


def measure(fn):
    """(CUDA-event ms, peak bytes above the start) of one call"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    fx, ux = flow_inputs(), up_inputs()
    legs = {"flow_loss_forward": lambda nat: flow(fx, nat, False), "flow_loss_forward_backward": lambda nat: flow(fx, nat, True),
            "upsample_disp_x15_forward_backward": lambda nat: upsample(ux, nat)}
    out = {"card": card(), "shape": "B=1 N=7 384x512, %d iterates; upsample 7 x 48x64 x %d calls" % (ITERS, ITERS), "legs": {}}
    for leg, fn in legs.items():
        for nat in (True, False):
            fn(nat)                                                  # warm up
        t = {True: [], False: []}
        mem = {}
        for _ in range(args.rounds):
            for nat in (True, False):
                ms, peak = measure(lambda: fn(nat))
                t[nat].append(ms)
                mem[nat] = peak
        syncs = {nat: host_syncs(lambda: fn(nat))[0] for nat in (True, False)}
        out["legs"][leg] = {"native_ms": statistics.median(t[True]), "oracle_ms": statistics.median(t[False]),
                            "native_peak_MB": mem[True] / 2 ** 20, "oracle_peak_MB": mem[False] / 2 ** 20,
                            "native_host_syncs": syncs[True], "oracle_host_syncs": syncs[False]}
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
