"""Time the update operator's ConvGRU (droid_slam_b200.modules.conv_gru, csrc/gru_train.cu) against the reference's op sequence
(oracle/update.py conv_gru_forward: the same torch ops as modules/gru.py) on the same GPU, the legs alternating, with the card's name,
power limit and clocks read in the same run.

    python tools/bench_conv_gru.py --rounds 5 [--json out.json]

Workload: what one train.py step asks of the ConvGRU at its defaults -- 15 chained calls (net fed back, fresh inputs per call, as
DroidNet.forward's update iterations) and one backward through all of them, at 22 and 24 edges of 48 x 64.  Legs: native; the
reference's ops with torch's defaults (cuDNN may run its convolutions in single-pass TF32); the reference's ops under
torch.backends.cudnn.flags(allow_tf32=False), the precision class of the native path.  Each time is the CUDA-event median over the
rounds after one warm-up round; peak memory is torch.cuda.max_memory_allocated over one step above what was allocated before it;
host synchronisations of one step are counted with tests/util.host_syncs.  TFLOP/s: the multiply-adds of the layer shapes (both 3x3
convolutions and the 1x1 w forward; their data and weight gradients and the recomputed w backward; 2 FLOP each) over the step's time."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from conv_gru_cases import ConvGRU, load_params, make_cotangent, make_inputs, make_params  # noqa: E402
from droid_slam_b200 import modules  # noqa: E402
from oracle.update import conv_gru_forward  # noqa: E402
from util import card, host_syncs  # noqa: E402

CALLS = 15
HT, WD = 48, 64
LEGS = ("native", "reference_default", "reference_no_tf32")
CEILING = 495.0 / 3           # 3xTF32's effective rate on the H100 SXM's dense TF32 data-sheet figure, TFLOP/s


def step_flops(b):
    """FLOPs of one step (CALLS calls forward and backward) from the layer shapes"""
    px = b * HT * WD
    f3 = 2.0 * px * (256 + 128) * 448 * 9          # convz + convr (one GEMM), convq
    f1 = 2.0 * px * 128 * 128                      # w
    return CALLS * (3 * f3 + 4 * f1)               # forward, data gradient, weight gradient; w once more recomputed in the backward


def inputs(b):
    params = make_params(1)
    net, _ = make_inputs(b, HT, WD, 2)
    f = lambda t: t.cuda().float()  # noqa: E731
    ins = [[f(t).requires_grad_(True) for t in make_inputs(b, HT, WD, 10 + k)[1]] for k in range(CALLS)]
    cot = f(make_cotangent(b, HT, WD, 3))
    m = load_params(ConvGRU().cuda(), params)
    return dict(m=m, net=f(net).requires_grad_(True), ins=ins, cot=cot)


def step(x, leg):
    m = x["m"]
    params = dict(m.named_parameters())
    if leg == "native":
        fwd = lambda h, *i: modules.conv_gru(m, h, *i)  # noqa: E731
    else:
        fwd = lambda h, *i: conv_gru_forward(params, h, *i, prefix="")  # noqa: E731
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=(leg != "reference_no_tf32")):
        h = x["net"]
        for call in x["ins"]:
            h = fwd(h, *call)
        return torch.autograd.grad(h, [x["net"]] + [t for c in x["ins"] for t in c] + list(params.values()), x["cot"])


def measure(b, rounds):
    x = inputs(b)
    times = {leg: [] for leg in LEGS}
    peak, syncs = {}, {}
    for leg in LEGS:                      # warm-up round: modules load, cuDNN picks its algorithms
        step(x, leg)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        syncs[leg], _ = host_syncs(lambda: step(x, leg))
        torch.cuda.synchronize()
        peak[leg] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    for _ in range(rounds):
        for leg in LEGS:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            step(x, leg)
            e.record()
            torch.cuda.synchronize()
            times[leg].append(s.elapsed_time(e))
    flops = step_flops(b)
    out = {}
    for leg in LEGS:
        ms = statistics.median(times[leg])
        out[leg] = dict(ms=ms, peak_mib=peak[leg], host_syncs=syncs[leg], tflops=flops / ms / 1e9)
    out["native"]["share_of_3xtf32_ceiling"] = out["native"]["tflops"] / CEILING
    return dict(edges=b, ht=HT, wd=WD, calls=CALLS, step_gflop=flops / 1e9, legs=out)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_gru needs a CUDA device")
    res = dict(card=card(), results=[measure(b, a.rounds) for b in (22, 24)])
    for r in res["results"]:
        for leg, v in r["legs"].items():
            print("%2d edges %-18s %8.2f ms  %8.1f MiB peak  %d host syncs  %6.1f TFLOP/s" % (r["edges"], leg, v["ms"], v["peak_mib"],
                                                                                          v["host_syncs"], v["tflops"]))
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
