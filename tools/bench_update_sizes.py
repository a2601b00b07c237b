"""Update operator (UpdateModule, csrc/update_op.cu) at the feature-map sizes the reference's scripts produce, against the reference
formula (oracle/update.py, pinned against the reference's UpdateModule) through torch/cuDNN under fp16 autocast, as
bench.py:reference_update_operator_ms times it.

  43x70  ETH3D through evaluation_scripts/test_eth3d.py        44x69  raw EuRoC through demo.py      41x73  16:9 video through demo.py
  48x64, 30x40, 72x96: widths that are multiples of 8 (rectangular tiles), as controls

512 edges over 72 source frames, with flow and aggregation.  The two paths alternating, the median of --rounds rounds of --iters
calls.  TFLOP/s counts the useful FLOPs (SURVEY section 8d): 14.03 GFLOP per edge and 1.37 GFLOP per source frame at 48x64, scaled by
HW / 3072.  Prints the card, then one JSON line per size, then the card again.

  python tools/bench_update_sizes.py [--sizes 43x70,44x69] [--edges 512] [--frames 72] [--rounds 7] [--iters 5]
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
from util import card, timed  # noqa: E402

SIZES = "43x70,44x69,41x73,48x64,30x40,72x96"
GFLOP_EDGE, GFLOP_FRAME = 14.03, 1.37


def run_size(ht, wd, E, frames, rounds, iters, dev):
    import oracle
    from droid_slam_b200 import synth
    from droid_slam_b200.update import UpdateModule
    w = synth.make_update_weights(0)
    wd_dev = {k: v.to(dev) for k, v in w.items()}
    mod = UpdateModule().to(dev)
    mod.load_state_dict(w)
    g = torch.Generator(device=dev).manual_seed(7)
    net = torch.tanh(torch.randn(1, E, 128, ht, wd, generator=g, device=dev)).half()
    inp = torch.relu(torch.randn(1, E, 128, ht, wd, generator=g, device=dev)).half()
    corr = torch.randn(1, E, 196, ht, wd, generator=g, device=dev).half()
    flow = torch.randn(1, E, 4, ht, wd, generator=g, device=dev)
    ii = torch.arange(E, device=dev) % frames
    with torch.no_grad():
        native = lambda: mod(net, inp, corr, flow, ii)

        def reference():
            with torch.autocast("cuda", dtype=torch.float16):
                return oracle.update_module_forward(wd_dev, net, inp, corr, flow, ii)

        got, ref = native(), reference()
        diff = {k: float((a.float() - b.float()).abs().max()) for k, a, b in zip(("net", "delta", "weight", "eta", "upmask"), got, ref)}
        del got, ref
        for _ in range(2):
            native(); reference()
        t_nat, t_ref = [], []
        for _ in range(rounds):
            t_nat.append(timed(native, iters)[0])
            t_ref.append(timed(reference, iters)[0])
    n_src = min(E, frames)
    gflop = (GFLOP_EDGE * E + GFLOP_FRAME * n_src) * ht * wd / 3072.0
    ms_n, ms_r = statistics.median(t_nat), statistics.median(t_ref)
    return {"size": "%dx%d" % (ht, wd), "wd_mod_8": wd % 8, "edges": E, "source_frames": n_src, "useful_gflop": round(gflop, 1),
            "native_ms": round(ms_n, 3), "native_tflops": round(gflop / ms_n, 1), "reference_ms": round(ms_r, 3),
            "reference_tflops": round(gflop / ms_r, 1), "speedup": round(ms_r / ms_n, 2),
            "native_ms_rounds": [round(t, 3) for t in t_nat], "max_abs_diff_vs_reference": diff}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--sizes", default=SIZES)
    ap.add_argument("--edges", type=int, default=512)
    ap.add_argument("--frames", type=int, default=72)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_update_sizes.py needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.backends.cudnn.benchmark = True
    print(json.dumps({"card": card()}), flush=True)
    for s in args.sizes.split(","):
        ht, wd = (int(v) for v in s.lower().split("x"))
        print(json.dumps(run_size(ht, wd, args.edges, args.frames, args.rounds, args.iters, dev)), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
