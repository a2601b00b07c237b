"""Time droid_slam_b200.lietorch (csrc/lie.cu) against the same calls on the pure-PyTorch stand-in (oracle/shims/lietorch), both on the GPU,
the two alternating, with the card's name, power limit and clocks printed beside the numbers.

    python tools/bench_lietorch.py --reps 20 --warmup 3 [--json out.json]

Workloads, fp32: act4 forward and backward of Gij [1,E,1,1] on homogeneous points [1,E,48,64,4] (projective_transform's reprojection,
E = 512 and 2048); adjT forward and backward of Gij [1,E,1,1,1] on its Jacobians [1,E,48,64,2,6]; SE3(poses).inv() and .log() on buffers
of 512 and 4096 poses.  CUDA events around `--reps` calls after `--warmup`, the median of 5 such windows.  GB/s on algorithmic bytes:
each operand read once, each result written once (a forward reads the group elements and points, writes the result; a backward also
reads the upstream gradient and writes both gradients), nothing for broadcast copies; the share of the H100 SXM data sheet's 3.35 TB/s.
The stand-in expands the group elements to the points' batch (lietorch's kernels do the same with a copy); its backward is autograd.
A fwd+bwd call also includes autograd's own work: the ones_like upstream gradient and the graph; the operands are leaf tensors made once.
The reference's own lietorch cannot be built without its Eigen submodule, so it is not measured here."""
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
from oracle.lie_grad import shim  # noqa: E402
from util import card, timed  # noqa: E402

HBM = 3.35e12


def workloads(dev):
    g = torch.Generator(device=dev).manual_seed(0)
    ht, wd = 48, 64
    out = []
    for E in (512, 2048):
        G = 0.3 * torch.randn(1, E, 6, generator=g, device=dev)
        data = shim.SE3.exp(G).data
        p = torch.randn(1, E, ht, wd, 4, generator=g, device=dev)
        J = torch.randn(1, E, ht, wd, 2, 6, generator=g, device=dev)
        n = E * ht * wd
        out.append(("act4 fwd E=%d" % E, "act4", False, data[:, :, None, None], p, 4 * (7 * E + 4 * n + 4 * n)))
        out.append(("act4 fwd+bwd E=%d" % E, "act4", True, data[:, :, None, None], p, 4 * (7 * E + 4 * n + 4 * n) + 4 * (4 * n + 7 * E + 4 * n + 7 * E + 4 * n)))
        out.append(("adjT fwd E=%d" % E, "adjT", False, data[:, :, None, None, None], J, 4 * (7 * E + 24 * n)))
        out.append(("adjT fwd+bwd E=%d" % E, "adjT", True, data[:, :, None, None, None], J, 4 * (7 * E + 24 * n) + 4 * (12 * n + 7 * E + 12 * n + 7 * E + 12 * n)))
    for n in (512, 4096):
        poses = shim.SE3.exp(torch.randn(n, 6, generator=g, device=dev)).data
        out.append(("inv %d poses" % n, "inv", False, poses, None, 4 * 14 * n))
        out.append(("log %d poses" % n, "log", False, poses, None, 4 * 13 * n))
    return out


def call(mod, op, backward, X, b):
    """one call of op on module `mod` (the package or the stand-in); with backward (X and b leaf tensors requiring grad, made once outside
    the timed calls), the gradients of a sum-of-outputs loss too, into fresh .grad tensors"""
    if backward:
        X.grad = b.grad = None
    G = mod.SE3(X)
    out = {"act4": lambda: G.act(b), "adjT": lambda: G.adjT(b), "inv": lambda: G.inv().data, "log": lambda: G.log()}[op]()
    if backward:
        torch.autograd.backward(out, torch.ones_like(out))
        return X.grad
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lietorch needs a CUDA device")
    dev = "cuda"
    info = card()
    print("card:", info)
    rows = []
    for name, op, backward, X, b, nbytes in workloads(dev):
        if backward:
            X, b = X.clone().requires_grad_(True), b.clone().requires_grad_(True)
        times = {"native": [], "stand-in": []}
        diff = 0.0
        for _ in range(5):
            for tag, mod in (("native", lt), ("stand-in", shim)):
                ms, _, out = timed(lambda: call(mod, op, backward, X, b), calls=args.reps, warmup=args.warmup)
                times[tag].append(ms)
        with torch.no_grad():                                                          # forward values (the gradients use other conventions)
            got, want = call(lt, op, False, X, b), call(shim, op, False, X, b)
        diff = float((got - want).abs().max())
        t_n, t_s = statistics.median(times["native"]), statistics.median(times["stand-in"])
        row = dict(workload=name, native_ms=t_n, standin_ms=t_s, speedup=t_s / t_n, bytes=nbytes, native_GBps=nbytes / t_n / 1e6,
                   native_share_of_hbm=nbytes / t_n / 1e-3 / HBM, max_abs_diff_vs_standin=diff)
        rows.append(row)
        print("%-22s native %8.4f ms  stand-in %8.4f ms  x%6.2f  %7.1f GB/s (%4.1f%% of 3.35 TB/s)  max |diff| %.2e"
              % (name, t_n, t_s, t_s / t_n, row["native_GBps"], 100 * row["native_share_of_hbm"], diff))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=info, rows=rows, reps=args.reps, warmup=args.warmup), f, indent=1)


if __name__ == "__main__":
    main()
