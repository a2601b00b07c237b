"""Time DroidNet's feature / context encoders (BasicEncoder, modules/extractor.py:118-198) on the GPU: the fp32 oracle module under CUDA
autocast (cuDNN convolutions + ATen instance norms, as the reference runs) against the native `encoder_forward` (csrc/encoder.cu).

    python tools/bench_encoder.py [--reps 7] [--out result.json]
    python tools/bench_encoder.py --profile [--trace-dir DIR]     # one torch.profiler run of hooked fnet + cnet at n = 1, 384x512

Workloads, at 384x512 and 352x552: fnet n = 1 and cnet n = 1 (MotionFilter.track, per frame), fnet n = 16 (one PoseTrajectoryFiller
batch); plus native fnet + cnet at n = 1 (384x512) captured as one CUDA graph.  The two paths alternating, median of --reps rounds of
20 calls each after warm-up.  FLOP/s from the shape-derived FLOPs (2 MACs per conv tap, every convolution of the encoder).  Prints a
header line naming the card, then one JSON line per workload."""
import argparse
import json
import os
import statistics
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import droid_slam_b200  # noqa: E402
import oracle.encoder as oenc  # noqa: E402
from droid_slam_b200 import synth  # noqa: E402
from droid_slam_b200.encoder import pack_encoder_weights  # noqa: E402
from util import card, timed  # noqa: E402

be = droid_slam_b200.install()
dev = "cuda"
ENC = {"fnet": ("instance", 128, 1, 0), "cnet": ("none", 256, 0, 1)}   # norm_fn, output_dim, norm code, weight seed


def flops(H, W, output_dim):
    """FLOPs of one image: 2 x MACs of every convolution (stride-2 ones at their output resolution)"""
    f = 2 * 32 * 3 * 49 * (H // 2) * (W // 2)
    for cin, p, h, w in ((32, 32, H // 2, W // 2), (32, 64, H // 4, W // 4), (64, 128, H // 8, W // 8)):
        f += 2 * p * cin * 9 * h * w + 3 * 2 * p * p * 9 * h * w + (2 * p * cin * h * w if cin != p else 0)
    return f + 2 * output_dim * 128 * (H // 8) * (W // 8)


def time_rounds(fns, reps, calls=20):
    """fns: dict name -> callable; alternating rounds, returns median ms per call"""
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            ts[k].append(timed(f, calls)[0])
    return {k: statistics.median(v) for k, v in ts.items()}


def setup(name, n, H, W):
    norm_fn, od, code, seed = ENC[name]
    sd = synth.make_encoder_weights(seed, od)
    mod = oenc.BasicEncoder(od, norm_fn).to(dev).eval()
    mod.load_state_dict(sd)
    sdd = {k: v.to(dev) for k, v in sd.items()}
    pk = pack_encoder_weights(sd, norm_fn, od, dev)
    x = torch.randn(1, n, 3, H, W, device=dev)
    x0 = x[0].contiguous()

    def ref():
        with torch.autocast("cuda", dtype=torch.float16):
            return oenc.encoder_forward(sdd, x, norm_fn)

    def nat():
        return be.encoder_forward(x0, pk, code, od)
    return ref, nat, od


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--trace-dir", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder needs a CUDA device")
    torch.backends.cudnn.benchmark = False
    if a.profile:
        return profile(a.trace_dir)
    rows = []
    with torch.no_grad():
        for H, W in ((384, 512), (352, 552)):
            for name, n in (("fnet", 1), ("cnet", 1), ("fnet", 16)):
                ref, nat, od = setup(name, n, H, W)
                for _ in range(3):
                    ref(); nat()
                torch.cuda.synchronize()
                ms = time_rounds({"reference_autocast": ref, "native": nat}, a.reps)
                fl = flops(H, W, od) * n
                rows.append({"workload": "%s_n%d_%dx%d" % (name, n, H, W), "gflop": fl / 1e9, "reference_ms": ms["reference_autocast"],
                             "native_ms": ms["native"], "speedup": ms["reference_autocast"] / ms["native"],
                             "native_tflops": fl / ms["native"] / 1e9, "reference_tflops": fl / ms["reference_autocast"] / 1e9})
        # fnet + cnet at n = 1 as one CUDA graph against the same two native calls issued eagerly
        rf, nf, _ = setup("fnet", 1, 384, 512)
        rc, nc, _ = setup("cnet", 1, 384, 512)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            nf(); nc()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            nf(); nc()
        for _ in range(3):
            g.replay(); rf(); rc()
        torch.cuda.synchronize()
        ms = time_rounds({"reference_autocast": lambda: (rf(), rc()), "native_eager": lambda: (nf(), nc()), "native_graph": g.replay}, a.reps)
        fl = flops(384, 512, 128) + flops(384, 512, 256)
        rows.append({"workload": "fnet+cnet_n1_384x512_graph", "gflop": fl / 1e9, "reference_ms": ms["reference_autocast"], "native_ms": ms["native_graph"],
                     "native_eager_ms": ms["native_eager"], "speedup": ms["reference_autocast"] / ms["native_graph"],
                     "native_tflops": fl / ms["native_graph"] / 1e9, "reference_tflops": fl / ms["reference_autocast"] / 1e9})
    head = card()
    print(json.dumps(head))
    for r in rows:
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": head, "rows": rows}, f, indent=1)


def profile(trace_dir):
    """torch.profiler of hooked fnet + cnet (the stand-in module with install_encoder_hook, under autocast, as MotionFilter calls them)"""
    from torch.profiler import ProfilerActivity, profile as tprofile
    from droid_slam_b200.modules import install_encoder_hook
    ns = types.SimpleNamespace(BasicEncoder=type("BasicEncoder", (oenc.BasicEncoder,), {}))
    install_encoder_hook(ns)
    fnet = ns.BasicEncoder(128, "instance").to(dev).eval()
    fnet.load_state_dict(synth.make_encoder_weights(0, 128))
    cnet = ns.BasicEncoder(256, "none").to(dev).eval()
    cnet.load_state_dict(synth.make_encoder_weights(1, 256))
    x = torch.randn(1, 1, 3, 384, 512, device=dev)
    with torch.no_grad(), torch.autocast("cuda", enabled=True):
        for _ in range(3):
            fnet(x); cnet(x)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                fnet(x); cnet(x)
            torch.cuda.synchronize()
    print(json.dumps(card()))
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
    names = [e.key for e in prof.key_averages()]
    bad = [k for k in names if "cudnn" in k.lower() or k == "aten::convolution" or k == "aten::cudnn_convolution"]
    print("cuDNN / aten::convolution entries:", bad if bad else "none")
    if trace_dir:
        os.makedirs(trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(trace_dir, "encoder_trace.json"))


if __name__ == "__main__":
    main()
