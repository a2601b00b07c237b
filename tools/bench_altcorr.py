"""Time AltCorrBlock (modules/corr.py:89-117) on the GPU: the reference's call sequence on the drop-in ops (3x avg_pool2d for the pyramid;
per call 4x altcorr_forward + flatten + stack) against install_alt_corr_hook's path (altcorr_pyramid + altcorr_lookup_pyramid).

    python tools/bench_altcorr.py [--reps 5] [--out result.json]

Workloads (f16 feature maps, 128 channels):
  update_lowmem_c3   one FactorGraph.update_lowmem step's lookups on the c3 graph (synth "c3_global": 2048 edges, 400 frames, 48x64),
                     issued in chunks of 8 source frames in update_lowmem's order (factor_graph.py:284-296)
  single_512_48x64   one 512-edge call, 72 frames
  single_512_72x96   one 512-edge call at c5's image size, 128 frames
The pyramid build (AltCorrBlock.__init__ over all frames) and the lookups (__call__) are timed separately, the two paths alternating,
median of --reps rounds.  Outputs of both paths are compared with torch.equal in the same run.
MACs = 4 levels x HW x 64 taps x C per edge.  Compulsory bytes per edge = source level-0 map + target maps of all levels + coords +
output (the 0.79 MB per map at 48x64 of SURVEY section 8d; frames shared between edges are counted once per edge).
Prints a header line naming the card, then one JSON line per workload."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import droid_slam_b200  # noqa: E402
from droid_slam_b200 import synth  # noqa: E402
from droid_slam_b200.modules import install_alt_corr_hook  # noqa: E402
from util import card, timed  # noqa: E402

be = droid_slam_b200.install()
dev = "cuda"
LEVELS, C = 4, 128


def ref_pyramid(fmaps):
    """AltCorrBlock.__init__ of the reference: level l = avg_pool2d applied l times, viewed [B,N,C,H>>l,W>>l]"""
    B, N, Cc, H, W = fmaps.shape
    f = fmaps.view(B * N, Cc, H, W)
    pyr = []
    for l in range(LEVELS):
        pyr.append(f.view(B, N, Cc, H >> l, W >> l))
        f = F.avg_pool2d(f, 2, stride=2)
    return pyr


def ref_lookup(pyr, coords, ii, jj):
    """AltCorrBlock.__call__ of the reference: coords [B,M,H,W,2]"""
    c = coords.permute(0, 1, 4, 2, 3).contiguous()
    outs = [be.altcorr_forward(pyr[0], pyr[l], c / 2 ** l, ii, jj, 3)[0].flatten(2, 3) for l in range(LEVELS)]
    return torch.stack(outs, dim=2).flatten(2, 3)


class _Stub:
    def __init__(self, *a, **k):
        raise AssertionError("replaced by the hook")

    def __call__(self, *a):
        raise AssertionError("replaced by the hook")


Hooked = install_alt_corr_hook(type("m", (), {"AltCorrBlock": type("AltCorrBlock", (_Stub,), {})})).AltCorrBlock


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def workload(name, n_frames, ht, wd, ii, jj, coords, chunks, reps):
    """coords [1,E,ht,wd,2] f32; chunks: list of edge-index tensors, one lookup call each"""
    g = torch.Generator().manual_seed(0)
    fmaps = torch.randn(1, n_frames, C, ht, wd, generator=g).half().to(dev)
    calls = [(coords[:, v].contiguous(), ii[v].contiguous(), jj[v].contiguous()) for v in chunks]
    E = sum(int(c[1].numel()) for c in calls)
    with torch.no_grad():
        ref_pyr, blk = ref_pyramid(fmaps), Hooked(fmaps)
        equal = all(torch.equal(ref_lookup(ref_pyr, *a), blk(*a)) for a in calls)
        t = {"ref_pyramid": [], "hook_pyramid": [], "ref_lookup": [], "hook_lookup": []}
        for _ in range(reps):   # alternate the two paths so that drift on a shared host hits both
            t["ref_pyramid"].append(timed(lambda: ref_pyramid(fmaps), calls=3, warmup=2)[0])
            t["hook_pyramid"].append(timed(lambda: Hooked(fmaps), calls=3, warmup=2)[0])
            t["ref_lookup"].append(timed(lambda: [ref_lookup(ref_pyr, *a) for a in calls], calls=3, warmup=1)[0])
            t["hook_lookup"].append(timed(lambda: [blk(*a) for a in calls], calls=3, warmup=1)[0])
    t = {k: median(v) for k, v in t.items()}
    HW = ht * wd
    macs = E * LEVELS * HW * 64 * C
    lvl_px = sum((ht >> l) * (wd >> l) for l in range(LEVELS))
    byts = E * (HW * C * 2 + lvl_px * C * 2 + HW * 2 * 4 + LEVELS * 49 * HW * 2)
    res = {"workload": name, "frames": n_frames, "edges": E, "calls": len(calls), "ht": ht, "wd": wd, "equal": bool(equal)}
    for k, v in t.items():
        res[k + "_ms"] = round(v, 4)
    res["ref_total_ms"] = round(t["ref_pyramid"] + t["ref_lookup"], 4)
    res["hook_total_ms"] = round(t["hook_pyramid"] + t["hook_lookup"], 4)
    res["lookup_speedup"] = round(t["ref_lookup"] / t["hook_lookup"], 3)
    res["pyramid_speedup"] = round(t["ref_pyramid"] / t["hook_pyramid"], 3)
    res["total_speedup"] = round(res["ref_total_ms"] / res["hook_total_ms"], 3)
    res["lookup_GMAC"] = round(macs / 1e9, 2)
    res["ref_lookup_GMACps"] = round(macs / t["ref_lookup"] / 1e6, 1)
    res["hook_lookup_GMACps"] = round(macs / t["hook_lookup"] / 1e6, 1)
    res["compulsory_MB"] = round(byts / 1e6, 1)
    res["hook_lookup_compulsory_GBps"] = round(byts / t["hook_lookup"] / 1e6, 1)
    del fmaps, ref_pyr, blk, calls
    torch.cuda.empty_cache()
    return res


def lowmem_chunks(ii, jj, s=8):
    """the edge sets of update_lowmem's inner loop: source frames [i, i+8) from ii.min() to jj.max()"""
    out = []
    for i in range(int(ii.min()), int(jj.max()) + 1, s):
        v = ((ii >= i) & (ii < i + s)).nonzero().flatten()
        if v.numel():
            out.append(v.to(dev))
    return out


def random_graph(n_frames, E, ht, wd, seed):
    g = torch.Generator().manual_seed(seed)
    ii = torch.randint(0, n_frames, (E,), generator=g)
    jj = (ii + torch.randint(1, 6, (E,), generator=g)) % n_frames
    ys, xs = torch.meshgrid(torch.arange(ht, dtype=torch.float32), torch.arange(wd, dtype=torch.float32), indexing="ij")
    coords = torch.stack([xs, ys], -1)[None, None] + 3 * torch.randn(1, E, ht, wd, 2, generator=g)
    return ii.to(dev), jj.to(dev), coords.to(dev)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_altcorr needs a CUDA device")
    lines = [dict(card(), torch=torch.__version__)]
    s = synth.make_scene("c3_global")
    ii, jj = s["ii"].to(dev), s["jj"].to(dev)
    g = torch.Generator().manual_seed(1)
    coords = (s["coords_gt"] + 2 * torch.rand(s["coords_gt"].shape, generator=g) - 1)[None].to(dev)
    lines.append(workload("update_lowmem_c3", s["cfg"]["N"], 48, 64, ii, jj, coords, lowmem_chunks(ii, jj), args.reps))
    for name, n_frames, ht, wd in (("single_512_48x64", 72, 48, 64), ("single_512_72x96", 128, 72, 96)):
        ii, jj, coords = random_graph(n_frames, 512, ht, wd, seed=ht)
        lines.append(workload(name, n_frames, ht, wd, ii, jj, coords, [torch.arange(512, device=dev)], args.reps))
    text = "\n".join(json.dumps(l) for l in lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
