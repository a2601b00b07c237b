"""Time CorrBlock's pyramid build and lookup at the image sizes the reference's scripts produce (1/8-resolution feature maps), native
against the reference's call sequence on the GPU.

    python tools/bench_corr_sizes.py [--reps 5] [--edges 32 128] [--out result.json]

Sizes: TUM 240x320 -> 30x40, ETH3D 739x458 (area-preserving resize) -> 43x70, raw EuRoC 752x480 -> 44x69, 16:9 video 1280x720 -> 41x73,
bench config c5 -> 72x96, and 48x64 (TartanAir 384x512) as the control that runs on the wd = 64 kernel.  f16 feature maps, 128 channels.
  build:  corr_volume_pyramid (one launch; plus the staging copy when wd % 8 != 0) against torch.matmul of the /4-scaled maps +
          3x avg_pool2d (CorrBlock.__init__).  Reported as achieved GB/s over the 1.33 * HW^2 * 2 bytes of volume per edge.
  lookup: corr_lookup_pyramid (one launch, reference layout) against 4x corr_index_forward + cat (CorrBlock.__call__).
Each call timed on its own, the two paths alternating, median of --reps rounds.  The volumes are compared (max |diff| against the
cuBLAS pipeline, 6e-2 in f16) and the lookups with torch.equal in the same run.  The first line describes the card."""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import droid_slam_b200  # noqa: E402
from util import card, timed  # noqa: E402

be = droid_slam_b200.install()
dev = "cuda"
C = 128
SIZES = [("tum", 30, 40), ("eth3d", 43, 70), ("euroc_raw", 44, 69), ("video_16x9", 41, 73), ("c5", 72, 96), ("control_48x64", 48, 64)]


def ref_build(f, ii, jj):
    E, ht, wd = ii.shape[0], f.shape[2], f.shape[3]
    corr = torch.matmul((f[ii].reshape(E, C, -1) / 4.0).transpose(1, 2), f[jj].reshape(E, C, -1) / 4.0).reshape(E * ht * wd, 1, ht, wd)
    pyr = []
    for l in range(4):
        pyr.append(corr.view(E, ht, wd, ht >> l, wd >> l))
        corr = F.avg_pool2d(corr, 2, stride=2)
    return pyr


def ref_lookup(pyr, coords):
    E, _, ht, wd = coords.shape
    return torch.cat([be.corr_index_forward(pyr[l], coords / 2 ** l, 3)[0].view(E, 49, ht, wd) for l in range(4)], dim=1)


def run(name, ht, wd, E, reps, g):
    N = max(8, E // 4)
    f = torch.randn(N, C, ht, wd, generator=g).half().to(dev)
    ii = torch.randint(0, N, (E,), generator=g).to(dev)
    jj = torch.randint(0, N, (E,), generator=g).to(dev)
    coords = torch.stack([torch.rand(E, ht, wd, generator=g) * (wd + 8) - 4, torch.rand(E, ht, wd, generator=g) * (ht + 8) - 4], dim=1).contiguous().to(dev)
    nat = lambda: be.corr_volume_pyramid(f, f, ii, jj)
    ref = lambda: ref_build(f, ii, jj)
    for fn in (nat, ref):                                               # warm-up: module loads, cuBLAS algorithm choice
        fn()
    torch.cuda.synchronize()
    tb_n, tb_r = [], []
    for _ in range(reps):
        tb_n.append(timed(nat)[0])
        tb_r.append(timed(ref)[0])
    pyr, rpyr = nat(), ref()
    err = 0.0
    for l in range(4):
        for e0 in range(0, E, 8):
            err = max(err, float((pyr[l][e0:e0 + 8].float() - rpyr[l][e0:e0 + 8].float()).abs().max()))
    del rpyr
    torch.cuda.empty_cache()
    lk_n = lambda: be.corr_lookup_pyramid(pyr, coords, False)
    lk_r = lambda: ref_lookup(pyr, coords)
    lk_n(); lk_r()
    tl_n, tl_r = [], []
    for _ in range(reps):
        t, _, a = timed(lk_n); tl_n.append(t)
        t, _, b = timed(lk_r); tl_r.append(t)
    same = bool(torch.equal(a, b))
    HW = ht * wd
    vol_bytes = E * HW * HW * 2 * (1 + 1 / 4 + 1 / 16 + 1 / 64)
    bn, br, ln, lr = (statistics.median(x) for x in (tb_n, tb_r, tl_n, tl_r))
    res = {"size": name, "ht": ht, "wd": wd, "edges": E,
           "build_native_ms": bn, "build_reference_ms": br, "build_speedup": br / bn,
           "build_native_GBps": vol_bytes / bn / 1e6, "build_reference_GBps": vol_bytes / br / 1e6,
           "staging_bytes": be_staging_bytes(N, ht, wd), "volume_bytes": vol_bytes,
           "build_max_abs_diff_vs_cublas": err, "build_within_tolerance": err < 6e-2,
           "lookup_native_ms": ln, "lookup_reference_ms": lr, "lookup_speedup": lr / ln, "lookup_bit_identical": same}
    del pyr, f
    torch.cuda.empty_cache()
    return res


def be_staging_bytes(n_frames, ht, wd):
    from droid_slam_b200 import c_api
    return int(c_api.load().dba_corr_volume_workspace_bytes(n_frames, n_frames, C, ht, wd))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--edges", type=int, nargs="+", default=[32, 128])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    g = torch.Generator().manual_seed(0)
    lines = [card()]
    print(json.dumps(lines[0]), flush=True)
    for name, ht, wd in SIZES:
        for E in args.edges:
            r = run(name, ht, wd, E, args.reps, g)
            lines.append(r)
            print(json.dumps(r), flush=True)
    lines[0]["sm_clock_at_end"] = card()["sm_clock"]
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
