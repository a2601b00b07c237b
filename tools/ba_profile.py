"""Where the time of one native BA call goes, stage by stage and kernel by kernel.

For each config (synth.CONFIGS: metric, c3_global, c4_stereo) the scene bench.py builds is run through the C ABI:
  1. CUDA events around `dba_ba_prepare` (once per call) and around each Gauss-Newton iteration's `dba_ba_build` and `dba_ba_solve`,
     averaged over --reps calls of the config's iterations (poses and inverse depths are restored between calls, outside the events);
  2. in a separate run, torch.profiler with CUDA activities over --prof-reps calls: every kernel and memset with its time per
     Gauss-Newton iteration, written to OUT/<config>.txt when --out is given.

usage: python tools/ba_profile.py [--config metric c3_global c4_stereo] [--reps 50] [--prof-reps 20] [--out DIR]"""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
from droid_slam_b200 import c_api, synth  # noqa: E402
from util import card  # noqa: E402

dev = "cuda"


class Call:
    """one BA call of a config's scene, driven stage by stage through the C ABI"""

    def __init__(self, L, cfg):
        s = synth.make_scene(cfg)
        self.L, self.itrs = L, s["itrs"]
        g = lambda k: s[k].to(dev).contiguous()
        self.p0, self.d0 = g("poses"), g("disps")
        self.poses, self.disps = self.p0.clone(), self.d0.clone()
        self.keep = [g(k) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
        intr, ds, tg, wt, eta, ii, jj = self.keep
        N, ht, wd = self.disps.shape
        E = ii.shape[0]
        t0, t1 = s["t0"], s["t1"]
        M = s["M"]
        ws_bytes = L.dba_ba_workspace_bytes(N, E, ht, wd, t0, t1)
        self.ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        self.dx = torch.zeros(max(t1 - t0, 1), 6, device=dev)
        self.dz = torch.zeros(M, ht * wd, device=dev)
        self.a = c_api.ba_args(self.poses, self.disps, intr, ds, tg, wt, eta, ii, jj, t0, t1, s["lm"], s["ep"], self.dx, self.dz, self.ws,
                               torch.cuda.current_stream().cuda_stream)
        self.shape = "E=%d N=%d %dx%d, %d depth frames, window [%d, %d), %d Gauss-Newton iterations" % (E, N, ht, wd, M, t0, t1, self.itrs)

    def stage(self, fn):
        c_api.check(getattr(self.L, fn)(ctypes.byref(self.a)), fn)

    def restore(self):
        self.poses.copy_(self.p0)
        self.disps.copy_(self.d0)

    def run(self, ev=None):
        """prepare + itrs x (build, solve); ev: list of 2 itrs + 2 events recorded at each stage boundary"""
        rec = (lambda k: ev[k].record()) if ev else (lambda k: None)
        rec(0)
        self.stage("dba_ba_prepare")
        rec(1)
        for it in range(self.itrs):
            self.stage("dba_ba_build")
            rec(2 + 2 * it)
            self.stage("dba_ba_solve")
            rec(3 + 2 * it)


def stage_times(call, reps):
    """ms per call of prepare, and per Gauss-Newton iteration of build and solve (CUDA events, mean over reps calls)"""
    n_ev = 2 + 2 * call.itrs
    tot = dict(prepare=0.0, build=0.0, solve=0.0)
    for _ in range(3):
        call.run()
        call.restore()
    for _ in range(reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(n_ev)]
        call.run(ev)
        torch.cuda.synchronize()
        tot["prepare"] += ev[0].elapsed_time(ev[1])
        for it in range(call.itrs):
            tot["build"] += ev[1 + 2 * it].elapsed_time(ev[2 + 2 * it]) / call.itrs
            tot["solve"] += ev[2 + 2 * it].elapsed_time(ev[3 + 2 * it]) / call.itrs
        call.restore()
    return {k: v / reps for k, v in tot.items()}


def kernel_table(call, reps):
    """[(name, launches per iteration, us per iteration)] of every CUDA kernel and memset over reps calls, slowest first"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        call.run()
        call.restore()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call.run()
        torch.cuda.synchronize()
    call.restore()
    per_iter = reps * call.itrs
    rows = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        n, us = rows.get(name, (0, 0.0))
        rows[name] = (n + 1, us + e.device_time)
    return sorted(((k, n / per_iter, us / per_iter) for k, (n, us) in rows.items()), key=lambda r: -r[2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+", default=["metric", "c3_global", "c4_stereo"], choices=sorted(synth.CONFIGS))
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--prof-reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for the per-kernel tables (<config>.txt)")
    args = ap.parse_args()
    L = c_api.load()
    gpu = card()
    print("card:", gpu)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    for cfg in args.config:
        call = Call(L, cfg)
        t = stage_times(call, args.reps)
        print("%s (%s)" % (cfg, call.shape))
        print("  stages (CUDA events, mean of %d calls): prepare %.1f us per call; per iteration build %.1f us, solve %.1f us"
              % (args.reps, 1e3 * t["prepare"], 1e3 * t["build"], 1e3 * t["solve"]))
        rows = kernel_table(call, args.prof_reps)
        lines = ["%s (%s)" % (cfg, call.shape), "card: %s" % gpu,
                 "torch.profiler, %d calls; per Gauss-Newton iteration (prepare counted over the iterations of its call):" % args.prof_reps,
                 "  %10s %9s  %s" % ("us/iter", "launches", "kernel")]
        lines += ["  %10.2f %9.2f  %s" % (us, n, name[:150]) for name, n, us in rows]
        lines.append("  %10.2f %9s  total" % (sum(r[2] for r in rows), ""))
        print("\n".join(lines[2:]))
        if args.out:
            with open(os.path.join(args.out, cfg + ".txt"), "w") as f:
                f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
