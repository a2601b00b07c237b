"""Distribution of the elementwise deviation between this build's ba and the reference build's ba (oracle/_ref) on the same GPU,
and of both against the fp64 CPU oracle where that is affordable; prints quantiles of each."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
import torch
import droid_slam_b200
from droid_slam_b200 import synth
import oracle
import droid_backends_ref as ref

be = droid_slam_b200.install()
dev = "cuda"


def q(x):
    x = x.flatten().double()
    ks = [0.5, 0.99, 0.999, 0.9999]
    s = torch.sort(x).values
    return " ".join("p%g=%.2e" % (100 * k, float(s[min(len(s) - 1, int(k * len(s)))])) for k in ks) + " max=%.2e" % float(s[-1])


def run(name, itrs, with_oracle, rgbd=False):
    s = synth.make_scene(name, rgbd=rgbd)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    Pr, Dr = s["poses"].to(dev), s["disps"].to(dev)
    be.ba(P, D, *args, s["t0"], s["t1"], itrs, s["lm"], s["ep"], False)
    ref.ba(Pr, Dr, *args, s["t0"], s["t1"], itrs, s["lm"], s["ep"], False)
    torch.cuda.synchronize()
    kx = torch.unique(torch.cat([torch.arange(s["t0"], s["t1"]), s["ii"]]))
    D_, Dr_ = D[kx.to(dev)].cpu().double(), Dr[kx.to(dev)].cpu().double()
    print("== %s, %d GN iterations: ours vs reference build" % (name, itrs))
    print("   disps rel |a-b|/|b| : %s" % q((D_ - Dr_).abs() / Dr_.abs()))
    print("   disps abs           : %s   (values %.3f .. %.3f)" % (q((D_ - Dr_).abs()), float(Dr_.min()), float(Dr_.max())))
    print("   poses abs           : %s" % q((P.cpu().double() - Pr.cpu().double()).abs()))
    if with_oracle:
        t = time.time()
        P64, D64 = s["poses"].double(), s["disps"].double()
        oracle.ba(P64, D64, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"], s["t0"], s["t1"], itrs, s["lm"], s["ep"], False, dtype=torch.float64)
        D64_ = D64[kx]
        print("   fp64 oracle (%.0f s): ours rel %s" % (time.time() - t, q((D_ - D64_).abs() / D64_.abs())))
        print("                        ref  rel %s" % q((Dr_ - D64_).abs() / D64_.abs()))
        print("                        ours poses abs %s | ref poses abs %s" % (q((P.cpu().double() - P64).abs()), q((Pr.cpu().double() - P64).abs())))
    sys.stdout.flush()


torch.set_num_threads(min(32, os.cpu_count() or 8))
run("metric", 2, True)
run("c4_stereo", 2, True)
run("c2_frontend", 2, True, rgbd=True)
run("c3_global", 2, False)
run("c3_global", 10, False)
if os.environ.get("C3_ORACLE"):
    run("c3_global", 10, True)
