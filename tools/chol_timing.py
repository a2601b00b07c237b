"""CUDA-event timing of the damped SPD solve (`dba_solve_spd`): 20 warm-up solves, then 200 back-to-back solves of one seeded system,
printed with the card.  usage: python tools/chol_timing.py [n ...]   (default 426; n <= 448 runs the resident kernel, larger n the
cluster kernel)."""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
from droid_slam_b200 import c_api  # noqa: E402
from util import card, timed  # noqa: E402


def time_solve(L, n):
    g = torch.Generator().manual_seed(0)
    A = torch.randn(n, n + 8, generator=g, dtype=torch.float64)
    Hc = A @ A.t() + 1e-3 * torch.eye(n, dtype=torch.float64)
    bc = torch.randn(n, generator=g, dtype=torch.float64)
    H, b = Hc.cuda(), bc.cuda()
    ws = torch.empty(L.dba_solve_workspace_bytes(n), dtype=torch.uint8, device="cuda")
    x = torch.zeros(n, device="cuda")
    fail = torch.zeros(1, dtype=torch.int32, device="cuda")

    def solve():
        c_api.check(L.dba_solve_spd(ctypes.c_void_p(H.data_ptr()), ctypes.c_void_p(b.data_ptr()), n, ctypes.c_float(1e-4), ctypes.c_float(0.1),
                                    ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(fail.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ws.numel(), None),
                    "dba_solve_spd")

    ms, _, _ = timed(solve, calls=200, warmup=20)
    Hd = Hc.clone()
    Hd.diagonal().add_(0.1 + 1e-4 * Hc.diagonal())
    ref = torch.linalg.solve(Hd, bc)
    err = float((x.cpu().double() - ref).abs().max() / ref.abs().max())
    return 1e3 * ms, int(fail), err


def main():
    L = c_api.load()
    gpu = card()
    for n in [int(a) for a in sys.argv[1:]] or [426]:
        us, fail, err = time_solve(L, n)
        print("n=%d  %s kernel: %.1f us per solve (200 back-to-back), fail=%d, max rel err vs fp64 LAPACK %.2e  [%s]"
              % (n, "resident" if n <= 448 else "cluster", us, fail, err, gpu))


if __name__ == "__main__":
    main()
