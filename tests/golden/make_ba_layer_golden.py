"""Golden vectors of the dense BA layer from the reference's own Python, imported UNMODIFIED from /root/reference and run in fp64 on the CPU:

    python tests/golden/make_ba_layer_golden.py        -> tests/golden/ba_layer.pt

droid_slam/geom/ba.py BA, with geom/chol.py and geom/projective_ops.py, on the lietorch / torch_scatter stand-ins (oracle/shims), with
projective_ops.py's `torch.as_tensor(..., device="cuda")` served on the CPU (reference.cuda_on_cpu).  The default
dtype is fp64 while it runs, so that constant lands in the inputs' dtype.  Per case (tests/ba_layer_cases.py: inputs regenerated from
seeds, only outputs stored): the outputs of every chained call and the gradients of target, weight, eta, poses (lietorch's left-tangent
gradient, through poses = Exp(eps) X to first order: oracle.ba_layer.left_perturbed) and disps of loss = sum(a * log(poses')) + sum(b * disps') over the calls.
"""
import contextlib
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from ba_layer_cases import cases, loss_weights  # noqa: E402
from oracle.ba_layer import left_perturbed  # noqa: E402
from oracle.shims.lietorch import SE3  # noqa: E402
from reference import cuda_on_cpu, reference_modules  # noqa: E402

NAMES = ("target", "weight", "eta", "poses", "disps")


def import_reference_ba():
    """the reference's geom/ba.py BA function, on the stand-ins"""
    with reference_modules("geom.ba") as (ba,):
        return ba.BA


def run(BA, SE3, c):
    """[outputs of each call..., gradients of NAMES...] in fp64 on the CPU; BA(target, weight, eta, poses, disps, intrinsics, ii, jj,
    fixedp) and SE3 the stand-in class"""
    B, N, ht, wd = c["disps"].shape
    a, b = loss_weights(B, N, ht, wd)
    x = {k: c[k].clone().requires_grad_(k in NAMES and k != "poses") for k in NAMES + ("intrinsics",)}
    eps = torch.zeros(B, N, 6, dtype=torch.float64, requires_grad=True)
    P, D, outs, loss = SE3(left_perturbed(x["poses"], eps)), x["disps"], [], 0.0
    for _ in range(c["chain"]):
        with contextlib.redirect_stdout(io.StringIO()):           # the reference prints a failed Cholesky's exception
            P, D = BA(x["target"], x["weight"], x["eta"], P, D, x["intrinsics"], c["ii"], c["jj"], fixedp=c["fixedp"])
        outs += [P.data.detach(), D.detach()]
        loss = loss + (a[..., :6] * P.log()).sum() + (b * D).sum()
    grads = torch.autograd.grad(loss, [x[k] if k != "poses" else eps for k in NAMES])
    return outs + list(grads)


def generate():
    BA = import_reference_ba()
    dt = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with cuda_on_cpu():
            return {name: run(BA, SE3, c) for name, c in cases().items()}
    finally:
        torch.set_default_dtype(dt)


if __name__ == "__main__":
    out = generate()
    torch.save(out, os.path.join(HERE, "ba_layer.pt"))
    print("wrote", {k: len(v) for k, v in out.items()})
