"""Golden vectors of training's flow loss and upsample_disp from the reference's own Python, imported UNMODIFIED from /root/reference
and run in fp64 on the CPU:

    python tests/golden/make_flow_loss_golden.py        -> tests/golden/flow_loss.pt

droid_slam/geom/losses.py flow_loss (with geom/projective_ops.py) and droid_slam/droid_net.py upsample_disp on the lietorch /
torch_scatter stand-ins (oracle/shims), droid_backends an empty module (neither function calls it), projective_ops.py's
`torch.as_tensor(..., device="cuda")` served on the CPU (reference.cuda_on_cpu).  Per flow case (tests/flow_loss_cases.py: inputs
regenerated from seeds, only outputs stored): the loss, the metrics and the gradients of every disps_est[i] and poses_est[i] (lietorch's
left-tangent gradient through poses = Exp(eps) X to first order: oracle.ba_layer.left_perturbed, 7th entry 0).  Per upsample case: the
loss sum(cot * upsample_disp(disp, mask)) and the gradients of disp and mask.
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from flow_loss_cases import cases, upsample_cases  # noqa: E402
from oracle.ba_layer import left_perturbed  # noqa: E402
from oracle.shims.lietorch import SE3  # noqa: E402
from reference import cuda_on_cpu, reference_modules  # noqa: E402


def import_reference():
    """(losses.flow_loss, droid_net.upsample_disp) of the reference, on the stand-ins"""
    with reference_modules("geom.losses", "droid_net", stubs={"droid_backends": types.ModuleType("droid_backends")}) as (losses, net):
        return losses.flow_loss, net.upsample_disp


def run_flow(flow_loss, c):
    """dict(loss, metrics, grad_disps_est [n], grad_poses_est [n]) in fp64"""
    n = len(c["poses_est"])
    d = [x.clone().requires_grad_(True) for x in c["disps_est"]]
    eps = [torch.zeros(*p.shape[:-1], 6, dtype=torch.float64, requires_grad=True) for p in c["poses_est"]]
    P = [SE3(left_perturbed(p, e)) for p, e in zip(c["poses_est"], eps)]
    loss, metrics = flow_loss(SE3(c["Ps"]), c["disps"], P, d, c["intrinsics"], None)
    g = torch.autograd.grad(loss, d + eps)
    gp = [torch.cat([x, torch.zeros_like(x[..., :1])], -1) for x in g[n:]]
    return dict(loss=loss.detach(), metrics=metrics, grad_disps_est=list(g[:n]), grad_poses_est=gp)


def run_upsample(upsample_disp, c):
    disp, mask = c["disp"].clone().requires_grad_(True), c["mask"].clone().requires_grad_(True)
    loss = (c["cot"] * upsample_disp(disp, mask)).sum()
    gd, gm = torch.autograd.grad(loss, [disp, mask])
    return dict(loss=loss.detach(), grad_disp=gd, grad_mask=gm)


def generate():
    flow_loss, upsample_disp = import_reference()
    dt = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with cuda_on_cpu():
            flow = {name: run_flow(flow_loss, c) for name, c in cases().items()}
            up = {name: run_upsample(upsample_disp, c) for name, c in upsample_cases().items()}
        return dict(flow=flow, upsample=up)
    finally:
        torch.set_default_dtype(dt)


if __name__ == "__main__":
    out = generate()
    torch.save(out, os.path.join(HERE, "flow_loss.pt"))
    print("wrote", sorted(out["flow"]), sorted(out["upsample"]))
