"""Golden vectors of the update operator's ConvGRU from the reference's own module, imported UNMODIFIED from /root/reference and run in
fp64 on the CPU:

    python tests/golden/make_conv_gru_golden.py        -> tests/golden/conv_gru.pt

droid_slam/modules/gru.py ConvGRU(128, 128+128+64), as UpdateModule builds it, with the seeded parameters and inputs of
tests/conv_gru_cases.py (regenerated from the seeds; only results stored).  Per case: every call's output (a chain feeds net back) and
the gradients of loss = sum_k <cot_k, out_k> with respect to the first net, every call's inputs and the 14 parameters (a fixed strided
sample of each weight gradient, conv_gru_cases.param_sample, to keep the file small).
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from conv_gru_cases import CASES, case_inputs, load_params, run_chain  # noqa: E402
from reference import reference_modules  # noqa: E402


def import_reference():
    """modules.gru.ConvGRU of the reference"""
    with reference_modules("modules.gru") as (gru,):
        return gru.ConvGRU


def generate():
    ConvGRU = import_reference()
    out = {}
    for name in CASES:
        params, net, ins, cots = case_inputs(name)
        module = load_params(ConvGRU(128, 128 + 128 + 64).double(), params)
        out[name] = run_chain(module, dict(module.named_parameters()), net, ins, cots)
    return out


if __name__ == "__main__":
    out = generate()
    torch.save(out, os.path.join(HERE, "conv_gru.pt"))
    print("wrote", sorted(out))
