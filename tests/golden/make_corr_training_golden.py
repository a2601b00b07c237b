"""Golden vectors of the training CorrBlock from the reference's own modules/corr.py, imported UNMODIFIED from /root/reference and run
on CPU in fp64 on an oracle-backed `droid_backends` stub (make_reference_python_golden.import_reference):

    python tests/golden/make_corr_training_golden.py        -> tests/golden/corr_training.pt

Per case of tests/corr_training_cases.FIXTURE: CorrBlock(fmap1, fmap2, num_levels=4, radius=3) on fp64 maps, every call's lookup, and
autograd's backward of sum_k (w_k * out_k).sum() over the calls that feed the loss -> every 31st element of each level and call output,
every 7th of both map gradients.  Inputs are regenerated from seeds; only outputs are stored."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from corr_training_cases import FIXTURE, fixture_record, make_inputs, run  # noqa: E402
from make_reference_python_golden import import_reference  # noqa: E402


def main(out_path):
    _, corr = import_reference()
    G = {}
    for name, (B, N, C, ht, wd, calls, used) in FIXTURE.items():
        f1, f2, coords, weights = make_inputs(B, N, ht, wd, calls, seed=11, C=C)
        G[name] = fixture_record(*run(corr.CorrBlock, f1, f2, coords, weights, used, torch.float64))
    torch.save(G, out_path)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(os.path.join(HERE, "corr_training.pt"))
