"""Regenerate tests/golden/encoder.pt: outputs of the reference's own BasicEncoder (droid_slam/modules/extractor.py, imported unmodified;
it needs only torch) for DroidNet's two instances, fp32 on the CPU, with seeded weights (synth.make_encoder_weights, nonzero biases).

    python tests/golden/make_encoder_golden.py

Cases: fnet (128, 'instance') and cnet (256, 'none') on [1,2,3,64,96] and [1,1,3,40,56] images, plus [1,1,3,64,96] images + 40 (every
instance norm then sees |mean| >> std)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from droid_slam_b200 import synth  # noqa: E402
from reference import reference_modules  # noqa: E402

CASES = [("fnet", (1, 2, 3, 64, 96), 0.0), ("cnet", (1, 2, 3, 64, 96), 0.0), ("fnet", (1, 1, 3, 40, 56), 0.0), ("cnet", (1, 1, 3, 40, 56), 0.0),
         ("fnet", (1, 1, 3, 64, 96), 40.0), ("cnet", (1, 1, 3, 64, 96), 40.0)]
ENCODERS = {"fnet": ("instance", 128, 0), "cnet": ("none", 256, 1)}   # norm_fn, output_dim, weight seed


def import_reference():
    """the reference's modules/extractor.py, imported unmodified"""
    with reference_modules("modules.extractor") as (ext,):
        return ext


def main():
    ext = import_reference()
    torch.manual_seed(0)
    out = {"cases": []}
    for i, (name, shape, shift) in enumerate(CASES):
        norm_fn, od, wseed = ENCODERS[name]
        enc = ext.BasicEncoder(output_dim=od, norm_fn=norm_fn).eval()
        enc.load_state_dict(synth.make_encoder_weights(wseed, od))
        x = torch.randn(*shape, generator=torch.Generator().manual_seed(100 + i)) + shift
        with torch.no_grad():
            y = enc(x)
        out["cases"].append({"name": name, "norm_fn": norm_fn, "output_dim": od, "weight_seed": wseed, "images": x, "out": y})
    path = os.path.join(ROOT, "tests", "golden", "encoder.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
