"""Golden vectors for the update operator (row A6) from the REFERENCE module itself, run on CPU in this container.

    python tests/golden/make_update_golden.py            -> tests/golden/update_module.pt

`droid_slam/droid_net.py` is imported unmodified from /root/reference on the stand-ins of oracle/shims (tests/golden/reference.py):
`lietorch` (unused by UpdateModule) and `torch_scatter` (its `scatter_mean` with the documented semantics: out[:, k] = mean of
src[:, e] over e with index[e] == k); `droid_backends`, which modules/corr.py imports, is an empty module.  Everything
UpdateModule.forward executes besides that one call -- the 19 convolutions, the GRU gating, GradientClip, Softplus, views and
permutes -- is the reference's own code.  Weights and inputs are regenerated from seeds (droid_slam_b200/synth.py); only outputs are stored.
"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from reference import reference_modules  # noqa: E402


def import_reference():
    """the reference's droid_net module, imported unmodified; `import droid_backends` in modules/corr.py finds an empty stub"""
    with reference_modules("droid_net", stubs={"droid_backends": types.ModuleType("droid_backends")}) as (droid_net,):
        return droid_net


def upmask_sample_index(n):
    return torch.randperm(n, generator=torch.Generator().manual_seed(0))[:n // 4]


def main(out_path):
    from droid_slam_b200 import synth
    droid_net = import_reference()
    torch.manual_seed(0)
    mod = droid_net.UpdateModule().eval()
    w = synth.make_update_weights(0)
    missing = mod.load_state_dict(w, strict=True)
    G = {"state_dict_keys": sorted(mod.state_dict().keys()), "load": str(missing)}
    with torch.no_grad():
        for name, kw in (("a", dict(E=5, ht=6, wd=8, seed=0, n_src=3)), ("b", dict(E=7, ht=5, wd=9, seed=1, n_src=4))):
            net, inp, corr, flow, ii = synth.make_update_inputs(**kw)
            o = mod(net, inp, corr, flow, ii)
            for k, t in zip(("net", "delta", "weight", "eta", "upmask"), o):
                G["%s_%s" % (name, k)] = t.clone()
            up = G.pop("%s_upmask" % name)                             # the largest output: a seeded quarter of it (file < 1 MB)
            G["%s_upmask_shape" % name] = tuple(up.shape)
            G["%s_upmask_sample" % name] = up.reshape(-1)[upmask_sample_index(up.numel())].clone()
            o2 = mod(net, inp, corr, None, None)                       # no flow, no aggregation
            for k, t in zip(("net", "delta", "weight"), o2):
                G["%s_noflow_%s" % (name, k)] = t.clone()
    # cvx_upsample (droid_net.py:21-35), the reference function itself, on seeded inputs
    g = torch.Generator().manual_seed(321)
    d = torch.rand(3, 6, 10, 1, generator=g) + 0.2
    m = 2.0 * torch.randn(3, 576, 6, 10, generator=g)
    G["cvx_upsample"] = droid_net.cvx_upsample(d, m).clone()
    torch.save(G, out_path)
    print("saved", out_path, os.path.getsize(out_path), "bytes;", len(G["state_dict_keys"]), "parameters")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "update_module.pt"))
