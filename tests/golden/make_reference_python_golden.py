"""Golden vectors from the reference's own PYTHON call sites, imported UNMODIFIED from /root/reference and run on CPU in this container:

    python tests/golden/make_reference_python_golden.py        -> tests/golden/reference_python.pt

  * droid_slam/geom/projective_ops.py  : projective_transform(jacobian=False) -- what DepthVideo.reproject calls
    (depth_video.py:171-179) -> pins oracle.reproject and the dba_reproject kernel (row A5);
  * droid_slam/modules/corr.py         : CorrBlock / AltCorrBlock / CorrSampler on a CPU `droid_backends` whose two correlation
    ops are the oracle's (the reference classes only need those) -> pins the call pattern, layouts and the pyramid construction.

What is substituted, and only for the import / CPU execution: `lietorch` and `torch_scatter` are the pure-PyTorch stand-ins of
oracle/shims (the real packages are CUDA extensions that cannot be built here), `droid_backends` is an oracle-backed stub while
modules/corr.py runs on CPU tensors, and `torch.as_tensor(..., device="cuda")` inside projective_ops.py:176 (a hard-coded device)
is served on the CPU.  Every line of the reference files themselves executes as written.  Inputs are regenerated from seeds
(tests/golden/cases.py, droid_slam_b200/synth.py); only outputs are stored.
"""
import hashlib
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from reference import cuda_on_cpu, reference_modules  # noqa: E402


def import_reference():
    """returns (pops, corr_module) = the reference's geom/projective_ops.py and modules/corr.py, imported unmodified"""
    import oracle
    stub = types.ModuleType("droid_backends")
    stub.corr_index_forward = lambda v, c, r: oracle.corr_index_forward(v, c.contiguous(), r)
    stub.corr_index_backward = lambda v, c, g, r: oracle.corr_index_backward(v, c.contiguous(), g, r)
    stub.altcorr_forward = lambda f1, f2, c, ii, jj, r: oracle.altcorr_forward(f1, f2, c, ii, jj, r)
    stub.altcorr_backward = lambda f1, f2, c, g, ii, jj, r: oracle.altcorr_backward(f1, f2, c, g, ii, jj, r)
    with reference_modules("geom.projective_ops", "modules.corr", stubs={"droid_backends": stub}) as (pops, corr):
        return pops, corr


def reproject_cases():
    """(name, poses [N,7], disps [N,ht,wd], intrinsics [N,4], ii, jj): mono, stereo (ii == jj edges), per-frame intrinsics, points
    behind / close to the camera (Z < MIN_DEPTH and Z < 0.1 branches of geom/projective_ops.py:52,185)"""
    from droid_slam_b200 import synth
    out = []
    s = synth.make_scene(dict(E=20, N=8, ht=12, wd=16, stereo=False, itrs=1, lm=1e-4, ep=0.1), seed=7)
    intr = s["intrinsics"][None].repeat(8, 1)
    out.append(("mono", s["poses"], s["disps"], intr, s["ii"], s["jj"]))
    s = synth.make_scene(dict(E=30, N=9, ht=12, wd=16, stereo=True, itrs=1, lm=1e-4, ep=0.1), seed=4)
    intr = s["intrinsics"][None].repeat(9, 1) * (1.0 + 0.05 * torch.arange(9.0)[:, None])     # per-frame intrinsics
    out.append(("stereo_perframe_intr", s["poses"], s["disps"], intr, s["ii"], s["jj"]))
    s = synth.make_scene(dict(E=16, N=6, ht=10, wd=14, stereo=False, itrs=1, lm=1e-4, ep=0.1), seed=11)
    g = torch.Generator().manual_seed(5)
    poses = s["poses"].clone()
    poses[:, 2] += torch.linspace(-1.5, 1.5, 6)                                               # large forward/backward motion: points end up behind the camera
    disps = s["disps"] * (0.2 + 3.0 * torch.rand(s["disps"].shape, generator=g))
    out.append(("near_plane", poses, disps, s["intrinsics"][None].repeat(6, 1), s["ii"], s["jj"]))
    return out


def corr_cases():
    g = torch.Generator().manual_seed(77)
    B, E, C, H, W = 1, 5, 16, 8, 16
    f1 = torch.randn(B, E, C, H, W, generator=g)
    f2 = torch.randn(B, E, C, H, W, generator=g)
    coords = torch.rand(B, E, H, W, 2, generator=g) * torch.tensor([W + 4.0, H + 4.0]) - 2
    N = 4
    fm = torch.randn(B, N, C, H, W, generator=g)
    ii = torch.tensor([0, 1, 2, 3, 0]); jj = torch.tensor([1, 2, 3, 3, 3])
    return (f1, f2, coords), (fm, coords, ii, jj)


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def main(out_path):
    pops, corr = import_reference()
    from oracle.shims.lietorch import SE3
    G = {}
    with torch.no_grad(), cuda_on_cpu():
        for name, poses, disps, intr, ii, jj in reproject_cases():
            coords, valid = pops.projective_transform(SE3(poses[None]), disps[None], intr[None], ii, jj)
            G["reproject_%s_coords" % name] = coords.clone()
            G["reproject_%s_valid" % name] = valid.clone()
        (f1, f2, coords), (fm, coords_a, ii, jj) = corr_cases()
        blk = corr.CorrBlock(f1, f2, num_levels=3, radius=3)
        for l, v in enumerate(blk.corr_pyramid):
            G["corrblock_pyr%d" % l] = v.clone() if l >= 2 else digest(v)     # levels 0, 1 as digests (file < 1 MB)
        G["corrblock_lookup"] = blk(coords).clone()
        alt = corr.AltCorrBlock(fm, num_levels=3, radius=3)
        G["altcorrblock_lookup"] = alt(coords_a, ii, jj).clone()
    torch.save(G, out_path)
    print("saved", out_path, os.path.getsize(out_path), "bytes,", len(G), "tensors")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "reference_python.pt"))
