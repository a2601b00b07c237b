"""Outputs of the UNMODIFIED reference CUDA build on the inputs of tests/test_vs_reference_build_gpu.py -> reference_build.pt.

The reference build is oracle/_ref/droid_backends_ref (reference src/{droid.cpp,droid_kernels.cu,correlation_kernels.cu,
altcorr_kernel.cu} compiled for sm_90a by oracle/build_ref.sh against the Eigen stand-in).  Regenerate on an H100 with it present:
    python tests/golden/make_reference_build_golden.py [out.pt]
or, to add one group of entries to the existing file and leave the others as they are:
    python tests/golden/make_reference_build_golden.py --add geometry_edges [out.pt]
Outputs the tests require to be bit-identical are stored as SHA-256 digests of their bytes plus a seeded sample of values (for the
failure message); frame distances in full; bundle adjustment as the updated poses and a seeded sample of the inverse depths.
The geometry_edges group is kept small: digests alone, and frame distances in full up to N_FD_SAMPLE pairs, else a seeded sample of
that many.  The sample positions are not stored: sample_index regenerates them from their seeds."""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from droid_slam_b200 import synth  # noqa: E402
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import geometry_cases  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_build.pt")
N_SAMPLE = 4096
N_DISP_SAMPLE = 16384
N_FD_SAMPLE = 2048
BA_CASES = {  # name: (scene, scene kwargs, iterations, motion_only)
    "ba_metric": ("metric", {}, 2, False),
    "ba_c4_stereo": ("c4_stereo", {}, 2, False),
    "ba_c2_rgbd": ("c2_frontend", {"rgbd": True}, 2, False),
    "ba_c2_rgbd_motion_only": ("c2_frontend", {"rgbd": True}, 2, True),
    "ba_c3_global": ("c3_global", {}, 10, False),
}


def digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def sample_index(n, k, seed=0):
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:min(k, n)].clone()   # not a view of the whole permutation


def corr_metric(be, dev, chunk=None):
    """512 edges x 48x64 f16 volumes, all four levels (CorrBlock.__call__, modules/corr.py:40-50); the reference's 32-bit accessors
    cannot address 512 level-0 planes at once, so it is called in chunks of `chunk` edges"""
    s = synth.make_scene("metric")
    pyr, coords, _ = synth.make_corr_inputs(s, dtype=torch.float16, device=dev)
    out = {}
    for lvl, vol in enumerate(pyr):
        c = (coords / 2 ** lvl).contiguous()
        if chunk is None:
            out["corr_metric_l%d" % lvl], = be.corr_index_forward(vol, c, 3)
        else:
            out["corr_metric_l%d" % lvl] = torch.cat([be.corr_index_forward(vol[a:a + chunk], c[a:a + chunk].contiguous(), 3)[0]
                                                      for a in range(0, vol.shape[0], chunk)])
    return out


def corr_f32(be, dev):
    """config 2 (fp32 volumes), 96 edges: forward at every level, backward at levels 2 and 3"""
    s = synth.make_scene("c2_frontend")
    sub = dict(s); sub["ii"] = s["ii"][:96]; sub["jj"] = s["jj"][:96]; sub["coords_gt"] = s["coords_gt"][:96]; sub["cfg"] = dict(s["cfg"], E=96)
    pyr, coords, _ = synth.make_corr_inputs(sub, dtype=torch.float32, device=dev)
    g = torch.Generator(device=dev).manual_seed(3)
    out = {}
    for lvl, vol in enumerate(pyr):
        c = (coords / 2 ** lvl).contiguous()
        out["corr_f32_fwd_l%d" % lvl], = be.corr_index_forward(vol, c, 3)
        if lvl >= 2:
            grad = torch.randn(96, 7, 7, 48, 64, device=dev, generator=g)
            out["corr_f32_bwd_l%d" % lvl], = be.corr_index_backward(vol, c, grad, 3)
    return out


def altcorr(be, dev):
    """AltCorrBlock.__call__ (modules/corr.py:104-117) on 48x64 f16 feature maps, 4 levels, a chunk of 24 edges"""
    g = torch.Generator().manual_seed(5)
    N, M = 8, 24
    fmaps = torch.randn(1, N, 128, 48, 64, generator=g).half().to(dev)
    s = synth.make_scene(dict(E=M, N=N, ht=48, wd=64, stereo=False, itrs=1, lm=1e-4, ep=0.1), seed=3)
    coords = (s["coords_gt"] + 2 * torch.rand(M, 48, 64, 2, generator=g) - 1).permute(0, 3, 1, 2)[None].contiguous().to(dev)
    ii, jj = s["ii"].to(dev), s["jj"].to(dev)
    f = fmaps[0]
    out = {}
    for lvl in range(4):
        f2 = f[None].contiguous()
        c = (coords / 2 ** lvl).contiguous()
        out["altcorr_l%d" % lvl] = be.altcorr_forward(fmaps, f2, c, ii, jj, 3)[0].contiguous()
        f = torch.nn.functional.avg_pool2d(f, 2, stride=2)
    return out


def geometry(be, dev):
    s = synth.make_scene("metric")
    P, D, K, ii, jj = [s[k].to(dev) for k in ("poses", "disps", "intrinsics", "ii", "jj")]
    out = {}
    out["projmap_coords"], out["projmap_valid"] = be.projmap(P, D, K, ii, jj)
    out["iproj"] = be.iproj(P, D, K)
    ix = torch.arange(72, device=dev); th = torch.full((72,), 0.05, device=dev)
    out["depth_filter"] = be.depth_filter(P, D, K, ix, th)
    a, b = torch.meshgrid(torch.arange(72), torch.arange(72), indexing="ij")
    out["frame_distance"] = be.frame_distance(P, D, K, a.reshape(-1).to(dev), b.reshape(-1).to(dev), 0.3)   # DepthVideo.distance
    return out


GEOMETRY_EDGE_CASES = [n for n in geometry_cases.CASES if n != "empty"] + ["many_edges"]   # hw = 0 launches nothing in the reference


def geometry_edges_case(be, dev, name):
    """projmap, iproj, depth_filter and frame_distance (every beta of the case) on one case of tests/geometry_cases.py"""
    c = geometry_cases.case(name)
    P, D, K, ii, jj, ix, th = [c[k].to(dev).contiguous() for k in ("poses", "disps", "intr", "ii", "jj", "df_ix", "df_thresh")]
    out = {}
    out["projmap_coords"], out["projmap_valid"] = be.projmap(P, D, K, ii, jj)
    out["iproj"] = be.iproj(P, D, K)
    out["depth_filter"] = be.depth_filter(P, D, K, ix, th)
    for beta in c["betas"]:
        out["frame_distance beta=%g" % beta] = be.frame_distance(P, D, K, ii, jj, beta)
    return out


def geometry_edges(be, dev):
    out = {}
    for name in GEOMETRY_EDGE_CASES:
        for k, v in geometry_edges_case(be, dev, name).items():
            out["geometry_edges/%s/%s" % (name, k)] = v
    return out


def ba(be, dev, name):
    scene, kw, itrs, motion_only = BA_CASES[name]
    s = synth.make_scene(scene, **kw)
    args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
    P, D = s["poses"].to(dev), s["disps"].to(dev)
    o = be.ba(P, D, *args, s["t0"], s["t1"], itrs, s["lm"], s["ep"], motion_only)
    torch.cuda.synchronize()
    return P, D, o


def record_identical(t):
    flat = t.detach().reshape(-1).cpu()
    idx = sample_index(flat.numel(), N_SAMPLE)
    return {"sha256": digest(t), "shape": tuple(t.shape), "dtype": str(t.dtype), "val": flat[idx].clone()}


def _record(k, v):
    return {"full": v.cpu()} if "frame_distance" in k else record_identical(v)


def fd_sample_index(n):
    return sample_index(n, N_FD_SAMPLE, seed=2)


def record_edge(k, v):
    """a geometry_edges entry: the digest of a bit-identical output; a frame-distance vector's length and its values at
    fd_sample_index (all of them, permuted, when there are at most N_FD_SAMPLE)"""
    if "frame_distance" in k:
        flat = v.detach().reshape(-1).cpu()
        return {"n": flat.numel(), "val": flat[fd_sample_index(flat.numel())].clone()}
    return {"sha256": digest(v), "shape": tuple(v.shape), "dtype": str(v.dtype)}


def add_group(path, group):
    """add one group's keys to an existing fixture file; every entry already in it stays as it is"""
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import droid_backends_ref as ref
    gold = torch.load(path, weights_only=False)
    new = {k: record_edge(k, v) for k, v in {"geometry_edges": geometry_edges}[group](ref, "cuda").items()}
    assert not set(new) & set(gold), "only adds keys"
    gold.update(new)
    torch.save(gold, path)
    print("added", len(new), "entries to", path, os.path.getsize(path), "bytes")


def main(path):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import droid_backends_ref as ref
    dev = "cuda"
    gold = {"meta": {"note": "reference src/*.cu + droid.cpp unmodified, built for sm_90a (oracle/build_ref.sh), Eigen stand-in",
                     "gpu": torch.cuda.get_device_name(0), "torch": torch.__version__}}
    for k, v in corr_metric(ref, dev, chunk=128).items():
        gold[k] = record_identical(v)
    torch.cuda.empty_cache()
    for fn in (corr_f32, altcorr, geometry):
        for k, v in fn(ref, dev).items():
            gold[k] = _record(k, v)
    for k, v in geometry_edges(ref, dev).items():
        gold[k] = record_edge(k, v)
    for name in BA_CASES:
        P, D, o = ba(ref, dev, name)
        Df = D.reshape(-1).cpu()
        idx = sample_index(Df.numel(), N_DISP_SAMPLE, seed=1)
        gold[name] = {"poses": P.cpu(), "disp_val": Df[idx].clone(), "disp_absmax": float(Df.abs().max()),
                      "disp_sha256": digest(D), "out_shapes": [tuple(t.shape) if torch.is_tensor(t) else None for t in o]}
    torch.save(gold, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--add":      # --add geometry_edges [out.pt]
        add_group(sys.argv[3] if len(sys.argv) > 3 else GOLD, sys.argv[2])
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else GOLD)
