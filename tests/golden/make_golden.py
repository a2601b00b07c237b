"""Generate golden vectors by running the UNMODIFIED reference CUDA build (oracle/_ref/droid_backends_ref, built by
oracle/build_ref.sh from the reference's src/ with the Eigen stand-in) on an H100.

    python tests/golden/make_golden.py tests/golden/reference_h100.pt

The file holds only the reference's OUTPUTS (fp32/fp16 tensors, < 1 MB); inputs are regenerated from seeds by
tests/golden/cases.py.  It also stores our kernels' max deviation from the reference for the record.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import cases  # noqa: E402


def main(out_path):
    import droid_backends_ref as ref
    import droid_slam_b200
    ours = droid_slam_b200.install()
    dev = "cuda"
    G = {}
    dev_report = {}

    def cmp(name, a, b):
        a = a.double().cpu(); b = b.double().cpu()
        dev_report[name] = dict(max_abs=float((a - b).abs().max()), frac_equal=float((a == b).float().mean()))

    for si, shape in enumerate(cases.CORR_SHAPES):
        for dt in (torch.float16, torch.float32):
            vol, coords, grad = cases.corr_case(shape, dt, si)
            key = "corr_%d_%s" % (si, str(dt).split(".")[-1])
            o, = ref.corr_index_forward(vol.to(dev), coords.to(dev), 3)
            G[key + "_fwd"] = o.cpu()
            cmp(key + "_fwd", ours.corr_index_forward(vol.to(dev), coords.to(dev), 3)[0], o)
            b, = ref.corr_index_backward(vol.to(dev), coords.to(dev), grad.to(dev), 3)
            G[key + "_bwd"] = b.cpu()
            cmp(key + "_bwd", ours.corr_index_backward(vol.to(dev), coords.to(dev), grad.to(dev), 3)[0], b)
    for dt in (torch.float16, torch.float32):
        fmaps, coords, ii, jj = cases.altcorr_case(dt)
        f2 = torch.nn.functional.avg_pool2d(fmaps[0], 2, stride=2)[None].contiguous()
        for lvl, fm2 in enumerate((fmaps, f2)):
            c = (coords / 2 ** lvl).contiguous()
            o, = ref.altcorr_forward(fmaps.to(dev), fm2.to(dev), c.to(dev), ii.to(dev), jj.to(dev), 3)
            key = "altcorr_%s_l%d" % (str(dt).split(".")[-1], lvl)
            G[key] = o.contiguous().cpu()
            cmp(key, ours.altcorr_forward(fmaps.to(dev), fm2.to(dev), c.to(dev), ii.to(dev), jj.to(dev), 3)[0], o)
    s = cases.geom_scene()
    P, D, K, ii, jj = [s[k].to(dev) for k in ("poses", "disps", "intrinsics", "ii", "jj")]
    c, v = ref.projmap(P, D, K, ii, jj)
    G["projmap_coords"], G["projmap_valid"] = c.cpu(), v.cpu()
    oc, ov = ours.projmap(P, D, K, ii, jj); cmp("projmap_coords", oc, c); cmp("projmap_valid", ov, v)
    G["iproj"] = ref.iproj(P, D, K).cpu(); cmp("iproj", ours.iproj(P, D, K), G["iproj"])
    G["frame_distance"] = ref.frame_distance(P, D, K, ii, jj, 0.3).cpu(); cmp("frame_distance", ours.frame_distance(P, D, K, ii, jj, 0.3), G["frame_distance"])
    ix = torch.arange(8, device=dev); th = torch.full((8,), 0.05, device=dev)
    G["depth_filter"] = ref.depth_filter(P, D, K, ix, th).cpu(); cmp("depth_filter", ours.depth_filter(P, D, K, ix, th), G["depth_filter"])
    for name in cases.BA_CASES:
        s, c = cases.ba_scene(name)
        args = [s[k].to(dev) for k in ("intrinsics", "disps_sens", "targets", "weights", "eta", "ii", "jj")]
        P, D = s["poses"].to(dev), s["disps"].to(dev)
        out = ref.ba(P, D, *args, s["t0"], s["t1"], c["itrs"], s["lm"], s["ep"], c["motion_only"])
        torch.cuda.synchronize()
        G["ba_%s_poses" % name], G["ba_%s_disps" % name], G["ba_%s_dx" % name] = P.cpu(), D.cpu(), out[0].cpu()
        if not c["motion_only"]:
            G["ba_%s_dz" % name] = out[1].cpu()
        P2, D2 = s["poses"].to(dev), s["disps"].to(dev)
        o2 = ours.ba(P2, D2, *args, s["t0"], s["t1"], c["itrs"], s["lm"], s["ep"], c["motion_only"])
        cmp("ba_%s_poses" % name, P2, P); cmp("ba_%s_disps" % name, D2, D); cmp("ba_%s_dx" % name, o2[0], out[0])
    G["_meta"] = dict(gpu=torch.cuda.get_device_name(0), torch=torch.__version__, ours_vs_reference=dev_report,
                      note="reference = src/*.cu unmodified, sm_90a, Eigen stand-in (dense fp64 LLT)")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    torch.save(G, out_path)
    for k, v in sorted(dev_report.items()):
        print("%-32s max_abs %.3e  identical %.4f" % (k, v["max_abs"], v["frac_equal"]))
    print("saved", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_h100.pt"))
