"""Pin the CPU oracle against outputs of the UNMODIFIED reference CUDA build run on an H100
(tests/golden/reference_h100.pt, produced by tests/golden/make_golden.py; the reference ships no golden vectors of
its own for this path, SURVEY.md section 8c)."""
import os
import sys

import pytest
import torch

import oracle

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import cases  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_h100.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, map_location="cpu", weights_only=False)


def _rel(a, b, floor=1.0):
    return float(((a.double() - b.double()).abs() / b.double().abs().clamp(min=floor)).max())


def test_golden_file_describes_reference(gold):
    m = gold["_meta"]
    assert "H100" in m["gpu"] and "unmodified" in m["note"]
    # our kernels vs the reference on the same GPU, recorded when the file was made
    for k, v in m["ours_vs_reference"].items():
        if k.startswith(("corr_", "altcorr_", "projmap", "iproj", "depth_filter")):
            assert v["frac_equal"] == 1.0, (k, v)           # bit-identical to the reference build
        else:
            assert v["max_abs"] < 1e-5, (k, v)


@pytest.mark.parametrize("si", range(len(cases.CORR_SHAPES)))
@pytest.mark.parametrize("dt", [torch.float16, torch.float32])
def test_corr_index_oracle_bit_exact_vs_reference(gold, si, dt):
    vol, coords, grad = cases.corr_case(cases.CORR_SHAPES[si], dt, si)
    key = "corr_%d_%s" % (si, str(dt).split(".")[-1])
    o, = oracle.corr_index_forward(vol, coords, 3)
    assert torch.equal(o, gold[key + "_fwd"])               # the oracle's rounding-order restatement is exact
    b, = oracle.corr_index_backward(vol, coords, grad, 3)
    assert torch.equal(b, gold[key + "_bwd"])


@pytest.mark.parametrize("dt", [torch.float16, torch.float32])
def test_altcorr_oracle_vs_reference(gold, dt):
    fmaps, coords, ii, jj = cases.altcorr_case(dt)
    f2 = torch.nn.functional.avg_pool2d(fmaps[0].float(), 2, stride=2).to(dt)[None].contiguous()
    for lvl, fm2 in enumerate((fmaps, f2)):
        o, = oracle.altcorr_forward(fmaps, fm2, (coords / 2 ** lvl).contiguous(), ii, jj, 3)
        ref = gold["altcorr_%s_l%d" % (str(dt).split(".")[-1], lvl)]
        assert o.shape == ref.shape
        assert _rel(o, ref) < (2e-2 if dt == torch.float16 else 1e-5)    # channel-sum order of the oracle (torch.sum) differs


def test_geometry_oracle_vs_reference(gold):
    s = cases.geom_scene()
    P, D, K, ii, jj = [s[k] for k in ("poses", "disps", "intrinsics", "ii", "jj")]
    c, v = oracle.projmap(P, D, K, ii, jj)
    assert _rel(c, gold["projmap_coords"]) < 1e-5 and torch.equal(v, gold["projmap_valid"])
    assert _rel(oracle.iproj(P, D, K), gold["iproj"]) < 1e-5
    assert _rel(oracle.frame_distance(P, D, K, ii, jj, 0.3), gold["frame_distance"]) < 1e-5
    cnt = oracle.depth_filter(P, D, K, torch.arange(8), torch.full((8,), 0.05))
    assert float((cnt == gold["depth_filter"]).float().mean()) > 0.999


@pytest.mark.parametrize("name", list(cases.BA_CASES))
def test_ba_oracle_vs_reference(gold, name):
    s, c = cases.ba_scene(name)
    for dtype, tol in ((torch.float32, 1e-4), (torch.float64, 1e-4)):
        P = s["poses"].clone().to(dtype); D = s["disps"].clone().to(dtype)
        dx, dz = oracle.ba(P, D, s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], s["eta"], s["ii"], s["jj"],
                           s["t0"], s["t1"], c["itrs"], s["lm"], s["ep"], c["motion_only"], dtype=dtype)
        assert _rel(P, gold["ba_%s_poses" % name]) < tol
        assert _rel(D, gold["ba_%s_disps" % name]) < tol
        assert _rel(dx, gold["ba_%s_dx" % name], floor=1e-2) < 1e-3
        if not c["motion_only"]:
            assert _rel(dz, gold["ba_%s_dz" % name]) < tol
