"""PoseTrajectoryFiller without a GPU: the restatement (oracle/trajectory_filler.py) bit-exact against what the unmodified reference
methods computed on CPU stand-ins (tests/golden/trajectory_filler.pt), its pose interpolation on the lietorch stand-in, and the C ABI of
the two filler kernels (exported, arguments rejected before any launch)."""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.shims import lietorch  # noqa: E402
from oracle import trajectory_filler as otf  # noqa: E402
from droid_slam_b200 import c_api  # noqa: E402


def _keyframes(n, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    xi = 0.3 * torch.randn(n, 6, generator=g, dtype=dtype)
    return lietorch.SE3.exp(xi).data, g


def test_bracket_search_and_quirks():
    """t0 counts keyframes stamped at or before t in an unsorted ts; t before every keyframe gives t0 = -1 (keyframe N-1 is used),
    after the last keyframe t1 = t0"""
    poses, _ = _keyframes(4, 0)
    ts = torch.tensor([0.0, 10.0, 5.0, 20.0], dtype=torch.float64)       # not sorted
    t0, t1, G = otf.interpolate(poses, ts, [-3.0, 0.0, 5.0, 7.0, 10.0, 25.0], lietorch.SE3)
    assert t0.tolist() == [-1, 0, 1, 1, 2, 3]
    assert t1.tolist() == [0, 1, 2, 2, 3, 3]
    # at keyframe t0's own stamp the interpolation is that keyframe (w = 0); with an unsorted ts, t0 need not be the keyframe stamped t
    assert torch.allclose(G[1], poses[0], atol=1e-12)
    assert not torch.allclose(G[4], poses[2], atol=1e-6)
    # t0 = -1 interpolates from keyframe N-1 (ts[-1] = 20) towards keyframe 0
    dt = ts[0] - ts[3] + 1e-3
    w = (lietorch.SE3(poses[0:1]) * lietorch.SE3(poses[3:4]).inv()).log() / dt * (-3.0 - ts[3])
    want = (lietorch.SE3.exp(w) * lietorch.SE3(poses[3:4])).data[0]
    assert torch.allclose(G[0], want, atol=1e-12)


def test_interpolation_is_linear_in_the_tangent_space():
    """pure translations interpolate linearly (dt carries the reference's + 1e-3); a rotation's angle grows linearly"""
    poses = torch.zeros(2, 7, dtype=torch.float64)
    poses[:, 6] = 1
    poses[1, :3] = torch.tensor([1.0, -2.0, 0.5])
    ts = torch.tensor([0.0, 4.0], dtype=torch.float64)
    _, _, G = otf.interpolate(poses, ts, [1.0, 3.0], lietorch.SE3)
    for k, t in enumerate((1.0, 3.0)):
        assert torch.allclose(G[k, :3], poses[1, :3] * t / (4.0 + 1e-3), atol=1e-12)
    rot = lietorch.SE3.exp(torch.tensor([[0.0, 0.0, 0.0, 0.0, 0.0, 0.8]], dtype=torch.float64)).data
    poses[1] = rot[0]
    _, _, G = otf.interpolate(poses, ts, [2.0], lietorch.SE3)
    ang = 2 * torch.atan2(G[0, 3:6].norm(), G[0, 6])
    assert abs(float(ang) - 0.8 * 2.0 / (4.0 + 1e-3)) < 1e-12


def test_fp32_interpolation_error_of_the_stand_in():
    """lietorch's formulas in fp32 against fp64, the yardstick of the device kernel's bound (tests/test_trajectory_filler_gpu.py): about
    1e-7 of (1 + |t|) between keyframes; frames extrapolated far beyond a bracket (large tangent steps) lose up to a few 1e-5"""
    poses, g = _keyframes(12, 3)
    ts = torch.sort(torch.rand(12, generator=g, dtype=torch.float64) * 100).values
    tq = (torch.rand(64, generator=g, dtype=torch.float64) * 110 - 5).tolist()
    _, _, G64 = otf.interpolate(poses, ts, tq, lietorch.SE3)
    _, _, G32 = otf.interpolate(poses.float(), ts.float(), tq, lietorch.SE3)
    err = (G32.double() - G64).abs().amax(dim=1) / (1 + G64[:, :3].norm(dim=1))
    assert float(err.median()) < 2e-7 and float(err.max()) < 1e-4, (float(err.median()), float(err.max()))


def test_capi_filler_symbols_and_argument_checks():
    L = c_api.load()
    for name in ("dba_fill_interpolate", "dba_pose_only_ba"):
        assert name in c_api.SYMBOLS and hasattr(L, name)
    assert L.dba_fill_interpolate(None, None, 0, None, 0, None, None, None, None) == 0           # nothing to do: no launch
    assert L.dba_fill_interpolate(None, None, 0, None, 3, None, None, None, None) == 1           # no keyframe
    assert b"no keyframe" in L.dba_last_error()
    assert L.dba_fill_interpolate(None, None, 2, None, 3, None, None, None, None) == 1           # null pointers
    assert L.dba_fill_interpolate(None, None, 2, None, -1, None, None, None, None) == 1          # negative extent
    args = lambda **kw: [kw.get(k, d) for k, d in (("poses", 8), ("disps", 8), ("intr", 8), ("tg", 8), ("wt", 8), ("ii", 8), ("jj", 8),
                                                   ("n", 10), ("nd", 10), ("E", 4), ("ht", 4), ("wd", 4), ("t0", 6), ("t1", 10), ("it", 2),
                                                   ("lm", 1e-4), ("ep", 0.1), ("st", 8), ("sys", None), ("dx", None), ("stream", None))]
    assert L.dba_pose_only_ba(*args(st=None)) == 1 and b"status" in L.dba_last_error()
    assert L.dba_pose_only_ba(*args(t0=7, t1=6)) == 1 and b"window" in L.dba_last_error()
    assert L.dba_pose_only_ba(*args(t1=11)) == 1
    assert L.dba_pose_only_ba(*args(ht=0)) == 1
    assert L.dba_pose_only_ba(*args(ii=None)) == 1 and b"edge" in L.dba_last_error()
    assert L.dba_pose_only_ba(*args(poses=None)) == 1


# ---- the restatement against the unmodified reference methods (tests/golden/make_trajectory_filler_golden.py) ----
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import pytest  # noqa: E402
import oracle.factor_graph as ofg  # noqa: E402
import make_trajectory_filler_golden as mtf  # noqa: E402

FILL_CASES = {c[0]: c for c in mtf.cases()}


@pytest.fixture(scope="module")
def filler_gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "trajectory_filler.pt"))


def _run_oracle(case, seed=0):
    name, n_kf, stamps = case
    video, fnet, update, mean, stdv = mtf.filler_parts(seed, n_kf)
    filler = types.SimpleNamespace(fnet=fnet, update=update, video=video, MEAN=mean, STDV=stdv)
    graph = lambda v, op: otf.FillerGraph(v, op, mtf.CorrBlock, ofg.update)
    with torch.no_grad():
        poses, edges = otf.fill(filler, mtf.stream(seed, video, stamps), graph, lietorch.SE3)
    return mtf.stored(poses, edges, video)


@pytest.mark.parametrize("name", list(FILL_CASES))
def test_restatement_matches_the_reference_filler(filler_gold, name):
    """edge lists, stamps and counter bit for bit; poses bit for bit on the CPU the fixture was made on.  Elsewhere the fp64 LAPACK
    Cholesky inside oracle.ba may round differently (CPU instruction set), so poses are held to 1e-6 (1 + |t|) there."""
    got = _run_oracle(FILL_CASES[name])
    for k, t in got.items():
        want = filler_gold[name + "/" + k]
        if k in ("poses", "video_poses"):
            err = (t.double() - want.double()).abs().amax(dim=1) / (1 + want[:, :3].double().norm(dim=1))
            assert float(err.max()) <= 1e-6, (name, k, float(err.max()))
        else:
            assert torch.equal(t, want), (name, k)


def test_filler_cases_exercise_the_reference_behaviours(filler_gold):
    g = filler_gold
    assert int(g["mixed_19/n_batches"]) == 2 and g["mixed_19/poses"].shape == (19, 7)         # 16 + 3 frames
    assert int(g["before_first_17/ii0"].min()) == -1                                          # t0 = -1: the buffer's last slot
    n = len(FILL_CASES["after_last_5"][2])
    assert g["after_last_5/ii0"].numel() < 2 * n                                              # t0 == t1 drops the duplicate edge
    assert int(g["mixed_19/counter"]) == FILL_CASES["mixed_19"][1]                            # counter restored
