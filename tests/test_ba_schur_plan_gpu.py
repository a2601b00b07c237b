"""The one-launch Schur complement's work split, every stage against fp64 (tests/test_ba_stages_gpu.py's checks and bounds).

ba_schur_tc_kernel runs one CTA per SM.  The packed and single-tile frames form one cost line (one unit per 64-pixel packed chunk, two
per 32-pixel single-tile chunk), and CTA b takes the chunks that start in [b T / SMs, (b + 1) T / SMs).  The tile pairs of frames above
21 rows are a flat list that the CTAs take round-robin.  Each case below puts that split at an edge: more frames than SMs, fewer chunks
than SMs, one frame spread over many CTAs, CTAs whose share crosses a packed and a single-tile frame, and all three routes in one
launch.  `plan` restates the split, so that each case checks that it reaches the edge it is named for."""
import pytest
import torch

from droid_slam_b200 import synth
from test_ba_stages_cpu import _sliding, _targets, boundary_graph, route, rows_per_frame
from test_ba_stages_gpu import _report, run_stages

pytestmark = pytest.mark.gpu


def _graph(N, big=None):
    """sliding window of radius 2, with frames f of `big` given big[f] rows instead (targets inside [1, N))"""
    big = big or {}
    e = _sliding(N, skip=big)
    for f, r in big.items():
        e += [(f, j) for j in _targets(f, r - 1, 1, N)]
    return [a for a, _ in e], [b for _, b in e]


def plan(ii, jj, N, t0, t1, HW, sms):
    """(routes of the depth frames, [per CTA: the (frame, route) parts of its cost interval], tile-pair items per CTA)"""
    ii, jj = torch.as_tensor(ii), torch.as_tensor(jj)
    kx = torch.unique(torch.cat([torch.arange(t0, t1), ii])).tolist()
    rows, deg = rows_per_frame(ii, jj, N, t0, t1), torch.bincount(ii, minlength=N)
    routes = [route(int(rows[f]), int(deg[f])) for f in kx]
    cdiv = lambda a, b: -(-a // b)
    cost = [0 if r in (None, "pair") else cdiv(HW, 64) if r == "packed" else 2 * cdiv(HW, 32) for r in routes]
    off = [sum(cost[:m]) for m in range(len(cost) + 1)]
    T = off[-1]
    parts = []
    for b in range(sms):
        lo, hi = b * T // sms, (b + 1) * T // sms
        w = lambda m: 1 if routes[m] == "packed" else 2
        parts.append([(kx[m], routes[m]) for m in range(len(kx)) if cost[m] and
                      any(lo <= off[m] + c * w(m) < hi for c in range(cost[m] // w(m)))])
    tiles = lambda m: cdiv(int(rows[kx[m]]), 10)
    npair = sum(tiles(m) * (tiles(m) - 1) // 2 for m in range(len(kx)) if routes[m] == "pair")
    return routes, parts, [len(range(b, npair, sms)) for b in range(sms)]


def _case(ii, jj, N, ht, wd, seed, t0=1, t1=None):
    t1 = N if t1 is None else t1
    s = synth.make_scene(dict(E=len(ii), N=N, ht=ht, wd=wd, stereo=False, itrs=2, lm=1e-4, ep=0.1, graph=(torch.tensor(ii), torch.tensor(jj)),
                              t0=t0, t1=t1), seed=seed)
    s.update(itrs=2, eta_by_frame=False, ws_fill=None, kx=torch.unique(torch.cat([torch.arange(t0, t1), s["ii"]])))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return s, plan(ii, jj, N, t0, t1, ht * wd, sms)


def test_more_depth_frames_than_sms(capi):
    N = 200
    s, (routes, parts, _) = _case(*_graph(N), N, 8, 12, seed=11)
    assert len(routes) > len(parts) and set(routes) == {"packed"}
    assert max(len(p) for p in parts) >= 2            # 2 chunks per frame: CTAs take parts of several frames
    _report("plan_200_frames_8x12", run_stages(capi, s))


def test_fewer_chunks_than_sms_one_frame(capi):
    N = 5
    ii, jj = [2, 2, 2, 2], [0, 1, 3, 4]
    s, (routes, parts, _) = _case(ii, jj, N, 3, 5, seed=12)
    assert [r for r in routes if r] == ["packed"]
    assert sum(1 for p in parts if p) == 1             # the one 64-pixel chunk: one CTA works, the others find nothing
    _report("plan_one_frame_3x5", run_stages(capi, s))


@pytest.mark.parametrize("rows", [6, 16], ids=["packed", "single"])
def test_one_frame_over_many_ctas(capi, rows):
    N = 20
    ii, jj = [5] * (rows - 1), _targets(5, rows - 1, 1, N)
    s, (routes, parts, _) = _case(ii, jj, N, 96, 128, seed=13)
    assert [r for r in routes if r] == ["packed" if rows <= 10 else "single"]
    assert sum(1 for p in parts if p) >= 96            # 192 packed / 768 single-tile cost units over the SMs
    _report("plan_one_frame_%d_rows_96x128" % rows, run_stages(capi, s))


def test_cta_share_crosses_packed_and_single_frames(capi):
    N = 40
    s, (routes, parts, _) = _case(*_graph(N, {f: 16 for f in range(4, 36, 3)}), N, 16, 24, seed=14)
    assert {"packed", "single"} <= set(routes)
    assert any({"packed", "single"} <= {r for _, r in p} for p in parts)
    _report("plan_packed_single_crossing_16x24", run_stages(capi, s))


def test_pair_frames_with_packed_and_single_in_one_launch(capi):
    N = 40
    ii, jj, _ = boundary_graph(N)
    s, (routes, parts, items) = _case(ii, jj, N, 12, 16, seed=15)
    assert {"packed", "single", "pair"} <= set(routes)
    assert max(items) >= 2 and any(p and n for p, n in zip(parts, items))   # CTAs with a cost share and tile pairs
    _report("plan_all_routes_12x16", run_stages(capi, s))
