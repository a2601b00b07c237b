"""The update operator (`dba_update_forward`) stage by stage against fp64 on the GPU: every case of tests/test_update_stages_cpu.py
runs through the C ABI on a NaN-filled workspace with every output inside a NaN-filled buffer with guard margins, and every stage of
that table is checked on the intermediates the kernels left in the workspace (located by `dba_update_workspace_layout`), with the fp64
references computed on the GPU.  The guards must come back untouched and no output may keep a NaN.  The 512-edge cases check the
per-edge stages on 16 edges: the first, the last and those whose tiles straddle a wave of the persistent z|r and q convolutions; the
global context, the segment means and the aggregation outputs on every row.

Non-finite inputs: a NaN in corr or net propagates like it does through the reference (torch.relu keeps NaN), to exactly the pixels
whose receptive field holds it; every other output is bit-identical to the call without the NaN.

Worst kappa per stage over the case table (|err| past the output's rounding interval, or the fp32 |err|, in units of u times: A for
the convolutions, sum |h| over the slot for gate_partial, |b| + sum |W g| for global_context, sum |Y| + |b| for delta, the mean |term|
for segment_mean, 1 for weight and eta) and the smallest fraction of f16 outputs equal to the correctly rounded fp64 value, measured on
one H100 80GB HBM3 at a 700 W power limit (the committed bounds are derived, tests/test_update_stages_cpu.py; none is tightened):
  corr_encoder.0   3.12  0.9993      z              4.16  0.9832      segment_mean   1.25  0.9982
  corr_encoder.2   6.01  0.9970      rh             4.81  0.9824      agg.conv2      5.16  0.9966
  flow_encoder.0   2.44  0.9993      hidden        18.6   0.9855      upmask         3.52  0.9983
  flow_encoder.2   5.47  0.9969      stems          5.11  0.9971      eta_partials   4.98
  gate_partial    49.5               head_partials  4.91              eta            0.357
  global_context  17.9               delta          3.12              layout         0     1 (bit-equal)
                                     weight         1.61
The convolutions stay near 0.1 sqrt(K), as in tests/test_tensor_core_fp64_gpu.py.  gate_partial (bound ~ EPS_S / u = 4100 plus the
conv term) and hidden (whose bound carries EPS_T |q|) are dominated by tanh.approx, far inside its documented error.  A scratch build
whose glo_kernel leaves out slot 0 fails 21 of the 23 table and NaN cases here (at global_context); the end-to-end tests catch it
only at 10x40, 9x13 and in the 16x64 emulation comparison.  A scratch build whose segment mean divides by n + 1 for segments of more
than one edge fails 16 here (at segment_mean) and 11 end-to-end tests.
"""
import ctypes
import json
import os

import pytest
import torch

from droid_slam_b200 import c_api
from droid_slam_b200.update import PACKED_ORDER, UpdateModule
from test_tensor_core_fp64_cpu import conv_plan
from test_tensor_core_fp64_gpu import Guarded
from test_update_stages_cpu import CASE_IDS, CASES, UPWS, case_inputs, case_segments, case_weights, check_stages, slot_of_pixel, workspace_layout
from util import assert_bit_identical

pytestmark = pytest.mark.gpu
DEV = "cuda"
DT = {torch.float16: c_api.DBA_F16, torch.float32: c_api.DBA_F32}

# dtype and row shape of each workspace intermediate (channels-last rows of HW pixels; partial / glo per edge)
WS_VIEWS = dict(hin=(torch.float16, 128), x320=(torch.float16, 320), c1=(torch.float16, 128), f1=(torch.float16, 128), z=(torch.float16, 128),
                rh=(torch.float16, 128), s=(torch.float16, 384), am=(torch.float16, 128), b2=(torch.float16, 128), yh=(torch.float32, 36),
                ye=(torch.float32, 12))


def _report(name, res):
    stats = {k: [None if v[0] != v[0] else round(v[0], 4), float("%.3g" % v[1])] for k, v in res.items()}
    print("UPDATE_STAGES %s %s" % (name, json.dumps(stats)))
    out = os.environ.get("UPDATE_STAGES_REPORT")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(dict(case=name, **stats)) + "\n")


def run_forward(L, pk, net, inp, corr, flow, seg, n_src, layout):
    """one dba_update_forward call on a NaN-filled workspace, outputs in guarded NaN buffers -> (workspace views, outputs, guards)"""
    E = inp.shape[0]
    ht, wd = inp.shape[2:]
    HW = ht * wd
    W = c_api.UpdateWeights(*[pk[k].data_ptr() for k in PACKED_ORDER])
    nbytes = L.dba_update_workspace_bytes(E, n_src, ht, wd)
    ws = torch.full((nbytes,), 255, dtype=torch.uint8, device=DEV)             # every f16 and f32 in it NaN
    assert ws.data_ptr() % 256 == 0
    g = dict(net_out=Guarded(E, ht, wd, 128), delta=Guarded(E, ht, wd, 2, dtype=torch.float32), weight=Guarded(E, ht, wd, 2, dtype=torch.float32))
    if n_src:
        g.update(eta=Guarded(n_src, ht, wd, dtype=torch.float32), upmask=Guarded(n_src, 576, ht, wd))
    p = lambda k: g[k].t.data_ptr() if k in g else None
    a = c_api.UpdateArgs(E, ht, wd, net.data_ptr(), DT[net.dtype], layout, inp.data_ptr(), DT[inp.dtype], corr.data_ptr(), DT[corr.dtype],
                         flow.data_ptr() if flow is not None else None, seg.data_ptr() if seg is not None else None, n_src, ctypes.pointer(W),
                         p("net_out"), p("delta"), p("weight"), p("eta"), p("upmask"), ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream)
    c_api.check(L.dba_update_forward(ctypes.byref(a)), "update_forward")
    torch.cuda.synchronize()
    offs, slots = workspace_layout(L, E, n_src, ht, wd)

    def view(k, dt, n, rows):
        nb = rows * n * torch.finfo(dt).bits // 8
        return ws[offs[k]:offs[k] + nb].view(dt).view(rows, n)

    st = {}
    for k, (dt, c) in WS_VIEWS.items():
        rows = (max(n_src, 1) if k in ("am", "b2", "ye") else E) * HW
        st[k] = view(k, dt, c, rows).view(-1, ht, wd, c)
    st["partial"] = view("partial", torch.float32, 128, E * slots).view(E, slots, 128)
    st["glo"] = view("glo", torch.float32, 384, E)
    return st, {k: v.t for k, v in g.items()}, g


def sample_edges(L, E, ht, wd, k):
    """k edges: the first, the last and the edges of the tiles on either side of each wave boundary of the persistent z|r and q
    convolutions (grid = min(tiles, SMs)), then evenly spread ones"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pick = [0, E - 1]
    for c0, c1, n in ((128, 320, 256), (128, 320, 128), (128, 0, 384)):
        p = conv_plan(L, ht, wd, c0, c1, 3, n)
        tpi = p["tiles"]
        total = p["n_ntiles"] * E * tpi
        grid = min(total, sms)
        for w in range(1, 4):
            for t in (w * grid - 1, w * grid):
                if t < total:
                    pick.append((t % (E * tpi)) // tpi)
    pick = list(dict.fromkeys(pick))
    for e in torch.linspace(0, E - 1, k).round().long().tolist():
        if len(pick) >= k:
            break
        if e not in pick:
            pick.append(e)
    return sorted(pick[:max(k, 2)])


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_update_stages_match_fp64(capi, case):
    name, E, ht, wd, segs, n_src, opt = case
    sd, pk = case_weights(case)
    pk = {k: v.to(DEV) for k, v in pk.items()}
    seg, n_src = case_segments(case)
    seg = seg.to(DEV) if seg is not None else None
    net, inp, corr, flow = case_inputs(case, device=DEV)
    layout = opt.get("layout", 0)
    if layout == 1:
        net = net.half().permute(0, 2, 3, 1).contiguous()
    st, out, guards = run_forward(capi, pk, net, inp, corr, flow, seg, n_src, layout)
    for k, gd in guards.items():
        gd.check_guards("update_forward %s %s" % (name, k))
        assert not bool(torch.isnan(gd.t).any()), "%s: %s keeps a NaN" % (name, k)
    if n_src == 0:
        # MotionFilter's call: stems 256 wide, nothing aggregated
        assert bool((st["s"][..., 256:].contiguous().view(torch.int16) == -1).all()), "%s: stems wider than 256 without aggregation" % name
        assert bool((st["am"].contiguous().view(torch.int16) == -1).all()), "%s: segment mean written without aggregation" % name
    edges = sample_edges(capi, E, ht, wd, opt["sample"]) if opt.get("sample") else None
    ins = dict(net=net, inp=inp, corr=corr, flow=flow, layout=layout, seg=seg, n_src=n_src)
    res = check_stages(pk, ins, st, out, slot_of_pixel(capi, ht, wd), edges)
    _report(name, res)


# ---- non-finite inputs -------------------------------------------------------------------------------------------------------
def _dilate(mask, r):
    """[N,H,W] bool -> pixels within Chebyshev distance r (the receptive field of r stacked 3x3 convolutions)"""
    if r == 0:
        return mask
    return torch.nn.functional.max_pool2d(mask.float()[:, None], 2 * r + 1, stride=1, padding=r)[:, 0] > 0


@pytest.mark.parametrize("where", ["corr", "net"])
def test_nan_input_propagates_like_the_reference(capi, where):
    """A NaN in corr reaches exactly the pixels whose receptive field holds it (the reference's torch.relu keeps NaN; the encoders'
    ReLU must not turn it into 0); a NaN in net makes its edge's global context NaN, so that edge's outputs and its segment's
    aggregation outputs are NaN everywhere.  Every other output is bit-identical to the call without the NaN."""
    case = ("nan", 6, 20, 40, "rand", 3, {})
    sd, pk = case_weights(case)
    pk = {k: v.to(DEV) for k, v in pk.items()}
    seg, n_src = case_segments(case)
    seg = seg.to(DEV)
    net, inp, corr, flow = case_inputs(case, device=DEV)
    e, y, x = 2, 7, 33
    clean = run_forward(capi, pk, net, inp, corr, flow, seg, n_src, 0)[1]
    bad_net, bad_corr = net.clone(), corr.clone()
    if where == "corr":
        bad_corr[e, 5, y, x] = float("nan")
    else:
        bad_net[e, 7, y, x] = float("nan")
    got = run_forward(capi, pk, bad_net, inp, bad_corr, flow, seg, n_src, 0)[1]
    E, ht, wd = 6, 20, 40
    px = torch.zeros(E, ht, wd, dtype=torch.bool, device=DEV)
    px[e, y, x] = True
    src = torch.zeros(n_src, ht, wd, dtype=torch.bool, device=DEV)
    if where == "corr":
        # c1 at the pixel, X320 1, z / r*h 2, net_out 3, stems 4, delta / weight 5; segment mean 4, agg.conv2 and upmask 5, eta 6
        src[seg[e]] = _dilate(px, 4)[e]
        want = dict(net_out=_dilate(px, 3), delta=_dilate(px, 5), weight=_dilate(px, 5), eta=_dilate(src, 2), upmask=_dilate(src, 1))
    else:
        full = torch.zeros_like(px)
        full[e] = True
        src[seg[e]] = True
        want = dict(net_out=full, delta=full, weight=full, eta=src, upmask=src)
    for k, m in want.items():
        a, b = got[k], clean[k]
        m = m[..., None] if k in ("net_out", "delta", "weight") else (m[:, None] if k == "upmask" else m)
        m = m.expand(a.shape)
        assert torch.equal(torch.isnan(a), m), "%s: NaN in %s reaches %d outputs, the reference %d" % (k, where, int(torch.isnan(a).sum()), int(m.sum()))
        assert_bit_identical(a[~m], b[~m], "%s outside the NaN's receptive field" % k)


# ---- batches -----------------------------------------------------------------------------------------------------------------
def test_update_module_batch_of_two_equals_two_calls():
    """UpdateModule.forward with batch = 2 offsets the second batch's segments by the number of sources (update.py): the result is
    the two batch-1 calls, bit for bit"""
    case = ("batch", 7, 24, 32, "uneven", 3, {})
    sd, _ = case_weights(case)
    mod = UpdateModule().to(DEV)
    mod.load_state_dict(sd)
    ii = torch.tensor([4, 9, 4, 2, 9, 9, 4], device=DEV)
    ins = [case_inputs(case, device=DEV, seed=s) for s in (0, 1)]
    with torch.no_grad():
        both = mod(*[torch.stack([a, b]).half() if i < 3 else torch.stack([a, b]) for i, (a, b) in enumerate(zip(*ins))], ii)
        one = [mod(*[t[None].half() if i < 3 else t[None] for i, t in enumerate(x)], ii) for x in ins]
    torch.cuda.synchronize()
    assert both[3].shape == (2, 3, 24, 32) and both[4].shape == (2, 3, 576, 24, 32)
    for k in range(5):
        assert_bit_identical(both[k], torch.cat([one[0][k], one[1][k]]), "output %d" % k)
