"""The update operator (`dba_update_forward`, csrc/update_op.cu) stage by stage against fp64: the case table, the per-stage fp64
references and their error bounds, which tests/test_update_stages_gpu.py applies to the intermediates the kernels leave in the
workspace (located by `dba_update_workspace_layout`).  Each stage is checked from its own inputs as the previous kernel left them,
so errors do not compound; here the same checks run on an fp32 restatement of the kernels (their roundings, tanh.approx perturbed
by its documented error) and must accept it, and must reject each of a list of planted faults by the name of the stage it breaks.

Notation: u = 2^-24; for a convolution A = conv(|x|, |w|) + |b| (the sum of the magnitudes of its terms, |glo| added where the
global context enters) and c = 0.5 sqrt(K) u A, the bound tests/test_tensor_core_fp64_gpu.py holds the convolution engine to.
EPS_T is the maximum relative error the PTX ISA documents for tanh.approx.f32, 2^-10.987; sigmoid_fast(x) = fma(0.5,
tanh.approx(x / 2), 0.5) is then within EPS_S = EPS_T / 2 + u.  __expf is within 2 + floor(1.173 |x|) ulp and log1pf within 1 ulp
(CUDA C++ Programming Guide, mathematical functions).

  stage            output                    fp64 reference from                               bound
  layout           HIN, X320[:128]           f16(net), f16(inp)                                bit-equal
  corr_encoder.0   C1                        relu(conv1x1(f16 corr))                           faithful f16, beta = c (ReLU is 1-Lipschitz)
  corr_encoder.2   X320[128:256]             relu(conv3x3(C1))                                 faithful, c
  flow_encoder.0   F1                        relu(conv7x7(f16 flow)), flow None = zeros         faithful, c
  flow_encoder.2   X320[256:320]             relu(conv3x3(F1))                                 faithful, c
  gate_partial     PARTIAL [E,slots,128]     sum over each 16-pixel slot of sigmoid(conv1x1(h)) h   sum |h| (EPS_S + c/4) + 5u sum |sigma h|
  global_context   GLO [E,384] f32           b_glo + W_glo (sum of the slots / HW)            sum_k |W| (slots + 2) u sum|slots| / HW + 130 u (|b| + sum |W g|)
  z, rh            Z, RH                     sigmoid(conv3x3([h | X320]) + GLO)(, * h)         faithful, EPS_S + c/4 (times |h|, plus u |rh|)
  hidden           net_out                   (1 - z) h + z tanh(conv3x3([RH | X320]) + GLO_q)  faithful, z (EPS_T |q| + c) + 3u (|h| + |z h| + |z q|)
  stems            S[:256 or 384]            relu(conv3x3(net_out))                            faithful, c
  head_partials    YH [E,HW,36] f32          per-tap 1x1 partials of S[:256]                   gamma_K A (fp32 sums of K = 256 terms)
  delta, weight    [E,HW,2] f32              b + 9-tap gather of YH; sigmoid                   10 u (sum |Y| + |b|); sigma (1 - sigma) (that + __expf) + 2u sigma
  segment_mean     AM                        scatter-mean of S[256:384] over each segment      faithful, (n_e + 2) u mean |terms|
  agg.conv2        B2                        relu(conv3x3(AM))                                 faithful, c
  upmask           [n_src,576,HW] f16        conv1x1(B2), NCHW                                 faithful, c
  eta_partials     YE [n_src,HW,12] f32      per-tap 1x1 partials of B2                        gamma_K A
  eta              [n_src,HW] f32            0.01 softplus(b + gather of YE), threshold 20     0.01 (sigma (gather + __expf) + 2^-23 sp) + 2u eta
The global context is checked in two steps, the slot partials and then their sum, which keeps each bound at its own stage's rounding:
one 16-pixel slot left out of the sum moves GLO by |W| |slot| / HW, thousands of times that summation bound.

No convolution of the operator is planned with MT = 4 (that takes n_out <= 64, a 3x3 kernel and >= 4 K blocks), so the route
coverage asks for MT 1 and 2 on both tilings, and fails if a retune makes MT 4 reachable without a case for it."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from droid_slam_b200 import c_api, synth
from droid_slam_b200.update import pack_update_weights
from test_tensor_core_fp64_cpu import H100_SMS, conv_plan
from util import assert_faithful_f16

U = 2.0 ** -24
EPS_T = 2.0 ** -10.987
EPS_S = EPS_T / 2 + U
F32_TINY = 2.0 ** -126                    # __expf / ex2.approx flush results below the smallest normal to zero
C01 = abs(float(np.float32(0.01)) - 0.01) / 0.01     # relative error of the constant 0.01f
KAPPA_CONV = 0.5                          # c = KAPPA_CONV sqrt(K) u A

UPWS = ("hin", "x320", "cc", "f0", "c1", "f1", "z", "rh", "s", "partial", "glo", "am", "b2", "yh", "ye")

# the operator's convolutions: (name, c0, c1, ksize, n_out as planned)
OPERATOR_CONVS = [("corr0", 196, 0, 1, 128), ("corr2", 128, 0, 3, 128), ("flow0", 196, 0, 1, 128), ("flow2", 128, 0, 3, 64),
                  ("gate", 128, 0, 1, 128), ("zr", 128, 320, 3, 256), ("q", 128, 320, 3, 128), ("stem", 128, 0, 3, 384),
                  ("heads", 256, 0, 1, 64), ("agg2", 128, 0, 3, 128), ("eta", 128, 0, 1, 32), ("upmask", 128, 0, 1, 192)]
AGG_CONVS = ("agg2", "eta", "upmask")


# ---- case table --------------------------------------------------------------------------------------------------------------
# (name, E, ht, wd, segments, options).  segments: "rand" (synth's unsorted, non-contiguous frame numbers over n_src sources),
# "one" (one segment), "single" (every edge its own source), "uneven" (sizes 1..9 over unsorted, non-contiguous frames), "bench"
# (every one of n_src sources, ~E / n_src edges each), "none" (n_src = 0: no aggregation).  Options: net / inp / corr dtype and
# net layout, flow None, "large" (corr x 8, inp x 4 as real features are: saturates the gates), "eta_bias" (agg.eta.0 bias 20: its
# pre-activation on both sides of the softplus threshold), "weight_bias" (weight.2 biases +-90: __expf overflows), "sample" (per-edge
# stages on a sample of edges).
def _case(name, E, ht, wd, segs, n_src, **opt):
    return (name, E, ht, wd, segs, n_src, opt)


CASES = [
    _case("tw64_48x64", 6, 48, 64, "rand", 3),
    _case("tw64_16x64_f32_net", 5, 16, 64, "rand", 3, net="f32"),
    _case("tw32_72x96", 6, 72, 96, "uneven", 4, inp="f32", corr="f32"),
    _case("tw32_24x32_channels_last", 6, 24, 32, "rand", 3, layout=1),
    _case("flat_43x70", 6, 43, 70, "rand", 3),
    _case("flat_44x69_no_flow", 6, 44, 69, "one", 1, flow=False),
    _case("flat_41x73_odd_hw", 6, 41, 73, "single", 6, net="f32"),
    _case("flat_9x13", 6, 9, 13, "rand", 3),
    _case("tiny_1x1", 6, 1, 1, "rand", 2),
    _case("e1_16x64", 1, 16, 64, "rand", 1),
    _case("e1_9x13_odd", 1, 9, 13, "rand", 1, net="f32", layout=0),
    _case("one_segment_40_edges", 40, 12, 40, "one", 1),
    _case("uneven_segments_43x70", 30, 43, 70, "uneven", 7),
    _case("no_aggregation_48x64", 6, 48, 64, "none", 0),
    _case("no_aggregation_41x73", 5, 41, 73, "none", 0, flow=False),
    _case("large_features_48x64", 6, 48, 64, "rand", 3, large=True),
    _case("large_features_43x70", 6, 43, 70, "rand", 3, large=True, layout=1),
    _case("eta_threshold_16x64", 6, 16, 64, "rand", 3, eta_bias=True),
    _case("weight_overflow_24x32", 6, 24, 32, "rand", 3, weight_bias=True),
    _case("bench_512_edges_48x64", 512, 48, 64, "bench", 72, sample=16),
    _case("c5_rank_512_edges_72x96", 512, 72, 96, "bench", 63, sample=16),
]
CASE_IDS = [c[0] for c in CASES]


def case_weights(case):
    """state dict (synth.make_update_weights(0) with the case's bias changes) and its packed form"""
    opt = case[6]
    sd = synth.make_update_weights(0)
    if opt.get("eta_bias"):
        sd["agg.eta.0.bias"] = sd["agg.eta.0.bias"] + 20.0
    if opt.get("weight_bias"):
        sd["weight.2.bias"] = sd["weight.2.bias"] + torch.tensor([90.0, -90.0])
    return sd, pack_update_weights(sd)


def case_segments(case, seed=0):
    """ii [E] (frame numbers, unsorted and non-contiguous) -> (seg = rank among the distinct sources, n_src), or (None, 0)"""
    name, E, ht, wd, segs, n_src, opt = case
    g = torch.Generator().manual_seed(7 + E + seed)
    if segs == "none":
        return None, 0
    if segs == "one":
        ii = torch.full((E,), 5)
    elif segs == "single":
        ii = torch.randperm(E, generator=g) * 2 + 1
    elif segs == "uneven":
        sizes = [1 + (3 * k) % 9 for k in range(n_src)]
        while sum(sizes) > E:
            sizes[sizes.index(max(sizes))] -= 1
        sizes[-1] += E - sum(sizes)
        assert min(sizes) >= 1
        ii = torch.cat([torch.full((s,), 11 * k + 3) for k, s in enumerate(sizes)])[torch.randperm(E, generator=g)]
    elif segs == "bench":
        ii = torch.cat([torch.arange(n_src), torch.randint(0, n_src, (E - n_src,), generator=g)])[torch.randperm(E, generator=g)] * 3 + 2
    else:
        ii = torch.randint(0, n_src, (E,), generator=g) * 3 + 2
        ii[torch.randperm(E, generator=g)[:n_src]] = torch.arange(n_src) * 3 + 2        # every source present
    uniq, seg = torch.unique(ii, return_inverse=True)
    assert uniq.numel() == n_src
    return seg, n_src


def case_inputs(case, device="cpu", seed=0):
    """net, inp [E,128,ht,wd], corr [E,196,ht,wd] in the case's dtypes, flow [E,4,ht,wd] f32 or None (the synth distribution)"""
    name, E, ht, wd, segs, n_src, opt = case
    g = torch.Generator(device=device).manual_seed(1000 * E + 10 * ht + wd + seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=device)
    net = torch.tanh(rn(E, 128, ht, wd))
    inp = torch.relu(rn(E, 128, ht, wd))
    corr = rn(E, 196, ht, wd)
    flow = 4.0 * rn(E, 4, ht, wd)
    if opt.get("large"):
        corr, inp = corr * 8, inp * 4
    dt = lambda k: torch.float32 if opt.get(k, "f16") == "f32" else torch.float16
    return net.to(dt("net")), inp.to(dt("inp")), corr.to(dt("corr")), (flow if opt.get("flow", True) else None)


# ---- layouts and plans --------------------------------------------------------------------------------------------------------
def workspace_layout(L, E, n_src, ht, wd):
    offs = (ctypes.c_size_t * len(UPWS))()
    slots = ctypes.c_int(0)
    c_api.check(L.dba_update_workspace_layout(E, n_src, ht, wd, ctypes.cast(offs, ctypes.c_void_p), ctypes.byref(slots)), "update_workspace_layout")
    return dict(zip(UPWS, list(offs))), slots.value


def slot_of_pixel(L, ht, wd):
    """[ht*wd] EPI_GATE slot of every pixel (conv_engine.cuh: slot = ((ty tiles_x + tx) MT + t) 8 + the warp's 16 of the M tile's
    128 pixels), from the plan of the gate convolution, and the slot count"""
    p = conv_plan(L, ht, wd, 128, 0, 1, 128)
    y, x = torch.meshgrid(torch.arange(ht), torch.arange(wd), indexing="ij")
    y, x = y.reshape(-1), x.reshape(-1)
    if p["flat"]:
        return (y * p["TW"] + x) // 16, p["tiles"] * p["MT"] * 8           # flat index on the row pitch, 128 MT per CTA tile
    tw, mt = p["TW"], p["MT"]
    rm = 128 // tw
    tiles_x = (wd + tw - 1) // tw
    ty, r = y // (mt * rm), y % (mt * rm)
    t, my = r // rm, r % rm
    tx, mx = x // tw, x % tw
    return ((ty * tiles_x + tx) * mt + t) * 8 + (my * tw + mx) // 16, p["tiles"] * mt * 8


# ---- fp64 references and checks ----------------------------------------------------------------------------------------------
def wconv(pk, name, k, cin):
    """packed [k*k][N][Kpad] f16 -> reference layout [N, cin, k, k] fp64"""
    w = pk[name]
    return w.view(k, k, w.shape[1], w.shape[2]).permute(2, 3, 0, 1)[:, :cin].double()


def conv_ref(x, w, b, extra=None):
    """channels-last x [N,H,W,C] (any float dtype; values taken exactly), w [Co,C,k,k] fp64, b [Co] -> fp64 exact and A, [N,H,W,Co]"""
    k = w.shape[-1]
    xd = x.double().permute(0, 3, 1, 2)
    bd = b.double().to(xd.device)
    w = w.to(xd.device)
    ex = F.conv2d(xd, w, bd, padding=k // 2).permute(0, 2, 3, 1)
    A = F.conv2d(xd.abs(), w.abs(), bd.abs(), padding=k // 2).permute(0, 2, 3, 1)
    if extra is not None:
        ex, A = ex + extra, A + extra.abs()
    return ex, A


def cbound(A, K):
    return KAPPA_CONV * math.sqrt(K) * U * A


def sigmoid(x):
    return torch.sigmoid(x)


def gather9(y, no):
    """y [N,H,W,9 no] per-tap partials -> [N,H,W,no] and sum of magnitudes: out[p] = sum_t y[p + shift_t][t no + o] (zero outside)"""
    N, H, W, _ = y.shape
    yp = F.pad(y, (0, 0, 1, 1, 1, 1))
    out, mag = 0, 0
    for t in range(9):
        dy, dx = t // 3, t % 3
        v = yp[:, dy:dy + H, dx:dx + W, t * no:(t + 1) * no]
        out, mag = out + v, mag + v.abs()
    return out, mag


def assert_f32(got, exact, bound, what, unit):
    """|got - exact| <= bound elementwise (NaN only where exact is NaN); returns the worst |err| / unit"""
    got, exact = got.double(), exact.to(got.device).double()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=got.device).expand(got.shape)
    err = (got - exact).abs()
    both_nan = torch.isnan(got) & torch.isnan(exact)
    ok = (err <= bound) | both_nan
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:4].tolist()
        detail = ["%s: got %.9g exact %.9g bound %.3g" % (tuple(i), float(got[tuple(i)]), float(exact[tuple(i)]), float(bound[tuple(i)])) for i in bad]
        raise AssertionError("%s: %d of %d fp32 outputs outside the bound; %s" % (what, int((~ok).sum()), got.numel(), "; ".join(detail)))
    unit = torch.as_tensor(unit, dtype=torch.float64, device=got.device).expand(got.shape)
    need = torch.where(both_nan | (err == 0), torch.zeros_like(err), err / unit)
    return float(need.max()) if need.numel() else 0.0


def faithful(got, exact, beta, what, A=None):
    """assert_faithful_f16 with kappa reported in units of u A when A is given (u otherwise)"""
    unit = U * A if A is not None else torch.full_like(exact, U)
    return assert_faithful_f16(got, exact, beta, what, unit=unit)


def bitequal(got, want, what):
    g, w = got.contiguous().view(torch.int16), want.to(got.device).contiguous().view(torch.int16)
    same = (g == w) | (torch.isnan(got) & torch.isnan(want.to(got.device)))
    assert bool(same.all()), "%s: %d of %d elements differ from the f16 rounding of the input" % (what, int((~same).sum()), got.numel())
    return 1.0, 0.0


def check_stages(pk, ins, st, out, slot_map, edges=None):
    """Check every stage of one dba_update_forward call from its own inputs as the kernels left them.
    pk: packed weights (any device); ins: dict net, inp, corr, flow (as passed: [E,C,ht,wd]; net channels-last f16 [E,ht,wd,128] when
    layout == 1), layout, seg, n_src; st: the workspace intermediates, channels-last [E,ht,wd,C] (partial [E,slots,128], glo [E,384]);
    out: net_out [E,ht,wd,128], delta, weight [E,ht,wd,2], eta [n_src,ht,wd], upmask [n_src,576,ht,wd]; slot_map: (slot of every
    pixel, slot count); edges: the edges whose per-edge stages are checked (None: all; the global context, the segment means and the
    aggregation outputs are always checked for every row).  Returns {stage: (fraction correctly rounded, worst kappa)}; raises
    AssertionError naming the stage that fails."""
    dev = st["x320"].device
    pk = {k: v.to(dev) for k, v in pk.items()}
    E = st["x320"].shape[0]
    ht, wd = st["x320"].shape[1:3]
    HW = ht * wd
    ed = torch.arange(E, device=dev) if edges is None else torch.as_tensor(edges, device=dev)
    cl = lambda t: t.permute(0, 2, 3, 1)
    res = {}
    # layout
    H_all = ins["net"].to(dev) if ins["layout"] == 1 else st["hin"]
    if ins["layout"] == 0:
        res["layout.hin"] = bitequal(st["hin"][ed], cl(ins["net"][ed.cpu()].to(dev).half()), "layout.hin")
    res["layout.inp"] = bitequal(st["x320"][ed][..., :128], cl(ins["inp"][ed.cpu()].to(dev).half()), "layout.inp")
    H, X = H_all[ed], st["x320"][ed]
    # corr encoder
    ex, A = conv_ref(cl(ins["corr"][ed.cpu()].to(dev).half()), wconv(pk, "w_corr0", 1, 196), pk["b_corr0"])
    res["corr_encoder.0"] = faithful(st["c1"][ed], ex.clamp(min=0), cbound(A, 196), "corr_encoder.0", A)
    ex, A = conv_ref(st["c1"][ed], wconv(pk, "w_corr2", 3, 128), pk["b_corr2"])
    res["corr_encoder.2"] = faithful(X[..., 128:256], ex.clamp(min=0), cbound(A, 1152), "corr_encoder.2", A)
    # flow encoder: the 7x7 convolution with weights unfolded from K = (dy*7+dx)*4 + c
    flow = ins["flow"]
    f16flow = torch.zeros(len(ed), ht, wd, 4, dtype=torch.float16, device=dev) if flow is None else cl(flow[ed.cpu()].to(dev).half())
    w7 = pk["w_flow0"][0, :, :196].view(128, 7, 7, 4).permute(0, 3, 1, 2).double()
    ex, A = conv_ref(f16flow, w7, pk["b_flow0"])
    res["flow_encoder.0"] = faithful(st["f1"][ed], ex.clamp(min=0), cbound(A, 196), "flow_encoder.0", A)
    ex, A = conv_ref(st["f1"][ed], wconv(pk, "w_flow2", 3, 128), pk["b_flow2"])
    res["flow_encoder.2"] = faithful(X[..., 256:320], ex.clamp(min=0), cbound(A, 1152), "flow_encoder.2", A)
    # global context, every edge (in chunks): slot partials from h, then GLO from the partials
    smap, nslots = slot_map
    smap = smap.to(dev)
    part = st["partial"]
    assert part.shape[1] == nslots
    kap, kap_g = 0.0, 0.0
    wg = pk["w_glo"].double()
    for e0 in range(0, E, 32):
        hh = H_all[e0:e0 + 32]
        ex, A = conv_ref(hh, wconv(pk, "w_gate", 1, 128), pk["b_gate"])
        sg = sigmoid(ex)
        h64 = hh.double()
        n = hh.shape[0]
        flat = lambda t: t.reshape(n, HW, 128)
        exact = torch.zeros(n, nslots, 128, dtype=torch.float64, device=dev).index_add_(1, smap, flat(sg * h64))
        bound = torch.zeros_like(exact).index_add_(1, smap, flat(h64.abs() * (EPS_S + cbound(A, 128) / 4) + 5 * U * (sg * h64).abs()))
        kap = max(kap, assert_f32(part[e0:e0 + n], exact, bound, "gate_partial", U * torch.zeros_like(exact).index_add_(1, smap, flat(h64.abs()))))
        p64 = part[e0:e0 + n].double()
        g = p64.sum(1) / HW
        gm = (nslots + 2) * U * p64.abs().sum(1) / HW
        exact = g @ wg.t() + pk["b_glo"].double()
        bound = gm @ wg.abs().t() + 130 * U * (pk["b_glo"].double().abs() + g.abs() @ wg.abs().t())
        kap_g = max(kap_g, assert_f32(st["glo"][e0:e0 + n], exact, bound, "global_context", U * (pk["b_glo"].double().abs() + g.abs() @ wg.abs().t())))
    res["gate_partial"] = (float("nan"), kap)
    res["global_context"] = (float("nan"), kap_g)
    glo = st["glo"][ed].double()[:, None, None, :]
    # z, r*h
    ex, A = conv_ref(torch.cat([H, X], -1), wconv(pk, "w_zr", 3, 448), pk["b_zr"], glo[..., :256])
    sg = sigmoid(ex)
    bz = EPS_S + cbound(A, 4032) / 4
    res["z"] = faithful(st["z"][ed], sg[..., :128], bz[..., :128], "z", A[..., :128])
    h64 = H.double()
    rh = sg[..., 128:] * h64
    res["rh"] = faithful(st["rh"][ed], rh, h64.abs() * bz[..., 128:] + U * rh.abs(), "rh", A[..., 128:] * h64.abs())
    # hidden update, with z and r*h from the workspace
    ex, A = conv_ref(torch.cat([st["rh"][ed], X], -1), wconv(pk, "w_q", 3, 448), pk["b_q"], glo[..., 256:])
    q = torch.tanh(ex)
    z = st["z"][ed].double()
    hn = (1 - z) * h64 + z * q
    beta = z.abs() * (EPS_T * q.abs() + cbound(A, 4032)) + 3 * U * (h64.abs() + (z * h64).abs() + (z * q).abs())
    res["hidden"] = faithful(out["net_out"][ed], hn, beta, "hidden", A)
    # stems, heads
    n_stem = 384 if ins["n_src"] > 0 else 256
    ex, A = conv_ref(out["net_out"][ed], wconv(pk, "w_stem", 3, 128)[:n_stem], pk["b_stem"][:n_stem])
    res["stems"] = faithful(st["s"][ed][..., :n_stem], ex.clamp(min=0), cbound(A, 1152), "stems", A)
    s64 = st["s"][ed][..., :256].double()
    wh = pk["w_heads"][0, :36].double()
    exact, A = s64 @ wh.t(), s64.abs() @ wh.abs().t()
    res["head_partials"] = (float("nan"), assert_f32(st["yh"][ed], exact, 256 * U / (1 - 256 * U) * A, "head_partials", U * A))
    y, mag = gather9(st["yh"][ed].double(), 4)
    bh = pk["b_heads"].double()
    x = y + bh
    dx = 10 * U * (mag + bh.abs())
    res["delta"] = (float("nan"), assert_f32(out["delta"][ed], x[..., :2], dx[..., :2], "delta", U * (mag + bh.abs())[..., :2]))
    xw, dw = x[..., 2:], dx[..., 2:]
    sw = sigmoid(xw)
    dexp = (2 + torch.floor(1.173 * (xw.abs() + dw))) * 2.0 ** -23
    bound = 1.01 * sw * (1 - sw) * (dw + dexp) + 2 * U * sw + F32_TINY
    res["weight"] = (float("nan"), assert_f32(out["weight"][ed], sw, bound, "weight", torch.full_like(sw, U)))
    if ins["n_src"] == 0:
        return res
    # aggregation: every segment
    seg, n_src = ins["seg"].to(dev), ins["n_src"]
    a1 = st["s"][..., 256:384].double()
    ssum = torch.zeros(n_src, ht, wd, 128, dtype=torch.float64, device=dev).index_add_(0, seg, a1)
    smag = torch.zeros_like(ssum).index_add_(0, seg, a1.abs())
    cnt = torch.bincount(seg, minlength=n_src).double().view(-1, 1, 1, 1)
    del a1
    am = ssum / cnt.clamp(min=1)
    res["segment_mean"] = faithful(st["am"], am, (cnt + 2) * U * smag / cnt.clamp(min=1), "segment_mean", smag / cnt.clamp(min=1))
    del ssum, smag
    ex, A = conv_ref(st["am"], wconv(pk, "w_agg2", 3, 128), pk["b_agg2"])
    res["agg.conv2"] = faithful(st["b2"], ex.clamp(min=0), cbound(A, 1152), "agg.conv2", A)
    ex, A = conv_ref(st["b2"], wconv(pk, "w_upmask", 1, 128), pk["b_upmask"])
    res["upmask"] = faithful(out["upmask"], ex.permute(0, 3, 1, 2), cbound(A, 128).permute(0, 3, 1, 2), "upmask", A.permute(0, 3, 1, 2))
    b64 = st["b2"].double()
    we = pk["w_eta"][0, :9].double()
    exact, A = b64 @ we.t(), b64.abs() @ we.abs().t()
    res["eta_partials"] = (float("nan"), assert_f32(st["ye"][..., :9], exact, 128 * U / (1 - 128 * U) * A, "eta_partials", U * A))
    y, mag = gather9(st["ye"][..., :9].double(), 1)
    be = pk["b_eta"].double()
    x = (y + be)[..., 0]
    dx = 10 * U * (mag + be.abs())[..., 0]
    sp = torch.where(x > 20, x, torch.log1p(torch.exp(x)))
    dexp = (2 + torch.floor(1.173 * (x.abs() + dx))) * 2.0 ** -23
    bound = 0.01 * (sigmoid(x) * (dx + dexp) + 2.0 ** -23 * sp + 3e-9) + (U + C01) * 0.01 * sp + F32_TINY
    res["eta"] = (float("nan"), assert_f32(out["eta"], 0.01 * sp, bound, "eta", torch.full_like(sp, U)))
    return res


# ---- an fp32 restatement of the kernels, and planted faults ------------------------------------------------------------------
FAULTS = {
    "gate_slot_dropped": "global_context",         # glo_kernel skips one 16-pixel slot of the sum
    "glo_of_neighbour_edge": "z",                  # EPI_ZR reads the next edge's global context
    "rh_formed_with_z": "rh",                      # r*h formed with z
    "sigma_before_glo": "z",                       # sigmoid(conv) + glo instead of sigmoid(conv + glo)
    "z_unrounded_in_q": "hidden",                  # EPI_Q uses the fp32 z, the workspace holds its f16 rounding
    "flow_halo_shift_at_x64": "flow_encoder.0",    # the 7x7 im2col of the 64-pixel block at x0 = 64 shifted by one column
    "segment_mean_wrong_count": "segment_mean",    # a mean divided by n + 1
    "segment_mean_wrong_edges": "segment_mean",    # one segment summed over another segment's first edge
    "head_tap_missing_at_border": "delta",         # the gather drops tap dx = -1 of the pixels at x = 1 (reading column 0)
    "softplus_threshold_wrong_side": "eta",        # x if x < 20 else softplus(x)
    "upmask_channel_off_by_one": "upmask",         # NCHW channel 100 gets channel 101
}


def restate(pk, ins, slot_map, tanh_sign=0, fault=None):
    """the kernels' dataflow in fp32 with their f16 roundings and tanh.approx perturbed by tanh_sign * EPS_T (relative): the
    intermediates and outputs in the layout check_stages reads"""
    pk = {k: v.float() for k, v in pk.items()}
    r16 = lambda t: t.half()
    cl = lambda t: t.permute(0, 2, 3, 1)
    tanh = lambda x: torch.tanh(x) * (1 + tanh_sign * EPS_T)
    sig = lambda x: 0.5 + 0.5 * tanh(0.5 * x)

    def conv(x, name, k, cin, b, n=None):
        w = wconv(pk, name, k, cin).float()
        if n is not None:
            w, b = w[:n], b[:n]
        return F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=k // 2).permute(0, 2, 3, 1)

    st, out = {}, {}
    E, _, ht, wd = ins["inp"].shape
    HW = ht * wd
    H = ins["net"] if ins["layout"] == 1 else r16(cl(ins["net"]))
    st["hin"] = H
    inp16 = r16(cl(ins["inp"]))
    st["c1"] = r16(conv(r16(cl(ins["corr"])), "w_corr0", 1, 196, pk["b_corr0"]).relu())
    c2 = r16(conv(st["c1"], "w_corr2", 3, 128, pk["b_corr2"]).relu())
    flow = torch.zeros(E, 4, ht, wd) if ins["flow"] is None else ins["flow"]
    w7 = pk["w_flow0"][0, :, :196].view(128, 7, 7, 4).permute(0, 3, 1, 2)
    f16flow = r16(flow).float()
    f1 = F.conv2d(f16flow, w7, pk["b_flow0"], padding=3).permute(0, 2, 3, 1)
    if fault == "flow_halo_shift_at_x64":
        shifted = F.conv2d(torch.roll(f16flow, 1, dims=3), w7, pk["b_flow0"], padding=3).permute(0, 2, 3, 1)
        f1[:, :, 64:128] = shifted[:, :, 64:128]
    st["f1"] = r16(f1.relu())
    f2 = r16(conv(st["f1"], "w_flow2", 3, 128, pk["b_flow2"]).relu())
    st["x320"] = torch.cat([inp16, c2, f2], -1)
    X = st["x320"]
    smap, nslots = slot_map
    g = sig(conv(H, "w_gate", 1, 128, pk["b_gate"])) * H.float()
    st["partial"] = torch.zeros(E, nslots, 128).index_add_(1, smap, g.reshape(E, HW, 128))
    psum = st["partial"]
    if fault == "gate_slot_dropped":
        psum = psum.clone()
        psum[:, 0] = 0
    st["glo"] = (psum.sum(1) * (1.0 / HW)) @ pk["w_glo"].t() + pk["b_glo"]
    glo = st["glo"][:, None, None, :]
    if fault == "glo_of_neighbour_edge":
        glo = torch.roll(glo, 1, dims=0)
    pre = conv(torch.cat([H, X], -1), "w_zr", 3, 448, pk["b_zr"])
    zr = sig(pre) + glo[..., :256] if fault == "sigma_before_glo" else sig(pre + glo[..., :256])
    z32 = zr[..., :128]
    st["z"] = r16(z32)
    st["rh"] = r16((z32 if fault == "rh_formed_with_z" else zr[..., 128:]) * H.float())
    q = tanh(conv(torch.cat([st["rh"], X], -1), "w_q", 3, 448, pk["b_q"]) + glo[..., 256:])
    z = z32 if fault == "z_unrounded_in_q" else st["z"].float()
    out["net_out"] = r16((1 - z) * H.float() + z * q)
    n_stem = 384 if ins["n_src"] > 0 else 256
    s = torch.full((E, ht, wd, 384), float("nan"), dtype=torch.float16)
    s[..., :n_stem] = r16(conv(out["net_out"], "w_stem", 3, 128, pk["b_stem"], n_stem).relu())
    st["s"] = s
    st["yh"] = s[..., :256].float() @ pk["w_heads"][0, :36].t()
    yp = F.pad(st["yh"], (0, 0, 1, 1, 1, 1))
    acc = 0
    for t in range(9):
        dy, dx = t // 3, t % 3
        v = yp[:, dy:dy + ht, dx:dx + wd, 4 * t:4 * t + 4]
        if fault == "head_tap_missing_at_border" and dx == 0 and wd > 1:
            v = v.clone()
            v[:, :, 1] = 0
        acc = acc + v
    hd = acc + pk["b_heads"]
    out["delta"] = hd[..., :2]
    out["weight"] = 1.0 / (1.0 + torch.exp(-hd[..., 2:]))
    if ins["n_src"] == 0:
        return st, out
    seg, n_src = ins["seg"], ins["n_src"]
    a1 = s[..., 256:384].float()
    if fault == "segment_mean_wrong_edges":
        seg = seg.clone()
        seg[(seg != seg[0]).nonzero()[0, 0]] = seg[0]
    cnt = torch.bincount(seg, minlength=n_src).float()
    if fault == "segment_mean_wrong_count":
        cnt[0] += 1
    st["am"] = r16(torch.zeros(n_src, ht, wd, 128).index_add_(0, seg, a1) * (1.0 / cnt).view(-1, 1, 1, 1))
    st["b2"] = r16(conv(st["am"], "w_agg2", 3, 128, pk["b_agg2"]).relu())
    up = r16(conv(st["b2"], "w_upmask", 1, 128, pk["b_upmask"])).permute(0, 3, 1, 2).contiguous()
    if fault == "upmask_channel_off_by_one":
        up[:, 100] = up[:, 101]
    out["upmask"] = up
    st["ye"] = torch.cat([st["b2"].float() @ pk["w_eta"][0, :9].t(), torch.zeros(n_src, ht, wd, 3)], -1)
    y, _ = gather9(st["ye"][..., :9], 1)
    x = (y + pk["b_eta"])[..., 0]
    sp = torch.where(x < 20, x, torch.log1p(torch.exp(x))) if fault == "softplus_threshold_wrong_side" else torch.where(x > 20, x, torch.log1p(torch.exp(x)))
    out["eta"] = np.float32(0.01) * sp
    return st, out


def cpu_inputs(case):
    seg, n_src = case_segments(case)
    net, inp, corr, flow = case_inputs(case)
    if case[6].get("layout") == 1:
        net = net.half().permute(0, 2, 3, 1).contiguous()
    return dict(net=net, inp=inp, corr=corr, flow=flow, layout=case[6].get("layout", 0), seg=seg, n_src=n_src)


# the restatement's cases: a 64-wide image, one past the x0 = 64 block boundary of the flow im2col, large features with both sides of
# the softplus threshold and the weight overflow, and no aggregation
SELF_CASES = [
    _case("cpu_16x64", 5, 16, 64, "rand", 3),
    _case("cpu_8x70_large", 4, 8, 70, "uneven", 2, large=True, eta_bias=True, weight_bias=True, layout=1),
    _case("cpu_6x20_no_agg", 3, 6, 20, "none", 0, flow=False, net="f32"),
]


@pytest.mark.parametrize("tanh_sign", [-1, 0, 1])
@pytest.mark.parametrize("case", SELF_CASES, ids=[c[0] for c in SELF_CASES])
def test_bounds_accept_the_fp32_restatement(capi, case, tanh_sign):
    sd, pk = case_weights(case)
    ins = cpu_inputs(case)
    smap = slot_of_pixel(capi, case[2], case[3])
    st, out = restate(pk, ins, smap, tanh_sign)
    res = check_stages(pk, ins, st, out, smap)
    want = {"layout.inp", "corr_encoder.0", "corr_encoder.2", "flow_encoder.0", "flow_encoder.2", "gate_partial", "global_context", "z", "rh",
            "hidden", "stems", "head_partials", "delta", "weight"}
    if ins["layout"] == 0:
        want.add("layout.hin")
    if ins["n_src"]:
        want |= {"segment_mean", "agg.conv2", "upmask", "eta_partials", "eta"}
    assert set(res) == want


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_bounds_reject_planted_fault(capi, fault):
    case = SELF_CASES[1] if fault == "flow_halo_shift_at_x64" else SELF_CASES[0]
    sd, pk = case_weights(case)
    ins = cpu_inputs(case)
    smap = slot_of_pixel(capi, case[2], case[3])
    st, out = restate(pk, ins, smap, 0, fault)
    with pytest.raises(AssertionError, match="^%s:" % FAULTS[fault].replace(".", r"\.")):
        check_stages(pk, ins, st, out, smap)


def test_workspace_layout_matches_the_operator(capi):
    for E, n_src, ht, wd in ((6, 3, 48, 64), (5, 0, 41, 73), (512, 72, 48, 64), (1, 1, 1, 1)):
        offs, slots = workspace_layout(capi, E, n_src, ht, wd)
        total = capi.dba_update_workspace_bytes(E, n_src, ht, wd)
        HW = ht * wd
        sizes = dict(hin=E * HW * 256, x320=E * HW * 640, cc=E * HW * 400, f0=E * HW * 400, c1=E * HW * 256, f1=E * HW * 256, z=E * HW * 256,
                     rh=E * HW * 256, s=E * HW * 768, partial=E * slots * 512, glo=E * 384 * 4, am=max(n_src, 1) * HW * 256, b2=max(n_src, 1) * HW * 256)
        spans = sorted((offs[k], offs[k] + sizes[k], k) for k in sizes)
        for (a0, a1, ka), (b0, b1, kb) in zip(spans, spans[1:]):
            assert a1 <= b0, (ka, kb)
        assert spans[-1][1] <= total and all(v % 256 == 0 for v in offs.values())
        assert offs["yh"] == offs["cc"] and E * HW * 144 <= sizes["cc"]          # the head partials reuse the corr staging buffer
        assert offs["ye"] == offs["f0"] and max(n_src, 1) * HW * 48 <= sizes["f0"]
        smap, n = slot_of_pixel(capi, ht, wd)
        assert n == slots and int(smap.max()) < slots
        assert torch.bincount(smap, minlength=slots).max() <= 16                  # 16 pixels per slot at most
    bad = (ctypes.c_size_t * len(UPWS))()
    assert capi.dba_update_workspace_layout(0, 1, 8, 8, ctypes.cast(bad, ctypes.c_void_p), ctypes.byref(ctypes.c_int())) == 1


def test_case_table_covers_every_route(capi):
    routes, mts, flags = set(), set(), set()
    for name, E, ht, wd, segs, n_src, opt in CASES:
        for cname, c0, c1, ks, n in OPERATOR_CONVS:
            if cname in AGG_CONVS and n_src == 0:
                continue
            p = conv_plan(capi, ht, wd, c0, c1, ks, n)
            routes.add("flat" if p["flat"] else "tw%d" % p["TW"])
            mts.add((p["flat"], p["MT"]))
            if p["n_ntiles"] * (n_src if cname in AGG_CONVS else E) * p["tiles"] > H100_SMS:
                flags.add("more_tiles_than_sms")
        flags.add(("segs", segs))
        flags |= {(k, v) for k, v in opt.items() if k != "sample"}
        if (ht * wd) % 2:
            flags.add("odd_hw")
        if E == 1:
            flags.add("one_edge")
        if (ht, wd) == (1, 1):
            flags.add("1x1")
    assert routes == {"tw64", "tw32", "flat"}
    assert mts == {(f, m) for f in (0, 1) for m in (1, 2)}
    for name, c0, c1, ks, n in OPERATOR_CONVS:                             # MT 4 needs n_out <= 64, 3x3 and >= 4 K blocks
        assert not (n <= 64 and ks == 3 and (c0 + 63) // 64 + (c1 + 63) // 64 >= 4), name
    assert {"more_tiles_than_sms", "odd_hw", "one_edge", "1x1", ("net", "f32"), ("inp", "f32"), ("corr", "f32"), ("layout", 1), ("flow", False),
            ("large", True), ("eta_bias", True), ("weight_bias", True)} <= flags
    assert {("segs", s) for s in ("rand", "one", "single", "uneven", "bench", "none")} <= flags
