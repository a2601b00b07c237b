"""The feature / context encoders (csrc/encoder.cu, `dba_encoder_forward`) stage by stage: the table of their launches, the fp64
reference and the derived bound of every stage, an fp32 restatement that must meet every bound, planted faults that must be rejected at
the stage they break, the workspace sweep and the coverage of the case table.  No GPU is needed here; tests/test_encoder_stages_gpu.py
runs `check_stage` below on what the kernels leave in the workspace after each launch (`dba_encoder_forward_prefix`).

Every stage is checked from its own stored inputs (the fp16 / fp32 bits in the workspace before the launch), so errors do not compound:
  im2col, gather   bit-equal to the copy they define; the 5 pad columns of the 152 pitch +0; nothing written past the level's rows.
  convolution      fp64 of the fp16 inputs, the fp16 weights of the state dict (not the packed tensors: a packing the kernel reads
                   differently fails here) and the fp32 bias; `assert_faithful_f16` with beta = 0.5 sqrt(K) 2^-24 A,
                   A = conv(|x|, |w|) + |b| (K = C for the downsample columns of a merged GEMM, whose other rows hold zeros).
                   EPI_RELU_RES: ReLU on relu_cols only, then relu(v + res) with beta + 2^-24 (|v| + |res|) for the fp32 add.
                   EPI_NCHW: the same values at the NCHW address.
  EPI_STATS slots  counts exactly the valid pixels of each 16-pixel slot; (mean, M2) against fp64 of the exact convolution, with
                   tol_mean = mean(beta) + 6u mean(|x| + beta) and tol_M2 = sum 2|d| g + sum g^2 + 8u M2, g = beta + tol_mean + 2u|x|
                   (u = 2^-24: the fp32 rounding of acc + bias, of a 16-term tree sum and of the deviations).
  finalize         (mean, rstd) against fp64 two ways, both required.  From the native slots (isolates the Chan merge), with
                   D = ceil(slots / 32) + 31 the merge depth: tol_mean = (D + 4) u max|slot mean|, tol_var = (D + 8) u var +
                   4 tol_mean sqrt(var) + tol_mean^2, tol_rstd = rstd^3 tol_var / 2 + 6u rstd.  From the exact convolution over the
                   whole image (isolates a lost or doubled slot, the biased variance, eps): the same plus the slot tolerances averaged.
  act              fp64 of relu(relu((a - m) r) + res) on the stored a, (m, r) and residual, beta = 4u (|a - m| r + |res|).

What the bounds cannot see is said where the fault is planted (FAULTS): the unbiased variance and a missing eps are visible only where 1 / pixels and eps / var exceed the merge tolerance (small levels, small variance), and K 32..63
of a 32-channel activation read as data meets zero weight rows, so it changes no finite value: it is seen only because the workspace
starts NaN-filled and the bytes after the last pixel of X are the still untouched T1 (0 x NaN = NaN in that pixel)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from droid_slam_b200 import c_api, synth
from droid_slam_b200.encoder import ENCODER_CONVS, pack_encoder_weights
from util import assert_faithful_f16

U = 2.0 ** -24
KAPPA_PER_SQRT_K = 0.5
REGIONS = ("big", "X", "T1", "T2", "partial", "counts", "msA", "msB")
ENCODERS = {"fnet": (1, 128), "cnet": (0, 256)}
STEM_TAPS, STEM_PITCH = 147, 152


# ---- the layout and the launch table -------------------------------------------------------------------------------------------
def layout(L, n, H, W, norm):
    offs, sizes = (ctypes.c_size_t * len(REGIONS))(), (ctypes.c_size_t * len(REGIONS))()
    nl, plans = ctypes.c_int(0), (ctypes.c_int * (len(ENCODER_CONVS) * 5))()
    c_api.check(L.dba_encoder_workspace_layout(n, H, W, norm, offs, sizes, ctypes.byref(nl), plans), "encoder_workspace_layout")
    keys = ("TW", "MT", "tiles_x", "tiles_y", "slots")
    return dict(off=dict(zip(REGIONS, offs)), size=dict(zip(REGIONS, sizes)), n_launches=nl.value, n=n, H=H, W=W,
                plans=[dict(zip(keys, plans[5 * k:5 * k + 5])) for k in range(len(ENCODER_CONVS))],
                total=L.dba_encoder_workspace_bytes(n, H, W, 128 if norm else 256))


def stage_table(norm):
    """One row per launch of dba_encoder_forward, in launch order.  lvl: the resolution level H / 2^lvl of the stage's pixels.
    conv rows: k (index into ENCODER_CONVS), ks, src (region, channels read, channel pitch), n outputs, dst (region or 'out', pitch),
    epi, relu_cols, res (region, first column, pitch).  act rows: a / b (region, first column, pitch), ms_a / ms_b (region, first
    channel, channels per image), x (region) and out (region, pitch) over c channels.  writes: the regions the launch owns."""
    rows = []

    def conv(k, lvl, ks, src, n, dst, epi, relu_cols=0, res=None):
        writes = (dst[0], "partial", "counts") if epi == "stats" else (dst[0],)
        rows.append(dict(name=ENCODER_CONVS[k], kernel="conv_tc_kernel<%s>" % epi, kind="conv", k=k, lvl=lvl, ks=ks, src=src, n=n, dst=dst,
                         epi=epi, relu_cols=relu_cols, res=res, reads=(src[0],) + ((res[0],) if res else ()), writes=writes))

    def conv_stats(k, lvl, ks, src, n, dst, ms):
        conv(k, lvl, ks, src, n, (dst, n), "stats")
        rows.append(dict(name=ENCODER_CONVS[k] + ".finalize", kernel="inorm_finalize_kernel", kind="finalize", k=k, lvl=lvl, n=n, ms=ms,
                         reads=("partial", "counts"), writes=(ms,)))

    def act(name, lvl, c, a, ms_a, out, b=None, ms_b=None, x=None):
        rows.append(dict(name=name + ".act", kernel="inorm_act_kernel", kind="act", lvl=lvl, c=c, a=a, ms_a=ms_a, b=b, ms_b=ms_b, x=x, out=out,
                         reads=(a[0], ms_a[0]) + ((b[0], ms_b[0]) if b else ()) + ((x,) if x else ()), writes=(out[0],)))

    def block_s1(k, lvl, P):
        if norm:
            conv_stats(k, lvl, 3, ("X", P, P), P, "T1", "msA")
            act(ENCODER_CONVS[k], lvl, P, ("T1", 0, P), ("msA", 0, P), ("T2", P))
            conv_stats(k + 1, lvl, 3, ("T2", P, P), P, "T1", "msB")
            act(ENCODER_CONVS[k + 1], lvl, P, ("T1", 0, P), ("msB", 0, P), ("X", P), x="X")                    # in place: out == x
        else:
            conv(k, lvl, 3, ("X", P, P), P, ("T1", P), "relu_res", P)
            conv(k + 1, lvl, 3, ("T1", P, P), P, ("X", P), "relu_res", P, ("X", 0, P))                          # in place: out == res

    def block_s2(k, lvl, C, P):
        rows.append(dict(name=ENCODER_CONVS[k] + ".gather", kernel="s2_gather_kernel", kind="gather", lvl=lvl, c=C, reads=("X",), writes=("big",)))
        if norm:
            conv_stats(k, lvl, 1, ("big", 9 * C, 9 * C), 2 * P, "T1", "msA")
            act(ENCODER_CONVS[k], lvl, P, ("T1", 0, 2 * P), ("msA", 0, 2 * P), ("T2", P))
            conv_stats(k + 1, lvl, 3, ("T2", P, P), P, "X", "msB")
            act(ENCODER_CONVS[k + 1], lvl, P, ("X", 0, P), ("msB", 0, P), ("X", P), b=("T1", P, 2 * P), ms_b=("msA", P, 2 * P))   # out == a
        else:
            conv(k, lvl, 1, ("big", 9 * C, 9 * C), 2 * P, ("T1", 2 * P), "relu_res", P)
            conv(k + 1, lvl, 3, ("T1", P, 2 * P), P, ("X", P), "relu_res", P, ("T1", P, 2 * P))

    rows.append(dict(name="conv1.im2col", kernel="image_im2col_kernel", kind="im2col", lvl=1, reads=(), writes=("big",)))
    if norm:
        conv_stats(0, 1, 1, ("big", STEM_TAPS, STEM_PITCH), 32, "T1", "msA")
        act("conv1", 1, 32, ("T1", 0, 32), ("msA", 0, 32), ("X", 32))
    else:
        conv(0, 1, 1, ("big", STEM_TAPS, STEM_PITCH), 32, ("X", 32), "relu_res", 32)
    block_s1(1, 1, 32)
    block_s1(3, 1, 32)
    block_s2(5, 2, 32, 64)
    block_s1(7, 2, 64)
    block_s2(9, 3, 64, 128)
    block_s1(11, 3, 128)
    conv(13, 3, 1, ("X", 128, 128), 128 if norm else 256, ("out", 0), "nchw")
    return rows


def conv_taps(row):
    """K of the accumulation per output column of a conv row (the downsample half of a merged GEMM has C nonzero rows)"""
    if row["ks"] == 3:
        return [9 * row["src"][1]] * row["n"]
    if row["k"] in (5, 9):
        C = row["src"][1] // 9
        return [9 * C] * (row["n"] // 2) + [C] * (row["n"] // 2)
    return [row["src"][1]] * row["n"]


# ---- views of a workspace snapshot (a uint8 tensor on any device) ------------------------------------------------------------------
def region(ws, lay, name, dtype, count):
    o = lay["off"][name]
    return ws[o:o + count * torch.empty(0, dtype=dtype).element_size()].view(dtype)


def dims(lay, lvl):
    return lay["n"], lay["H"] >> lvl, lay["W"] >> lvl


def act_view(ws, lay, name, lvl, pitch):
    E, ht, wd = dims(lay, lvl)
    return region(ws, lay, name, torch.float16, E * ht * wd * pitch).view(E, ht, wd, pitch)


def ms_view(ws, lay, name, stride):
    return region(ws, lay, name, torch.float32, lay["n"] * stride * 2).view(lay["n"], stride, 2)


def extent_bytes(row, lay):
    """bytes from the start of each region this launch may write"""
    E, ht, wd = dims(lay, row["lvl"])
    px = E * ht * wd
    if row["kind"] == "im2col":
        return {"big": px * STEM_PITCH * 2}
    if row["kind"] == "gather":
        return {"big": px * 9 * row["c"] * 2}
    if row["kind"] == "finalize":
        return {row["ms"]: E * row["n"] * 8}
    if row["kind"] == "act":
        return {row["out"][0]: px * row["out"][1] * 2}
    ext = {} if row["dst"][0] == "out" else {row["dst"][0]: px * row["dst"][1] * 2}
    if row["epi"] == "stats":
        s = lay["plans"][row["k"]]["slots"]
        ext.update(partial=E * s * row["n"] * 8, counts=E * s * 4)
    return ext


# ---- fp64 references -------------------------------------------------------------------------------------------------------------
def im2col_rows(img16):
    """[E,3,H,W] f16 -> [E,H/2,W/2,152] f16: K = (dy*7 + dx)*3 + c of the 7x7 / stride 2 / pad 3 window, K 147..151 = +0"""
    E, _, H, W = img16.shape
    cols = F.unfold(img16.float(), 7, padding=3, stride=2).view(E, 3, 49, H // 2, W // 2)       # f16 -> f32 -> f16 is exact
    rows = cols.permute(0, 3, 4, 2, 1).reshape(E, H // 2, W // 2, STEM_TAPS)
    return F.pad(rows, (0, STEM_PITCH - STEM_TAPS)).half()


def gather_rows(x):
    """[E,h,w,C] f16 -> [E,h/2,w/2,9C]: K = (dy*3 + dx)*C + c of the 3x3 / stride 2 / pad 1 window"""
    E, h, w, C = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    taps = [xp[:, dy:dy + h:2, dx:dx + w:2] for dy in range(3) for dx in range(3)]
    return torch.cat(taps, -1)


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def conv_exact(row, before, lay, sd):
    """fp64 result [E,ht,wd,n] of the convolution of `row` on its stored inputs (before ReLU / residual), and A, the sum of the
    magnitudes of its terms.  Weights: the state dict's, rounded to fp16."""
    name, k = row["name"], row["k"]
    src, c, pitch = row["src"]
    x = act_view(before, lay, src, row["lvl"], pitch)[..., :c].double()
    w = sd[name + ".weight"].to(x.device).half().double()
    b = sd[name + ".bias"].to(x.device).double()
    if k == 0:
        wm = w.permute(0, 2, 3, 1).reshape(32, STEM_TAPS)
        return x @ wm.t() + b, x.abs() @ wm.abs().t() + b.abs()
    if k in (5, 9):
        blk = name[:-len(".conv1")]
        P, C = w.shape[0], w.shape[1]
        wm = w.permute(0, 2, 3, 1).reshape(P, 9 * C)
        wds = sd[blk + ".downsample.0.weight"].to(x.device).half().double()[:, :, 0, 0]
        bds = sd[blk + ".downsample.0.bias"].to(x.device).double()
        xc = x[..., 4 * C:5 * C]
        # a non-finite tap anywhere in the window makes the downsample columns NaN too (0 x NaN in the merged GEMM, where the
        # reference's 1x1 / 2 reads the centre only); conv1 reads the same window, so the block's output is NaN there either way
        ex = torch.cat([x @ wm.t() + b, xc @ wds.t() + bds + (x * 0).sum(-1, keepdim=True)], -1)
        mag = torch.cat([x.abs() @ wm.abs().t() + b.abs(), xc.abs() @ wds.abs().t() + bds.abs()], -1)
        return ex, mag
    xn = x.permute(0, 3, 1, 2)
    ex = F.conv2d(xn, w, b, padding=row["ks"] // 2)
    mag = F.conv2d(xn.abs(), w.abs(), b.abs(), padding=row["ks"] // 2)
    return ex.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)


def slot_reference(ex, g_beta, plan, ht, wd):
    """fp64 (count [slots], mean, M2 [E,slots,n]) of the 16-pixel EPI_STATS slots of the exact convolution ex [E,ht,wd,n], and their
    tolerances.  Slot ((ty tiles_x + tx) MT + t) 8 + j holds pixels 16 j .. 16 j + 15 of M tile t of CTA tile (ty, tx): pixel m of an M
    tile is row m / TW, column m mod TW of its RM x TW rectangle."""
    TW, MT, tiles_x, tiles_y = plan["TW"], plan["MT"], plan["tiles_x"], plan["tiles_y"]
    RM = 128 // TW
    E, _, _, n = ex.shape
    Y, X = tiles_y * MT * RM, tiles_x * TW
    pad = lambda t: F.pad(t, (0, 0, 0, X - wd, 0, Y - ht)).view(t.shape[0], Y, X // 16, 16, t.shape[3])
    valid = pad(torch.ones_like(ex[:1, :, :, :1]))[0, :, :, :, 0]                         # [Y, X/16, 16]
    cnt = valid.sum(-1)
    v, x, beta = valid[None, ..., None], pad(ex), pad(g_beta)
    den = cnt.clamp(min=1)[None, ..., None]
    mean = (x * v).sum(3) / den
    d = (x - mean.unsqueeze(3)) * v
    m2 = (d * d).sum(3)
    tol_mean = ((beta * v).sum(3) + 6 * U * ((x.abs() + beta) * v).sum(3)) / den
    g = (beta + tol_mean.unsqueeze(3) + 2 * U * x.abs()) * v
    tol_m2 = (2 * d.abs() * g).sum(3) + (g * g).sum(3) + 8 * U * m2
    y, xs = torch.meshgrid(torch.arange(Y, device=ex.device), torch.arange(X // 16, device=ex.device), indexing="ij")
    ty, t, my = y // (MT * RM), (y % (MT * RM)) // RM, y % RM
    tx, mx = (xs * 16) // TW, (xs * 16) % TW
    slot = ((ty * tiles_x + tx) * MT + t) * 8 + (my * TW + mx) // 16
    order = slot.reshape(-1).argsort()
    assert bool((slot.reshape(-1)[order] == torch.arange(plan["slots"], device=ex.device)).all()), "slot map is not a bijection"
    pick = lambda a: a.reshape(E, -1, n)[:, order]
    return cnt.reshape(-1)[order], pick(mean), pick(m2), pick(tol_mean), pick(tol_m2)


def image_statistics(cnt, mean, m2):
    """fp64 merge of slots: cnt [slots], mean / m2 [E,slots,n] -> (mean, biased variance) [E,n]"""
    w = cnt[None, :, None]
    n = cnt.sum()
    mu = (w * mean).sum(1) / n
    var = (m2.sum(1) + (w * (mean - mu[:, None]) ** 2).sum(1)) / n
    return mu, var


def _ratio(got, want, tol):
    """worst |got - want| / tol (0 where both are NaN, as a NaN input makes them; inf where only one is, or past the tolerance)"""
    err = (got - want).abs()
    r = torch.where(err <= tol, err / tol.clamp(min=1e-300), torch.full_like(err, float("inf")))
    r = torch.where(torch.isnan(got) & torch.isnan(want), torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


def check_stage(row, before, after, lay, sd, images, out_before=None, out_after=None, cache=None):
    """stage `row` on the snapshots around its launch: raises AssertionError when an output is outside its bound, returns the stage's
    statistics (worst kappa, fraction correctly rounded, worst ratio to a tolerance).  cache: carries a statistics convolution's fp64
    result to its finalize row."""
    E, ht, wd = dims(lay, row["lvl"])
    what = "%s (%s)" % (row["name"], row["kernel"])
    kind = row["kind"]
    stats = {}
    if kind == "im2col":
        got = act_view(after, lay, "big", 1, STEM_PITCH)
        want = im2col_rows(images.to(got.device).half())
        assert torch.equal(bits(got), bits(want)), "%s: %d im2col elements differ" % (what, int((bits(got) != bits(want)).sum()))
    elif kind == "gather":
        C = row["c"]
        got = act_view(after, lay, "big", row["lvl"], 9 * C)
        want = gather_rows(act_view(before, lay, "X", row["lvl"] - 1, C))
        assert torch.equal(bits(got), bits(want)), "%s: %d gathered elements differ" % (what, int((bits(got) != bits(want)).sum()))
    elif kind == "conv":
        ex, mag = conv_exact(row, before, lay, sd)
        kk = torch.tensor(conv_taps(row), dtype=torch.float64, device=ex.device)
        unit = U * mag
        beta = KAPPA_PER_SQRT_K * kk.sqrt() * unit
        n = row["n"]
        if row["epi"] == "stats" and cache is not None:
            cache[row["k"]] = (ex, beta)
        if row["epi"] == "relu_res":
            rc = row["relu_cols"]
            ex = torch.cat([ex[..., :rc].clamp(min=0), ex[..., rc:]], -1)
            if row["res"]:
                r, c0, rp = row["res"]
                res = act_view(before, lay, r, row["lvl"], rp)[..., c0:c0 + n].double()
                beta = beta + U * (ex.abs() + res.abs())
                ex = (ex + res).clamp(min=0)
        if row["dst"][0] == "out":
            got = out_after.view(E, n, ht, wd).permute(0, 2, 3, 1)
        else:
            got = act_view(after, lay, row["dst"][0], row["lvl"], row["dst"][1])[..., :n]
        frac, kappa = assert_faithful_f16(got, ex, beta, what, unit=unit)
        stats.update(kappa=kappa, kappa_per_sqrt_k=kappa / max(conv_taps(row)) ** 0.5, correct=frac, K=max(conv_taps(row)))
        if row["epi"] == "stats":
            ex, beta = cache[row["k"]] if cache is not None else (ex, beta)
            plan = lay["plans"][row["k"]]
            S = plan["slots"]
            cnt, mean, m2, tol_mean, tol_m2 = slot_reference(ex, beta, plan, ht, wd)
            counts = region(after, lay, "counts", torch.float32, E * S).view(E, S).double()
            assert torch.equal(counts, cnt[None].expand(E, S)), "%s: %d slot counts differ from the valid pixels of the slot" % (
                what, int((counts != cnt[None]).sum()))
            part = region(after, lay, "partial", torch.float32, E * S * n * 2).view(E, S, n, 2).double()
            live = cnt > 0
            r_mean = _ratio(part[..., 0][:, live], mean[:, live], tol_mean[:, live])
            r_m2 = _ratio(part[..., 1][:, live], m2[:, live], tol_m2[:, live])
            assert r_mean <= 1 and r_m2 <= 1, "%s: slot statistics outside their tolerance (mean %.3g, M2 %.3g of it)" % (what, r_mean, r_m2)
            stats.update(slot_mean=r_mean, slot_m2=r_m2)
    elif kind == "finalize":
        n, S = row["n"], lay["plans"][row["k"]]["slots"]
        counts = region(before, lay, "counts", torch.float32, E * S).view(E, S).double()
        part = region(before, lay, "partial", torch.float32, E * S * n * 2).view(E, S, n, 2).double()
        assert bool((counts == counts[:1]).all())
        cnt = counts[0]
        live = cnt > 0
        got = ms_view(after, lay, row["ms"], n).double()
        depth = -(-S // 32) + 31
        # from the native slots: only the merge differs
        mu, var = image_statistics(cnt[live], part[:, live, :, 0], part[:, live, :, 1])
        tol_mu = (depth + 4) * U * part[:, live, :, 0].abs().amax(1)
        tol_var = (depth + 8) * U * var + 4 * tol_mu * var.sqrt() + tol_mu ** 2
        rstd = (var + 1e-5) ** -0.5
        tol_rstd = 0.5 * rstd ** 3 * tol_var + 6 * U * rstd
        r1 = max(_ratio(got[..., 0], mu, tol_mu), _ratio(got[..., 1], rstd, tol_rstd))
        assert r1 <= 1, "%s: (mean, rstd) outside the merge tolerance of the native slots (%.3g of it)" % (what, r1)
        stats.update(merge=r1)
        if cache is not None and row["k"] in cache:
            # from the exact convolution over the whole image: a slot lost or doubled, the variance's divisor, eps
            ex, beta = cache.pop(row["k"])
            g = beta + 8 * U * ex.abs()
            mu_x = ex.mean((1, 2))
            d = ex - mu_x[:, None, None]
            var_x = (d * d).mean((1, 2))
            tol_mu_x = tol_mu + g.mean((1, 2))
            tol_var_x = tol_var + (2 * d.abs() * (g + tol_mu_x[:, None, None])).mean((1, 2)) + ((g + tol_mu_x[:, None, None]) ** 2).mean((1, 2))
            rstd_x = (var_x + 1e-5) ** -0.5
            tol_rstd_x = 0.5 * rstd_x ** 3 * tol_var_x + 6 * U * rstd_x
            r2 = max(_ratio(got[..., 0], mu_x, tol_mu_x), _ratio(got[..., 1], rstd_x, tol_rstd_x))
            assert r2 <= 1, "%s: (mean, rstd) outside the tolerance of the exact convolution's statistics (%.3g of it)" % (what, r2)
            stats.update(exact=r2)
    elif kind == "act":
        C = row["c"]
        a = act_view(before, lay, row["a"][0], row["lvl"], row["a"][2])[..., row["a"][1]:row["a"][1] + C].double()
        ms = ms_view(before, lay, row["ms_a"][0], row["ms_a"][2])[:, row["ms_a"][1]:row["ms_a"][1] + C].double()[:, None, None]
        t = (a - ms[..., 0]) * ms[..., 1]
        mag = t.abs()
        v = t.clamp(min=0)
        if row["b"]:
            b = act_view(before, lay, row["b"][0], row["lvl"], row["b"][2])[..., row["b"][1]:row["b"][1] + C].double()
            mb = ms_view(before, lay, row["ms_b"][0], row["ms_b"][2])[:, row["ms_b"][1]:row["ms_b"][1] + C].double()[:, None, None]
            r = (b - mb[..., 0]) * mb[..., 1]
            v, mag = v + r, mag + r.abs()
        elif row["x"]:
            r = act_view(before, lay, row["x"], row["lvl"], C).double()
            v, mag = v + r, mag + r.abs()
        got = act_view(after, lay, row["out"][0], row["lvl"], row["out"][1])[..., :C]
        unit = U * mag
        frac, kappa = assert_faithful_f16(got, v.clamp(min=0), 4 * unit, what, unit=unit)
        stats.update(kappa=kappa, correct=frac)
    # what the launch does not own is bit-identical: every other region, and its own regions past the extent of its output
    ext = extent_bytes(row, lay)
    for name in REGIONS:
        o, s = lay["off"][name], lay["size"][name]
        lo = o + ext.get(name, 0)
        assert torch.equal(before[lo:o + s], after[lo:o + s]), "%s wrote %s" % (what, "past its output in " + name if name in ext else "region " + name)
    if out_before is not None and not (kind == "conv" and row["dst"][0] == "out"):
        assert torch.equal(bits(out_before), bits(out_after)), "%s wrote the encoder's output" % what
    return stats


# ---- fp32 restatement of every launch, writing the same workspace (and the faults planted into it) --------------------------------
def _rn16(x):
    return x.float().half()


def _matmul_f32(x, w, g):
    """fp32 x [.., K] @ w [n, K]^T summed over K in blocks of 16 columns taken in a random order"""
    K = x.shape[-1]
    blocks = [torch.arange(i, min(i + 16, K)) for i in range(0, K, 16)]
    acc = torch.zeros(x.shape[:-1] + (w.shape[0],), dtype=torch.float32)
    for i in torch.randperm(len(blocks), generator=g).tolist():
        acc = acc + x[..., blocks[i]].float() @ w[:, blocks[i]].float().t()
    return acc


def _relu_keep_nan(v):
    return torch.where(torch.isnan(v), v, v.clamp(min=0))


def emulate(norm, lay, sd, images, faults=(), seed=0):
    """Runs the launch table in fp32 on the CPU into a NaN-filled workspace of the native layout; yields (row, before, after,
    out_before, out_after) per launch.  The packed weights are read the way the kernels read them ([taps][N][Kpad] f16)."""
    g = torch.Generator().manual_seed(seed)
    od = 128 if norm else 256
    pk = pack_encoder_weights(sd, "instance" if norm else "none", od)
    if "downsample_on_tap_0" in faults:
        for k, C in ((5, 32), (9, 64)):
            P = pk[k].shape[1] // 2
            centre = pk[k][0, P:, 4 * C:5 * C].clone()
            pk[k][0, P:, 4 * C:5 * C] = 0
            pk[k][0, P:, 0:C] = centre
    E = lay["n"]
    ws = torch.full((lay["total"],), 255, dtype=torch.uint8)
    out = torch.full((E, od, lay["H"] // 8, lay["W"] // 8), float("nan"), dtype=torch.float16)
    relu = _relu_keep_nan
    if "fmaxf_relu" in faults:                                                               # fmaxf(NaN, 0) = 0
        relu = lambda v: torch.nan_to_num(v, nan=0.0, posinf=float("inf"), neginf=float("-inf")).clamp(min=0)
    for row in stage_table(norm):
        before, out_before = ws.clone(), out.clone()
        _, ht, wd = dims(lay, row["lvl"])
        kind = row["kind"]
        if kind == "im2col":
            rows = im2col_rows(images.half())
            if "im2col_dy_dx_swapped" in faults:
                rows[..., :STEM_TAPS] = rows[..., :STEM_TAPS].reshape(E, ht, wd, 7, 7, 3).transpose(3, 4).reshape(E, ht, wd, STEM_TAPS)
            if "im2col_pad_nonzero" in faults:
                rows[..., STEM_TAPS + 2] = 2.0 ** -24
            act_view(ws, lay, "big", 1, STEM_PITCH).copy_(rows)
        elif kind == "gather":
            act_view(ws, lay, "big", row["lvl"], 9 * row["c"]).copy_(gather_rows(act_view(before, lay, "X", row["lvl"] - 1, row["c"])))
        elif kind == "conv":
            k, n = row["k"], row["n"]
            src, c, pitch = row["src"]
            x = act_view(before, lay, src, row["lvl"], pitch)[..., :c]
            w, b = pk[k], pk[14 + k]
            if row["ks"] == 1:
                acc = _matmul_f32(x, w[0][:, :c], g)
            else:
                if c == 32 and "k32_read_as_data" in faults:
                    # the 64-channel box over a 32-channel pitch: K 32..63 of a pixel are the next pixel's channels in memory
                    flat = region(before, lay, src, torch.float16, E * ht * wd * 32 + 32).clone()
                    nxt = flat[32:].view(E, ht, wd, 32)
                    x = torch.cat([x, nxt], -1)
                    c = 64
                xp = F.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1))
                cols = torch.cat([xp[:, :, dy:dy + ht, dx:dx + wd] for dy in range(3) for dx in range(3)], 1).permute(0, 2, 3, 1)   # K = tap*c + ch
                acc = _matmul_f32(cols, w[:, :, :c].permute(1, 0, 2).reshape(n, 9 * c), g)
            v = acc + b
            if row["epi"] == "stats":
                plan = lay["plans"][k]
                S = plan["slots"]
                src_stats = _rn16(v).float() if "stats_from_f16_output" in faults else v
                cnt, mean, m2, _, _ = slot_reference(src_stats, torch.zeros_like(v), plan, ht, wd)          # in fp32
                cnt = cnt.clone()
                if "last_partial_slot_counted_16" in faults:
                    part_slots = ((cnt > 0) & (cnt < 16)).nonzero()
                    if part_slots.numel():
                        cnt[part_slots[-1]] = 16
                region(ws, lay, "counts", torch.float32, E * S).view(E, S).copy_(cnt[None].expand(E, S))
                region(ws, lay, "partial", torch.float32, E * S * n * 2).view(E, S, n, 2).copy_(torch.stack([mean, m2], -1))
            elif row["epi"] == "relu_res":
                rc = n if "relu_on_all_columns" in faults else row["relu_cols"]
                v = torch.cat([relu(v[..., :rc]), v[..., rc:]], -1)
                if row["res"]:
                    r, c0, rp = row["res"]
                    if "residual_from_conv1_half" in faults and c0:
                        c0 = 0
                    v = relu(v + act_view(before, lay, r, row["lvl"], rp)[..., c0:c0 + n].float())
            if row["dst"][0] == "out":
                out.copy_(_rn16(v).permute(0, 3, 1, 2))
            else:
                act_view(ws, lay, row["dst"][0], row["lvl"], row["dst"][1])[..., :n] = _rn16(v)
        elif kind == "finalize":
            n, S = row["n"], lay["plans"][row["k"]]["slots"]
            cnt = region(before, lay, "counts", torch.float32, E * S).view(E, S)[0].double()
            part = region(before, lay, "partial", torch.float32, E * S * n * 2).view(E, S, n, 2)
            live = (cnt > 0).nonzero()[:, 0]
            live = live[torch.randperm(len(live), generator=g)]
            if "one_slot_skipped" in faults:
                live = live[live != int((cnt > 0).nonzero()[len(live) // 2, 0])]
            cn = torch.zeros((), dtype=torch.float32)
            mean = torch.zeros(E, n)
            m2 = torch.zeros(E, n)
            for s in live.tolist():                                                          # Chan's update, fp32, in a random order
                nb = cnt[s].float()
                nab = cn + nb
                d, f = part[:, s, :, 0] - mean, nb / nab
                mean = mean + d * f
                m2 = m2 + part[:, s, :, 1] + d * d * cn * f
                cn = nab
            var = m2 / ((cn - 1) if "unbiased_variance" in faults else cn)
            rstd = (var + (0.0 if "eps_missing" in faults else 1e-5)) ** -0.5
            ms_view(ws, lay, row["ms"], n).copy_(torch.stack([mean, rstd], -1))
        elif kind == "act":
            C = row["c"]
            a = act_view(before, lay, row["a"][0], row["lvl"], row["a"][2])[..., row["a"][1]:row["a"][1] + C].float()
            ms = ms_view(before, lay, row["ms_a"][0], row["ms_a"][2])[:, row["ms_a"][1]:row["ms_a"][1] + C][:, None, None]
            v = relu((a - ms[..., 0]) * ms[..., 1])
            if row["b"]:
                b = act_view(before, lay, row["b"][0], row["lvl"], row["b"][2])[..., row["b"][1]:row["b"][1] + C].float()
                mb = ms_view(before, lay, row["ms_b"][0], row["ms_b"][2])
                if "ms_b_stride_P" in faults:                                                 # image e read at (e P + P) instead of (e 2P + P)
                    mb = mb.reshape(-1, 2)[torch.arange(E)[:, None] * C + C + torch.arange(C)[None]]
                else:
                    mb = mb[:, row["ms_b"][1]:row["ms_b"][1] + C]
                mb = mb[:, None, None]
                v = v + (b - mb[..., 0]) * mb[..., 1]
            elif row["x"]:
                v = v + act_view(before, lay, row["x"], row["lvl"], C).float()
            act_view(ws, lay, row["out"][0], row["lvl"], row["out"][1])[..., :C] = _rn16(relu(v))
        yield row, before, ws, out_before, out


def first_rejected(norm, lay, sd, images, faults=(), seed=0):
    """name of the first stage whose check fails on the emulation (None when every stage passes), and the per-stage statistics"""
    cache, report = {}, []
    for row, before, after, ob, oa in emulate(norm, lay, sd, images, faults, seed):
        try:
            report.append((row["name"], check_stage(row, before, after, lay, sd, images, ob, oa, cache)))
        except AssertionError as e:
            return row["name"], report, str(e)
    return None, report, ""


# ---- cases -----------------------------------------------------------------------------------------------------------------------
# (name, n, H, W, image kind, image dtype, weights).  Image kinds: randn; shift40 (+ 40: |mean| >> std in every norm); const1 (image 1
# constant); overflow (fp32 values beyond the fp16 range at a few pixels: end to end only, see the GPU file); weights: 'synth'
# (synth.make_encoder_weights) or 'bias' (the same with biases x 30 so the bias dominates A)
CASES = [
    ("384x512", 1, 384, 512, "randn", torch.float32, "synth"),
    ("352x552", 1, 352, 552, "randn", torch.float32, "synth"),
    ("384x512_shift40", 1, 384, 512, "shift40", torch.float32, "synth"),
    ("240x320_f16", 1, 240, 320, "randn", torch.float16, "synth"),
    ("8x8_n16", 16, 8, 8, "randn", torch.float32, "synth"),
    ("8x520_n2", 2, 8, 520, "randn", torch.float32, "synth"),
    ("24x72_n2_const1", 2, 24, 72, "const1", torch.float32, "synth"),
    ("40x128_n2", 2, 40, 128, "randn", torch.float32, "synth"),          # W/2 = 64 takes 64-wide tiles, W/4 = 32 does not
    ("64x96_n2_bias", 2, 64, 96, "randn", torch.float32, "bias"),
    ("64x96_n16_f16_shift40", 16, 64, 96, "shift40", torch.float16, "synth"),
    ("128x256_n2", 2, 128, 256, "randn", torch.float32, "synth"),       # 64-wide tiles at H/2 and H/4
]
CASE_IDS = [c[0] for c in CASES]


def case_images(case):
    name, n, H, W, kind, dtype, _ = case
    g = torch.Generator().manual_seed(1000 * H + W + n)
    x = torch.randn(n, 3, H, W, generator=g)
    if kind == "shift40":
        x = x + 40.0
    if kind == "const1":
        x[1] = 0.75
    return x.to(dtype)


def case_weights(case, norm):
    sd = synth.make_encoder_weights(3, 128 if norm else 256)
    if case[6] == "bias":
        sd = {k: (v * 30 if k.endswith(".bias") else v) for k, v in sd.items()}
    return sd


# ---- tests -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["fnet", "cnet"])
def test_stage_table_has_one_row_per_launch(capi, name):
    norm, _ = ENCODERS[name]
    rows = stage_table(norm)
    for n, H, W in ((1, 8, 8), (2, 64, 96), (1, 384, 512)):
        lay = layout(capi, n, H, W, norm)
        assert lay["n_launches"] == len(rows) == (43 if norm else 17)
        stats = [r["k"] for r in rows if r["kind"] == "conv" and r["epi"] == "stats"]
        assert [k for k in range(14) if lay["plans"][k]["slots"]] == stats
    assert sum(r["kind"] == "conv" for r in rows) == 14 and [r["k"] for r in rows if r["kind"] == "conv"] == list(range(14))
    bad = (ctypes.c_size_t * 8)()
    assert capi.dba_encoder_workspace_layout(1, 12, 8, norm, bad, bad, ctypes.byref(ctypes.c_int()), (ctypes.c_int * 70)()) == 1
    assert capi.dba_encoder_workspace_layout(1, 8, 8, 2, bad, bad, ctypes.byref(ctypes.c_int()), (ctypes.c_int * 70)()) == 1


def _sweep(capi, norm, n, sizes):
    rows = stage_table(norm)
    for H, W in sizes:
        lay = layout(capi, n, H, W, norm)
        ends = sorted((lay["off"][r], lay["off"][r] + lay["size"][r]) for r in REGIONS)
        assert ends[0][0] == 0 and all(a[1] <= b[0] for a, b in zip(ends, ends[1:])), (n, H, W, "regions overlap")
        assert ends[-1][1] == lay["total"], (n, H, W, "workspace_bytes is not the end of the last region")
        for row in rows:
            for name, nbytes in extent_bytes(row, lay).items():
                assert nbytes <= lay["size"][name], (n, H, W, row["name"], name, nbytes, lay["size"][name])


@pytest.mark.parametrize("name", ["fnet", "cnet"])
def test_workspace_sweep_every_stage_fits_its_region(capi, name):
    """every H, W in multiples of 8 up to 1024 x 1024 at n = 1 (the extents scale with n; n = 2 and 16 on a coarser grid)"""
    norm, _ = ENCODERS[name]
    r8 = range(8, 1025, 8)
    _sweep(capi, norm, 1, [(H, W) for H in r8 for W in r8])
    coarse = [8, 16, 24, 40, 64, 72, 120, 128, 136, 248, 256, 264, 352, 384, 504, 512, 520, 552, 1016, 1024]
    for n in (2, 16):
        _sweep(capi, norm, n, [(H, W) for H in coarse for W in r8])


def test_case_table_covers_the_tilings(capi):
    seen, flags = set(), set()
    for name, n, H, W, kind, dtype, wts in CASES:
        for norm in (0, 1):
            lay = layout(capi, n, H, W, norm)
            for row in stage_table(norm):
                if row["kind"] != "conv":
                    continue
                p = lay["plans"][row["k"]]
                _, ht, wd = dims(lay, row["lvl"])
                seen.add((row["lvl"], p["TW"]))
                seen.add(("MT", p["MT"]))
                if ht % (p["MT"] * (128 // p["TW"])) and wd % p["TW"]:
                    flags.add("partial_tiles_both_ways")
                if wd % 16:
                    flags.add("partial_slot")
        if (W // 8) % 8:
            flags.add("eighth_width_not_multiple_of_8")
        if (W // 2) % 64 == 0 and (W // 4) % 64:
            flags.add("tw64_then_tw32")
        flags.add((kind, dtype))
        flags.add(wts)
        flags.add("n%d" % n)
    assert {(lvl, tw) for lvl in (1, 2, 3) for tw in (32, 64)} <= seen
    # MT = 4 needs nk >= 4 K blocks of a 3x3 convolution with N <= 64; the encoder's N <= 64 layers have 1 K block, so it plans 1 and 2
    assert {m for t, m in seen if t == "MT"} == {1, 2}
    assert {"partial_tiles_both_ways", "partial_slot", "eighth_width_not_multiple_of_8", "tw64_then_tw32", ("shift40", torch.float32),
            ("randn", torch.float16), ("const1", torch.float32), "bias", "n1", "n2", "n16"} <= flags


EMUL_CASES = [("24x72_n2_const1", 2, 24, 72, "const1", torch.float32, "synth"), ("8x8_n2", 2, 8, 8, "randn", torch.float32, "synth"),
              ("64x96_n2_bias", 2, 64, 96, "randn", torch.float32, "bias"), ("16x136_shift40", 1, 16, 136, "shift40", torch.float16, "synth")]


@pytest.mark.parametrize("name", ["fnet", "cnet"])
@pytest.mark.parametrize("case", EMUL_CASES, ids=[c[0] for c in EMUL_CASES])
def test_fp32_restatement_meets_every_bound(capi, name, case):
    norm, _ = ENCODERS[name]
    lay = layout(capi, case[1], case[2], case[3], norm)
    for seed in (0, 1):
        bad, report, msg = first_rejected(norm, lay, case_weights(case, norm), case_images(case), seed=seed)
        assert bad is None, msg
        assert len(report) == lay["n_launches"]


# (fault, encoder, case, the stage that must reject it: that one and no earlier one)
_SMALL = ("24x72_n2", 2, 24, 72, "randn", torch.float32, "synth")
_SMALLVAR = ("24x72_n2_small", 2, 24, 72, "small", torch.float32, "synth")
_SHIFT = ("24x72_n2_shift40", 2, 24, 72, "shift40", torch.float32, "synth")
FAULTS = [
    ("one_slot_skipped", "fnet", _SMALL, "conv1.finalize"),
    ("last_partial_slot_counted_16", "fnet", _SMALL, "conv1"),
    ("unbiased_variance", "fnet", _SMALL, "conv1.finalize"),                 # 1 / 432 pixels at this level; not visible from ~ 2^16 pixels up
    ("eps_missing", "fnet", _SMALLVAR, "conv1.finalize"),                    # images x 0.02: eps / var is large; not visible at var ~ 1
    ("stats_from_f16_output", "fnet", _SHIFT, "conv1"),                      # the slot tolerance sees the fp16 rounding (2^-11 |x|, against
    ("stats_from_f16_output", "fnet", _SMALL, "conv1"),                      # ~ 6 2^-24 |x|) at images + 40 and on centred data alike
    ("downsample_on_tap_0", "fnet", _SMALL, "layer2.0.conv1"),
    ("downsample_on_tap_0", "cnet", _SMALL, "layer2.0.conv1"),
    ("residual_from_conv1_half", "cnet", _SMALL, "layer2.0.conv2"),
    ("relu_on_all_columns", "cnet", _SMALL, "layer2.0.conv1"),
    ("ms_b_stride_P", "fnet", _SMALL, "layer2.0.conv2.act"),
    ("im2col_dy_dx_swapped", "cnet", _SMALL, "conv1.im2col"),
    ("im2col_pad_nonzero", "fnet", _SMALL, "conv1.im2col"),
    ("k32_read_as_data", "cnet", _SMALL, "layer1.0.conv1"),                  # through the NaN fill after the last pixel only
]


def _fault_images(case):
    if case[4] == "small":
        return case_images(case[:4] + ("randn",) + case[5:]) * 0.02
    return case_images(case)


@pytest.mark.parametrize("fault, name, case, stage", FAULTS, ids=["%s-%s-%s" % (f[0], f[1], f[2][0]) for f in FAULTS])
def test_planted_fault_is_rejected_at_its_stage(capi, fault, name, case, stage):
    norm, _ = ENCODERS[name]
    lay = layout(capi, case[1], case[2], case[3], norm)
    sd, img = case_weights(case, norm), _fault_images(case)
    assert first_rejected(norm, lay, sd, img)[0] is None                                  # the same run without the fault passes
    bad, report, msg = first_rejected(norm, lay, sd, img, faults=(fault,))
    assert bad == stage, (fault, bad, msg)


@pytest.mark.parametrize("name", ["fnet", "cnet"])
def test_fmaxf_relu_is_rejected_where_the_nan_is_dropped(capi, name):
    """a ReLU that turns NaN into 0 (fmaxf) fails at the first stage that applies it to a NaN; the NaN-keeping one passes everywhere"""
    norm, _ = ENCODERS[name]
    lay = layout(capi, 2, 24, 72, norm)
    sd, img = case_weights(_SMALL, norm), case_images(_SMALL)
    img[1, 1, 10, 30] = float("nan")
    bad, report, msg = first_rejected(norm, lay, sd, img)
    assert bad is None, msg
    bad, report, msg = first_rejected(norm, lay, sd, img, faults=("fmaxf_relu",))
    assert bad == ("conv1.act" if norm else "conv1"), (bad, msg)
