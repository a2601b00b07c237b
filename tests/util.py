"""helpers shared by the parity tests and the bench tools: calling the C ABI with torch CUDA tensors, comparison metrics, counting host
synchronisations, reading the card and timing calls"""
import contextlib
import ctypes
import subprocess
import time
import warnings

import torch

from droid_slam_b200 import c_api

DT = {torch.float32: c_api.DBA_F32, torch.float16: c_api.DBA_F16, torch.float64: c_api.DBA_F64, torch.bfloat16: c_api.DBA_BF16}


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def c_corr_index_forward(L, volume, coords, r):
    n, h1, w1, h2, w2 = volume.shape
    out = torch.full((n, 2 * r + 1, 2 * r + 1, h1, w1), float("nan"), dtype=volume.dtype, device=volume.device)
    c_api.check(L.dba_corr_index_forward(ptr(volume), ptr(coords), ptr(out), n, h1, w1, h2, w2, r, DT[volume.dtype], stream()), "corr_index_forward")
    return out


def c_corr_index_backward(L, volume, coords, grad, r):
    n, h1, w1, h2, w2 = volume.shape
    out = torch.full_like(volume, float("nan"))
    c_api.check(L.dba_corr_index_backward(ptr(coords), ptr(grad), ptr(out), n, h1, w1, h2, w2, r, DT[volume.dtype], stream()), "corr_index_backward")
    return out


def c_ba(L, poses, disps, intr, disps_sens, targets, weights, eta, ii, jj, t0, t1, itrs, lm, ep, motion_only, M, ws_fill=None):
    """dba_ba through ctypes; ws_fill: byte value the workspace starts with (255 makes every float in it NaN) instead of torch.empty's"""
    N, ht, wd = disps.shape
    E = ii.shape[0]
    ws_bytes = L.dba_ba_workspace_bytes(N, E, ht, wd, t0, t1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=poses.device)
    if ws_fill is not None:
        ws.fill_(ws_fill)
    dx = torch.full((t1 - t0, 6), float("nan"), device=poses.device)
    dz = torch.full((M, ht * wd), float("nan"), device=poses.device)
    a = c_api.ba_args(poses, disps, intr, disps_sens, targets, weights, eta, ii, jj, t0, t1, lm, ep, dx, dz, ws,
                      torch.cuda.current_stream().cuda_stream, motion_only=motion_only)
    c_api.check(L.dba_ba(ctypes.byref(a), itrs) if itrs > 0 else L.dba_ba_prepare(ctypes.byref(a)), "ba")
    m = ctypes.c_int(0); st = ctypes.c_int(0)
    c_api.check(L.dba_ba_read_info(ctypes.byref(a), ctypes.byref(m), ctypes.byref(st)), "ba_read_info")
    return dx, dz, m.value, st.value, (a, ws)


def rel_err(a, b, floor=1.0):
    """max |a-b| / max(|b|, floor): the '1e-4 rel' of BASELINE.json with an absolute floor for values near zero"""
    a = a.double().cpu(); b = b.double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=floor)).max())


def frac_equal(a, b):
    a = a.cpu(); b = b.cpu()
    return float((a == b).float().mean())


F16_OVERFLOW = 65520.0          # the midpoint between 65504, the largest finite fp16, and 2^16: from here on round-to-nearest gives inf


def f16_rounding_interval(h):
    """for fp16 values h: the fp64 bounds (lo, hi) of the reals that round to h under round-to-nearest-even, and whether they belong to
    it (h's significand even: ties round to h).  Computed exactly from h's exponent; ±0 -> ±2^-25; ±inf -> [65520, inf] and its negative
    (NaN gives NaN bounds)."""
    x = h.double()
    a = x.abs()
    m, e = torch.frexp(a)                                       # a = m 2^e, 0.5 <= m < 1
    tiny = 2.0 ** -24
    up = torch.ldexp(torch.ones_like(a), e - 11).clamp(min=tiny)                 # gap to the next larger magnitude
    down = torch.where((m == 0.5) & (e - 1 > -14), up / 2, up)                     # a normal power of two above 2^-14: finer below
    down = torch.where(a == 0, torch.full_like(a, tiny), down)
    up = torch.where(a == 0, torch.full_like(a, tiny), up)
    mag_lo, mag_hi = a - down / 2, a + up / 2
    mag_lo = torch.where(a == 0, -mag_hi, mag_lo)                                  # zero: symmetric about 0
    inf = torch.isinf(a)
    mag_lo = torch.where(inf, torch.full_like(a, F16_OVERFLOW), mag_lo)
    mag_hi = torch.where(inf, torch.full_like(a, float("inf")), mag_hi)
    neg = torch.signbit(x) & (a != 0)
    lo = torch.where(neg, -mag_hi, mag_lo)
    hi = torch.where(neg, -mag_lo, mag_hi)
    even = (h.view(torch.int16) & 1) == 0
    return lo, hi, even | inf


def faithful_f16(got, exact, beta):
    """elementwise: is the fp16 value `got` round-to-nearest-even of some real in [exact - beta, exact + beta]?  Also returns the
    distance from `exact` to the rounding interval of `got` (0 inside it; inf for NaN).  fp64 arithmetic on got's device."""
    assert got.dtype == torch.float16 and got.shape == exact.shape == beta.shape, (got.dtype, got.shape, exact.shape, beta.shape)
    exact = exact.to(got.device, torch.float64)
    beta = beta.to(got.device, torch.float64)
    lo, hi, closed = f16_rounding_interval(got)
    a, b = exact - beta, exact + beta
    ok = torch.where(closed, (lo <= b) & (hi >= a), (lo < b) & (hi > a))
    ok &= ~torch.isnan(got) & ~torch.isnan(beta) & (beta >= 0)                     # NaN is never a rounding of a finite value
    both_nan = torch.isnan(got) & torch.isnan(exact)
    ok |= both_nan
    dist = torch.clamp(torch.maximum(lo - exact, exact - hi), min=0)
    dist = torch.where(torch.isnan(got), torch.full_like(dist, float("inf")), dist)
    dist = torch.where(both_nan, torch.zeros_like(dist), dist)
    return ok, dist


def assert_faithful_f16(got, exact, beta, what="", unit=None):
    """Every fp16 output h must equal round-to-nearest fp16 of some real in [exact - beta, exact + beta] (exact, beta: fp64 or anything
    torch converts exactly; the expected value is never formed by a cast, which may round twice).  Returns (fraction of outputs equal
    to the correctly rounded `exact`, smallest multiple of `unit` that would serve as beta -- the smallest passing kappa when
    beta = kappa * unit; max dist / beta without a unit)."""
    beta = torch.as_tensor(beta, dtype=torch.float64, device=got.device).expand(got.shape)
    ok, dist = faithful_f16(got, exact, beta)
    correct, _ = faithful_f16(got, exact, torch.zeros_like(beta))
    scale = beta if unit is None else torch.as_tensor(unit, dtype=torch.float64, device=got.device).expand(got.shape)
    need = torch.where(dist > 0, dist / scale, torch.zeros_like(dist))
    worst = float(need.max()) if need.numel() else 0.0
    frac = float(correct.double().mean()) if correct.numel() else 1.0
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        first = [tuple(int(v) for v in i) for i in bad[:4].tolist()]
        detail = ["%s: got %r exact %.9g beta %.3g" % (i, float(got[i]), float(exact[i]), float(beta[i])) for i in first]
        raise AssertionError("%s: %d of %d fp16 outputs are not a rounding of a value within beta of the fp64 reference (needs %.3g); %s"
                             % (what, bad.shape[0], got.numel(), worst, "; ".join(detail)))
    return frac, worst


def assert_bit_identical(a, b, what=""):
    """torch.equal with a useful message (how many elements differ and by how much)"""
    a = a.cpu(); b = b.cpu()
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    if not torch.equal(a, b):
        neq = (a != b) & ~(torch.isnan(a) & torch.isnan(b))          # NaN in the same place on both sides (NaN coordinates) counts as identical
        if bool(neq.any()):
            d = (a.double() - b.double()).abs()
            raise AssertionError("%s: %d of %d elements differ, max |diff| %.3e" % (what, int(neq.sum()), a.numel(), float(d[neq].max())))


SYNC_WARNING = "called a synchronizing CUDA operation"      # torch's warning per synchronising operation in sync debug mode "warn"


def host_syncs(fn):
    """(host synchronisations fn() makes, its result).  Counts torch's per-operation warnings only, not its one-time notice that the
    debug mode is a prototype, so a count does not depend on whether an earlier window in the process already raised that notice."""
    torch.cuda.synchronize()
    mode = torch.cuda.get_sync_debug_mode()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode(mode)
    return sum(str(w.message).startswith(SYNC_WARNING) for w in caught), out


@contextlib.contextmanager
def syncs_not_counted():
    """synchronisations inside the block are not counted by an enclosing host_syncs"""
    mode = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode(0)
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(mode)


def card():
    """name, power limit and SM clocks of torch's current device, read (never set) with nvidia-smi.  The device is named to nvidia-smi
    by its PCI bus id: nvidia-smi's indices ignore CUDA_VISIBLE_DEVICES.  Never raises; when nvidia-smi cannot answer, the name comes
    from torch and the other fields say why they are unknown."""
    d = torch.cuda.current_device()
    p = torch.cuda.get_device_properties(d)
    bus = "%08X:%02X:%02X.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
    keys = ("name", "power_limit", "sm_clock", "max_sm_clock")
    try:
        r = subprocess.run(["nvidia-smi", "-i", bus, "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().split(",")]
        if r.returncode == 0 and len(vals) == len(keys):
            return dict(zip(keys, vals))
        why = "nvidia-smi -i %s exited %d: %s" % (bus, r.returncode, (r.stderr or r.stdout).strip()[:200])
    except (OSError, subprocess.SubprocessError) as e:
        why = "%s: %s" % (type(e).__name__, e)
    return dict(name=torch.cuda.get_device_name(d), **{k: "unknown (%s)" % why for k in keys[1:]})


def timed(fn, calls=1, warmup=0):
    """(CUDA-event ms per call, host-clock ms per call, the last call's result) over `calls` calls of fn after `warmup` calls.  The
    device is synchronised before both clocks start and after the last call, so they cover the work, not only its launch."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    start.record()
    out = None
    for _ in range(calls):
        out = fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / calls, 1e3 * (time.perf_counter() - t0) / calls, out
