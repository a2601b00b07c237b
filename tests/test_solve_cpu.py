"""The damped fp64 pose solve (`dba_solve_spd`, csrc/chol.cu): the case builders, fp64 LAPACK references and acceptance criteria that
tests/test_solve_gpu.py holds every route of the kernel to, and the CPU tests that pin them -- including proof that each criterion
rejects the kind of error it is there to catch.

The solve factors Hd = H + diag(ep + lm * diag(H)) (lm, ep rounded to fp32: they are C floats) in fp64 and returns x in fp32.  With
nt = ceil(n / 32) tile rows it takes one of three routes:
  resident  chol_resident_kernel, nt <= 14: one owner warp per tile, a cluster of 1 / 2 / 4 / 8 / 16 CTAs for nt = 1 / 2 / 3-4 / 5-8 /
            9-14, the tile placement computed on the host (`dba_solve_tile_placement`)
  envelope  chol_cluster_kernel, 15 <= nt <= 255: per tile row the first nonzero tile column `first[i]`; tiles left of it are skipped
  dense     chol_cluster_kernel, nt >= 256: the envelope is off (one thread per tile row scans it)

Criteria, all evaluated in fp64, with u = 2^-53 and gamma = 4 (n + 32) u:
  factor    e_L = max_{i>=j} |(L L^T - Hd)_ij| / sqrt(Hd_ii Hd_jj) <= gamma.  The Cholesky backward-error bound: |L||L^T|_ij <=
            sqrt(Hd_ii Hd_jj) by Cauchy-Schwarz, so it does not depend on the condition number.  L must also be exactly zero left of
            the envelope (no arithmetic can fill it in).
  residual  |Hd x - b|_i <= 2^-23 (|Hd||x|)_i + gamma (sum_j sqrt(Hd_ii Hd_jj) |x_j| + |b_i|): one fp32 rounding of x plus the fp64
            solve; again independent of the condition number.
  forward   |x_i - x*_i| <= 2^-23 |x*_i| + kappa gamma max|x*|, x* the LAPACK solution, where kappa is known by construction (a
            prescribed spectrum, or a Gershgorin bound for a diagonally dominant Hd): each element within about one fp32 rounding.
Rounding x* to fp32 alone can take half of the residual and forward bounds (a round-to-nearest error is at most 2^-24 |x|), so the
margins asserted below are: LAPACK's factor within gamma / 10, LAPACK's fp64 x* within a tenth of the gamma term of the residual, and
fl32(x*) within half of both the residual and the forward bound."""
import ctypes
import functools

import numpy as np
import pytest
import scipy.linalg as sla
import torch

from droid_slam_b200 import c_api

T = 32                    # tile edge (kT)
RES_MAX_NT = 14           # largest system of the resident kernel, in tile rows (kResMaxNt)
ENVELOPE_MAX_NT = 255     # the cluster kernel tracks the envelope below kCholThreads = 256 tile rows
U = 2.0 ** -53
EPS32 = 2.0 ** -23
FRONTEND = (1e-4, 0.1)    # (lm, ep) of the frontend windows
GLOBAL = (1e-5, 1e-2)     # (lm, ep) of global BA (update_lowmem)


def cdiv(a, b):
    return (a + b - 1) // b


def gamma(n):
    return 4 * (n + T) * U


def f32(v):
    return float(np.float32(v))


def damp(H, lm, ep):
    """Hd = H + diag(ep32 + lm32 * H_ii), lm and ep rounded to fp32 first, as the kernel's load phase does"""
    Hd = np.array(H, dtype=np.float64, copy=True)
    d = np.diagonal(H).copy()
    Hd[np.diag_indices_from(Hd)] = d + (f32(ep) + f32(lm) * d)
    return Hd


# ---- matrix families ------------------------------------------------------------------------------------------------------------------
def spectrum(n, kappa, seed):
    """Q diag(lambda) Q^T with lambda spread geometrically over [1 / kappa, 1]: condition number kappa by construction"""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = float(kappa) ** -np.linspace(0.0, 1.0, n)
    H = (Q * lam) @ Q.T
    return 0.5 * (H + H.T), rng.standard_normal(n)


def dominant(n, lower, seed, diag_extra=1.0):
    """symmetric matrix from strictly-lower entries {(r, c): v}, diagonal = off-diagonal row sum of |.| + diag_extra (SPD, Gershgorin)"""
    rng = np.random.default_rng(seed)
    H = np.zeros((n, n))
    for (r, c), v in lower.items():
        assert r > c
        H[r, c] = H[c, r] = v                                           # -0.0 stays -0.0 on both sides
    H[np.diag_indices(n)] = np.abs(H).sum(1) + diag_extra
    return H, rng.standard_normal(n)


def banded(n, bw, seed):
    """diagonally dominant, half bandwidth bw elements, couplings decaying away from the diagonal"""
    rng = np.random.default_rng(seed)
    H = np.zeros((n, n))
    for d in range(1, bw + 1):
        i = np.arange(n - d)
        H[i + d, i] = rng.standard_normal(n - d) * 0.5 ** (d / 16)
    H = H + H.T
    H[np.diag_indices(n)] = np.abs(H).sum(1) + 1.0
    return H, rng.standard_normal(n)


def ba_like(P, w, loops, seed, free_pose):
    """Sum over edges of J^T J, J = [G, -G] (8 x 12) on poses (i, j): a window graph |i - j| <= w plus loop closures.  Every edge is
    blind to moving both poses together, so H is only positive semi-definite (the gauge); damping makes it definite.  Pose
    `free_pose` has no edges: its rows and columns are exactly zero."""
    rng = np.random.default_rng(seed)
    H = np.zeros((6 * P, 6 * P))
    edges = [(i, j) for i in range(P) for j in range(i + 1, min(P, i + w + 1))] + list(loops)
    for i, j in edges:
        if free_pose in (i, j):
            continue
        G = rng.standard_normal((8, 6)) * rng.uniform(0.3, 3.0)
        A = G.T @ G
        si, sj = slice(6 * i, 6 * i + 6), slice(6 * j, 6 * j + 6)
        H[si, si] += A; H[sj, sj] += A; H[si, sj] -= A; H[sj, si] -= A
    assert not H[6 * free_pose:6 * free_pose + 6].any()
    return H, rng.standard_normal(6 * P)


def old_random(n):
    """the matrices the solver was first checked with: A A^T + 1e-3 I, A [n, n + 8] (torch generator seeded with n)"""
    g = torch.Generator().manual_seed(n)
    A = torch.randn(n, n + 8, generator=g, dtype=torch.float64)
    H = A @ A.t() + 1e-3 * torch.eye(n, dtype=torch.float64)
    return H.numpy(), torch.randn(n, generator=g, dtype=torch.float64).numpy()


def old_banded(n, band, far):
    """block-banded, diagonally dominant systems shaped like a sliding-window pose system, with `far` couplings deep in the matrix
    that widen the envelope of single rows (torch generator seeded with n + band)"""
    g = torch.Generator().manual_seed(n + band)
    H = torch.zeros(n, n, dtype=torch.float64)
    blk = 6
    nb = n // blk
    for d in range(0, band // blk + 1):
        w = torch.randn(nb - d, blk, blk, generator=g, dtype=torch.float64) * (0.5 ** d)
        for t in range(nb - d):
            H[(t + d) * blk:(t + d + 1) * blk, t * blk:(t + 1) * blk] = w[t]
    for f in range(far):
        r, c = nb - 5 - 7 * f, 3 + 11 * f
        H[r * blk:(r + 1) * blk, c * blk:(c + 1) * blk] = 0.3 * torch.randn(blk, blk, generator=g, dtype=torch.float64)
    H = torch.tril(H); H = H + H.t()
    H.diagonal().add_(H.abs().sum(1) + 1.0)
    return H.numpy(), torch.randn(n, generator=g, dtype=torch.float64).numpy()


def _band_lower(n, bw, seed):
    rng = np.random.default_rng(seed)
    return {(r, c): rng.standard_normal() for r in range(n) for c in range(max(0, r - bw), r)}


def pattern(kind, n=640, seed=0):
    """envelope patterns for the cluster kernel (n = 640: 20 tile rows).  The property each is named for is asserted in
    test_pattern_cases_have_their_property."""
    rng = np.random.default_rng(seed + 1)
    low = {}
    if kind == "arrow":                       # last tile row couples to tile column 0; the zero tiles in between fill in
        low = _band_lower(n, 40, seed)
        for r in range(n - T, n):
            for c in range(T):
                low[(r, c)] = 0.2 * rng.standard_normal()
    elif kind == "blockdiag":                 # dense diagonal tiles only: first[i] = i, no trailing work
        for t in range(cdiv(n, T)):
            for r in range(t * T, min(n, t * T + T)):
                for c in range(t * T, r):
                    low[(r, c)] = rng.standard_normal()
    elif kind == "boundary":                  # row 351 starts at column 127 = 32*4 - 1, row 352 (next tile row) at column 128 = 32*4
        low = _band_lower(n, 4, seed)
        low[(351, 127)] = 0.5
        low[(352, 128)] = -0.5
    elif kind == "nonmonotone":               # tile row 12 reaches tile 1, tile row 13 only its neighbour, tile row 14 tile 2
        low = _band_lower(n, 4, seed)
        low[(12 * T + 5, 40)] = 0.7
        low[(14 * T + 9, 2 * T + 3)] = -0.4
    elif kind == "negzero":                   # -0.0 left of the envelope must not widen it
        low = _band_lower(n, 4, seed)
        for rc in ((500, 10), (501, 11), (600, 300)):
            low[rc] = -0.0
    elif kind == "single":                    # tile (18, 2) holds a single nonzero
        low = _band_lower(n, 4, seed)
        low[(600, 70)] = 0.9
    else:
        raise ValueError(kind)
    return dominant(n, low, seed)


@functools.lru_cache(maxsize=None)
def real_system(name):
    """the fp64 reduced pose system of a BA configuration's first Gauss-Newton iteration (test_ba_stages_cpu.ref_system), symmetric
    from its lower triangle"""
    from test_ba_stages_cpu import make_case, ref_system, eta_for_kx, symmetric_from_lower
    s = make_case(name)
    ref = ref_system(s["poses"], s["disps"], s["intrinsics"], s["disps_sens"], s["targets"], s["weights"], eta_for_kx(s), s["ii"], s["jj"],
                     s["t0"], s["t1"])
    return symmetric_from_lower(ref["H"]).numpy(), ref["b"].numpy(), s["lm"], s["ep"]


# ---- the case table -------------------------------------------------------------------------------------------------------------------
# every nt from 1 to 14 at n = 32 nt and 32 nt - 1; the smallest sizes; both sides of the resident / cluster switch; nt = 32, 75, 188,
# 255 (the largest system with an envelope) and 256 (the dense path, banded so that the references stay cheap)
SIZES = sorted({*range(1, 7), 33, 144, 426, *(T * t for t in range(1, RES_MAX_NT + 1)), *(T * t - 1 for t in range(1, RES_MAX_NT + 1)),
                449, 480, 1024, 2394, 6016, 8160, 8161, 8192})
OLD_RANDOM_N = [6, 30, 42, 100, 200, 426, 448, 449, 1000, 2394]
OLD_BANDED = [(700, 100, 0), (1200, 150, 3), (2394, 160, 0), (5994, 150, 2)]
PATTERNS = ["arrow", "blockdiag", "boundary", "nonmonotone", "negzero", "single"]


def _size_case(n):
    if n <= 2394:                                                       # prescribed spectrum, undamped: kappa is exact
        kappa = 1e8 if n % T == 0 else 1e2
        return dict(build=lambda: spectrum(n, kappa, seed=n), lm=0.0, ep=0.0, kappa=kappa)
    return dict(build=lambda: banded(n, 96 if n > 8160 else 150, seed=n), lm=GLOBAL[0], ep=GLOBAL[1])


def _ba_case(P, w, loops, settings, seed):
    return dict(build=lambda: ba_like(P, w, loops, seed, free_pose=P // 3), lm=settings[0], ep=settings[1], free_pose=P // 3)


CASES = {}
for _n in SIZES:
    CASES["size_%d" % _n] = _size_case(_n)
CASES["ba_frontend_72"] = _ba_case(12, 3, [(0, 11)], FRONTEND, 1)
CASES["ba_frontend_426"] = _ba_case(71, 3, [(2, 60), (10, 70), (0, 35)], FRONTEND, 2)
CASES["ba_global_2400"] = _ba_case(400, 4, [(5, 390), (20, 300), (100, 399)], GLOBAL, 3)
CASES["ba_global_8166"] = _ba_case(1361, 4, [(i, i + 40) for i in range(0, 1300, 97)], GLOBAL, 4)   # nt = 256: the dense path
for _k in PATTERNS:
    CASES["pattern_" + _k] = dict(build=functools.partial(pattern, _k), lm=FRONTEND[0], ep=FRONTEND[1])
for _name in ("metric", "c3_global"):
    CASES["real_" + _name] = dict(real=_name)
for _n in OLD_RANDOM_N:
    CASES["old_random_%d" % _n] = dict(build=functools.partial(old_random, _n), lm=FRONTEND[0], ep=FRONTEND[1])
for _n, _band, _far in OLD_BANDED:
    CASES["old_banded_%d_%d_%d" % (_n, _band, _far)] = dict(build=functools.partial(old_banded, _n, _band, _far), lm=GLOBAL[0], ep=GLOBAL[1])


@functools.lru_cache(maxsize=2)
def make_case(name):
    """dict(H (full symmetric, fp64), b, lm, ep, Hd (damped), n, first (tile envelope of Hd), kappa (None if not known))"""
    c = CASES[name]
    if "real" in c:
        H, b, lm, ep = real_system(c["real"])
    else:
        (H, b), lm, ep = c["build"](), c["lm"], c["ep"]
    H, b = np.ascontiguousarray(H, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    Hd = damp(H, lm, ep)
    kappa = c.get("kappa") or gershgorin_kappa(Hd)
    return dict(name=name, H=H, b=b, lm=lm, ep=ep, Hd=Hd, n=H.shape[0], first=tile_first(Hd), kappa=kappa, free_pose=c.get("free_pose"))


# ---- routes ---------------------------------------------------------------------------------------------------------------------------
def tile_placement(n):
    """(cluster size, map_i, map_j) of the resident kernel from the library's host code; cluster size 0: the cluster kernel"""
    L = c_api.load()
    mi = (ctypes.c_ubyte * 128)(); mj = (ctypes.c_ubyte * 128)()
    cs = L.dba_solve_tile_placement(n, ctypes.cast(mi, ctypes.c_void_p), ctypes.cast(mj, ctypes.c_void_p))
    return cs, list(mi), list(mj)


def route(n):
    """'resident', 'envelope' or 'dense' (see the module docstring) and the resident kernel's cluster size"""
    nt = cdiv(n, T)
    cs, _, _ = tile_placement(n)
    if cs:
        return "resident", cs
    return ("envelope" if nt <= ENVELOPE_MAX_NT else "dense"), 0


def tile_first(Hd):
    """numpy restatement of the cluster kernel's envelope: for tile row i, the first tile column < i holding an element != 0.0 of the
    lower triangle (NaN counts, -0.0 does not), else i"""
    n = Hd.shape[0]
    nt = cdiv(n, T)
    first = np.arange(nt)
    for i in range(1, nt):
        blk = Hd[i * T:min(n, i * T + T), :i * T] != 0
        cols = np.flatnonzero(blk.any(0))
        if cols.size:
            first[i] = cols[0] // T
    return first


def gershgorin_kappa(Hd):
    """an upper bound of the condition number when Hd is strictly diagonally dominant with a positive diagonal, else None"""
    d = np.diagonal(Hd)
    off = np.abs(Hd).sum(1) - np.abs(d)
    lo = d - off
    if not np.all(np.isfinite(lo)) or lo.min() <= 0:
        return None
    return float((d + off).max() / lo.min())


# ---- fp64 references ------------------------------------------------------------------------------------------------------------------
def elem_bandwidth(Hd):
    nz = Hd != 0
    n = Hd.shape[0]
    firstcol = np.where(nz.any(1), nz.argmax(1), np.arange(n))
    return int((np.arange(n) - firstcol).max())


def _band_form(Hd, kd):
    n = Hd.shape[0]
    ab = np.zeros((kd + 1, n))
    for k in range(kd + 1):
        ab[k, :n - k] = np.diagonal(Hd, -k)
    return ab


def lapack_factor(Hd):
    """LAPACK's Cholesky factor (dpbtrf for narrow bands, dpotrf otherwise), dense lower triangular"""
    n = Hd.shape[0]
    kd = elem_bandwidth(Hd)
    if 4 * kd >= n:
        return sla.cholesky(Hd, lower=True)
    cb = sla.cholesky_banded(_band_form(Hd, kd), lower=True)
    L = np.zeros_like(Hd)
    for k in range(kd + 1):
        i = np.arange(n - k)
        L[i + k, i] = cb[k, :n - k]
    return L


def lapack_solve(Hd, b):
    n = Hd.shape[0]
    kd = elem_bandwidth(Hd)
    if 4 * kd >= n:
        return sla.cho_solve(sla.cho_factor(Hd, lower=True), b)
    return sla.cho_solve_banded((sla.cholesky_banded(_band_form(Hd, kd), lower=True), True), b)


def tiled_cholesky(Hd, first, dtype=np.float64, skip=None):
    """right-looking tiled Cholesky over the envelope, like chol_cluster_kernel: per panel k, TRSM of the rows with first[i] <= k, then
    A_ij -= L_ik L_jk^T for those rows.  skip=(i, j, k): leave tile (i, j) without the update of panel k"""
    n = Hd.shape[0]
    nt = cdiv(n, T)
    A = np.eye(nt * T, dtype=dtype)
    A[:n, :n] = np.tril(Hd)
    t = lambda i, j: (slice(i * T, i * T + T), slice(j * T, j * T + T))
    for k in range(nt):
        Lkk = np.linalg.cholesky(np.tril(A[t(k, k)]) + np.tril(A[t(k, k)], -1).T).astype(dtype)
        A[t(k, k)] = Lkk
        act = [i for i in range(k + 1, nt) if first[i] <= k]
        for i in act:
            A[t(i, k)] = sla.solve_triangular(Lkk, A[t(i, k)].T, lower=True).T.astype(dtype)
        for a, i in enumerate(act):
            for j in act[:a + 1]:
                if skip != (i, j, k):
                    A[t(i, j)] -= A[t(i, k)] @ A[t(j, k)].T
    return np.tril(A)[:n, :n]


def tiled_solve(L, b, first, skip=None):
    """L L^T x = b with the tiled factor: forward substitution, then the kernel's backward substitution over the envelope
    (x_k = L_kk^-T y_k, then y_i -= L_ki^T x_k for first[k] <= i < k).  skip=k: leave out tile (k, first[k]) in that step"""
    n = L.shape[0]
    nt = cdiv(n, T)
    Lp = np.eye(nt * T); Lp[:n, :n] = L
    y = np.zeros(nt * T); y[:n] = sla.solve_triangular(L, b, lower=True)
    s = lambda i: slice(i * T, i * T + T)
    for k in range(nt - 1, -1, -1):
        y[s(k)] = sla.solve_triangular(Lp[s(k), s(k)], y[s(k)], lower=True, trans="T")
        for i in range(first[k], k):
            if skip == k and i == first[k]:
                continue
            y[s(i)] -= Lp[s(k), s(i)].T @ y[s(k)]
    return y[:n]


# ---- criteria ---------------------------------------------------------------------------------------------------------------------------
def factor_error(Lhat, Hd, first):
    """e_L / gamma (module docstring), from the lower triangle of Lhat only; inf if Lhat is not zero left of the envelope.  The
    product is taken tile row by tile row over the envelope: L L^T of tile row i needs only columns from 32 first[i] on."""
    n = Hd.shape[0]
    s = np.sqrt(np.diagonal(Hd))
    worst = 0.0
    for i in range(cdiv(n, T)):
        r0, r1 = i * T, min(n, i * T + T)
        c0 = first[i] * T
        if np.any(Lhat[r0:r1, :c0] != 0):
            return float("inf")
        Li = np.tril(Lhat[r0:r1, c0:r1], k=r0 - c0)
        Lj = np.tril(Lhat[c0:r1, c0:r1])
        E = np.abs(Li @ Lj.T - Hd[r0:r1, c0:r1]) / (s[r0:r1, None] * s[None, c0:r1])
        E = np.tril(E, k=r0 - c0)
        worst = max(worst, float(np.max(E)) if not np.isnan(E).any() else float("inf"))
    return worst / gamma(n)


def residual_ratio(Hd, x, b, gamma_only=False):
    """max_i |Hd x - b|_i over the residual bound (module docstring); gamma_only: over the fp64 (gamma) term of the bound alone"""
    n = Hd.shape[0]
    x = np.asarray(x, dtype=np.float64)
    r = np.abs(Hd @ x - b)
    s = np.sqrt(np.diagonal(Hd))
    bound = gamma(n) * (s * float(s @ np.abs(x)) + np.abs(b))
    if not gamma_only:
        bound = bound + EPS32 * (np.abs(Hd) @ np.abs(x))
    if np.isnan(r).any():
        return float("inf")
    if np.any(r[bound == 0] != 0):
        return float("inf")
    return float(np.max(r[bound > 0] / bound[bound > 0])) if np.any(bound > 0) else 0.0


def forward_ratio(x, xs, kappa):
    """max_i |x_i - x*_i| over 2^-23 |x*_i| + kappa gamma max|x*|"""
    x = np.asarray(x, dtype=np.float64)
    bound = EPS32 * np.abs(xs) + kappa * gamma(len(xs)) * np.abs(xs).max()
    d = np.abs(x - xs)
    if np.isnan(d).any():
        return float("inf")
    if np.any(d[bound == 0] != 0):
        return float("inf")
    return float(np.max(d[bound > 0] / bound[bound > 0])) if np.any(bound > 0) else 0.0


def fl32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


# ---- tests ----------------------------------------------------------------------------------------------------------------------------
EXPECTED_CLUSTER = {1: 1, 2: 2, 3: 4, 4: 4, **{t: 8 for t in range(5, 9)}, **{t: 16 for t in range(9, 15)}}


def test_size_table_covers_every_route():
    nts = {cdiv(n, T) for n in SIZES}
    assert set(range(1, RES_MAX_NT + 1)) <= nts and {15, 32, 75, 188, 255, 256} <= nts
    for t in range(1, RES_MAX_NT + 1):
        assert T * t in SIZES and T * t - 1 in SIZES
    assert {route(n)[0] for n in SIZES} == {"resident", "envelope", "dense"}
    assert route(8160) == ("envelope", 0) and route(8161) == ("dense", 0) and route(8192) == ("dense", 0)
    assert "ba_global_8166" in CASES and route(6 * 1361) == ("dense", 0)


@pytest.mark.parametrize("n", SIZES)
def test_route_of_every_size(n):
    nt = cdiv(n, T)
    r, cs = route(n)
    if nt <= RES_MAX_NT:
        assert r == "resident" and cs == EXPECTED_CLUSTER[nt], (n, r, cs)
    else:
        assert r == ("envelope" if nt < 256 else "dense") and cs == 0


def test_resident_cholesky_tile_placement_invariants():
    """host logic of csrc/chol.cu (resident_tile_map), for every resident size of the table: every tile of the lower triangle and every
    right-hand-side piece has exactly one warp slot, diagonal tile s sits on CTA s, and a tile of column c shares an SM with diagonal
    tile s only if it is finished before potrf(s) runs (c < s) -- or the SM has no diagonal tile / is CTA 0 (potrf(0) runs before
    anything else has operands)."""
    resident = [n for n in SIZES if cdiv(n, T) <= RES_MAX_NT]
    assert len({cdiv(n, T) for n in resident}) == RES_MAX_NT
    for n in resident:
        ncta, mi, mj = tile_placement(n)
        nt = cdiv(n, T)
        assert ncta in (1, 2, 4, 8, 16) and ncta >= nt and ncta * 8 >= nt * (nt + 1) // 2 + nt
        seen = {}
        for slot in range(128):
            if mi[slot] == 0xFF:
                continue
            assert slot < ncta * 8
            i, j = mi[slot], mj[slot]
            assert 0 <= j < nt and j <= i <= nt and (i, j) not in seen
            seen[(i, j)] = slot // 8
        assert set(seen) == {(i, j) for j in range(nt) for i in range(j, nt + 1)}
        for (i, j), cta in seen.items():
            if i == j:
                assert cta == j
            else:
                assert cta > j or cta >= nt or cta == 0, (n, i, j, cta)
    for n in [n for n in SIZES if cdiv(n, T) > RES_MAX_NT]:
        assert tile_placement(n)[0] == 0          # the cluster kernel beyond 14 tile rows


def test_pattern_cases_have_their_property():
    f = {k: make_case("pattern_" + k)["first"] for k in PATTERNS}
    Hd = {k: make_case("pattern_" + k)["Hd"] for k in PATTERNS}
    nt = 20
    # arrow: the last tile row reaches column 0 across zero tiles that fill in
    a = Hd["arrow"]
    assert f["arrow"][nt - 1] == 0 and not a[(nt - 1) * T:, T:(nt - 3) * T].any() and a[T:2 * T, :T].any()
    # block diagonal: no tile row reaches left of its diagonal tile
    assert list(f["blockdiag"]) == list(range(nt))
    # boundary: row 351 starts at 32*4 - 1, row 352 at 32*4
    bd = Hd["boundary"]
    assert np.flatnonzero(bd[351])[0] == 4 * T - 1 and np.flatnonzero(bd[352])[0] == 4 * T
    assert f["boundary"][10] == 3 and f["boundary"][11] == 4
    # non-monotone: first[14] < first[13]
    assert f["nonmonotone"][12] == 1 and f["nonmonotone"][13] == 12 and f["nonmonotone"][14] == 2
    # -0.0 left of the envelope does not widen it
    nz = Hd["negzero"]
    assert np.signbit(nz[500, 10]) and nz[500, 10] == 0 and f["negzero"][500 // T] == 500 // T - 1
    assert np.signbit(nz[600, 300]) and f["negzero"][600 // T] > 300 // T
    # a tile with a single nonzero
    sg = Hd["single"]
    assert np.count_nonzero(sg[18 * T:19 * T, 2 * T:3 * T]) == 1 and f["single"][18] == 2


def test_ba_like_cases_are_gauge_deficient_with_a_free_pose():
    for name in ("ba_frontend_72", "ba_global_2400"):
        c = make_case(name)
        H, p = c["H"], c["free_pose"]
        assert not H[6 * p:6 * p + 6].any() and not H[:, 6 * p:6 * p + 6].any()
        v = np.tile(np.eye(6)[0], H.shape[0] // 6)                       # all poses moving together
        assert np.abs(H @ v).max() < 1e-9 * np.abs(H).max()
        assert c["Hd"][6 * p, 6 * p] == f32(c["ep"])


@pytest.mark.parametrize("name", list(CASES))
def test_criteria_accept_lapack(name):
    c = make_case(name)
    Hd, b, first = c["Hd"], c["b"], c["first"]
    L = lapack_factor(Hd)
    assert factor_error(L, Hd, first) <= 0.1, name
    xs = lapack_solve(Hd, b)
    assert residual_ratio(Hd, xs, b, gamma_only=True) <= 0.1, name
    assert residual_ratio(Hd, fl32(xs), b) <= 0.55, name
    if c["kappa"] is not None:
        assert forward_ratio(fl32(xs), xs, c["kappa"]) <= 0.5, name
    del L


def test_tiled_restatement_meets_the_criteria_on_the_envelope():
    for name in ("pattern_arrow", "pattern_nonmonotone", "size_449"):
        c = make_case(name)
        L = tiled_cholesky(c["Hd"], c["first"])
        assert factor_error(L, c["Hd"], c["first"]) <= 0.1
        x = tiled_solve(L, c["b"], c["first"])
        assert residual_ratio(c["Hd"], fl32(x), c["b"]) <= 0.55


def test_factor_criterion_rejects_fp32_factor():
    for name in ("size_449", "pattern_arrow", "ba_frontend_426"):
        c = make_case(name)
        L32 = sla.cholesky(c["Hd"].astype(np.float32), lower=True).astype(np.float64)
        assert factor_error(L32, c["Hd"], c["first"]) > 10, name


def test_factor_criterion_rejects_a_skipped_fill_in_update():
    c = make_case("pattern_arrow")
    nt = cdiv(c["n"], T)
    assert not c["Hd"][(nt - 1) * T:, T:2 * T].any()          # tile (nt-1, 1) is zero in Hd and fills in through panel 0
    L = tiled_cholesky(c["Hd"], c["first"], skip=(nt - 1, 1, 0))
    assert factor_error(L, c["Hd"], c["first"]) > 10


def test_residual_and_forward_reject_a_skipped_backward_tile():
    for name in ("pattern_arrow", "pattern_single", "size_449"):
        c = make_case(name)
        k = int(np.flatnonzero(c["first"] < np.arange(len(c["first"])))[-1])        # the last tile row with an off-diagonal tile
        L = lapack_factor(c["Hd"])
        x = fl32(tiled_solve(L, c["b"], c["first"], skip=k))
        assert residual_ratio(c["Hd"], x, c["b"]) > 10, name
        assert forward_ratio(x, lapack_solve(c["Hd"], c["b"]), c["kappa"]) > 10, name


def test_residual_and_forward_reject_an_fp32_solve():
    """The forward criterion catches an fp32 solve on every case with a known kappa.  The residual criterion is a backward-error
    check: on a dense, well-conditioned system an fp32 solve stays inside it (size_449: 0.63 of the bound), so it is held to
    rejecting one where the fp32 factor's error is not hidden by the rounding of x -- the banded, diagonally dominant ones (2.2-2.7x)."""
    for name in ("size_449", "size_2394", "old_banded_700_100_0", "pattern_arrow"):
        c = make_case(name)
        Hd32 = c["Hd"].astype(np.float32)
        x = sla.cho_solve(sla.cho_factor(Hd32, lower=True), c["b"].astype(np.float32)).astype(np.float64)
        assert forward_ratio(x, lapack_solve(c["Hd"], c["b"]), c["kappa"]) > 10, name
        if name in ("old_banded_700_100_0", "pattern_arrow"):
            assert residual_ratio(c["Hd"], x, c["b"]) > 2, name


def test_forward_rejects_four_ulps():
    c = make_case("size_449")
    xs = lapack_solve(c["Hd"], c["b"])
    x = np.asarray(xs, dtype=np.float32)
    i = int(np.abs(xs).argmax())
    for _ in range(4):
        x[i] = np.nextafter(x[i], np.float32(np.copysign(np.inf, x[i])))
    assert forward_ratio(x.astype(np.float64), xs, c["kappa"]) > 1
    assert forward_ratio(fl32(xs), xs, c["kappa"]) <= 0.5
