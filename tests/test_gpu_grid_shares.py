"""GPU: the per-share kernels of the norms, of the Cholesky and LU validations and of the Cholesky column-operand gather
at grid positions away from the origin, one share at a time on one GPU (the cflx_dbg_* hooks launch the production
kernels through the launch functions the grid paths call).  One GPU only ever runs the share at (0, 0) of a 1 x 1 grid,
which has no padding tiles on the Cholesky path; the shares here cross the kernels' block boundaries (Ml > 256 rows,
Nl > 128 columns and not a multiple of 128), use tiles that are not a power of two, hold Cholesky padding tiles (global
tile index >= Kappa), and sit on 1 x Py and Px x 1 grids.  Every entry a kernel must not read holds NaN (or a huge
value), every reference is plain numpy / math.fsum, and two calls must give the same bits."""
import math
from fractions import Fraction

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, cond_ref, hp_ref
from oracle import refine_ref as rr
from oracle import refinex_ref as rx
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
SUMSQ_PARTIALS = 1184                                                    # conflux_b200/csrc/kernels.h

# (v, Kappa, Px, Py, pi, pj): the share of a Kappa-tile Cholesky matrix (Ml = ceil(Kappa / Px) v rows, Nl = ceil(Kappa /
# Py) v columns) at (pi, pj); the LU-mode kernels read every entry of the same shares
SHARES = [
    (24, 90, 1, 1, 0, 0),   # the origin: 2160 x 2160, nine 256-row CTAs, Nl not a multiple of 128
    (48, 20, 3, 2, 2, 0),   # 336 x 480, v not a power of two, padding tile row 20 under every column
    (16, 29, 1, 3, 0, 2),   # 1 x Py: 464 x 160, padding tile column 29
    (15, 11, 2, 1, 1, 0),   # Px x 1: 90 x 165, odd v, padding tile row 11
    (32, 13, 2, 3, 1, 1),   # 224 x 160, padding tile row 13 and column 13
]
IDS = [f"v{s[0]}-K{s[1]}-{s[2]}x{s[3]}-at{s[4]}{s[5]}" for s in SHARES]


def _dims(v, Kappa, Px, Py):
    mt, nt = -(-Kappa // Px), -(-Kappa // Py)
    return mt * v, nt * v, max(mt * Px, nt * Py) * v


def _gidx(n, P, p, v):
    l = np.arange(n)
    return ((l // v) * P + p) * v + l % v


def _first_local_tile(g, p, P):
    return 0 if g <= p else (g - p + P - 1) // P


def _bits(x):
    return np.ascontiguousarray(x).view(np.int64)


def _same(a, b):
    """the same bits, except that any NaN matches any NaN (the device may produce its own NaN payload)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(_bits(a[~na]), _bits(b[~nb]))


_WORST = {}


@pytest.fixture
def margins():
    """margins(bound, m): m = the observed error over the bound; the worst of each is printed after the module"""
    def note(name, m):
        _WORST[name] = max(_WORST.get(name, 0.0), float(m))
    return note


@pytest.fixture(scope="module", autouse=True)
def _print_margins():
    yield
    for name, m in sorted(_WORST.items()):
        print(f"\nworst observed error / bound, {name}: {m:.3g}")


# ----------------------------------------------------------------------------------------------- norms
def _norm_ref(A, mode, v, Kappa, Px, Py, pi, pj, M):
    """out[g] = math.fsum of the entries the kernel must read (exact up to its final rounding), zeros elsewhere; and
    the mask of the global indices the share holds"""
    Ml, Nl = A.shape
    gr, gc = _gidx(Ml, Px, pi, v), _gidx(Nl, Py, pj, v)
    out, held = np.zeros(M), np.zeros(M, dtype=bool)
    a = np.abs(A)
    if mode == "row":
        for r in range(Ml):
            out[gr[r]] = math.fsum(a[r])
        held[gr] = True
    elif mode == "col":
        for c in range(Nl):
            out[gc[c]] = math.fsum(a[:, c])
        held[gc] = True
    else:
        mnn, mtn = rr.sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj)
        parts = [[] for _ in range(M)]
        for c in range(Nl):
            parts[gc[c]].append(a[mnn[:, c], c])
        for r in range(Ml):
            parts[gr[r]].append(a[r, mtn[r]])                           # a_ji = a_ij: strictly lower row sums
        for g in range(M):
            if parts[g]:
                out[g] = math.fsum(np.concatenate(parts[g]))
        held[gr] = held[gc] = True
    return out, held


def _norm_input(v, Kappa, Px, Py, pi, pj, mode, seed):
    """random magnitudes over 12 decades; column 0 and row 0 (of what the mode reads) hold one 1.0 and then 2^-54 in
    every other entry: a sequential sum in storage order rounds every 1 + 2^-54 back to 1 and loses them all"""
    Ml, Nl, _ = _dims(v, Kappa, Px, Py)
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((Ml, Nl)) * np.exp(rng.uniform(-14, 14, (Ml, Nl)))
    A[:, 0] = 2.0 ** -54
    A[0, :] = 2.0 ** -54
    A[0, 0] = 1.0
    if mode == "sym":
        mnn, _ = rr.sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj)
        g0 = _gidx(Nl, Py, pj, v)[0]     # global column g0: its lower column part and the row g0 (if held) all tiny,
        A[_gidx(Ml, Px, pi, v) == g0, :] = 2.0 ** -54                   # with 1.0 first in storage order
        A[0, 0] = 2.0 ** -54
        A[~mnn] = np.nan                 # upper triangles of the diagonal tiles, strictly upper tiles, padding tiles
        A[np.flatnonzero(mnn[:, 0])[0], 0] = 1.0
    return A


# The bound: every CTA's partial is a Neumaier sum (s + c within u |S| + O(n u^2) S of its exact sum S: the entries are
# non-negative, so sum |a| = S) rounded once to a double (u), and the partials are combined by a second Neumaier sum
# in a fixed order (u of the total, + O(n u^2)); the strictly lower row sums of "sym" go through the same pairwise tree
# of (s, c) pairs.  So |out - exact| <= 2u exact + O(n u^2) exact <= 3u exact for every n << 1 / u.
@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj", SHARES, ids=IDS)
@pytest.mark.parametrize("mode", ["col", "sym", "row"])
def test_norm_share(mode, v, Kappa, Px, Py, pi, pj, margins):
    Ml, Nl, M = _dims(v, Kappa, Px, Py)
    A = _norm_input(v, Kappa, Px, Py, pi, pj, mode, seed=Ml + Nl + pi)
    out = cb.dbg.norm_share(mode, A, v, Kappa, (Px, Py), (pi, pj), M=M)
    assert np.array_equal(_bits(out), _bits(cb.dbg.norm_share(mode, A, v, Kappa, (Px, Py), (pi, pj), M=M)))
    exact, held = _norm_ref(A, mode, v, Kappa, Px, Py, pi, pj, M)
    assert np.all(np.isfinite(out))
    assert np.all(out[~held] == 0.0)                                     # indices the share does not hold: exactly 0
    err = np.abs(out - exact)
    assert np.all(err <= 3 * U * exact), np.max(err / np.maximum(exact, 1e-300))
    margins("norm share 3u", float(np.max(err / np.maximum(exact, 1e-300)) / (3 * U)))
    # a sequential sum of the same entries in storage order misses the bound
    if mode == "sym":
        mnn, mtn = rr.sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj)
        g = _gidx(Nl, Py, pj, v)[0]
        rows = np.flatnonzero(_gidx(Ml, Px, pi, v) == g)
        first = np.concatenate([A[mnn[:, 0], 0]] + [A[r, mtn[r]] for r in rows])
    else:
        first = A[:, 0] if mode == "col" else A[0, :]
        g = _gidx(Nl, Py, pj, v)[0] if mode == "col" else _gidx(Ml, Px, pi, v)[0]
    naive = np.cumsum(np.abs(first))[-1]
    assert abs(naive - exact[g]) > 3 * U * exact[g]


@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj", SHARES, ids=IDS)
@pytest.mark.parametrize("mode", ["col", "row"])
def test_norm_share_nan_stays_in_its_line(mode, v, Kappa, Px, Py, pi, pj):
    Ml, Nl, M = _dims(v, Kappa, Px, Py)
    A = _norm_input(v, Kappa, Px, Py, pi, pj, mode, seed=7)
    base = cb.dbg.norm_share(mode, A, v, Kappa, (Px, Py), (pi, pj), M=M)
    r, c = Ml - 1 - v // 3, Nl // 2 + 1
    A[r, c] = np.nan
    out = cb.dbg.norm_share(mode, A, v, Kappa, (Px, Py), (pi, pj), M=M)
    g = _gidx(Nl, Py, pj, v)[c] if mode == "col" else _gidx(Ml, Px, pi, v)[r]
    assert np.isnan(out[g])
    keep = np.arange(M) != g
    assert np.array_equal(_bits(out[keep]), _bits(base[keep]))


def test_norm_share_is_the_public_anorm():
    """the pieces at 1 x 1 are what lu_rcond and cholesky.rcond take the maximum of"""
    N, v = 512, 32
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    A = gv.data.copy()
    cb.LU_rep(gv)
    _, anorm = cb.lu_rcond(gv)
    assert cb.dbg.norm_share("col", A, v).max() == anorm
    gv.free_comms()
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    ch.generateInputMatrixDistributed()
    A = ch.data.copy()
    ch.parallelCholesky()
    _, anorm = ch.rcond()
    assert cb.dbg.norm_share("sym", A, v, Kappa=N // v).max() == anorm
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- Cholesky validation
def _exact_sumsq(x):
    """the exact sum of squares, rounded once: Veltkamp's split makes every a^2 = h^2 + 2 h l + l^2 exact in doubles"""
    x = np.asarray(x, dtype=np.float64).ravel()
    t = x * (2.0 ** 27 + 1)
    h = t - (t - x)
    lo = x - h
    return math.fsum(np.concatenate([h * h, 2 * h * lo, lo * lo]))


def _sumsq_gamma_k(Ml, Nl):
    # The longest addition chain of one squared entry to the result: the fma chain of one thread's grid-stride loop
    # (SUMSQ_PARTIALS CTAs of 256 threads), the two shuffle trees of its CTA (5 levels each: 32 lanes, then the 8 warps'
    # sums padded to 32), launch_sum_partials' 1024 threads each adding ceil(SUMSQ_PARTIALS / 1024) partials in index
    # order, its two shuffle trees (5 + 5 levels), and the final += into the zeroed result.
    per_thread = -(-(Ml * Nl) // (SUMSQ_PARTIALS * 256))
    return per_thread + 5 + 5 + -(-SUMSQ_PARTIALS // 1024) + 5 + 5 + 1


def _gamma(k):
    return k * U / (1 - k * U)


@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj", SHARES, ids=IDS)
@pytest.mark.parametrize("fill", ["nan", "huge"])
def test_chol_validate_sumsq(fill, v, Kappa, Px, Py, pi, pj, margins):
    """the Frobenius norms of cholesky.validate read the lower triangle of the real tiles only: NaN or 1e150 in the
    padding tiles, in the strictly upper tiles and above the diagonal of the diagonal tiles does not reach them"""
    Ml, Nl, _ = _dims(v, Kappa, Px, Py)
    mnn, _ = rr.sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj)
    rng = np.random.default_rng(Ml * 7 + Nl)
    bad = np.nan if fill == "nan" else 1e150
    k = _sumsq_gamma_k(Ml, Nl)
    for data in ("random", "tiny"):
        if data == "random":
            A = rng.standard_normal((Ml, Nl)) * np.exp(rng.uniform(-10, 10, (Ml, Nl)))
        else:   # one 1 before thousands of 2^-27: every square 2^-54 is a tie a sequential sum rounds back to 1
            A = np.full((Ml, Nl), 2.0 ** -27)
            A.ravel()[np.flatnonzero(mnn.ravel())[0]] = 1.0
        A[~mnn] = bad
        _, s = cb.dbg.chol_validate_share(A, v, Kappa, (Px, Py), (pi, pj))
        _, s2 = cb.dbg.chol_validate_share(A, v, Kappa, (Px, Py), (pi, pj))
        assert _bits(np.float64(s)) == _bits(np.float64(s2))
        exact = _exact_sumsq(A[mnn])
        assert np.isfinite(s) and abs(s - exact) <= _gamma(k) * exact, (data, s, exact)
        margins("chol validate sumsq gamma_k", abs(s - exact) / (_gamma(k) * exact))
        if data == "tiny":
            x = A[mnn]
            naive = np.cumsum(x * x)[-1]
            assert abs(naive - exact) > _gamma(k) * exact


def _steps(v, Kappa, Px, Py, pi, pj):
    """steps t on both sides of the share's first tile row and column, and the last one"""
    return sorted({t for t in (0, 1, pi, pi + 1, pi + Px, pj, pj + Py, Kappa - 1) if 0 <= t < Kappa})


@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj", SHARES, ids=IDS)
def test_chol_validate_panel(v, Kappa, Px, Py, pi, pj):
    Ml, Nl, _ = _dims(v, Kappa, Px, Py)
    A = np.random.default_rng(3).standard_normal((Ml, Nl))
    mnn, _ = rr.sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj)
    A[~mnn] = np.nan                              # what the panel masks to zero must not be read (padding rows are copied)
    gr = _gidx(Ml, Px, pi, v)
    ldbuf = Ml + (Ml & 1) + 2
    for t in _steps(v, Kappa, Px, Py, pi, pj):
        PT, _ = cb.dbg.chol_validate_share(A, v, Kappa, (Px, Py), (pi, pj), t=t)
        PT2, _ = cb.dbg.chol_validate_share(A, v, Kappa, (Px, Py), (pi, pj), t=t)
        assert np.array_equal(_bits(PT), _bits(PT2))
        want = np.full(v * ldbuf, np.nan)
        if t % Py == pj:
            row0 = _first_local_tile(t, pi, Px) * v
            n = Ml - row0
            ldp = max(2, n + (n & 1))                                    # the broadcast piece's leading dimension
            if n > 0:
                col0 = (t // Py) * v
                gc = t * v + np.arange(v)
                blk = A[row0:, col0:col0 + v]                            # n x v
                keep = gr[row0:, None] >= gc[None, :]
                panel = np.where(keep, blk, 0.0).T                       # v x n
                for c in range(v):
                    want[c * ldp:c * ldp + n] = panel[c]
        assert np.array_equal(_bits(PT.ravel()), _bits(want)), t


# ----------------------------------------------------------------------------------------------- LU validation
@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj", SHARES, ids=IDS)
def test_lu_validate_extracts(v, Kappa, Px, Py, pi, pj):
    lcm = Px * Py // math.gcd(Px, Py)
    Nt = -(-Kappa // lcm) * lcm                                          # the LU's shares of an Nt v square matrix
    Ml, Nl = Nt // Px * v, Nt // Py * v
    C0 = np.random.default_rng(11).standard_normal((Ml, Nl))
    gr, gc = _gidx(Ml, Px, pi, v), _gidx(Nl, Py, pj, v)
    ldp = Ml + (Ml & 1)
    for t in sorted({x for x in _steps(v, Nt, Px, Py, pi, pj) + [Nt - 1] if 0 <= x < Nt}):
        row_lo = min(Ml, _first_local_tile(t, pi, Px) * v)
        col_lo = min(Nl, _first_local_tile(t, pj, Py) * v)
        lc0, lr0 = (t // Py) * v, (t // Px) * v
        readL = np.zeros((Ml, Nl), dtype=bool)
        readU = np.zeros((Ml, Nl), dtype=bool)
        wantL, wantU = np.full((v, ldp), np.nan), np.full((v, Nl), np.nan)
        if t % Py == pj and row_lo < Ml:
            tc = t * v + np.arange(v)
            q = gr[row_lo:, None]
            readL[row_lo:, lc0:lc0 + v] = q > tc[None, :]
            blk = C0[row_lo:, lc0:lc0 + v]
            wantL[:, row_lo:Ml] = np.where(q > tc, blk, np.where(q == tc, 1.0, 0.0)).T
        if t % Px == pi and col_lo < Nl:
            q = t * v + np.arange(v)[:, None]
            readU[lr0:lr0 + v, col_lo:] = gc[None, col_lo:] >= q
            wantU[:, col_lo:] = np.where(gc[None, col_lo:] >= q, C0[lr0:lr0 + v, col_lo:], 0.0)
        C = np.where(readL | readU, C0, np.nan)                          # nothing else may be read
        LT, Uo = cb.dbg.lu_validate_share(C, v, (Px, Py), (pi, pj), t=t)
        LT2, Uo2 = cb.dbg.lu_validate_share(C, v, (Px, Py), (pi, pj), t=t)
        assert np.array_equal(_bits(LT), _bits(LT2)) and np.array_equal(_bits(Uo), _bits(Uo2))
        assert np.array_equal(_bits(LT), _bits(wantL)), t
        assert np.array_equal(_bits(Uo), _bits(wantU)), t


# ----------------------------------------------------------------------------------------------- Cholesky gather
@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj", SHARES, ids=IDS)
def test_chol_gather_cols(v, Kappa, Px, Py, pi, pj):
    """Bc holds, for every real column tile j >= gfirst of the share (in local order from the first such tile),
    exactly the rows of tile j of the broadcast panel.  The panel entry of global row g, column c is g * 1024 + c (exact), so a wrong piece, row or column shows.
    Padding column tiles (j >= Kappa) have no contract: when Py differs from Px their row offset can run past the end of
    the piece's active rows (still inside its buffer); they only feed padding columns, so nothing is asserted there."""
    Ml, Nl, _ = _dims(v, Kappa, Px, Py)
    for gfirst in sorted({0, 1, pj, pi + 1, Kappa - 1}):
        if gfirst >= Kappa:
            continue
        pieces = []
        for p in range(Px):
            first = _first_local_tile(gfirst, p, Px)
            rows = Ml - first * v
            ld = max(2, rows + (rows & 1))
            piece = np.full((v, ld), np.nan)                             # the rounding-up row (odd rows) is NaN
            if rows > 0:
                g = _gidx(Ml, Px, p, v)[first * v:]
                piece[:, :rows] = g[None, :] * 1024.0 + np.arange(v)[:, None]
            pieces.append(piece)
        Bc = cb.dbg.chol_gather_cols(pieces, v, Px, Py, pj, Ml, Nl, gfirst)
        assert np.array_equal(_bits(Bc), _bits(cb.dbg.chol_gather_cols(pieces, v, Px, Py, pj, Ml, Nl, gfirst)))
        lj0 = _first_local_tile(gfirst, pj, Py)                          # Bc's tile t is local column tile lj0 + t
        assert np.all(np.isnan(Bc[:, (Nl // v - lj0) * v:]))             # nothing is written past the last one
        for lt in range(lj0, Nl // v):
            j = lt * Py + pj
            if j >= Kappa:
                continue
            want = (j * v + np.arange(v))[None, :] * 1024.0 + np.arange(v)[:, None]
            t = lt - lj0
            assert np.array_equal(Bc[:, t * v:(t + 1) * v], want), (gfirst, j)


# ----------------------------------------------------------------------------------------------- refinement assembly
def _safe(M):
    eps, safmin = 2.0 ** -53, 2.0 ** -1022
    nz = M + 1.0
    return nz * safmin, nz * safmin / eps, nz * eps


def _fma(a, b, c):
    """a * b + c rounded once (Fraction's float() rounds correctly)"""
    out = np.empty(np.broadcast(a, b, c).shape)
    for i, (x, y, z) in enumerate(zip(*(np.broadcast_to(t, out.shape).ravel() for t in (a, b, c)))):
        out.ravel()[i] = float(Fraction(x) * Fraction(y) + Fraction(z))
    return out


def _assembly_case(grid, v, kind, seed):
    """the Px Py Pz chunks (NaN on the layers pk != 0, in the columns past nrhs and in the rows no row g < M reads) and
    B, with rows of heavy cancellation, b = s = 0, and s < safe2"""
    Px, Py, Pz = grid
    nn, tn = kind in ("nn", "sym"), kind in ("tn", "sym")
    Nt = 6
    Ml, Nl, M = Nt // Px * v, Nt // Py * v, Nt * v - 5
    nrhs, ldn = 3, 8
    rows = (Ml if nn else 0) + (Nl if tn else 0)
    rng = np.random.default_rng(seed)
    ch = np.full((Px * Py * Pz, rows, 2 * ldn), np.nan)
    for pi in range(Px):
        for pj in range(Py):
            k = (pi * Py + pj) * Pz
            p = rng.standard_normal((rows, nrhs)) * np.exp(rng.uniform(-5, 5, (rows, nrhs)))
            ch[k, :, :nrhs] = p
            ch[k, :, ldn:ldn + nrhs] = np.abs(p) * (1 + rng.uniform(0, 1, p.shape))
    nnd = {(pi, pj): (ch[(pi * Py + pj) * Pz, :Ml, :nrhs], ch[(pi * Py + pj) * Pz, :Ml, ldn:ldn + nrhs])
           for pi in range(Px) for pj in range(Py)} if nn else None
    off = Ml if nn else 0
    tnd = {(pi, pj): (ch[(pi * Py + pj) * Pz, off:off + Nl, :nrhs], ch[(pi * Py + pj) * Pz, off:off + Nl, ldn:ldn + nrhs])
           for pi in range(Px) for pj in range(Py)} if tn else None
    P, _ = rr._assemble(nnd, tnd, M, v, Px, Py, Ml)
    B = np.full((M, ldn), np.nan)
    B[:, :nrhs] = P * (1 + 1e-14 * rng.standard_normal(P.shape))     # heavy cancellation: b close to the sum
    B[1::3, :nrhs] = rng.standard_normal(B[1::3, :nrhs].shape)

    def rows_of(g):                                                  # the (chunk, row) pairs row g reads
        T, e = divmod(g, v)
        out = [((T % Px * Py + pj) * Pz, (T // Px) * v + e) for pj in range(Py)] if nn else []
        return out + ([((pi * Py + T % Py) * Pz, off + (T // Py) * v + e) for pi in range(Px)] if tn else [])
    for k, r in rows_of(0):                                          # b = 0 with s = 0
        ch[k, r, [0, ldn]] = 0.0
    B[0, 0] = 0.0
    for k, r in rows_of(2):                                          # s < safe2
        ch[k, r, [1, ldn + 1]] = 1e-300
    B[2, 1] = 1e-300
    read = np.zeros(ch.shape[:2], dtype=bool)
    for g in range(M):
        for k, r in rows_of(g):
            read[k, r] = True
    ch[~read] = np.nan
    return dict(ch=ch, B=B, M=M, Ml=Ml, Nl=Nl, nn=nn, tn=tn, nrhs=nrhs, ldn=ldn, rows_of=rows_of)


GRIDS3 = [(1, 1, 1), (2, 3, 1), (3, 2, 2), (1, 3, 2), (2, 1, 1)]


@pytest.mark.parametrize("grid", GRIDS3, ids=lambda g: "x".join(map(str, g)))
@pytest.mark.parametrize("kind", ["nn", "tn", "sym"])
@pytest.mark.parametrize("mode", ["gerfs", "lin_berr"])
def test_refine_assemble(mode, kind, grid):
    v = 16
    c = _assembly_case(grid, v, kind, seed=len(kind) * 10 + sum(grid))
    M, nrhs = c["M"], c["nrhs"]
    args = (c["ch"], c["B"], grid, v, M, c["Ml"], c["Nl"], c["nn"], c["tn"], nrhs)
    o = cb.dbg.refine_assemble(mode, *args)
    o2 = cb.dbg.refine_assemble(mode, *args)
    for k in o:
        assert _same(o[k], o2[k])
    Px, Py, Pz = grid
    Ml, off, ldn = c["Ml"], c["Ml"] if c["nn"] else 0, c["ldn"]
    ch0 = lambda pi, pj: c["ch"][(pi * Py + pj) * Pz]                # noqa: E731
    nnd = {(i, j): (ch0(i, j)[:Ml, :nrhs], ch0(i, j)[:Ml, ldn:ldn + nrhs]) for i in range(Px) for j in range(Py)}
    tnd = {(i, j): (ch0(i, j)[off:off + c["Nl"], :nrhs], ch0(i, j)[off:off + c["Nl"], ldn:ldn + nrhs])
           for i in range(Px) for j in range(Py)}
    P, Q = rr._assemble(nnd if c["nn"] else None, tnd if c["tn"] else None, M, v, Px, Py, Ml)
    b = c["B"][:, :nrhs]
    safe1, safe2, nzeps = _safe(M)
    r, s = b - P, Q + np.abs(b)
    assert _same(o["R"][:, :nrhs], r)
    assert np.all(np.isnan(o["R"][:, nrhs:]))
    with np.errstate(divide="ignore", invalid="ignore"):
        if mode == "gerfs":
            ratio = np.where(s > safe2, np.abs(r) / s, (np.abs(r) + safe1) / (s + safe1))
            # W = |r| + nz eps s (+ safe1): the product may be contracted into one fused multiply-add
            fused, plain = _fma(nzeps, s, np.abs(r)), np.abs(r) + nzeps * s
            fused, plain = (np.where(s > safe2, x, x + safe1) for x in (fused, plain))
            W = o["W"][:, :nrhs]
            assert _same(W, fused) or _same(W, plain)
        else:
            ratio = np.where(s != 0, (np.abs(r) + safe1) / s, 0.0)
            assert _same(o["Q"][:, :nrhs], Q)
    assert _same(o["ratio"][:, :nrhs], ratio)
    assert o["ratio"][0, 0] == (1.0 if mode == "gerfs" else 0.0)   # b = s = 0
    # a NaN partial makes its row NaN and no other row
    k, row = c["rows_of"](4)[-1]
    c["ch"][k, row, 2] = np.nan
    o3 = cb.dbg.refine_assemble(mode, *args)
    assert np.isnan(o3["R"][4, 2])
    keep = np.ones(o3["R"].shape, dtype=bool)
    keep[4, 2] = False
    assert _same(o3["R"][keep], o["R"][keep])


@pytest.mark.parametrize("grid", GRIDS3, ids=lambda g: "x".join(map(str, g)))
@pytest.mark.parametrize("kind", ["nn", "tn", "sym"])
def test_refine_assemble_x(kind, grid, margins):
    """R = b - the double-double sum of the (hi, lo) partials, rounded once: bit for bit the restatement, and within
    u |r| + 4 u^2 sum |partials| of the exact b - sum (hi + lo)"""
    v = 16
    c = _assembly_case(grid, v, kind, seed=7 + sum(grid))
    ch, ldn, nrhs, M = c["ch"], c["ldn"], c["nrhs"], c["M"]
    rng = np.random.default_rng(3)
    lo = ch[:, :, :nrhs] * 2.0 ** -53 * rng.uniform(-1, 1, ch[:, :, :nrhs].shape)
    ch[:, :, ldn:ldn + nrhs] = lo                                    # (hi, lo) pairs; NaN stays NaN
    args = (ch, c["B"], grid, v, M, c["Ml"], c["Nl"], c["nn"], c["tn"], nrhs)
    R = cb.dbg.refine_assemble("x", *args)["R"]
    assert _same(R, cb.dbg.refine_assemble("x", *args)["R"])
    assert np.all(np.isnan(R[:, nrhs:]))
    Px, Py, Pz = grid
    Ml, off = c["Ml"], c["Ml"] if c["nn"] else 0
    worst, violated = 0.0, False
    for j in range(nrhs):
        ch0 = lambda i, jj: ch[(i * Py + jj) * Pz]                   # noqa: E731
        nnd = {(i, jj): (ch0(i, jj)[:Ml, j], ch0(i, jj)[:Ml, ldn + j]) for i in range(Px) for jj in range(Py)}
        tnd = {(i, jj): (ch0(i, jj)[off:off + c["Nl"], j], ch0(i, jj)[off:off + c["Nl"], ldn + j])
               for i in range(Px) for jj in range(Py)}
        H, L = rx._assemble_x(nnd if c["nn"] else None, tnd if c["tn"] else None, M, v, Px, Py)
        b = c["B"][:, j]
        s = b + (-H)
        bb = s - b
        e = (b - (s - bb)) + (-H - bb)
        assert _same(R[:, j], s + (e - L))
        for g in range(M):
            parts = [(ch[k, r, j], ch[k, r, ldn + j]) for k, r in c["rows_of"](g)]
            exact = Fraction(b[g]) - sum(Fraction(h) + Fraction(lw) for h, lw in parts)
            tol = U * abs(R[g, j]) + 4 * U * U * sum(abs(h) + abs(lw) for h, lw in parts)
            err = abs(float(Fraction(R[g, j]) - exact))
            assert err <= tol, (g, j, err, tol)
            worst = max(worst, err / tol if tol else 0.0)
            violated |= abs(float(Fraction(b[g] - sum(h for h, _ in parts)) - exact)) > tol   # hi only, in FP64
    margins("refine assemble_x u|r| + 4u^2 sum", worst)
    assert violated


# ----------------------------------------------------------------------------------------------- per-column steps
@pytest.mark.parametrize("M", [1, 255, 257, 1000])
def test_refine_columns(M):
    nrhs, ldn = 5, 8
    rng = np.random.default_rng(M)
    A = np.full((M, ldn), np.nan)
    D = np.full((M, ldn), np.nan)                                    # NaN in the ldn padding columns
    A[:, :nrhs] = rng.standard_normal((M, nrhs))
    D[:, :nrhs] = rng.standard_normal((M, nrhs)) * 1e-8
    A[M // 2, 1] = np.nan                                            # NaN wins
    A[M - 1, 2], D[M - 1, 2] = 0.0, 3.0                              # y = 0 != dy: +inf
    A[0, 3] = D[0, 3] = 0.0                                          # y = dy = 0: 0
    A[:, 4] = -np.abs(A[:, 4])                                       # every entry below the start value 0
    d = np.exp(rng.uniform(-3, 3, M))
    sel = np.array([2, 1, 0, 2, 1, 1, 2, 0], dtype=np.int32)
    T = np.full((M, ldn), np.nan)
    T[:, :nrhs] = A[:, :nrhs] * 2.0 ** -60 * rng.standard_normal((M, nrhs))
    for dd in (None, d):
        o = cb.dbg.refine_columns(A, D, sel, nrhs, d=dd, T=T)
        o2 = cb.dbg.refine_columns(A, D, sel, nrhs, d=dd, T=T)
        for k in o:
            assert _same(o[k], o2[k])
        a, dy = A[:, :nrhs], D[:, :nrhs]
        want_max = [np.nan if np.isnan(a[:, j]).any() else max(0.0, a[:, j].max()) for j in range(nrhs)]
        assert _same(o["max"], np.array(want_max))
        # rx.stats with numpy's max / min, which already let a NaN win
        want = np.array([rx.stats(a[:, j], dy[:, j], dd) for j in range(nrhs)])
        assert _same(o["stats"], want)
    assert np.isinf(o["stats"][2, 3]) and o["stats"][3, 3] >= 0 and np.isnan(o["stats"][1, 0])
    s = sel[:nrhs].astype(bool)
    assert _same(o["select"][:, :nrhs], np.where(s, a, 0.0))
    assert _same(o["add"][:, :nrhs], np.where(s, a + dy, a))
    t = T[:, :nrhs]
    yw, tw = rx.wwaddw(a, t, dy)
    how = sel[:nrhs]
    wantY = np.where(how == 2, yw, np.where(how == 1, a + dy, a))
    wantT = np.where(how == 2, tw, t)
    assert _same(o["Y"][:, :nrhs], wantY)
    assert _same(o["T"][:, :nrhs], wantT)


# ----------------------------------------------------------------------------------------------- refusals
_Z, _X = np.zeros((32, 32)), np.zeros((32, 1))
# each hook on the share of a 32-row tile-16 matrix at grid row pi = Px = 2 (chol_gather_cols: column pj = Py = 2), off
# the grid, with every other argument valid
OFF_GRID = {
    "residual": lambda: cb.dbg.residual(_Z, "nn", 16, grid=(2, 1), pos=(2, 0), Xc=_X),
    "residual_x": lambda: cb.dbg.residual_x(_Z, "nn", 16, grid=(2, 1), pos=(2, 0), Xc=_X),
    "equil": lambda: cb.dbg.equil(_Z, 16, grid=(2, 1), pos=(2, 0)),
    "growth_cols": lambda: cb.dbg.growth_cols("lu", _Z, _Z, 16, grid=(2, 1), pos=(2, 0)),
    "inverse_share": lambda: cb.dbg.inverse_share("lu", 16, (2, 1), (2, 0), 64, 0, 8, 32, 64),
    "solve_local_share": lambda: cb.dbg.solve_local_share("lu", 16, (2, 1), (2, 0), 64, 8, 0, 8, 32, B=_Z[:, :16]),
    "norm_share": lambda: cb.dbg.norm_share("col", _Z, 16, grid=(2, 1), pos=(2, 0)),
    "chol_validate_share": lambda: cb.dbg.chol_validate_share(_Z, 16, 2, (2, 1), (2, 0)),
    "lu_validate_share": lambda: cb.dbg.lu_validate_share(np.zeros((32, 64)), 16, (2, 1), (2, 0)),
    "chol_gather_cols": lambda: cb.dbg.chol_gather_cols([np.zeros((16, 32))], 16, 1, 2, 2, 32, 32, 0),
}


@pytest.mark.parametrize("hook", list(OFF_GRID))
def test_share_hooks_refuse_off_grid(hook):
    """a share off the grid is refused before any kernel runs, with an error that names the hook and the condition,
    not the text of an earlier failure"""
    with pytest.raises(cb.ConfluxError, match="unknown probe"):
        cb.dbg.fp64_peak_ex(99)
    with pytest.raises(cb.ConfluxError) as e:
        OFF_GRID[hook]()
    cond = "pj outside [0, Py)" if hook == "chol_gather_cols" else "pi outside [0, Px)"
    assert f"cflx_dbg_{hook}: refused, {cond}" in str(e.value)
    assert "unknown probe" not in str(e.value)


def test_hooks_refuse_null_inputs():
    """a missing input array is refused before anything is uploaded or launched; with no pivots to push, push_pivots
    reads no array and accepts NULL"""
    lib = cb.lib()
    with pytest.raises(cb.ConfluxError, match=r"push_pivots: refused, !A_inout \|\| !pivot_rows"):
        cb.check(lib.cflx_dbg_push_pivots(8, 8, None, 1, None, 0, None, None), "push_pivots")
    assert lib.cflx_dbg_push_pivots(8, 8, None, 0, None, 0, None, None) == 0
    with pytest.raises(cb.ConfluxError, match=r"ozaki_gemm: refused, !AT \|\| !B"):
        cb.check(lib.cflx_dbg_ozaki_gemm(2, 2, 128, 0, 0, 0, *[None] * 8, 1, None, None), "ozaki_gemm")


# ----------------------------------------------------------------------------------------------- end to end
def test_multi_gpu_chol_padded_grid():
    """N = 288, v = 32 on 2 x 1 x 1: Kappa = 9, so rank (1, 0) holds padding tile row 9 under every column.  With NaN in
    the padding tiles, above the diagonal and on no other layer, validate() stays finite and agrees with the residual
    of the assembled input, and rcond()'s anorm is the 1-norm of the symmetric matrix."""
    N, v, grid = 288, 32, (2, 1, 1)
    if n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    G = np.random.default_rng(21).standard_normal((N, N))
    A = G @ G.T + N * np.eye(N)
    As = np.where(np.tril(np.ones((N, N), dtype=bool)), A, np.nan)
    locs = chol_solve_ref.scatter(As, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        out = dict(L=ch.local_factor(), val=ch.validate(), rc=ch.rcond())
        ch.finalize()
        return out

    rs = run_ranks(2, body)
    L = np.tril(chol_ref.assemble([r["L"] for r in rs], N, v, *grid))[:N, :N]
    absr, rel = rs[0]["val"]
    assert all(r["val"] == (absr, rel) for r in rs)
    assert np.isfinite(absr) and np.isfinite(rel)
    R, LL = hp_ref.chol_residual(A, L)
    ref = float(np.sqrt(np.sum(np.asarray(R, dtype=np.float64) ** 2)))
    # the replayed residual differs from the exact one by at most gamma_{N+1} |L| |L^T| in every lower entry
    slack = float(np.sqrt(np.sum((_gamma(N + 1) * LL) ** 2)))
    assert abs(absr - ref) <= slack, (absr, ref, slack)
    assert abs(rel - absr / math.sqrt(_exact_sumsq(np.tril(A)))) <= _gamma(2 * _sumsq_gamma_k(N // 2, N)) * rel
    anorm = rs[0]["rc"][1]
    want = cond_ref.norm1_chol(locs, N, v, *grid)
    assert abs(anorm - want) <= 3 * U * want
