"""CPU: oracle/svx_ref.py (the restatement of cflx_*_equilibrate / cflx_*_svx) against scipy's LAPACK.

  * geequ / laqge equal scipy's dgeequ and the as / equed of dgesvx(fact='E') bit for bit, poequ / laqsy the s / a_s /
    equed of dposvx(fact='E', lower=1);
  * gesvx / posvx on LAPACK's own factors of the scaled matrix match dgesvx / dposvx(fact='E'): X to its forward-error
    bound, rcond within 2x, ferr within FERR_RATIO and berr within max(2 berr_LAPACK, 4u), the thresholds of
    tests/test_gpu_refine.py;
  * the rank-by-rank maxima and the diagonal gather equal the dense ones on the grids of the GPU tests, with NaN in
    every entry the device must not read."""
import numpy as np
import pytest
from scipy.linalg import lapack

from oracle import chol_ref, chol_solve_ref, layout
from oracle import svx_ref as sr

EPS = 2.0 ** -53
FERR_RATIO = 2.0
BERR_FLOOR = 4 * EPS


def scaled(n, kind, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    s = np.logspace(0, 12, n)
    rng.shuffle(s)
    t = np.logspace(0, 12, n)
    rng.shuffle(t)
    if kind == "rows":
        return A * s[:, None]
    if kind == "cols":
        return A * s[None, :]
    if kind == "both":
        return A * s[:, None] * t[None, :]
    if kind == "tiny":
        return A * 2.0 ** -1020
    if kind == "huge":
        return A * 2.0 ** 1020
    return A


KINDS = ["rows", "cols", "both", "plain", "tiny", "huge"]


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", [0, 1])
def test_geequ_laqge_bit_identical_to_lapack(kind, seed):
    A = scaled(64, kind, seed)
    g = sr.geequ(A)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequ(A)
    assert info == g["info"] == 0
    assert _same(r, g["r"]) and _same(c, g["c"]) and rowcnd == g["rowcnd"] and colcnd == g["colcnd"] and amax == g["amax"]
    As, equed = sr.laqge(A, g["r"], g["c"], g["rowcnd"], g["colcnd"], g["amax"])
    out = lapack.dgesvx(A, np.ones((64, 1)), fact="E")
    assert equed == (out[3].decode() if isinstance(out[3], bytes) else out[3])
    assert _same(As, out[0])
    expect = {"rows": "R", "cols": "C", "plain": "N"}
    if kind in expect:
        assert equed == expect[kind]


def test_geequ_zero_row_and_column():
    A = scaled(32, "plain", 3)
    A[5] = 0.0
    g = sr.geequ(A)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequ(A)
    assert g["info"] == info == 6 and _same(g["r"], r) and g["amax"] == amax
    A = scaled(32, "plain", 4)
    A[:, 9] = 0.0
    g = sr.geequ(A)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequ(A)
    assert g["info"] == info == 32 + 10 and _same(g["r"], r) and g["rowcnd"] == rowcnd and _same(g["c"], c)


def _spd(n, kind, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    A = G @ G.T / n + np.eye(n)
    if kind == "scaled":
        s = np.logspace(0, 6, n)
        rng.shuffle(s)
        A = A * s[:, None] * s[None, :]
    return A


@pytest.mark.parametrize("kind", ["plain", "scaled"])
def test_poequ_laqsy_bit_identical_to_lapack(kind):
    A = _spd(48, kind, 5)
    p = sr.poequ(A)
    As, equed = sr.laqsy(A, p["s"], p["scond"], p["amax"])
    out = lapack.dposvx(A, np.ones((48, 1)), fact="E", lower=1)
    eq = out[2].decode() if isinstance(out[2], bytes) else out[2]
    assert equed == eq == ("Y" if kind == "scaled" else "N")
    if equed == "Y":
        assert _same(p["s"], out[3])
    assert _same(np.tril(As), np.tril(out[0]))


def test_poequ_non_positive_diagonal():
    A = _spd(16, "plain", 6)
    A[4, 4] = 0.0
    A[7, 7] = -1.0
    assert sr.poequ(A)["info"] == 5


def _check_solution(got, lap, what):
    X, fe, be = got["X"], got["ferr"], got["berr"]
    Xl, rcl, fel, bel = lap
    assert np.all(np.max(np.abs(X - Xl), 0) <= 2 * (fe + fel) * np.max(np.abs(Xl), 0)), what
    assert max(got["rcond"] / rcl, rcl / got["rcond"]) <= 2.0, what
    assert np.all(np.maximum(fe / fel, fel / fe) <= FERR_RATIO), what
    assert np.all(be <= np.maximum(2 * bel, BERR_FLOOR)), what


@pytest.mark.parametrize("kind", ["rows", "cols", "both", "plain"])
@pytest.mark.parametrize("trans", [False, True])
def test_gesvx_matches_lapack(kind, trans):
    from scipy.linalg import lu_factor
    n = 96
    A = scaled(n, kind, 7)
    B = np.random.default_rng(8).standard_normal((n, 3))
    g = sr.geequ(A)
    As, equed = sr.laqge(A, g["r"], g["c"], g["rowcnd"], g["colcnd"], g["amax"])
    LU, piv = lu_factor(As)
    perm = np.arange(n)
    for i, p in enumerate(piv):
        perm[i], perm[p] = perm[p], perm[i]
    got = sr.gesvx(As, LU, perm, B, trans, g["r"], g["c"], equed, g["rowcnd"], g["colcnd"])
    out = lapack.dgesvx(A, B, fact="E", trans="T" if trans else "N")
    assert got["info"] == out[11] == 0
    _check_solution(got, (out[7], out[8], out[9], out[10]), f"gesvx {kind} trans={trans}")
    assert got["rpvgrw"] == sr.rpvgrw(As, LU)


@pytest.mark.parametrize("kind", ["plain", "scaled"])
def test_posvx_matches_lapack(kind):
    n = 80
    A = _spd(n, kind, 9)
    B = np.random.default_rng(10).standard_normal((n, 2))
    p = sr.poequ(A)
    As, equed = sr.laqsy(A, p["s"], p["scond"], p["amax"])
    L = np.linalg.cholesky(chol_ref.lower_sym(As))
    got = sr.posvx(chol_ref.lower_sym(As), L, B, p["s"], equed, p["scond"])
    out = lapack.dposvx(A, B, fact="E", lower=1)
    assert got["info"] == out[9] == 0
    _check_solution(got, (out[5], out[6], out[7], out[8]), f"posvx {kind}")


def test_gesvx_zero_pivot():
    n = 12
    rng = np.random.default_rng(11)
    A = np.triu(rng.integers(1, 9, (n, n)).astype(float))
    A[4, 4] = 0.0
    got = sr.gesvx(A, A.copy(), np.arange(n), np.ones((n, 1)))
    assert got["info"] == 5 and got["rcond"] == 0.0 and got["X"] is None
    assert got["rpvgrw"] == np.abs(A[:, :5]).max() / np.abs(np.triu(A[:5, :5])).max()


LU_GRIDS = [(64, 8, 2, 2, 1), (128, 16, 1, 1, 2), (128, 8, 2, 2, 2), (96, 16, 3, 3, 1), (100, 16, 1, 1, 1)]
CHOL_GRIDS = [(256, 32, (2, 2, 1)), (256, 32, (1, 1, 2)), (384, 32, (3, 2, 1)), (384, 32, (1, 3, 2)), (100, 16, (1, 1, 1))]


@pytest.mark.parametrize("N,v,Px,Py,Pz", LU_GRIDS)
def test_rank_by_rank_maxima_lu(N, v, Px, Py, Pz):
    d = layout.dims(N, v, Px, Py, Pz)
    A = scaled(d["M"], "both", N)
    locs = layout.scatter(A, v, Px, Py, Pz)
    for r in range(d["P"]):
        if r % Pz:
            locs[r][...] = np.nan                                      # layers pk != 0: never read
    rmax, cmax = sr.geequ_grid(locs, N, v, Px, Py, Pz)
    g = sr.geequ(A)
    assert _same(1.0 / np.minimum(np.maximum(rmax, sr.SAFMIN), 1 / sr.SAFMIN), g["r"])
    assert _same(1.0 / np.minimum(np.maximum(cmax, sr.SAFMIN), 1 / sr.SAFMIN), g["c"])
    As, equed = sr.laqge(A, g["r"], g["c"], g["rowcnd"], g["colcnd"], g["amax"])
    shares = [sr.apply_share(locs[layout.rank_of(pi, pj, 0, Px, Py, Pz)], v, Px, Py, pi, pj, g["r"], g["c"], equed)
              for pi in range(Px) for pj in range(Py)]
    full = [None] * d["P"]
    for (pi, pj), s in zip([(pi, pj) for pi in range(Px) for pj in range(Py)], shares):
        full[layout.rank_of(pi, pj, 0, Px, Py, Pz)] = s
    assert _same(layout.assemble(full, N, v, Px, Py, Pz), As)


@pytest.mark.parametrize("N,v,grid", CHOL_GRIDS)
def test_rank_by_rank_diagonal_chol(N, v, grid):
    d = chol_ref.dims(N, v, *grid)
    A = _spd(d["N"], "scaled", N)
    locs = chol_solve_ref.scatter(A, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)
    Px, Py, Pz = grid
    for r, loc in enumerate(locs):                                     # NaN in the diagonal tiles' upper triangle too
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        if r % Pz == 0:
            for t in range(d["Kappa"]):
                if t % Px == pi and t % Py == pj:
                    blk = loc[(t // Px) * v:(t // Px + 1) * v, (t // Py) * v:(t // Py + 1) * v]
                    blk[np.triu_indices(v, 1)] = np.nan
    assert _same(sr.diag_grid(locs, N, v, *grid), np.diag(A))
    p = sr.poequ(A)
    As, _ = sr.laqsy(A, p["s"], p["scond"], p["amax"])
    for r, loc in enumerate(locs):
        if r % Pz:
            continue
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        got = sr.sym_apply_share(loc, v, d["Kappa"], Px, Py, pi, pj, p["s"])
        ref = chol_solve_ref.scatter(As, N, v, *grid)[r]
        gr = ((np.arange(d["Ml"]) // v) * Px + pi) * v + np.arange(d["Ml"]) % v
        gc = ((np.arange(d["Nl"]) // v) * Py + pj) * v + np.arange(d["Nl"]) % v
        m = (gr[:, None] // v < d["Kappa"]) & (gc[None, :] // v < d["Kappa"]) & (gr[:, None] >= gc[None, :])
        assert _same(got[m], ref[m]) and np.all(np.isnan(got[~m]) | (got[~m] == loc[~m]))
