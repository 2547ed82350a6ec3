"""GPU: cflx_lu_equilibrate_b / cflx_lu_svxx and cflx_chol_equilibrate_b / cflx_chol_svxx (LAPACK dgeequb + dlaqge,
dgesvxx, dpoequb + dlaqsy, dposvxx on the grid).

  * exactness: the device's power-of-two scales, condition numbers, amax, equed and info equal scipy's dgeequb (LU) and
    OpenBLAS's dpoequb and the restatement oracle/svxx_ref.py (Cholesky) bit for bit; the scaled matrix is diag(r) A
    diag(c) exactly, and factoring after a device equilibrate_b gives the factors (and permutation) of the host-scaled
    matrix uploaded with set_local, bit for bit;
  * the drivers pinned to their parts: svxx's X, berr, bounds, rcond and info equal, bit for bit, the solve of the
    host-scaled B, refine_x of that, and the unscaling -- after equilibrate_b, equilibrate or no scaling;
  * growth: rpvgrw equals gerpvgrw / porpvgrw on the device's own factors, svx's rpvgrw is unchanged, and dbg.growth_cols
    equals the restatement exactly off the grid origin, with Kappa short of the share and NaN wherever it must not read;
  * behaviour: graded inputs get equed R / C / B and trusted bounds that hold against the double-double solution; the
    zero pivot (X untouched); kappa ~ 1e17 (info = M + j, untrusted); determinism, no side effects, the argument and
    state rules, and the multi-GPU grids (skipped on fewer GPUs)."""
import ctypes

import numpy as np
import pytest
from scipy.linalg import lapack

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, layout
from oracle import refine_ref as rr
from oracle import svx_ref as sr
from oracle import svxx_ref as xr
from tests._harness import n_gpus, run_ranks
from tests.test_refinex_ref import errors, true_solution
from tests.test_svxx_ref import lapack_dpoequb

pytestmark = pytest.mark.gpu
CFLX_ERR_ARG, CFLX_ERR_STATE = -1, -5                                     # include/conflux_b200.h
LU_GRIDS = [(64, 8, 2, 2, 1), (128, 16, 1, 1, 2), (128, 8, 2, 2, 2), (512, 64, 2, 2, 2)]
CHOL_GRIDS = [(256, 32, (2, 2, 1)), (256, 32, (1, 1, 2)), (384, 32, (3, 2, 1)), (512, 64, (2, 2, 2))]


def _scaled(n, kind, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    s = np.logspace(0, 12, n)
    rng.shuffle(s)
    t = np.logspace(0, 12, n)
    rng.shuffle(t)
    if kind == "pow2":                                                   # every maximum an exact power of two
        return np.exp2(rng.integers(-30, 30, (n, n)).astype(float)) * rng.choice([-1.0, 1.0], (n, n))
    return {"rows": A * s[:, None], "cols": A * s[None, :], "both": A * s[:, None] * t[None, :], "plain": A}[kind]


def _spd(n, kind, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    A = G @ G.T / n + np.eye(n)
    if kind == "scaled":
        s = np.logspace(0, 6, n)
        rng.shuffle(s)
        A = A * s[:, None] * s[None, :]
    if kind == "pow2":
        A = A + np.diag(np.exp2(rng.integers(0, 40, n).astype(float)))
    return A


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b))


def _lu_factors(gv):
    C, perm = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "get_factors")
    return C, perm


def _launches(gv):
    n = ctypes.c_int64()
    cb.check(cb.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n), 0), "launch_count")
    return n.value


# ----------------------------------------------------------------------------------------------- exactness
@pytest.mark.parametrize("N,v", [(16, 4), (100, 16), (512, 64), (1024, 128)])
@pytest.mark.parametrize("kind", ["rows", "cols", "both", "plain", "pow2"])
def test_lu_equilibrate_b_bit_identical(N, v, kind):
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    A = _scaled(gv.M, kind, N)
    gv.data[...] = A
    e = cb.lu_equilibrate_b(gv)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequb(A)
    g = xr.geequb(A)
    assert e["info"] == info == g["info"] == 0
    assert _same(e["r"], r) and _same(e["c"], c) and _same(e["r"], g["r"]) and _same(e["c"], g["c"]), kind
    assert (e["rowcnd"], e["colcnd"], e["amax"]) == (rowcnd, colcnd, amax)
    As, equed = sr.laqge(A, r, c, rowcnd, colcnd, amax)
    assert e["equed"] == equed
    assert _same(As, A * (r[:, None] if equed in "RB" else 1.0) * (c[None, :] if equed in "CB" else 1.0))
    cb.LU_rep(gv, upload=False)
    C1, p1 = _lu_factors(gv)
    gv.data[...] = As
    cb.LU_rep(gv)                                                        # the host-scaled matrix through set_local
    C2, p2 = _lu_factors(gv)
    assert _same(C1, C2) and _same(p1, p2), kind
    gv.free_comms()
    comm.close()


def test_lu_equilibrate_b_zero_row_and_column():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(64, 64, 16, 1, 1, 1, comm)
    for zero in ("row", "col"):
        A = _scaled(64, "both", 2)
        if zero == "row":
            A[7] = 0.0
        else:
            A[:, 11] = 0.0
        gv.data[...] = A
        e = cb.lu_equilibrate_b(gv)
        r, c, rowcnd, colcnd, amax, info = lapack.dgeequb(A)
        assert e["info"] == info == (8 if zero == "row" else 64 + 12) and e["equed"] == "N"
        assert _same(e["r"], r) and e["amax"] == amax
        if zero == "col":
            assert _same(e["c"], xr.geequb(A)["c"]) and e["rowcnd"] == rowcnd
    gv.free_comms()
    comm.close()


@pytest.mark.parametrize("N,v", [(16, 4), (100, 16), (512, 64), (1024, 128)])
@pytest.mark.parametrize("kind", ["plain", "scaled", "pow2"])
def test_chol_equilibrate_b_bit_identical(N, v, kind):
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    n = ch.N
    A = _spd(n, kind, N)
    ch.data[...] = chol_solve_ref.scatter(A, n, v, 1, 1, 1, upper=np.nan, pad=np.nan, layers=np.nan)[0]
    e = ch.equilibrate_b()
    p = xr.poequb(A)
    s, scond, amax, info = lapack_dpoequb(A)
    assert e["info"] == p["info"] == info == 0
    assert _same(e["s"], p["s"]) and _same(e["s"], s) and (e["scond"], e["amax"]) == (p["scond"], p["amax"]) == (scond, amax)
    As, equed = sr.laqsy(A, p["s"], p["scond"], p["amax"])
    assert e["equed"] == equed
    assert _same(np.tril(As), np.tril(A * s[:, None] * s[None, :]) if equed == "Y" else np.tril(A))
    ch.parallelCholesky(upload=False)
    L1 = ch.local_factor()
    ch.data[...] = chol_solve_ref.scatter(As, n, v, 1, 1, 1, upper=np.nan, pad=np.nan, layers=np.nan)[0]
    ch.parallelCholesky()
    assert _same(np.tril(L1), np.tril(ch.local_factor()))
    ch.finalize()
    comm.close()


def test_chol_equilibrate_b_non_positive_diagonal():
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(128, 32, (1, 1, 1), comm)
    A = _spd(ch.N, "scaled", 1)
    A[9, 9] = -1.0
    ch.data[...] = chol_solve_ref.scatter(A, ch.N, 32)[0]
    e = ch.equilibrate_b()
    p = xr.poequb(A)
    assert e["info"] == p["info"] == 10 and e["equed"] == "N" and _same(e["s"], p["s"])
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- LU driver
def _scale_rows(d, X):
    return X if d is None else d[:, None] * X


@pytest.mark.parametrize("scaling", ["b", "plain", "none"])
@pytest.mark.parametrize("kind", ["rows", "cols", "both", "plain"])
def test_lu_svxx_pinned_to_its_parts(kind, scaling):
    n, v = 256, 32
    A = _scaled(n, kind, 11)
    B = np.random.default_rng(5).standard_normal((n, 3))
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    gv.data[...] = A
    e = {"b": cb.lu_equilibrate_b, "plain": cb.lu_equilibrate}[scaling](gv) if scaling != "none" else None
    cb.LU_rep(gv, upload=scaling == "none")
    C, perm = _lu_factors(gv)
    equed = e["equed"] if e else "N"
    r = e["r"] if equed in "RB" else None
    c = e["c"] if equed in "CB" else None
    if scaling == "b" and kind in ("rows", "cols", "both"):
        assert equed == {"rows": "R", "cols": "C", "both": "B"}[kind]
    As = (A if r is None else r[:, None] * A) if c is None else (
        (c[None, :] * r[:, None]) * A if r is not None else c[None, :] * A)
    Xs, res_svx = cb.lu_svx(gv, B)
    for t in (False, True):
        pre, post = (c, r) if t else (r, c)
        n0 = _launches(gv)
        X, res = cb.lu_svxx(gv, B, trans=t)
        X2, res2 = cb.lu_svxx(gv, B, trans=t)
        assert _launches(gv) == n0
        assert _same(X, X2) and all(_same(res[k], res2[k]) for k in res)             # the same call, the same bits
        assert res["equed"] == equed and res["info"] in (0,) + tuple(range(n + 1, 2 * n + 1))
        Bs = _scale_rows(pre, B)
        Y0 = cb.lu_solve(gv, Bs, trans=t)
        Y, rx_ = cb.lu_refine_x(gv, Bs, Y0, trans=t)
        assert _same(X, _scale_rows(post, Y)), (kind, scaling, t)
        for k in ("rcond", "berr", "err_norm", "err_comp", "info"):
            assert _same(res[k], rx_[k]), (k, kind, scaling, t)
        assert res["rpvgrw"] == xr.gerpvgrw(As, C)
        assert np.array_equal(cb.lu_solve(gv, B, trans=t), cb.lu_solve(gv, B, trans=t))
        if scaling == "b" and res["info"] == 0:                          # exact unscaling: the bounds carry over
            solve, _ = rr.lu_solvers(C, perm, t)
            Yt, Tt = true_solution(As.T if t else As, Bs, solve)
            nw, cw = errors(Y, Yt, Tt, post)
            en, ec = res["err_norm"], res["err_comp"]
            print(f"svxx {kind} trans={int(t)}: equed={equed} err={nw.max():.2e} bound={en[:, 1].max():.2e} "
                  f"trust={en[:, 0].min():.0f} rpvgrw={res['rpvgrw']:.3e}")
            for j in range(B.shape[1]):
                if en[j, 0] == 1:
                    assert nw[j] <= en[j, 1]
                if ec[j, 0] == 1:
                    assert cw[j] <= ec[j, 1]
        Xc, resc = cb.lu_svxx(gv, B, trans=t, cwise=False)
        assert resc["err_comp"] is None and resc["err_norm"].shape == (3, 3)
    # no side effects: the factors, the permutation, svx and the scaling record
    C2, p2 = _lu_factors(gv)
    assert _same(C, C2) and _same(perm, p2)
    Xs2, res_svx2 = cb.lu_svx(gv, B)
    assert _same(Xs, Xs2) and all(_same(res_svx[k], res_svx2[k]) for k in res_svx)
    assert res_svx["rpvgrw"] == sr.rpvgrw(As, C)                         # svx's growth: unchanged
    gv.free_comms()
    comm.close()


def test_lu_svxx_zero_pivot_leaves_x():
    n, v = 64, 16
    rng = np.random.default_rng(12)
    A = np.triu(rng.integers(1, 9, (n, n)).astype(float)) + np.diag(np.full(n, 50.0))
    A[20, 20] = 0.0
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    gv.data[...] = A
    cb.LU_rep(gv)
    C, _ = _lu_factors(gv)
    B = np.ones((n, 2))
    for t in (0, 1):
        X = np.full((n, 2), 7.0)
        rcond, rpvgrw, info = ctypes.c_double(-1.0), ctypes.c_double(), ctypes.c_int()
        en, be = np.full((2, 3), 5.0), np.full(2, 5.0)
        cb.check(cb.lib().cflx_lu_svxx(gv._h, t, 2, B.ctypes.data, 2, X.ctypes.data, 2, ctypes.byref(rcond),
                                       ctypes.byref(rpvgrw), be.ctypes.data, en.ctypes.data, None, None,
                                       ctypes.byref(info)), "lu_svxx")
        assert info.value == 21 and rcond.value == 0.0 and np.all(X == 7.0) and np.all(en == 5.0) and np.all(be == 5.0)
        assert rpvgrw.value == xr.gerpvgrw(A, C, 21)
    X, res = cb.lu_svxx(gv, B)
    assert X is None and res["info"] == 21
    gv.free_comms()
    comm.close()


def test_lu_svxx_singular_to_working_precision():
    n, v = 128, 32
    rng = np.random.default_rng(13)
    Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
    Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q1 * np.logspace(0, -17, n)) @ Q2.T
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    gv.data[...] = A
    cb.lu_equilibrate_b(gv)
    cb.LU_rep(gv, upload=False)
    for t in (False, True):
        X, res = cb.lu_svxx(gv, rng.standard_normal((n, 2)), trans=t)
        assert res["info"] == n + 1 and np.all(res["err_norm"][:, 0] == 0) and np.all(np.isfinite(X))
    gv.free_comms()
    comm.close()


def test_lu_svxx_arguments_and_state():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(128, 128, 32, 1, 1, 1, comm)
    B = np.random.default_rng(3).standard_normal((gv.M, 2))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_svxx(gv, B)                                                # no factorisation yet
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_equilibrate_b(gv, upload=False)                            # no input yet
    gv.data[...] = _scaled(gv.M, "rows", 1)
    assert cb.lu_equilibrate_b(gv)["equed"] == "R"
    with pytest.raises(cb.ConfluxError, match="already scaled"):
        cb.lu_equilibrate_b(gv, upload=False)
    with pytest.raises(cb.ConfluxError, match="already scaled"):
        cb.lu_equilibrate(gv, upload=False)
    q = cb.lu_equilibrate_b(gv, apply=False, upload=False)               # a query leaves the record
    assert q["equed"] == "N"
    cb.LU_rep(gv, upload=False)
    X = np.zeros_like(B)
    rc, en, info = ctypes.c_double(), np.zeros((2, 3)), ctypes.c_int()
    L = cb.lib()
    args = lambda **kw: dict(dict(h=gv._h, t=0, nrhs=2, B=B.ctypes.data, ldb=2, X=X.ctypes.data, ldx=2,
                                  rc=ctypes.byref(rc), rp=None, be=None, en=en.ctypes.data, ec=None, eq=None,
                                  info=ctypes.byref(info)), **kw)
    for bad in (dict(t=2), dict(nrhs=0), dict(ldb=1), dict(ldx=1), dict(B=None), dict(X=None), dict(rc=None),
                dict(en=None), dict(info=None)):
        assert L.cflx_lu_svxx(*args(**bad).values()) == CFLX_ERR_ARG, bad
    assert L.cflx_lu_svxx(*args().values()) == 0 and info.value == 0
    _, res = cb.lu_svxx(gv, B)
    assert res["equed"] == "R"
    gv.free_comms()
    comm.close()


# ----------------------------------------------------------------------------------------------- Cholesky driver
@pytest.mark.parametrize("scaling", ["b", "plain", "none"])
@pytest.mark.parametrize("kind", ["plain", "scaled"])
def test_chol_svxx_pinned_to_its_parts(kind, scaling):
    N, v = 256, 32
    A = _spd(N, kind, 21)
    B = np.random.default_rng(22).standard_normal((N, 3))
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    ch.data[...] = chol_solve_ref.scatter(A, N, v, upper=np.nan, pad=np.nan, layers=np.nan)[0]
    e = {"b": ch.equilibrate_b, "plain": ch.equilibrate}[scaling]() if scaling != "none" else None
    ch.parallelCholesky(upload=scaling == "none")
    s = e["s"] if e and e["equed"] == "Y" else None
    if kind == "scaled" and scaling != "none":
        assert e["equed"] == "Y"
    Lf = ch.local_factor()
    X, res = ch.svxx(B)
    X2, res2 = ch.svxx(B)
    assert _same(X, X2) and all(_same(res[k], res2[k]) for k in res)
    Bs = _scale_rows(s, B)
    Y, rx_ = ch.refine_x(Bs, ch.solve(Bs))
    assert _same(X, _scale_rows(s, Y))
    for k in ("rcond", "berr", "err_norm", "err_comp", "info"):
        assert _same(res[k], rx_[k]), k
    As = A if s is None else sr.laqsy(A, s, 0.0, 1.0)[0]
    L = np.tril(chol_ref.assemble([Lf], N, v, 1, 1, 1))
    assert res["rpvgrw"] == xr.porpvgrw(np.tril(As), L)
    assert np.array_equal(Lf, ch.local_factor(), equal_nan=True)         # the input's NaN above the diagonal stays
    ch.finalize()
    comm.close()


def test_chol_svxx_state_rules():
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(128, 32, (1, 1, 1), comm)
    B = np.ones((ch.N, 1))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.svxx(B)
    A = _spd(ch.N, "scaled", 1)
    ch.data[...] = chol_solve_ref.scatter(A, ch.N, 32)[0]
    assert ch.equilibrate_b()["equed"] == "Y"
    with pytest.raises(cb.ConfluxError, match="already scaled"):
        ch.equilibrate_b(upload=False)
    ch.parallelCholesky(upload=False)
    assert ch.svxx(B)[1]["equed"] == "Y"
    A[9, 9] = -A[9, 9]                                                   # a failed factorisation stays refused
    ch.data[...] = chol_solve_ref.scatter(A, ch.N, 32)[0]
    with pytest.raises(cb.ConfluxError, match="positive definite"):
        ch.parallelCholesky()
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.svxx(B)
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- dbg.growth_cols
@pytest.mark.parametrize("mode", ["lu", "chol"])
def test_dbg_growth_cols_share(mode):
    v, Kappa, Px, Py, pi, pj, mt, nt = 8, 9, 2, 3, 1, 2, 5, 4
    Ml, Nl = mt * v, nt * v
    M = max(mt * Px, nt * Py) * v
    rng = np.random.default_rng(31)
    A = rng.standard_normal((Ml, Nl)) * np.exp(rng.uniform(-20, 20, (Ml, Nl)))
    F = rng.standard_normal((Ml, Nl)) * np.exp(rng.uniform(-20, 20, (Ml, Nl)))
    for ncols in (M, M // 2 + 3):
        ma, mf = xr.growth_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj, ncols, mode == "chol")
        An, Fn = np.where(ma, A, np.nan), np.where(mf, F, np.nan)        # NaN wherever the kernel must not read
        amax, fmax = cb.dbg.growth_cols(mode, Fn, An, v, Kappa, (Px, Py), (pi, pj), M, ncols)
        ra, rf = xr.growth_cols_share(Fn, An, M, v, Kappa, Px, Py, pi, pj, ncols, mode == "chol")
        assert _same(amax, ra) and _same(fmax, rf), (mode, ncols)
        assert np.count_nonzero(amax) > 0 and np.count_nonzero(fmax) > 0


# ----------------------------------------------------------------------------------------------- multi-GPU
@pytest.mark.parametrize("N,v,Px,Py,Pz", LU_GRIDS)
def test_multi_gpu_lu_svxx(N, v, Px, Py, Pz):
    if n_gpus() < Px * Py * Pz:
        pytest.skip(f"needs {Px * Py * Pz} GPUs")
    d = layout.dims(N, v, Px, Py, Pz)
    A = _scaled(d["M"], "both", N)
    locs = layout.scatter(A, v, Px, Py, Pz)
    B = np.random.default_rng(N).standard_normal((d["M"], 3))

    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        gv.data[...] = locs[gv.rank]
        e = cb.lu_equilibrate_b(gv)
        cb.LU_rep(gv, upload=False)
        out = [e[k] for k in ("r", "c", "rowcnd", "colcnd", "amax", "equed", "info")]
        for t in (False, True):
            X, res = cb.lu_svxx(gv, B, trans=t)
            out += [X] + [res[k] for k in ("rcond", "rpvgrw", "berr", "err_norm", "err_comp", "info")]
        gv.free_comms()
        return out

    rs = run_ranks(Px * Py * Pz, body)
    for r in rs[1:]:
        assert all(_same(a, b) for a, b in zip(r, rs[0]))
    g = xr.geequb(A)
    assert _same(rs[0][0], g["r"]) and _same(rs[0][1], g["c"]) and rs[0][2:5] == [g["rowcnd"], g["colcnd"], g["amax"]]


@pytest.mark.parametrize("N,v,grid", CHOL_GRIDS)
def test_multi_gpu_chol_svxx(N, v, grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    n = chol_ref.dims(N, v, *grid)["N"]
    A = _spd(n, "scaled", N)
    # layers pk != 0 hold zeros: the factorisation sums every layer's share into layer 0's tiles
    locs = chol_solve_ref.scatter(A, N, v, *grid, upper=np.nan, pad=np.nan, layers=0.0)
    B = np.random.default_rng(N).standard_normal((n, 3))

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = locs[ch.rank]
        e = ch.equilibrate_b()
        ch.parallelCholesky(upload=False)
        X, res = ch.svxx(B)
        ch.finalize()
        return [e[k] for k in ("s", "scond", "amax", "equed", "info")] + [X] + [
            res[k] for k in ("rcond", "rpvgrw", "berr", "err_norm", "err_comp", "info")]

    rs = run_ranks(P, body)
    for r in rs[1:]:
        assert all(_same(a, b) for a, b in zip(r, rs[0]))
    p = xr.poequb(A)
    assert _same(rs[0][0], p["s"]) and rs[0][1:3] == [p["scond"], p["amax"]]
