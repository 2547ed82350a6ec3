"""GPU: cflx_lu_equilibrate / cflx_lu_svx and cflx_chol_equilibrate / cflx_chol_svx (LAPACK dgeequ + dlaqge, dgesvx,
dpoequ + dlaqsy, dposvx on the grid).

  * exactness: the device's scales, condition numbers, amax, equed and info equal scipy's dgeequ (LU) and the numpy
    restatement oracle/svx_ref.py (Cholesky) bit for bit; factoring after a device equilibration gives the factors and
    permutation of factoring the host-scaled matrix uploaded with set_local, bit for bit (this pins the apply pass);
  * the drivers against LAPACK on the device's own factors: rpvgrw equals svx_ref.rpvgrw bit for bit; rcond equals
    cflx_lu_rcond (trans 0) bit for bit, or gecon_inf (trans 1) to n u kappa_inf; ferr / berr within the bounds of
    tests/test_gpu_refine.py against svx_ref.gesvx / posvx; ferr at least the true forward error;
  * behaviour: row / column scaled matrices are equilibrated ('R' / 'C') and their rcond grows by more than 1e6; an exactly
    zero pivot gives info = k, rcond = 0 and the leading-k rpvgrw; kappa ~ 1e17 gives info = M + 1 with X; the
    generator matrix is left unscaled and its factors unchanged;
  * dbg.equil: every per-share kernel at several grid positions equals the restatement exactly, with NaN or sentinels in
    every entry a kernel must not read or write;
  * the state rules (a query after scaling leaves the scaling the factors get) and the multi-GPU grids (skipped without
    enough GPUs)."""
import numpy as np
import pytest
from scipy.linalg import lapack

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, layout
from oracle import svx_ref as sr
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
FERR_RATIO = 2.0
BERR_FLOOR = 4 * U
LU_GRIDS = [(64, 8, 2, 2, 1), (128, 16, 1, 1, 2), (128, 8, 2, 2, 2), (512, 64, 2, 2, 2)]
CHOL_GRIDS = [(256, 32, (2, 2, 1)), (256, 32, (1, 1, 2)), (384, 32, (3, 2, 1)), (512, 64, (2, 2, 2))]


def _scaled(n, kind, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    s = np.logspace(0, 12, n)
    rng.shuffle(s)
    t = np.logspace(0, 12, n)
    rng.shuffle(t)
    return {"rows": A * s[:, None], "cols": A * s[None, :], "both": A * s[:, None] * t[None, :], "plain": A}[kind]


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b))


def _lu_factors(gv):
    C, perm = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "get_factors")
    return C, perm


# ----------------------------------------------------------------------------------------------- LU exactness
@pytest.mark.parametrize("N,v", [(16, 4), (100, 16), (512, 64), (1024, 128)])
@pytest.mark.parametrize("kind", ["rows", "cols", "both", "plain"])
def test_lu_equilibrate_bit_identical(N, v, kind):
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    A = _scaled(gv.M, kind, N)
    gv.data[...] = A
    e = cb.lu_equilibrate(gv)
    r, c, rowcnd, colcnd, amax, info = lapack.dgeequ(A)
    assert e["info"] == info == 0
    assert _same(e["r"], r) and _same(e["c"], c), kind
    assert (e["rowcnd"], e["colcnd"], e["amax"]) == (rowcnd, colcnd, amax)
    As, equed = sr.laqge(A, r, c, rowcnd, colcnd, amax)
    assert e["equed"] == equed
    cb.LU_rep(gv, upload=False)
    C1, p1 = _lu_factors(gv)
    gv.data[...] = As
    cb.LU_rep(gv)                                                        # the host-scaled matrix through set_local
    C2, p2 = _lu_factors(gv)
    assert _same(C1, C2) and _same(p1, p2), kind
    gv.free_comms()
    comm.close()


def test_lu_equilibrate_zero_row_and_column():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(64, 64, 16, 1, 1, 1, comm)
    for zero in ("row", "col"):
        A = _scaled(64, "plain", 2)
        if zero == "row":
            A[7] = 0.0
        else:
            A[:, 11] = 0.0
        gv.data[...] = A
        e = cb.lu_equilibrate(gv)
        g = sr.geequ(A)
        assert e["info"] == g["info"] == (8 if zero == "row" else 64 + 12) and e["equed"] == "N"
        assert _same(e["r"], g["r"]) and e["amax"] == g["amax"]
        cb.LU_rep(gv, upload=False)                                      # nothing was scaled
        C1, p1 = _lu_factors(gv)
        cb.LU_rep(gv)
        assert all(_same(a, b) for a, b in zip((C1, p1), _lu_factors(gv)))
    gv.free_comms()
    comm.close()


# ----------------------------------------------------------------------------------------------- LU drivers
def _lu_svx_case(A, v, B, trans_list=(False, True), equilibrate=True):
    n = A.shape[0]
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    gv.data[...] = A
    cb.LU_rep(gv)
    rc_plain = cb.lu_rcond(gv)[0]
    e = cb.lu_equilibrate(gv, apply=equilibrate)
    cb.LU_rep(gv, upload=False)
    C, perm = _lu_factors(gv)
    out = dict(e=e, rc_plain=rc_plain, C=C, perm=perm, rcond=cb.lu_rcond(gv))
    for t in trans_list:
        X, res = cb.lu_svx(gv, B, trans=t)
        X2, res2 = cb.lu_svx(gv, B, trans=t)
        assert _same(X, X2) and all(_same(res[k], res2[k]) for k in res)  # the same call, the same bits
        out[t] = (X, res)
    gv.free_comms()
    comm.close()
    return out


def _true_solution(A, B, trans):
    Ao = (A.T if trans else A)
    Xt = np.linalg.solve(Ao, B)
    AoL = Ao.astype(np.longdouble)
    for _ in range(3):
        Xt = Xt + np.linalg.solve(Ao, np.asarray(B - AoL @ Xt.astype(np.longdouble), dtype=np.float64))
    return Xt


def _true_scaled(As, B, t, e, equed):
    """the exact solution of the scaled system the factors solve, unscaled: c (As^-1 (r B)) for trans 0, r (As^-T (c B))
    for trans 1 (r B and c B rounded as the device rounds them)"""
    rowequ, colequ = equed in "RB", equed in "CB"
    if not t:
        Y = _true_solution(As, e["r"][:, None] * B if rowequ else B, False)
        return e["c"][:, None] * Y if colequ else Y
    Y = _true_solution(As, e["c"][:, None] * B if colequ else B, True)
    return e["r"][:, None] * Y if rowequ else Y


@pytest.mark.parametrize("kind", ["rows", "cols", "both", "plain"])
def test_lu_svx_against_lapack(kind):
    n, v = 256, 32
    A = _scaled(n, kind, 11)
    B = np.random.default_rng(5).standard_normal((n, 3))
    o = _lu_svx_case(A, v, B)
    e = o["e"]
    As, equed = sr.laqge(A, e["r"], e["c"], e["rowcnd"], e["colcnd"], e["amax"])
    assert e["equed"] == equed
    LU = o["C"]
    for t in (False, True):
        X, res = o[t]
        ref = sr.gesvx(As, LU, o["perm"], B, t, e["r"], e["c"], equed, e["rowcnd"], e["colcnd"])
        assert res["equed"] == equed and res["info"] == ref["info"] == 0
        assert res["rpvgrw"] == ref["rpvgrw"] == sr.rpvgrw(As, LU)
        if not t:
            assert res["rcond"] == o["rcond"][0]                            # the bits of cflx_lu_rcond
        kinf = np.abs(As).sum(1).max() * np.abs(np.linalg.inv(As)).sum(1).max()
        margin = abs(res["rcond"] - ref["rcond"]) / (ref["rcond"] * n * U * kinf)
        fwd = np.max(np.abs(X - _true_scaled(As, B, t, e, equed)), 0) / np.max(np.abs(X), 0)
        print(f"svx {kind} trans={int(t)}: equed={equed} rcond={res['rcond']:.3e} plain={o['rc_plain']:.3e} "
              f"margin={margin:.2e} ferr={res['ferr'].max():.2e} ref={ref['ferr'].max():.2e} fwd={fwd.max():.2e} "
              f"berr={res['berr'].max():.2e} ref={ref['berr'].max():.2e}")
        assert margin <= 1.0
        assert np.all(np.maximum(res["ferr"] / ref["ferr"], ref["ferr"] / res["ferr"]) <= FERR_RATIO)
        assert np.all(res["berr"] <= np.maximum(2 * ref["berr"], BERR_FLOOR))
        assert np.all(res["ferr"] >= fwd)
    if kind in ("rows", "cols"):
        assert equed == {"rows": "R", "cols": "C"}[kind]
        assert o[False][1]["rcond"] >= 1e6 * o["rc_plain"]


def test_lu_svx_zero_pivot():
    n, v = 64, 16
    rng = np.random.default_rng(12)
    A = np.triu(rng.integers(1, 9, (n, n)).astype(float)) + np.diag(np.full(n, 50.0))
    A[20, 20] = 0.0                                                      # row 20 and column 20 stay non-zero
    B = np.ones((n, 2))
    o = _lu_svx_case(A, v, B, trans_list=(False, True), equilibrate=False)
    assert _same(np.triu(o["C"]), A) and _same(o["perm"], np.arange(n))  # partial pivoting keeps every row: U = A
    for t in (False, True):
        X, res = o[t]
        assert X is None and res["info"] == 21 and res["rcond"] == 0.0
        assert res["rpvgrw"] == sr.rpvgrw(A, o["C"], 21)


def test_lu_svx_singular_to_working_precision():
    n, v = 128, 32
    rng = np.random.default_rng(13)
    Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
    Q2, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q1 * np.logspace(0, -17, n)) @ Q2.T
    o = _lu_svx_case(A, v, rng.standard_normal((n, 1)), trans_list=(False,))
    X, res = o[False]
    assert res["info"] == n + 1 and X is not None and np.all(np.isfinite(X)) and res["rcond"] < U


def test_lu_svx_generator_matrix_is_left_alone():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(16384, 16384, 256, 1, 1, 1, comm)                    # C2
    cb.LU_rep(gv)
    C0, p0 = _lu_factors(gv)
    e = cb.lu_equilibrate(gv)
    assert e["equed"] == "N" and e["info"] == 0
    cb.LU_rep(gv, upload=False)
    C1, p1 = _lu_factors(gv)
    assert _same(C0, C1) and _same(p0, p1)
    B = np.random.default_rng(1).standard_normal((gv.M, 2))
    X, res = cb.lu_svx(gv, B)
    assert res["equed"] == "N" and res["info"] == 0 and res["rcond"] == cb.lu_rcond(gv)[0]
    assert np.all(res["berr"] <= 1e-14)
    gv.free_comms()
    comm.close()


def test_lu_svx_state_rules():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(256, 256, 32, 1, 1, 1, comm)
    B = np.random.default_rng(3).standard_normal((gv.M, 2))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_svx(gv, B)                                                 # no factorisation yet
    gv.data[...] = _scaled(gv.M, "rows", 1)
    cb.LU_rep(gv)
    cb.lu_svx(gv, B)
    e = cb.lu_equilibrate(gv, upload=False)
    assert e["equed"] == "R"
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_svx(gv, B)                                                 # equilibrate dropped the factorisation
    with pytest.raises(cb.ConfluxError, match="already scaled"):
        cb.lu_equilibrate(gv, upload=False)
    # streamed next input: it carries no scaling, and svx of the run that handed A0 on is refused
    mats = [cb.pinned_empty((gv.Ml, gv.Nl)) for _ in range(2)]
    mats[0][...] = _scaled(gv.M, "rows", 2)
    mats[1][...] = _scaled(gv.M, "cols", 3)
    gv.data = mats[0]
    e = cb.lu_equilibrate(gv)
    assert e["equed"] == "R"
    cb.LU_rep(gv, upload=False, next_data=mats[1])
    with pytest.raises(cb.ConfluxError, match="queued next matrix"):
        cb.lu_svx(gv, B)
    cb.LU_rep(gv, upload=False)                                          # the streamed matrix's own run
    X, res = cb.lu_svx(gv, B)
    assert res["equed"] == "N" and res["info"] == 0
    for m in mats:
        cb.pinned_free(m)
    gv.free_comms()
    comm.close()


@pytest.mark.parametrize("N,v,Px,Py,Pz", LU_GRIDS)
def test_multi_gpu_lu_svx(N, v, Px, Py, Pz):
    if n_gpus() < Px * Py * Pz:
        pytest.skip(f"needs {Px * Py * Pz} GPUs")
    d = layout.dims(N, v, Px, Py, Pz)
    A = _scaled(d["M"], "both", N)
    locs = layout.scatter(A, v, Px, Py, Pz)
    B = np.random.default_rng(N).standard_normal((d["M"], 3))

    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        gv.data[...] = locs[gv.rank]
        e = cb.lu_equilibrate(gv)
        cb.LU_rep(gv, upload=False)
        out = [e[k] for k in ("r", "c", "rowcnd", "colcnd", "amax", "equed", "info")]
        for t in (False, True):
            X, res = cb.lu_svx(gv, B, trans=t)
            out += [X] + [res[k] for k in ("rcond", "ferr", "berr", "rpvgrw", "info")]
        gv.free_comms()
        return out

    rs = run_ranks(Px * Py * Pz, body)
    for r in rs[1:]:
        assert all(_same(a, b) for a, b in zip(r, rs[0]))
    g = sr.geequ(A)
    assert _same(rs[0][0], g["r"]) and _same(rs[0][1], g["c"]) and rs[0][2:5] == [g["rowcnd"], g["colcnd"], g["amax"]]


# ----------------------------------------------------------------------------------------------- Cholesky
def _spd(n, kind, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    A = G @ G.T / n + np.eye(n)
    if kind == "scaled":
        s = np.logspace(0, 6, n)
        rng.shuffle(s)
        A = A * s[:, None] * s[None, :]
    return A


@pytest.mark.parametrize("N,v", [(16, 4), (100, 16), (512, 64), (1024, 128)])
@pytest.mark.parametrize("kind", ["plain", "scaled"])
def test_chol_equilibrate_bit_identical_and_svx(N, v, kind):
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    n = ch.N
    A = _spd(n, kind, N)
    ch.data[...] = chol_solve_ref.scatter(A, n, v, 1, 1, 1, upper=np.nan, pad=np.nan, layers=np.nan)[0]
    e = ch.equilibrate()
    p = sr.poequ(A)
    As, equed = sr.laqsy(A, p["s"], p["scond"], p["amax"])
    assert e["info"] == 0 and e["equed"] == equed == ("Y" if kind == "scaled" else "N")
    assert _same(e["s"], p["s"]) and (e["scond"], e["amax"]) == (p["scond"], p["amax"])
    ch.parallelCholesky(upload=False)
    L1 = ch.local_factor()
    B = np.random.default_rng(N).standard_normal((n, 3))
    X, res = ch.svx(B)
    X2, res2 = ch.svx(B)
    assert _same(X, X2) and all(_same(res[k], res2[k]) for k in res)
    assert res["rcond"] == ch.rcond()[0] and res["equed"] == equed and res["info"] == 0
    ch.data[...] = chol_solve_ref.scatter(As, n, v, 1, 1, 1, upper=np.nan, pad=np.nan, layers=np.nan)[0]
    ch.parallelCholesky()
    assert _same(np.tril(L1), np.tril(ch.local_factor()))                # the apply pass: bit for bit
    L = np.tril(chol_ref.assemble([L1], n, v, 1, 1, 1))
    ref = sr.posvx(chol_ref.lower_sym(As), L, B, p["s"], equed, p["scond"])
    Y = _true_solution(chol_ref.lower_sym(As), p["s"][:, None] * B if equed == "Y" else B, False)
    fwd = np.max(np.abs(X - (p["s"][:, None] * Y if equed == "Y" else Y)), 0) / np.max(np.abs(X), 0)
    print(f"chol svx {N}/{v} {kind}: rcond={res['rcond']:.3e} ferr={res['ferr'].max():.2e} ref={ref['ferr'].max():.2e} "
          f"fwd={fwd.max():.2e} berr={res['berr'].max():.2e} ref={ref['berr'].max():.2e}")
    assert np.all(np.maximum(res["ferr"] / ref["ferr"], ref["ferr"] / res["ferr"]) <= FERR_RATIO)
    assert np.all(res["berr"] <= np.maximum(2 * ref["berr"], BERR_FLOOR))
    assert np.all(res["ferr"] >= fwd)
    ch.finalize()
    comm.close()


def test_chol_equilibrate_non_positive_diagonal_and_state_rules():
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(128, 32, (1, 1, 1), comm)
    B = np.ones((ch.N, 1))
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.svx(B)
    A = _spd(ch.N, "scaled", 1)
    a99 = A[9, 9]
    A[9, 9] = -1.0
    ch.data[...] = chol_solve_ref.scatter(A, ch.N, 32)[0]
    e = ch.equilibrate()
    assert e["info"] == 10 and e["equed"] == "N"
    A[9, 9] = a99
    ch.data[...] = chol_solve_ref.scatter(A, ch.N, 32)[0]
    ch.parallelCholesky()
    ch.svx(B)
    assert ch.equilibrate(upload=False)["equed"] == "Y"
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.svx(B)                                                        # equilibrate dropped the factorisation
    ch.parallelCholesky(upload=False)
    assert ch.svx(B)[1]["equed"] == "Y"
    ch.parallelCholesky()                                                # a new upload carries no scaling
    assert ch.svx(B)[1]["equed"] == "N"
    ch.finalize()
    comm.close()


@pytest.mark.parametrize("N,v,grid", CHOL_GRIDS)
def test_multi_gpu_chol_svx(N, v, grid):
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
        e = ch.equilibrate()
        ch.parallelCholesky(upload=False)
        X, res = ch.svx(B)
        ch.finalize()
        return [e[k] for k in ("s", "scond", "amax", "equed", "info")] + [X] + [res[k] for k in ("rcond", "ferr", "berr")]

    rs = run_ranks(P, body)
    for r in rs[1:]:
        assert all(_same(a, b) for a, b in zip(r, rs[0]))
    p = sr.poequ(A)
    assert _same(rs[0][0], p["s"]) and rs[0][1:3] == [p["scond"], p["amax"]]


# ----------------------------------------------------------------------------------------------- a query after scaling
def test_lu_query_after_scaling_keeps_the_record():
    n, v = 256, 32
    A = _scaled(n, "both", 21)
    B = np.random.default_rng(22).standard_normal((n, 3))
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    gv.data[...] = A
    e1 = cb.lu_equilibrate(gv)                                           # scales A0: equed 'B'
    cb.LU_rep(gv, upload=False)
    straight = {t: cb.lu_svx(gv, B, trans=t) for t in (False, True)}
    e1b = cb.lu_equilibrate(gv)
    assert e1b["equed"] == "B" and all(_same(e1[k], e1b[k]) for k in e1)
    q = cb.lu_equilibrate(gv, apply=False, upload=False)                 # a query of the scaled matrix
    As, equed = sr.laqge(A, e1["r"], e1["c"], e1["rowcnd"], e1["colcnd"], e1["amax"])
    g = sr.geequ(As)
    assert q["equed"] == "N" and _same(q["r"], g["r"]) and _same(q["c"], g["c"]) and not _same(q["r"], e1["r"])
    cb.LU_rep(gv, upload=False)
    C, perm = _lu_factors(gv)
    for t in (False, True):
        X, res = cb.lu_svx(gv, B, trans=t)
        X0, res0 = straight[t]
        assert res["equed"] == "B" and _same(X, X0) and all(_same(res[k], res0[k]) for k in res)
        ref = sr.gesvx(As, C, perm, B, t, e1["r"], e1["c"], equed, e1["rowcnd"], e1["colcnd"])
        assert np.all(np.max(np.abs(X - ref["X"]), 0) <= 2 * (res["ferr"] + ref["ferr"]) * np.max(np.abs(X), 0))
    gv.free_comms()
    comm.close()


def test_chol_query_after_scaling_keeps_the_record():
    N, v = 256, 32
    A = _spd(N, "scaled", 23)
    B = np.random.default_rng(24).standard_normal((N, 2))
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    ch.data[...] = chol_solve_ref.scatter(A, N, v)[0]
    e1 = ch.equilibrate()
    assert e1["equed"] == "Y"
    ch.parallelCholesky(upload=False)
    X0, res0 = ch.svx(B)
    ch.equilibrate()
    q = ch.equilibrate(apply=False, upload=False)
    p = sr.poequ(A)
    As, _ = sr.laqsy(A, p["s"], p["scond"], p["amax"])
    assert q["equed"] == "N" and _same(q["s"], sr.poequ(chol_ref.lower_sym(As))["s"]) and not _same(q["s"], e1["s"])
    ch.parallelCholesky(upload=False)
    X, res = ch.svx(B)
    assert res["equed"] == "Y" and _same(X, X0) and all(_same(res[k], res0[k]) for k in res)
    L = np.tril(chol_ref.assemble([ch.local_factor()], N, v, 1, 1, 1))
    ref = sr.posvx(chol_ref.lower_sym(As), L, B, p["s"], "Y", p["scond"])
    assert np.all(np.max(np.abs(X - ref["X"]), 0) <= 2 * (res["ferr"] + ref["ferr"]) * np.max(np.abs(X), 0))
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- dbg.equil
SHARES = [(4, 9, 2, 3, 1, 2, 5, 3), (16, 5, 2, 2, 0, 1, 3, 3), (16, 3, 1, 1, 0, 0, 4, 4), (8, 7, 3, 2, 2, 1, 3, 4),
          (32, 4, 2, 2, 1, 1, 2, 2)]


@pytest.mark.parametrize("v,Kappa,Px,Py,pi,pj,mt,nt", SHARES)
def test_dbg_equil_share_kernels(v, Kappa, Px, Py, pi, pj, mt, nt):
    Ml, Nl = mt * v, nt * v
    M = max(mt * Px, nt * Py) * v
    rng = np.random.default_rng(v * 1000 + pi * 10 + pj)
    A = rng.standard_normal((Ml, Nl)) * np.exp(rng.uniform(-20, 20, (Ml, Nl)))
    r, c = np.exp(rng.uniform(-30, 30, M)), np.exp(rng.uniform(-30, 30, M))
    gr = sr._gidx(np.arange(Ml), Px, pi, v)[:, None]
    gc = sr._gidx(np.arange(Nl), Py, pj, v)[None, :]
    # the LU passes read every local entry: maxima and the scaling against the restatement, bit for bit
    o = cb.dbg.equil(A, v, Kappa, (Px, Py), (pi, pj), M, r, c, "N")
    assert _same(o["rowmax"], sr.row_max_share(A, M, v, Px, pi))
    assert _same(o["colmax"], sr.col_max_share(A, M, v, Px, Py, pi, pj, r))
    for equed in "NRCB":
        o = cb.dbg.equil(A, v, Kappa, (Px, Py), (pi, pj), M, r, c, equed)
        assert _same(o["scaled"], sr.apply_share(A, v, Px, Py, pi, pj, r, c, equed)), equed
    # the diagonal: NaN everywhere but the real diagonal tiles' diagonals
    real = (gr // v < Kappa) & (gc // v < Kappa)
    D = np.where(real & (gr == gc), A, np.nan)
    assert _same(cb.dbg.equil(D, v, Kappa, (Px, Py), (pi, pj), M, r, c)["diag"],
                 sr.diag_share(D, M, v, Kappa, Px, Py, pi, pj))
    # the symmetric apply pass: a sentinel (3.0) in every entry it must not write, which any scaling would change
    low = real & (gr >= gc)
    S = np.where(low, A, 3.0)
    s_ = np.exp(rng.uniform(-5, 5, M))
    got = cb.dbg.equil(S, v, Kappa, (Px, Py), (pi, pj), M, s_, c)["sym_scaled"]
    assert _same(got, sr.sym_apply_share(S, v, Kappa, Px, Py, pi, pj, s_)) and np.all(got[~low] == 3.0)
    # the pivot growth: 1e300 in the columns >= ncols (read, it would win every maximum), the lower triangle larger than
    # the upper (read as U, it would win max |triu|), and exact zeros on some diagonal entries the share holds
    ncols = M // 2 + v // 2
    G = np.abs(A) + 1.0
    G = np.where(gr > gc, G * 1e6, G)
    G = np.where(gc >= ncols, 1e300, G)
    diag_rows = [l for l in range(Ml) if (sr._gidx(l, Px, pi, v) // v) % Py == pj]
    for l in diag_rows[3::7]:
        g = int(sr._gidx(l, Px, pi, v))
        cols = np.nonzero(gc[0] == g)[0]
        if len(cols):
            G[l, cols[0]] = 0.0
    o = cb.dbg.equil(G, v, Kappa, (Px, Py), (pi, pj), M, r, c, "N", ncols)
    assert tuple(o["growth"]) == sr.growth_share(G, G, v, Px, Py, pi, pj, ncols)
    assert o["growth"][1] < 1e300
    assert o["zero_pivot"] == sr.zero_pivot_share(G, M, v, Px, Py, pi, pj)
    assert cb.dbg.equil(np.abs(A) + 1.0, v, Kappa, (Px, Py), (pi, pj), M)["zero_pivot"] == 0
