"""GPU: the signed Cholesky A = R S R^T (cflx_chol_factor_ldlt), the symmetric butterflies (cflx_chol_rbt and its
solves) and every call on a signed factor, against oracle/ldlt_ref.py, numpy and the plain Cholesky's bits.  The grid
cases run on real GPUs when present, and on one device through a child pytest under the NCCL loopback."""
import ctypes
import os
import subprocess
import sys
import xml.etree.ElementTree as ET

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import chol_ref, hp_ref, ldlt_ref, rbt_ref
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BERR_TOL = 1e-13


def scatter(A, v, Px, Py, Pz):
    """the conflux shares (Ml x Nl) of the global N x N matrix A; layers pk != 0 zero"""
    N = A.shape[0]
    d = chol_ref.dims(N, v, Px, Py, Pz)
    out = [np.zeros((d["Ml"], d["Nl"])) for _ in range(d["P"])]
    for r, loc in enumerate(out):
        if r % Pz:
            continue
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        for lti in range(d["Ml"] // v):
            for ltj in range(d["Nl"] // v):
                gi, gj = lti * Px + pi, ltj * Py + pj
                if gi < d["Kappa"] and gj < d["Kappa"]:
                    loc[lti * v:(lti + 1) * v, ltj * v:(ltj + 1) * v] = A[gi * v:(gi + 1) * v, gj * v:(gj + 1) * v]
    return out


def _one(N, v, A, body):
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky(N, v, (1, 1, 1), comm)
    try:
        if A is not None:
            ch.data[...] = A
        return body(ch)
    finally:
        ch.finalize()
        comm.close()


def _berr(A, X, B):
    S = ldlt_ref.mirror(A)
    X2, B2 = X.reshape(len(B), -1), B.reshape(len(B), -1)
    return np.max(np.abs(S @ X2 - B2) / (np.abs(S) @ np.abs(X2) + np.abs(B2)))


def _kkt_padded(N, n, seed, c_zero=False):
    return ldlt_ref.kkt(n, N - n, seed=seed, c_zero=c_zero)


# --------------------------------------------------------------------------------------------------- 1. tile kernels
@pytest.mark.parametrize("v,variant", [(64, 0), (128, 0), (256, 0), (512, 0), (128, 1), (256, 2), (512, 2)])
def test_tile_kernel_matches_the_restatement(v, variant):
    A = ldlt_ref.kkt(v // 2 + 3, v // 2 - 3, seed=v + variant)
    r = cb.dbg.ldlt_tile(A, variant=variant)
    f = ldlt_ref.factor(A)
    assert np.array_equal(r["s"], f["s"])
    assert r["inertia"] == f["inertia"] == (v // 2 + 3, v // 2 - 3, 0)
    assert r["nrepl"] == 0 and r["info"] == 0
    R = np.tril(r["R"])
    assert np.array_equal(r["R"], R)
    assert np.array_equal(r["SRT"], r["s"][:, None] * R.T)
    assert ldlt_ref.componentwise_ok(A, R, r["s"])


@pytest.mark.parametrize("v,variant", [(64, 0), (128, 0), (256, 0), (512, 0), (128, 1), (256, 2), (512, 2)])
def test_tile_kernel_on_spd_is_the_cholesky(v, variant):
    A = hp_ref.random_spd(v, 1e4, np.random.default_rng(v))
    r = cb.dbg.ldlt_tile(A, variant=variant)
    L, LT, info = cb.dbg.potrf_tile(A, variant=variant)
    assert info == 0 and r["info"] == 0 and np.all(r["s"] == 1.0) and r["inertia"] == (v, 0, 0)
    assert np.array_equal(r["R"], L) and np.array_equal(r["SRT"], LT)


@pytest.mark.parametrize("variant,v", [(0, 64), (1, 128), (2, 256)])
def test_tile_kernel_zero_pivot_and_tiny(variant, v):
    A = ldlt_ref.kkt(v - 8, 8, seed=1)
    A[0, 0] = 0.0
    r = cb.dbg.ldlt_tile(A, variant=variant)
    assert r["info"] == 1 and r["inertia"][2] >= 1
    t = cb.dbg.ldlt_tile(A, tiny=1e-6, variant=variant)
    f = ldlt_ref.factor(A, tiny=1e-6)
    assert t["info"] == 0 and t["nrepl"] == f["nrepl"] >= 1
    assert np.array_equal(t["s"], f["s"])


# ------------------------------------------------------------------------------------------- 2. same bits on SPD
@pytest.mark.parametrize("ozaki", [False, True])
@pytest.mark.parametrize("kind,N,v", [("generator", 1024, 128), ("generator", 2048, 256), ("spd", 1536, 256),
                                      ("spd", 1024, 512)])
def test_spd_gives_the_cholesky_bits(kind, N, v, ozaki, monkeypatch):
    if ozaki:
        monkeypatch.setenv("CFLX_GEMM", "ozaki")                     # read when the object is created
    A = None if kind == "generator" else np.tril(hp_ref.random_spd(N, 1e5, np.random.default_rng(N)))

    def body(ch):
        ch.parallelCholesky()
        L = ch.local_factor()
        nrepl, inertia, info, _ = ch.factor_ldlt()
        assert (nrepl, inertia, info) == (0, (N, 0, 0), 0)
        assert np.array_equal(ch.local_factor(), L)
        assert np.all(ch.signs() == 1.0)
    _one(N, v, A, body)


# ---------------------------------------------------------------------------------- 3. indefinite without transform
@pytest.mark.parametrize("N,v,n,c_zero", [(1024, 128, 640, False), (1024, 256, 768, True), (768, 64, 300, False)])
def test_kkt_factors_without_pivoting(N, v, n, c_zero):
    K = _kkt_padded(N, n, seed=N + n, c_zero=c_zero)

    def body(ch):
        nrepl, inertia, info, _ = ch.factor_ldlt()
        assert (nrepl, inertia, info) == (0, (n, N - n, 0), 0)
        R, s = np.tril(ch.local_factor()), ch.signs()
        assert np.array_equal(s, ldlt_ref.factor(K)["s"])
        assert ldlt_ref.normwise_ok(K, R, s, hp_ref.diag_block_kappa(R, 128))
        a, rel = ch.validate()
        assert rel <= 1e-13, rel
        B = np.random.default_rng(1).standard_normal((N, 3))
        X = ch.solve(B)
        X2, _, be = ch.refine(B, X)
        assert be.max() <= BERR_TOL and _berr(K, X2, B) <= BERR_TOL
    _one(N, v, np.tril(K), body)


# ------------------------------------------------------------------------------------- 4. zero pivot and transform
def test_zero_pivot_then_transform():
    N, v = 1024, 128
    A = ldlt_ref.with_inertia(N, 600, 424, seed=5)
    A[0, 0] = 0.0
    want = ldlt_ref.inertia(A)

    def body(ch):
        nrepl, inertia, info, _ = ch.factor_ldlt()
        assert info == 1
        nrepl, inertia, info, _ = ch.factor_ldlt(tiny=1e-10)
        assert nrepl >= 1 and info == 0
        ch.rbt(depth=2, seed=3)
        nrepl, inertia, info, _ = ch.factor_ldlt(upload=False)
        assert (nrepl, info) == (0, 0) and inertia == want
        B = np.random.default_rng(2).standard_normal((N, 2))
        X, fe, be = ch.rbt_solve(B)
        assert _berr(A, X, B) <= BERR_TOL
    _one(N, v, np.tril(A), body)


@pytest.mark.parametrize("npos,seed", [(1024, 1), (0, 2), (333, 3), (900, 4)])
def test_inertia_matches_eigvalsh(npos, seed):
    N, v = 1024, 256
    A = ldlt_ref.with_inertia(N, npos, N - npos, seed=seed)

    def body(ch):
        ch.rbt(depth=2, seed=seed)
        nrepl, inertia, info, _ = ch.factor_ldlt(upload=False)
        assert info == 0 and inertia == ldlt_ref.inertia(A) == (npos, N - npos, 0)
    _one(N, v, np.tril(A), body)


# -------------------------------------------------------------------------------------------- 5. mirror, transform
@pytest.mark.parametrize("depth", [1, 2, 3])
def test_transform_bits(depth):
    N, v = 1024, 128
    A = ldlt_ref.with_inertia(N, 500, 524, seed=depth)
    stored = np.tril(A) + np.triu(np.full((N, N), np.nan), 1)

    def body(ch):
        u = ch.rbt(depth=depth, seed=11)
        assert np.array_equal(u, rbt_ref.multipliers(N, depth, 11)[0])
        W = ch.local_input()
        want = rbt_ref.global_w(ldlt_ref.mirror(stored), u, u)
        assert np.array_equal(np.tril(W), np.tril(want))
        assert np.array_equal(W, want)                      # the whole share: the mirror fills every NaN
    _one(N, v, stored, body)


def test_transform_bits_more_tiles_than_a_grid_dimension():
    """v = 8, N = 3072: 73536 tile pairs above the diagonal, more than a grid's 65535 y extent; the mirror and the
    transform still give the restatement's bits, and the refined solve is backward stable on A"""
    N, v = 3072, 8
    A = ldlt_ref.with_inertia(N, 1500, 1572, seed=8, lo=1.0, hi=3.0)
    stored = np.tril(A) + np.triu(np.full((N, N), np.nan), 1)
    B = np.random.default_rng(5).standard_normal((N, 1))

    def body(ch):
        u = ch.rbt(depth=2, seed=4)
        want = rbt_ref.global_w(ldlt_ref.mirror(stored), u, u)
        assert np.array_equal(ch.local_input(), want)
        nrepl, inertia, info, _ = ch.factor_ldlt(upload=False)
        assert info == 0 and inertia == (1500, 1572, 0)
        X, fe, be = ch.rbt_solve(B)
        assert _berr(A, X, B) <= BERR_TOL
    _one(N, v, stored, body)


@pytest.mark.parametrize("M", [140000, 139000])
def test_sign_pass_on_a_share_wider_than_a_grid_dimension(M):
    """the solves' sign pass on a share of 70000 local columns (grid column 1 of 2, v = 8): every column of a real
    tile is scaled by its global column's sign, the columns at or beyond M are left alone"""
    v, Nl, ldn = 8, 70000, 8
    rng = np.random.default_rng(M)
    Z = rng.standard_normal((Nl, ldn))
    sgn = np.where(rng.random(M) < 0.5, -1.0, 1.0)
    got = cb.dbg.solve_signs(Z, sgn, v, grid=(1, 2), pos=(0, 1), M=M)
    cols = rbt_ref.global_index(Nl, v, 2, 1)
    want = Z.copy()
    real = cols < M
    want[real] *= sgn[cols[real]][:, None]
    assert np.array_equal(got, want)
    assert (not real.all()) == (M < 140000)


# ------------------------------------------------------------------------------------- 6. every call, signed factor
def test_every_call_on_a_signed_factor():
    """a quasi-definite KKT matrix, factored without a transform: the represented matrix is the input's lower triangle"""
    N, v = 1024, 128
    K = ldlt_ref.kkt(640, 384, seed=9)
    rng = np.random.default_rng(4)
    B = rng.standard_normal((N, 5))

    def body(ch):
        assert ch.factor_ldlt()[:3] == (0, (640, 384, 0), 0)
        W = np.tril(ch.local_input())
        assert np.array_equal(W, np.tril(K))
        S = ldlt_ref.mirror(W)
        X = ch.solve(B)
        assert _berr(W, X, B) <= 1e-14
        ncl = cb.rhs_local_cols(5, v, 1)
        Bs = np.zeros((N, ncl))
        Bs[:, :5] = B
        Xl = ch.solve_local(Bs, 5)
        assert np.array_equal(Xl[:, :5], X)
        rc, anorm = ch.rcond()
        true = 1.0 / (np.linalg.norm(S, 1) * np.linalg.norm(np.linalg.inv(S), 1))
        assert anorm == pytest.approx(np.linalg.norm(S, 1), rel=1e-14)
        assert true * (1 - 1e-10) <= rc <= 10 * true
        X2, fe, be = ch.refine(B, X)
        assert be.max() <= BERR_TOL
        X3, d = ch.refine_x(B, X)
        assert d["berr"].max() <= BERR_TOL
        X4, d = ch.svx(B)
        assert d["berr"].max() <= BERR_TOL and d["info"] == 0
        X5, d = ch.svxx(B)
        assert d["berr"].max() <= BERR_TOL
        Ainv = ch.inverse()
        Iv = ldlt_ref.mirror(Ainv)
        assert np.abs(S @ Iv - np.eye(N)).max() <= 1e-10
        det = ch.det()
        sign, logabs = np.linalg.slogdet(S)
        assert np.sign(det["mantissa"]) == sign
        assert det["logdet"] == pytest.approx(logabs, rel=1e-12)
        a, rel = ch.validate()
        assert rel <= 1e-13
    _one(N, v, np.tril(K), body)


def test_transformed_solves():
    """rbt_apply_local(0) -> solve_local -> rbt_apply_local(1) is rbt_solve(refine = 0); the refined rbt_solve is
    backward stable on A itself"""
    N, v = 1024, 128
    A = ldlt_ref.with_inertia(N, 700, 324, seed=9, lo=1.5, hi=4.0)
    B = np.random.default_rng(4).standard_normal((N, 5))

    def body(ch):
        ch.rbt(depth=2, seed=21)
        assert ch.factor_ldlt(upload=False)[2] == 0
        ncl = cb.rhs_local_cols(5, v, 1)
        Bs = np.zeros((N, ncl))
        Bs[:, :5] = B
        Y, fe, be = ch.rbt_solve(B, refine=False)
        Bl = Bs.copy()
        ch.rbt_apply_local(0, Bl, 5)
        Xl = ch.solve_local(Bl, 5)
        ch.rbt_apply_local(1, Xl, 5)
        assert np.array_equal(Xl[:, :5], Y)
        X6, fe, be = ch.rbt_solve(B)
        assert be.max() <= BERR_TOL and _berr(A, X6, B) <= BERR_TOL
    _one(N, v, np.tril(A), body)


# ------------------------------------------------------------------------------------------------------ 7. refusals
def _refused(fn, status, *words):
    rc = fn()
    assert rc == status, (rc, cb._lib.lib().cflx_last_error())
    msg = cb._lib.lib().cflx_last_error().decode()
    for w in words:
        assert w in msg, msg


def test_refusals():
    L = cb._lib.lib()
    N, v = 512, 128
    ARG, UNSUP, STATE = -1, -4, -5            # CFLX_ERR_ARG, CFLX_ERR_UNSUPPORTED, CFLX_ERR_STATE

    def body(ch):
        h = ch._h
        info, nrepl = ctypes.c_int(), ctypes.c_int()
        B = np.ones((N, 1))
        X = np.empty((N, 1))
        s = np.empty(N)
        A = np.empty((ch.Ml, ch.Nl))
        _refused(lambda: L.cflx_chol_factor_ldlt(h, 0.0, None, None, ctypes.byref(info), None), STATE,
                 "cflx_chol_factor_ldlt:")
        _refused(lambda: L.cflx_chol_get_input(h, A.ctypes.data), STATE, "cflx_chol_get_input:")
        _refused(lambda: L.cflx_chol_rbt(h, 2, 0, None), STATE, "cflx_chol_rbt:")
        a = np.ascontiguousarray(ch.data)
        L.cflx_chol_set_local(h, a.ctypes.data)
        _refused(lambda: L.cflx_chol_factor_ldlt(h, -1.0, None, None, ctypes.byref(info), None), ARG,
                 "cflx_chol_factor_ldlt:", "tiny")
        _refused(lambda: L.cflx_chol_factor_ldlt(h, float("nan"), None, None, ctypes.byref(info), None), ARG,
                 "cflx_chol_factor_ldlt:", "tiny")
        _refused(lambda: L.cflx_chol_factor_ldlt(h, 0.0, None, None, None, None), ARG, "cflx_chol_factor_ldlt:",
                 "info_out")
        _refused(lambda: L.cflx_chol_get_signs(h, s.ctypes.data), STATE, "cflx_chol_get_signs:")
        _refused(lambda: L.cflx_chol_rbt(h, 0, 0, None), ARG, "cflx_chol_rbt:", "depth")
        _refused(lambda: L.cflx_chol_rbt(h, 5, 0, None), ARG, "cflx_chol_rbt:", "depth")
        _refused(lambda: L.cflx_chol_rbt(h, 3, 0, None), UNSUP, "cflx_chol_rbt:", "smallest N that works is 1024")
        assert L.cflx_chol_factor_ldlt(h, 0.0, None, None, ctypes.byref(info), None) == 0
        _refused(lambda: L.cflx_chol_rbt_solve(h, 1, B.ctypes.data, 1, X.ctypes.data, 1, 0, None, None), STATE,
                 "cflx_chol_rbt_solve:", "no random butterfly")
        _refused(lambda: L.cflx_chol_rbt_apply_local(h, 0, 1, X.ctypes.data, ch.Nl), STATE,
                 "cflx_chol_rbt_apply_local:", "no random butterfly")
        _refused(lambda: L.cflx_chol_rbt_apply_local(h, 2, 1, X.ctypes.data, ch.Nl), ARG, "cflx_chol_rbt_apply_local:",
                 "op")
        _refused(lambda: L.cflx_chol_rbt_apply_local(h, 0, 0, X.ctypes.data, ch.Nl), ARG, "cflx_chol_rbt_apply_local:",
                 "nrhs")
        _refused(lambda: L.cflx_chol_rbt_apply_local(h, 0, 1, None, ch.Nl), ARG, "cflx_chol_rbt_apply_local:", "B_local")
        _refused(lambda: L.cflx_chol_rbt_apply_local(h, 0, 1, X.ctypes.data, 1), ARG, "cflx_chol_rbt_apply_local:", "ldb")
        _refused(lambda: L.cflx_chol_rbt_solve(h, 1, B.ctypes.data, 1, X.ctypes.data, 1, 2, None, None), ARG,
                 "cflx_chol_rbt_solve:", "refine")
        _refused(lambda: L.cflx_chol_rbt_solve(h, 0, B.ctypes.data, 1, X.ctypes.data, 1, 0, None, None), ARG,
                 "cflx_chol_rbt_solve:", "nrhs")
        _refused(lambda: L.cflx_chol_get_signs(h, None), ARG, "cflx_chol_get_signs:", "s_out")
        _refused(lambda: L.cflx_chol_get_input(h, None), ARG, "cflx_chol_get_input:", "A_host")
        assert L.cflx_chol_rbt(h, 2, 0, None) == 0
        _refused(lambda: L.cflx_chol_rbt(h, 2, 0, None), STATE, "cflx_chol_rbt:", "already transformed")
        eq = ch._equilibrate
        with pytest.raises(cb.ConfluxError, match="random butterfly"):
            eq(True, False, L.cflx_chol_equilibrate, "chol_equilibrate")
        L.cflx_chol_set_local(h, a.ctypes.data)
        scond, amax, equed = ctypes.c_double(), ctypes.c_double(), ctypes.c_char()
        assert L.cflx_chol_equilibrate(h, 1, s.ctypes.data, ctypes.byref(scond), ctypes.byref(amax), ctypes.byref(equed),
                                       ctypes.byref(info)) == 0
        assert info.value == 0 and equed.value == b"Y" and scond.value < 0.1     # the diagonal spans 1 .. 1e6
        _refused(lambda: L.cflx_chol_rbt(h, 2, 0, None), STATE, "cflx_chol_rbt:", "scaled")
    # a positive diagonal from 1 to 1e6 (dpoequ's scond = 1e-3 < 0.1: it must scale), indefinite through the
    # off-diagonal entries
    G = np.random.default_rng(3).standard_normal((N, N))
    d = np.logspace(0, 6, N)
    A = np.tril((G + G.T) * np.sqrt(np.outer(d, d)))
    A[np.diag_indices(N)] = d
    _one(N, v, A, body)


# ---------------------------------------------------------------------------------------------------------- 8. grids
GRIDS = [(2, 2, 1), (2, 1, 1), (1, 2, 1), (2, 2, 2)]


def _grid_run(grid, N, v, A, depth, seed):
    Px, Py, Pz = grid
    shares = scatter(np.tril(A), v, Px, Py, Pz)
    B = np.random.default_rng(7).standard_normal((N, 2))

    def fn(comm):
        ch = cb.cholesky(N, v, grid, comm)
        try:
            ch.data[...] = shares[ch.rank]
            out = {}
            if depth:
                ch.rbt(depth=depth, seed=seed)
                out["W"] = ch.local_input()
            out["ldlt"] = ch.factor_ldlt(upload=not depth)[:3]
            out["s"] = ch.signs()
            out["R"] = ch.local_factor()
            out["X"] = ch.rbt_solve(B)[0] if depth else ch.solve(B)
            out["val"] = ch.validate()[1]
            out["det"] = ch.det()
            return out
        finally:
            ch.finalize()
    return run_ranks(Px * Py * Pz, fn), B


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "x".join(map(str, g)))
@pytest.mark.parametrize("depth", [0, 2])
def test_multi_gpu_ldlt_matches_one_gpu(grid, depth):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1024, 128
    A = ldlt_ref.kkt(600, 424, seed=17) if not depth else ldlt_ref.with_inertia(N, 500, 524, seed=17)
    res, B = _grid_run(grid, N, v, A, depth, 5)
    one, _ = _grid_run((1, 1, 1), N, v, A, depth, 5)
    for r in res:
        assert r["ldlt"] == one[0]["ldlt"] and r["ldlt"][2] == 0
        assert np.array_equal(r["s"], one[0]["s"])
        assert np.array_equal(r["X"], res[0]["X"])
        assert r["det"] == res[0]["det"]
    R = np.tril(chol_ref.assemble([r["R"] for r in res], N, v, *grid))
    s = res[0]["s"]
    if depth:
        W = chol_ref.assemble([r["W"] for r in res], N, v, *grid)
        u = rbt_ref.multipliers(N, depth, 5)[0]
        assert np.array_equal(np.tril(W), np.tril(rbt_ref.global_w(ldlt_ref.mirror(A), u, u)))
        target = np.tril(W)
    else:
        target = np.tril(A)
    kappa = hp_ref.diag_block_kappa(R, 128)
    E, Mabs = ldlt_ref.residual(target, R, s)
    assert ldlt_ref.normwise_ok(target, R, s, kappa, res=(E, Mabs))
    # validate's replay has the factorisation's own rounding: the same bound, relative to ||A||_F of the lower triangle
    assert res[0]["val"] * np.linalg.norm(target) <= 2 * hp_ref.chol_backward_bound(Mabs, kappa)
    assert _berr(A, res[0]["X"], B) <= BERR_TOL * 10


def test_grids_on_one_device(tmp_path):
    """the grid cases above in a child pytest under the NCCL loopback (P ranks as threads on device 0)"""
    from tests import _loopback
    if n_gpus() >= 8 and not os.environ.get("LD_PRELOAD"):
        pytest.skip("the grids ran on real GPUs")
    lib = _loopback.build()
    xml = tmp_path / "junit.xml"
    preload = " ".join(p for p in (lib, os.environ.get("LD_PRELOAD")) if p)
    env = dict(os.environ, LD_PRELOAD=preload, **{_loopback.STATS_ENV: str(tmp_path / "stats.json")})
    flags = ["-s"] if sys.flags.no_user_site else []
    cmd = [sys.executable] + flags + ["-m", "pytest", "-p", "tests._loopback", "-p", "no:cacheprovider", "-q", "-rA",
                                      f"--junitxml={xml}", "tests/test_gpu_ldlt.py::test_multi_gpu_ldlt_matches_one_gpu"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = r.stdout[-6000:] + "\n--- stderr ---\n" + r.stderr[-6000:]
    assert r.returncode == 0, tail
    cases = [[e.tag for e in c] for c in ET.parse(xml).iter("testcase")]
    assert len(cases) == 2 * len(GRIDS) and all(not t for t in cases), tail
