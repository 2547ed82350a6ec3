"""GPU: cflx_lu_factor_fixed / LU_rep_fixed, the LU in a prescribed row order without the pivot search, against the
restatement (oracle/fixed_ref.py), the pivoted factors of the same input, and every call that reads the factors."""
import os
import subprocess
import sys

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import fixed_ref, layout
from tests._harness import n_gpus, run_ranks
from tests.test_fixed_ref import integer_case

pytestmark = pytest.mark.gpu
RESIDUAL_TOL = 1e-12
FACTOR_TOL = 1e-10
EPS = np.finfo(float).eps
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _one(N, v, body):
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    try:
        return body(gv)
    finally:
        gv.free_comms()
        comm.close()


def _factors(gv, fixed=False, **kw):
    C, perm = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    out = cb.LU_rep_fixed(gv, C=C, permutation=perm, **kw) if fixed else cb.LU_rep(gv, C, perm, **kw)
    return C, perm, out


def _count(gv):
    import ctypes
    n = ctypes.c_int64()
    cb._lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(n), 1)
    return n.value


def _dominant(M, rng):
    return rng.standard_normal((M, M)) + 2.0 * M * np.eye(M)


# ---------------------------------------------------------------------------------------------------- the tile kernel
TILE_CASES = [(v, 0) for v in (4, 8, 16, 32, 128, 256, 512)] + [(256, 1), (512, 1)]


@pytest.mark.parametrize("v,variant", TILE_CASES)
def test_tile_hook_matches_the_restatement(v, variant):
    """variant 0: the one-CTA kernel on the whole tile; 1: the 128-block driver (what the factorisation runs at
    v = 256, 512)"""
    rng = np.random.default_rng(v)
    A = _dominant(v, rng) / v
    LU, nrepl, info = cb.dbg.getrf_nopiv_tile(A, variant=variant)
    ref, rn, ri = fixed_ref.tile_lu(A)
    assert (nrepl, info) == (rn, ri) == (0, 0)
    L, U = np.tril(ref, -1) + np.eye(v), np.triu(ref)
    # both LUs lie within the componentwise rounding bound of an LU (Higham 9.3) of the exact one: twice it apart
    bound = 8 * v * EPS * (np.abs(L) @ np.abs(U))
    assert (np.abs(LU - ref) <= bound + 1e-300).all()
    again, _, _ = cb.dbg.getrf_nopiv_tile(A, variant=variant)
    assert np.array_equal(again, LU)                            # deterministic


def bidiagonal_case(v, zeros, rng):
    """A = L U with unit lower-bidiagonal L and upper-bidiagonal U, entries in {-1, 0, 1}, U(j, j) = 0 at zeros (and
    L(j + 1, j) = 0 there): the inverses of every triangular block are integer too, so the driver's TRSMs with inverted
    diagonal blocks stay exact and the zero pivots come out exactly zero"""
    l = rng.integers(-1, 2, v - 1).astype(float)
    u = rng.integers(-1, 2, v - 1).astype(float)
    d = rng.choice([-1.0, 1.0], v)
    d[zeros] = 0.0
    for j in zeros:
        if j + 1 < v:
            l[j] = 0.0
    return (np.eye(v) + np.diag(l, -1)) @ (np.diag(d) + np.diag(u, 1))


@pytest.mark.parametrize("v", [256, 512])
def test_tile_driver_counts_and_first_zero(v):
    """the 128-block driver: zero pivots in different 128-blocks give the first one's column; the tiny rule replaces
    each, with the exact value"""
    rng = np.random.default_rng(v + 1)
    zeros = [130, v - 1]
    A = bidiagonal_case(v, zeros, rng)
    _, nrepl, info = cb.dbg.getrf_nopiv_tile(A, variant=1)
    assert (nrepl, info) == (0, zeros[0] + 1)
    got, nrepl, info = cb.dbg.getrf_nopiv_tile(A, tiny=0.5, variant=1)
    assert (nrepl, info) == (len(zeros), 0)
    assert all(got[j, j] == 0.5 for j in zeros)
    L, U = np.tril(got, -1) + np.eye(v), np.triu(got)
    E = np.zeros((v, v))
    E[zeros, zeros] = 0.5
    assert (np.abs(L @ U - A - E) <= 4 * v * EPS * (np.abs(L) @ np.abs(U))).all()


@pytest.mark.parametrize("v,zero", [(16, 0), (16, 5), (64, 31), (64, 32), (128, 127), (512, 300)])
def test_tile_hook_zero_and_tiny_pivots_are_exact(v, zero):
    rng = np.random.default_rng(v + zero)
    A, LU = integer_case(v, [zero], rng)
    _, nrepl, info = cb.dbg.getrf_nopiv_tile(A, variant=0)
    assert (nrepl, info) == (0, zero + 1)
    got, nrepl, info = cb.dbg.getrf_nopiv_tile(A, tiny=0.5, variant=0)
    want = LU.copy()
    want[zero, zero] = 0.5
    assert (nrepl, info) == (1, 0)
    assert np.array_equal(got, want)
    B, LB = integer_case(v, [], rng, small=[zero])
    got, nrepl, info = cb.dbg.getrf_nopiv_tile(B, tiny=0.5, variant=0)
    assert (nrepl, info) == (1, 0) and got[zero, zero] == -0.5
    assert np.array_equal(np.delete(got.ravel(), zero * v + zero), np.delete(LB.ravel(), zero * v + zero))


# ---------------------------------------------------------------------------------------------- whole factorisations
@pytest.mark.parametrize("N,v", [(16, 4), (64, 8), (96, 16), (256, 32), (512, 64), (1024, 128), (768, 256), (100, 16),
                                 (4096, 256)])
def test_same_input_last_permutation(N, v):
    def body(gv):
        C0, p0, _ = _factors(gv)
        C1, p1, (ms, nrepl, info) = _factors(gv, fixed=True, upload=False)
        assert (nrepl, info) == (0, 0) and ms > 0
        assert np.array_equal(p1, p0)
        assert np.abs(C1 - C0).max() <= FACTOR_TOL * np.abs(gv.data).max()
        assert cb.validate(gv)[1] <= RESIDUAL_TOL
    _one(N, v, body)


@pytest.mark.parametrize("N,v", [(256, 32), (1024, 128), (2048, 256)])
@pytest.mark.parametrize("order", ["identity", "random"])
def test_identity_and_random_orders_match_the_restatement(N, v, order):
    def body(gv):
        rng = np.random.default_rng(N + v)
        M = gv.M
        perm = np.arange(M, dtype=np.int32) if order == "identity" else rng.permutation(M).astype(np.int32)
        A = _dominant(M, rng)
        gv.data[...] = A[np.argsort(perm)]                     # rows scattered by perm^-1: A[perm] is dominant
        C, p, (_, nrepl, info) = _factors(gv, fixed=True, perm=perm)
        assert (nrepl, info) == (0, 0) and np.array_equal(p, perm)
        ref = fixed_ref.lu(gv.data, perm, v)["LU"]
        assert np.abs(C - ref).max() <= FACTOR_TOL * np.abs(A).max()
        assert cb.validate(gv)[1] <= RESIDUAL_TOL
    _one(N, v, body)


def test_nearby_matrix_with_the_last_pivots():
    def body(gv):
        rng = np.random.default_rng(3)
        A = gv.data.copy()
        _factors(gv)
        An = A + 1e-6 * rng.standard_normal(A.shape)
        B = rng.standard_normal((gv.M, 3))
        gv.data = An
        cb.LU_rep(gv)                                            # the pivoted factors of the nearby matrix
        _, _, berr_piv = cb.lu_refine(gv, B, cb.lu_solve(gv, B))
        gv.data = A
        cb.LU_rep(gv)
        gv.data = An
        _, _, (_, nrepl, info) = _factors(gv, fixed=True)        # perm = None: the last permutation, new upload
        assert (nrepl, info) == (0, 0)
        resid = cb.validate(gv)[1]
        assert resid <= RESIDUAL_TOL, resid
        X = cb.lu_solve(gv, B)
        berr = np.max(np.abs(B - An @ X) / (np.abs(An) @ np.abs(X) + np.abs(B)))
        assert berr <= 1e-13, berr
        X2, _, berr2 = cb.lu_refine(gv, B, X)
        # dgerfs stops at berr <= 2^-53, or when a correction no longer halves it; a column stopped by the second rule
        # ends at rounding level, and no further from 2^-53 than refinement with the pivoted factors gets
        ok = (berr2 <= 2.0 ** -53) | (berr2 <= np.maximum(2.0 ** -52, 2 * berr_piv))
        assert ok.all(), (berr2, berr_piv)
    _one(2048, 256, body)


def test_zero_pivot_info_is_the_first_column():
    N, v, zero = 128, 32, 40
    rng = np.random.default_rng(zero)
    A, _ = integer_case(N, [zero], rng)

    def body(gv):
        gv.data[...] = A
        _, _, (_, nrepl, info) = _factors(gv, fixed=True, perm=np.arange(N))
        assert (nrepl, info) == (0, zero + 1)
        assert cb.lu_det(gv)["info"] == zero + 1
    _one(N, v, body)


def test_tiny_pivots_perturb_only_the_replaced_diagonal():
    N, v = 256, 64
    rng = np.random.default_rng(5)
    zeros = [0, 63, 64, 200]
    A, LU = integer_case(N, zeros, rng)

    def body(gv):
        gv.data[...] = A
        C, p, (_, nrepl, info) = _factors(gv, fixed=True, perm=np.arange(N), tiny=0.5)
        assert (nrepl, info) == (len(zeros), 0)
        for j in zeros:
            assert C[j, j] == 0.5
        L, U = np.tril(C, -1) + np.eye(N), np.triu(C)
        E = np.zeros((N, N))
        E[zeros, zeros] = 0.5
        assert (np.abs(L @ U - A - E) <= 4 * N * EPS * (np.abs(L) @ np.abs(U))).all()
    _one(N, v, body)


def test_streaming_and_determinism():
    def body(gv):
        rng = np.random.default_rng(11)
        A0 = gv.data.copy()
        _factors(gv)
        mats = [cb.pinned_empty((gv.Ml, gv.Nl)) for _ in range(3)]
        for m in mats:
            m[...] = A0 + 1e-6 * rng.standard_normal(A0.shape)
        want = []
        for m in mats:                                           # separate uploads
            gv.data = m
            want.append(_factors(gv, fixed=True)[:2])
        gv.data = mats[0]
        got = []
        for i in range(3):                                       # streamed
            got.append(_factors(gv, fixed=True, upload=(i == 0), next_data=mats[i + 1] if i < 2 else None)[:2])
        for (c0, p0), (c1, p1) in zip(want, got):
            assert np.array_equal(p0, p1) and np.array_equal(c0, c1)
        a = _factors(gv, fixed=True)[:2]
        b = _factors(gv, fixed=True, upload=False)[:2]
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        for m in mats:
            cb.pinned_free(m)
    _one(1024, 128, body)


def test_downstream_calls_agree_with_the_pivoted_factors():
    def body(gv):
        rng = np.random.default_rng(2)
        B = rng.standard_normal((gv.M, 2))
        Bs = rng.standard_normal((gv.Ml, cb.rhs_local_cols(2, gv.v, gv.Py)))
        res = []
        for fixed in (False, True):
            if fixed:
                cb.LU_rep_fixed(gv, upload=False)
            else:
                cb.LU_rep(gv)
            X = cb.lu_solve(gv, B)
            XT = cb.lu_solve(gv, B, trans=True)
            rc = cb.lu_rcond(gv)[0]
            Xr, ferr, berr = cb.lu_refine(gv, B, X.copy())
            sv = cb.lu_svx(gv, B)
            det = cb.lu_det(gv)
            inv = cb.lu_inverse(gv)
            loc = cb.lu_solve_local(gv, Bs, 2)
            res.append((X, XT, rc, Xr, sv, det, inv, loc))
        (X0, XT0, r0, Xr0, sv0, d0, i0, l0), (X1, XT1, r1, Xr1, sv1, d1, i1, l1) = res
        scale = np.abs(X0).max()
        assert np.abs(X1 - X0).max() <= 1e-10 * scale and np.abs(XT1 - XT0).max() <= 1e-10 * np.abs(XT0).max()
        assert abs(r1 - r0) <= 1e-6 * r0
        assert np.abs(Xr1 - Xr0).max() <= 1e-9 * scale
        assert np.abs(np.asarray(sv1[0]) - np.asarray(sv0[0])).max() <= 1e-10 * scale
        _det_close(d0, d1)
        assert np.abs(_first(i1) - _first(i0)).max() <= 1e-9 * np.abs(_first(i0)).max()
        assert np.abs(_first(l1) - _first(l0)).max() <= 1e-10 * np.abs(_first(l0)).max()
    _one(1024, 128, body)


def _first(x):
    return np.asarray(x[0] if isinstance(x, tuple) else x)


def _det_close(d0, d1):
    assert d0["sign"] == d1["sign"] and d0["info"] == d1["info"] == 0
    assert abs(d0["logabsdet"] - d1["logabsdet"]) <= 1e-10 * max(1.0, abs(d0["logabsdet"]))


def test_no_effect_on_the_pivoted_path():
    def body(gv):
        C0, p0, _ = _factors(gv)
        n0 = _count(gv)
        _factors(gv, fixed=True, upload=False)
        _count(gv)
        C2, p2, _ = _factors(gv, upload=False)
        n2 = _count(gv)
        assert np.array_equal(p2, p0) and np.array_equal(C2.view(np.uint64), C0.view(np.uint64)) and n2 == n0
    _one(1024, 128, body)


def switch_factors(path):
    """the pivoted factorisation, then the fixed one of the same input with its permutation, saved to path (run in a
    child interpreter: CFLX_TRSM_NB and CFLX_GEMM_TILE are read once per process)"""
    def body(gv):
        cb.LU_rep(gv)
        C, p, _ = _factors(gv, fixed=True, upload=False)
        np.savez(path, C=C, p=p)
    _one(2048, 256, body)


def _child_factors(env, path):
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import test_gpu_lu_fixed as t; "
            f"t.switch_factors({path!r})")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=dict(os.environ, **env), cwd=ROOT, timeout=900,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    z = np.load(path)
    return z["C"], z["p"]


@pytest.mark.parametrize("env", [{"CFLX_LOOKAHEAD": "0"}, {"CFLX_PANEL_CTAS": "8"}, {"CFLX_TRSM_NB": "32"},
                                 {"CFLX_GEMM_TILE": "64"}, {"CFLX_GEMM": "ozaki"}],
                         ids=lambda e: "-".join(f"{k}={x}" for k, x in e.items()))
def test_switches(env, tmp_path):
    C0, p0 = _child_factors({}, os.path.join(str(tmp_path), "base.npz"))
    C1, p1 = _child_factors(env, os.path.join(str(tmp_path), "switch.npz"))
    assert np.array_equal(p1, p0)
    if set(env) <= {"CFLX_LOOKAHEAD", "CFLX_PANEL_CTAS"}:       # where and on how many SMs: the same operations
        assert np.array_equal(C1.view(np.uint64), C0.view(np.uint64))
    else:
        assert np.abs(C1 - C0).max() <= FACTOR_TOL * 6.0


def test_argument_and_state_rules():
    def body(gv):
        import ctypes
        L = cb._lib.lib()
        info = ctypes.c_int()
        M = gv.M
        with pytest.raises(cb.ConfluxError, match="status -5"):  # nothing uploaded yet
            cb.LU_rep_fixed(gv, perm=np.arange(M), upload=False)
        L.cflx_lu_set_local(gv._h, np.ascontiguousarray(gv.data).ctypes.data)
        with pytest.raises(cb.ConfluxError, match="status -5"):  # no completed factorisation: no last permutation
            cb.LU_rep_fixed(gv, upload=False)
        for bad in (np.zeros(M), np.arange(M)[::-1] + 1, np.r_[np.arange(M - 1), 0]):
            with pytest.raises(cb.ConfluxError, match="status -1"):
                cb.LU_rep_fixed(gv, perm=bad, upload=False)
        for tiny in (-1.0, float("nan")):
            with pytest.raises(cb.ConfluxError, match="status -1"):
                cb.LU_rep_fixed(gv, perm=np.arange(M), tiny=tiny, upload=False)
        p = np.arange(M, dtype=np.int32)
        assert L.cflx_lu_factor_fixed(gv._h, p.ctypes.data, 0.0, None, None, None) == -1     # info_out required
        assert L.cflx_lu_factor_fixed(gv._h, p.ctypes.data, 0.0, None, ctypes.byref(info), None) == 0
        cb.LU_rep(gv)
        _, p1, _ = _factors(gv, fixed=True)                     # NULL after set_local: allowed
        gv.data = gv.data * 2.0
        cb.lu_equilibrate(gv)                                   # equilibration keeps it too
        _, p2, _ = _factors(gv, fixed=True, upload=False)
        assert np.array_equal(p1, p2)
    _one(256, 32, body)


# ------------------------------------------------------------------------------------------------------- multi-GPU
@pytest.mark.parametrize("grid", [(1, 1, 2), (2, 2, 1), (2, 2, 2)], ids=lambda g: "x".join(map(str, g)))
def test_multi_gpu_same_input_refactor(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 512, 32

    def body(comm):
        gv = cb.lu_params(N, N, v, *grid, comm)
        C0, p0, _ = _factors(gv)
        C1, p1, (_, nrepl, info) = _factors(gv, fixed=True, upload=False)
        resid = cb.validate(gv)[1]
        bad = p0.copy()
        if gv.rank == 1:
            bad[[0, 1]] = bad[[1, 0]]
        try:
            cb.LU_rep_fixed(gv, perm=bad, upload=False)
            refused = False
        except cb.ConfluxError as e:
            refused = "status -1" in str(e)
        scale = np.abs(gv.data).max()
        gv.free_comms()
        return dict(same=np.array_equal(p0, p1), diff=np.abs(C1 - C0).max() / max(scale, 1e-300) if gv.pk == 0 else 0,
                    nrepl=nrepl, info=info, resid=resid, refused=refused)
    rs = run_ranks(P, body)
    for r in rs:
        assert r["same"] and r["diff"] <= FACTOR_TOL and (r["nrepl"], r["info"]) == (0, 0)
        assert r["resid"] <= RESIDUAL_TOL and r["refused"]


@pytest.mark.parametrize("grid", [(2, 2, 1), (2, 2, 2)], ids=lambda g: "x".join(map(str, g)))
def test_multi_gpu_zero_and_tiny_pivots_on_every_rank(grid):
    """zero pivots in tiles owned by different grid rows (different roots of the tile LU): info is the first one's column
    and nrepl counts all of them, identical on every rank; the replaced pivots hold exactly tiny"""
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 128, 16
    zeros = [37, 5 * v + 3, 110]                                 # tiles 2, 5, 6: grid rows 0, 1, 0
    A, _ = integer_case(N, zeros, np.random.default_rng(9))
    shares = layout.scatter(A, v, *grid)

    def body(comm):
        gv = cb.lu_params(N, N, v, *grid, comm)
        gv.data[...] = shares[gv.rank]
        _, _, (_, n0, i0) = _factors(gv, fixed=True, perm=np.arange(N))
        C, _, (_, n1, i1) = _factors(gv, fixed=True, perm=np.arange(N), tiny=0.5)
        gv.free_comms()
        return dict(n0=n0, i0=i0, n1=n1, i1=i1, C=C)
    rs = run_ranks(P, body)
    for r in rs:
        assert (r["n0"], r["i0"]) == (0, zeros[0] + 1)
        assert (r["n1"], r["i1"]) == (len(zeros), 0)
    F = layout.assemble([r["C"] for r in rs], N, v, *grid)
    assert all(F[j, j] == 0.5 for j in zeros)
