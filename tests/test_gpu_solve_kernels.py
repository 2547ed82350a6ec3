"""GPU: the solve engine (csrc/solve.cu) kernel by kernel against the extended-precision bounds of oracle/hp_ref.py: the
two narrow GEMMs at the windows the sweeps launch, the diagonal-tile solve in every triangle mode and block size, and the
one-GPU LU solves under the diagonal block-size switch.

Constants: every tolerance is one of the hp_ref bounds (gamma_n = n u / (1 - n u), u = 2^-53), or bit identity:
  * the narrow GEMMs (NN and TN):  |D^ - (beta C + alpha op(A) B)| <= gamma_{K+1} (|beta| |C| + |alpha| |op(A)| |B|)
                                   (gemm_ok), and the exact product bit for bit on small-integer inputs
  * diag_solve:                    ||T Y^ - R||_F <= gamma_{v+1} (1 + 4 kappa_max) || |T| |Y^| ||_F (trsm_left_ok); every
                                   cached inverse block |T_jj X^ - I| <= gamma_nb |T_jj| |X^|; and Y and the blocks bit
                                   for bit on tiles whose block inverses and products are exact
  * the whole solves:              the normwise backward error <= 1e-13 (as tests/test_gpu_solve.py), and X within
                                   100 eps / rcond of the reference solution or of the default block size's X (max norm,
                                   relative, per column), as tests/test_gpu_rbt.py bounds its forward error
Every buffer holds NaN outside the blocks a launch may read or write.  CFLX_TRSM_NB is read once per process: its solves
run in a child interpreter that writes its results to a temporary directory."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import hp_ref as hp, solve_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = np.nan
EPS = np.finfo(float).eps
ETA_TOL = 1e-13
AB = [(1.0, 0.0), (-1.0, 1.0)]          # every (alpha, beta) the engine launches


def _rup2(x):
    return x + (x & 1)


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint64),
                                                 np.ascontiguousarray(b).view(np.uint64))


def _canvas(shape, block, at):
    """a NaN array of `shape` with `block` at (row, column) `at`"""
    out = np.full(shape, NAN)
    out[at[0]:at[0] + block.shape[0], at[1]:at[1] + block.shape[1]] = block
    return out


def _padded(block, at):
    """block at `at` of a NaN buffer with a NaN margin on every side and an even leading dimension"""
    return _canvas((at[0] + block.shape[0] + 3, _rup2(at[1] + block.shape[1] + 3)), block, at)


# ----------------------------------------------------------------------------------------------- the narrow GEMMs
def _window(trans, Ablk, Bblk, Cwin, alpha, beta, in_place, a_buf=None, a_at=(3, 6), b_buf=None, b_at=(5, 3),
            c_buf=None, c_at=(7, 5)):
    """one launch through the window hook: Ablk (M x K, or K x M with trans) at a_at of a_buf (default: a NaN buffer
    around it), Bblk at b_at of b_buf, the C window Cwin (NaN when beta == 0: it must not be read) at c_at of c_buf.
    Checks that nothing outside the C window changed, and returns (D window, the reference AT)."""
    M, N = Cwin.shape
    K = Bblk.shape[0]
    a_buf = _padded(Ablk, a_at) if a_buf is None else a_buf
    b_buf = _padded(Bblk, b_at) if b_buf is None else b_buf
    Cin = np.full_like(Cwin, NAN) if beta == 0 else Cwin
    c_buf = _padded(Cin, c_at) if c_buf is None else c_buf.copy()
    c_buf[c_at[0]:c_at[0] + M, c_at[1]:c_at[1] + N] = Cin
    D, Cout = cb.dbg.gemm_narrow_window(a_buf, b_buf, c_buf, M, N, K, alpha, beta, a_at, b_at, c_at, trans, in_place)
    outside = np.ones(c_buf.shape, dtype=bool)
    outside[c_at[0]:c_at[0] + M, c_at[1]:c_at[1] + N] = False
    assert _same_bits(D[outside], c_buf[outside]), "the launch wrote outside its C window"
    if not in_place:
        assert _same_bits(Cout, c_buf), "the out-of-place launch wrote C"
    return D[c_at[0]:c_at[0] + M, c_at[1]:c_at[1] + N], (Ablk if trans else Ablk.T)


def _check_window(trans, M, N, K, seed, **kw):
    """gemm_ok for both (alpha, beta), in place and out of place, on standard normal blocks"""
    rng = np.random.default_rng(seed)
    Ablk = rng.standard_normal((K, M) if trans else (M, K))
    Bblk = rng.standard_normal((K, N))
    Cwin = rng.standard_normal((M, N))
    for alpha, beta in AB:
        for in_place in (True, False):
            D, AT = _window(trans, Ablk, Bblk, Cwin, alpha, beta, in_place, **kw)
            if K == 0:
                assert np.array_equal(D, beta * Cwin if beta else np.zeros((M, N))), (M, N, K, alpha, beta)
            else:
                assert hp.gemm_ok(AT, Bblk, Cwin, alpha, beta, D), (trans, M, N, K, alpha, beta, in_place)


TRANS = pytest.mark.parametrize("trans", [False, True], ids=["nn", "tn"])


@TRANS
@pytest.mark.parametrize("N", [1, 8, 9, 16, 17, 32, 33, 64, 65, 130, 2048])
def test_narrow_gemm_every_column_slab(trans, N):
    """every NT instantiation (N <= 8, 16, 32, wider) and several 64-column slabs, with K across two KC chunks and a
    partial 16-wide step"""
    _check_window(trans, 129 if not trans else 127, N, 68, N)


K_TAILS = [4, 12, 60, 64, 68, 128, 132, 512, 0]


@pytest.mark.parametrize("trans,K", [(False, K) for K in K_TAILS] + [(True, K) for K in K_TAILS + [1, 13, 67]],
                         ids=[f"nn-{K}" for K in K_TAILS] + [f"tn-{K}" for K in K_TAILS + [1, 13, 67]])
def test_narrow_gemm_every_k_tail(trans, K):
    """K across the KC = 64 chunks and the 16-wide steps (K % 16 != 0), and K = 0; odd K on the transposed kernel (the
    NN kernel takes K % 4 == 0 only: its refusal is tested below)"""
    for N in (9, 65):
        _check_window(trans, 65, N, K, K * 7 + N)


@TRANS
@pytest.mark.parametrize("M", [1, 15, 17, 63, 64, 65, 127, 129, 4097])
def test_narrow_gemm_every_row_tail(trans, M):
    """M around BM = 64 (NN) and BM_TN = 128 (TN), odd M (the TN kernel's last row pair)"""
    _check_window(trans, M, 17, 132, M)


# The launch forms solve.cu issues, on a share of Ml x Nl with lda = Nl: (name, trans, M, K, A block at, B rows at,
# C window rows at, the C buffer's rows, alpha, beta).  Sweep step t = 1 (t = 2 for the prefix) of v = 256 tiles on one
# GPU; the diagonal tile at (v, 2 v), nb = 32 (nblk = 8), and the inverse products at nb = 4, 32 and 128.
ML, NL, V = 768, 1024, 256
TILE = (V, 2 * V)


def _launch_forms():
    forms = [("row sweep, forward", False, ML - 2 * V, V, (2 * V, V), 0, 2 * V, ML, -1.0, 1.0),
             ("row sweep, backward", False, V, V, (0, V), 0, 0, ML, -1.0, 1.0),
             ("column sweep, suffix", True, NL - 2 * V, V, (V, 2 * V), 0, 2 * V, NL, -1.0, 1.0),
             ("column sweep, prefix", True, V, V, (2 * V, V), 0, V, NL, -1.0, 1.0)]
    for nb in (4, 32, 128):
        nblk = V // nb
        for j in sorted({0, nblk // 2, nblk - 1}):
            for half, row in (("forward", j * nb), ("backward", V + j * nb)):
                for trans in (False, True):
                    forms.append((f"inverse product nb={nb} j={j} {half} {'tn' if trans else 'nn'}", trans, nb, nb, ("inv", row), j * nb, j * nb,
                                  V, 1.0, 0.0))
    nb, nblk = 32, V // 32
    r0, c0 = TILE
    for j in (0, nblk // 2, nblk - 1):
        o, o1 = j * nb, (j + 1) * nb
        if j + 1 < nblk:
            forms.append((f"Lower update j={j}", False, V - o1, nb, (r0 + o1, c0 + o), o, o1, V, -1.0, 1.0))
            forms.append((f"UpperT update j={j}", True, V - o1, nb, (r0 + o, c0 + o1), o, o1, V, -1.0, 1.0))
        if j > 0:
            forms.append((f"Upper update j={j}", False, o, nb, (r0, c0 + o), o, 0, V, -1.0, 1.0))
            forms.append((f"LowerT update j={j}", True, o, nb, (r0 + o, c0), o, 0, V, -1.0, 1.0))
    return forms


LAUNCH_FORMS = _launch_forms()


@pytest.mark.parametrize("ldn", [8, 72])
@pytest.mark.parametrize("form", LAUNCH_FORMS, ids=[f[0] for f in LAUNCH_FORMS])
def test_narrow_gemm_at_the_engine_launch_forms(form, ldn):
    """each launch of the sweeps and of diag_solve with its own operand layout: A read in place from a share (lda = Nl)
    or from the cached inverse blocks (lda = nb), B the solved tile Y, the C window in W / Z / R (in place) or Y
    (beta = 0, out of place in the engine's sense: C is not read)"""
    name, trans, M, K, a_at, b_row, c_row, c_rows, alpha, beta = form
    rng = np.random.default_rng(sum(map(ord, name)) + ldn)
    Ablk = rng.standard_normal((K, M) if trans else (M, K))
    if a_at[0] == "inv":                                          # the tile's 2 v nb cached blocks, row-major nb wide
        a_buf, a_at = _canvas((2 * V, K if not trans else M), Ablk, (a_at[1], 0)), (a_at[1], 0)
    else:
        a_buf = _canvas((ML, NL), Ablk, a_at)
    Bblk = rng.standard_normal((K, ldn))
    b_buf = _canvas((V, ldn), Bblk, (b_row, 0))
    Cwin = rng.standard_normal((M, ldn))
    c_buf = np.full((c_rows, ldn), NAN)
    D, AT = _window(trans, Ablk, Bblk, Cwin, alpha, beta, True, a_buf=a_buf, a_at=a_at, b_buf=b_buf, b_at=(b_row, 0),
                    c_buf=c_buf, c_at=(c_row, 0))
    assert hp.gemm_ok(AT, Bblk, Cwin, alpha, beta, D), name


EXACT_SHAPES = [(129, 65, 132, (3, 6)), (4097, 9, 68, (0, 0)), (17, 2048, 12, (1, 2)), (64, 1, 512, (0, 0)),
                (63, 33, 64, (5, 4))]


@TRANS
@pytest.mark.parametrize("M,N,K,at", EXACT_SHAPES)
def test_narrow_gemm_exact_products(trans, M, N, K, at):
    """small-integer A, B and C whose every partial sum is exact (K max|a| max|b| + max|c| < 2^53): D must be the exact
    product bit for bit, dense (at the origin) and windowed; an epilogue that rounded alpha * acc before the add, a
    dropped or repeated k step, or a misplaced column would all show"""
    rng = np.random.default_rng(M + N + K)
    Ablk = rng.integers(-4, 5, (K, M) if trans else (M, K)).astype(np.float64)
    Bblk = rng.integers(-4, 5, (K, N)).astype(np.float64)
    Cwin = rng.integers(-4, 5, (M, N)).astype(np.float64)
    A_int = (Ablk.T if trans else Ablk).astype(np.int64)
    for alpha, beta in AB:
        want = (int(alpha) * (A_int @ Bblk.astype(np.int64)) + int(beta) * Cwin.astype(np.int64)).astype(np.float64)
        D, _ = _window(trans, Ablk, Bblk, Cwin, alpha, beta, True, a_at=at, b_at=at, c_at=at)
        assert np.array_equal(D, want), (trans, M, N, K, alpha, beta)
    if not trans:                                                 # the dense hook too
        D, _ = cb.dbg.gemm_narrow(Ablk, Bblk)
        assert np.array_equal(D, (A_int @ Bblk.astype(np.int64)).astype(np.float64))


# ----------------------------------------------------------------------------------------------- diag_solve
LU_MODES = ["lower", "upper", "unit_lower_t", "upper_t"]
CHOL_MODES = ["lower", "lower_t"]


@functools.lru_cache(maxsize=None)
def _lu_tile(v):
    """L\\U of a standard normal v x v block by the factorisation's panel kernel (a diagonal tile of a real factor)"""
    _, A00, _, _ = cb.dbg.panel(np.random.default_rng(v).standard_normal((v, v)))
    return A00


@functools.lru_cache(maxsize=None)
def _chol_tile(v):
    """L of an SPD matrix with kappa = 1e4 by the factorisation's tile kernel, zeros above its diagonal"""
    L, _, info = cb.dbg.potrf_tile(hp.random_spd(v, 1e4, np.random.default_rng(v + 1)), 0)
    assert info == 0
    return np.tril(L)


def _lu_parts(tile):
    return np.tril(tile, -1) + np.eye(len(tile)), np.triu(tile)


def _triangle(tile, mode, lower):
    """the T that diag_solve in `mode` solves with, on the LU tile L\\U or the Cholesky tile L"""
    if lower:
        return tile if mode == "lower" else tile.T
    L, U = _lu_parts(tile)
    return {"lower": L, "upper": U, "unit_lower_t": L.T, "upper_t": U.T}[mode]


def _share(tile):
    """a NaN share with the tile at a non-zero tile offset (its own row and twice its column)"""
    v = len(tile)
    return _canvas((2 * v + 3, _rup2(3 * v + 5)), tile, (v, 2 * v)), (v, 2 * v)


def _diag_solve(tile, lower, mode, nb, R):
    share, pos = _share(tile)
    return cb.dbg.diag_solve(mode, share, R, len(tile), nb, pos=pos, lower=lower)


def _blocks(T, nb):
    return [T[i:i + nb, i:i + nb] for i in range(0, len(T), nb)]


def _check_inverses(tile, lower, nb, inv):
    """every cached block against the diagonal block it inverts: forward inv(L_jj), backward inv(U_jj) (LU) or
    inv(L_jj)^T (Cholesky: checked as the inverse of L_jj^T, which the kernel computes; the forward half is its exact
    block transpose)"""
    fwd, bwd = inv
    if lower:
        for Ljj, F, Bk in zip(_blocks(tile, nb), fwd, bwd):
            assert hp.inverse_componentwise_ok(Ljj.T, Bk)
            assert _same_bits(F, np.ascontiguousarray(Bk.T))
    else:
        L, U = _lu_parts(tile)
        for Ljj, Ujj, F, Bk in zip(_blocks(L, nb), _blocks(U, nb), fwd, bwd):
            assert hp.inverse_componentwise_ok(Ljj, F)
            assert hp.inverse_componentwise_ok(Ujj, Bk)


def _check_tile(v, nb, ldn):
    rng = np.random.default_rng(v * 1000 + nb * 10 + ldn)
    R = rng.standard_normal((v, ldn))
    for lower, modes in ((False, LU_MODES), (True, CHOL_MODES)):
        tile = _chol_tile(v) if lower else _lu_tile(v)
        inv0 = None
        for mode in modes:
            Y, inv = _diag_solve(tile, lower, mode, nb, R)
            assert hp.trsm_left_ok(_triangle(tile, mode, lower), R, Y, nb), (v, nb, ldn, mode, lower)
            if inv0 is None:
                _check_inverses(tile, lower, nb, inv)
                inv0 = inv
            assert _same_bits(inv, inv0), "the cached inverses depend on the mode"


VNB = [(v, nb) for v in (64, 128, 256, 384, 512) for nb in (4, 8, 16, 32, 64, 128) if nb <= v and v % nb == 0]


@pytest.mark.parametrize("v,nb", VNB)
def test_diag_solve_every_block_size(v, nb):
    """the six (tile, mode) pairs the solves use, at every block size dividing v: nblk from 1 to 128, so every in-tile
    update runs at its first, interior and last block"""
    _check_tile(v, nb, 16)


@pytest.mark.parametrize("ldn", [8, 16, 32, 64, 136])
def test_diag_solve_every_rhs_width(ldn):
    _check_tile(512, 32, ldn)


def _exact_tile(v, nb, lower, rng):
    """A tile whose diagonal-block inverses and block products are exact in float64, and its exact inverse blocks:
    diagonal blocks 2^e (I + N) with N the sub- (lower) or superdiagonal (upper) of random signs, whose inverse
    2^-e (I + N)^-1 has entries 0 and +-2^-e, and the LU's unit L bidiagonal with -1 below the diagonal, whose inverse
    is the all-ones lower triangle; every other entry of the triangle a small integer"""
    def graded(upper):
        T = np.zeros((v, v))
        for j in range(0, v, nb):
            D = np.eye(nb) + np.diag(rng.choice([-1.0, 1.0], nb - 1), 1 if upper else -1)
            T[j:j + nb, j:j + nb] = 2.0 ** int(rng.integers(-1, 3)) * D
        return T

    def ints(k):
        M = rng.integers(-2, 3, (v, v)).astype(np.float64)
        for j in range(0, v, nb):
            M[j:j + nb, j:j + nb] = 0.0
        return np.tril(M, -1) if k == "lower" else np.triu(M, 1)

    if lower:
        L = graded(False) + ints("lower")
        bwd = [hp.tri_inverse(B.T, lower=False).astype(np.float64) for B in _blocks(L, nb)]
        return L, (np.stack([b.T for b in bwd]), np.stack(bwd))
    L = np.eye(v) - np.diag(np.ones(v - 1), -1)
    L = np.where(np.kron(np.eye(v // nb), np.ones((nb, nb))) > 0, L, 0.0) + ints("lower")
    U = graded(True) + ints("upper")
    fwd = [hp.tri_inverse(B, lower=True, unit=True).astype(np.float64) for B in _blocks(L, nb)]
    bwd = [hp.tri_inverse(B, lower=False).astype(np.float64) for B in _blocks(U, nb)]
    return np.tril(L, -1) + U, (np.stack(fwd), np.stack(bwd))


@pytest.mark.parametrize("v,nb,ldn", [(512, 4, 16), (384, 128, 8), (256, 32, 136), (128, 16, 33)])
def test_diag_solve_exact_tiles_bit_for_bit(v, nb, ldn):
    """Y = X bit for bit for R = T X with integer X, in every mode, and the cached inverse blocks bit for bit: a wrong
    block offset, a missing or repeated in-tile update or a wrong inverse block cannot hide in a rounding bound here"""
    rng = np.random.default_rng(v + nb + ldn)
    X = rng.integers(-3, 4, (v, ldn)).astype(np.float64)
    for lower, modes in ((False, LU_MODES), (True, CHOL_MODES)):
        tile, inv_want = _exact_tile(v, nb, lower, rng)
        for mode in modes:
            T = _triangle(tile, mode, lower)
            R = T @ X                                             # small dyadic sums: exact in any order
            Y, inv = _diag_solve(tile, lower, mode, nb, R)
            assert np.array_equal(Y, X), (v, nb, ldn, mode, lower, int(np.sum(Y != X)))
            assert np.array_equal(inv, inv_want), (v, nb, mode, lower)


# ----------------------------------------------------------------------------------------------- the whole solves
SWITCH_CASES = [(2048, 512), (1024, 256)]


@functools.lru_cache(maxsize=None)
def _solves(N, v):
    """the one-GPU LU of a seeded standard normal matrix of order N (tile v), then lu_solve, lu_solve(trans=True) and
    lu_rcond: dict(A, B, X, XT, rcond)"""
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    rng = np.random.default_rng(N + v)
    gv.data[...] = rng.standard_normal((gv.Ml, gv.Nl))
    A = gv.data.copy()
    cb.LU_rep(gv)
    B = rng.standard_normal((gv.M, 5))
    out = dict(A=A, B=B, X=cb.lu_solve(gv, B), XT=cb.lu_solve(gv, B, trans=True), rcond=cb.lu_rcond(gv)[0])
    gv.free_comms()
    comm.close()
    return out


def switch_solves(path):
    """X, XT and rcond of every SWITCH_CASES entry into the .npz file `path` (run in a child under CFLX_TRSM_NB)"""
    res = {}
    for N, v in SWITCH_CASES:
        s = _solves(N, v)
        res.update({f"X_{N}_{v}": s["X"], f"XT_{N}_{v}": s["XT"], f"rcond_{N}_{v}": s["rcond"]})
    np.savez(path, **res)


def _child(fn, env, tmp_path):
    """fn(path) of this module in a fresh interpreter with env added (switches read once per process); returns the
    arrays it saved to path"""
    path = os.path.join(str(tmp_path), f"{fn}.npz")
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import test_gpu_solve_kernels as t; "
            f"t.{fn}({path!r})")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=dict(os.environ, **env), cwd=ROOT, timeout=900,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return dict(np.load(path))


def _rel_cols(X, Xref):
    return float((np.abs(X - Xref).max(axis=0) / np.abs(Xref).max(axis=0)).max())


@pytest.mark.parametrize("N,v", SWITCH_CASES)
def test_default_block_solves(N, v):
    """the default block size (nb = 128: nblk = 4 at v = 512, 2 at v = 256) against LAPACK's solve"""
    s = _solves(N, v)
    A, B = s["A"], s["B"]
    assert s["rcond"] > 0
    for X, Ak in ((s["X"], A), (s["XT"], A.T)):
        assert solve_ref.backward_error(Ak, X, B) <= ETA_TOL
        assert _rel_cols(X, np.linalg.solve(Ak, B)) <= 100 * EPS / s["rcond"]


@pytest.mark.parametrize("nb", [4, 32])
def test_solves_under_the_block_size_switch(nb, tmp_path):
    """CFLX_TRSM_NB caps the solves' diagonal block size too: at nb = 4 a v = 512 tile runs 128 blocks of 4 x 4 inverses
    and the TN kernel reads them with ldat = 4.  Each solve meets the backward-error bound and stays within the forward
    bound of the default block size's X; the condition estimates agree"""
    got = _child("switch_solves", {"CFLX_TRSM_NB": str(nb)}, tmp_path)
    for N, v in SWITCH_CASES:
        s = _solves(N, v)
        rcond = float(got[f"rcond_{N}_{v}"])
        assert abs(rcond - s["rcond"]) <= 1e-3 * s["rcond"], (N, v, rcond, s["rcond"])
        for key, Ak in (("X", s["A"]), ("XT", s["A"].T)):
            X = got[f"{key}_{N}_{v}"]
            assert solve_ref.backward_error(Ak, X, s["B"]) <= ETA_TOL, (N, v, key)
            assert _rel_cols(X, s[key]) <= 100 * EPS / s["rcond"], (N, v, key)
            assert not _same_bits(X, s[key]), "the switch changed nothing"


# ----------------------------------------------------------------------------------------------- refusals
def _raw_window(**over):
    """cflx_dbg_gemm_narrow_window on 16 x 16 buffers with one argument changed; returns (status, error text)"""
    a = dict(trans=0, M=8, N=8, K=8, A=np.zeros((16, 16)), a_rows=16, lda=16, a_row=0, a_col=0, B=np.zeros((16, 16)),
             b_rows=16, ldb=16, b_row=0, b_col=0, C=np.zeros((16, 16)), c_rows=16, ldc=16, c_row=0, c_col=0)
    a.update(over)
    D = np.zeros((16, 16))
    ptr = lambda x: x.ctypes.data if x is not None else None  # noqa: E731
    rc = cb.lib().cflx_dbg_gemm_narrow_window(a["trans"], a["M"], a["N"], a["K"], ptr(a["A"]), a["a_rows"], a["lda"],
                                              a["a_row"], a["a_col"], ptr(a["B"]), a["b_rows"], a["ldb"], a["b_row"],
                                              a["b_col"], ptr(a["C"]), a["c_rows"], a["ldc"], a["c_row"], a["c_col"],
                                              1.0, 0.0, 1, D.ctypes.data, None)
    return rc, cb.lib().cflx_last_error().decode()


@pytest.mark.parametrize("over,what", [
    (dict(M=0), "M < 1, N < 1 or K < 0"), (dict(N=0), "M < 1, N < 1 or K < 0"), (dict(K=-4), "M < 1, N < 1 or K < 0"),
    (dict(A=None), "A, B or C is null"), (dict(C=None), "A, B or C is null"),
    (dict(ldb=0), "a leading dimension < 1"), (dict(c_row=-1), "negative offset"),
    (dict(K=6), "K not a multiple of 4"), (dict(a_col=1), "odd lda or A column offset"),
    (dict(lda=15, a_rows=17), "odd lda or A column offset"),
    (dict(a_row=9), "A block outside its buffer"), (dict(a_col=10), "A block outside its buffer"),
    (dict(trans=1, M=12, a_col=6), "A block outside its buffer"), (dict(b_row=9), "B block outside its buffer"),
    (dict(b_col=9), "B block outside its buffer"), (dict(c_row=9), "C window outside its buffer"),
    (dict(c_col=9), "C window outside its buffer")])
def test_gemm_narrow_window_refusals(over, what):
    rc, msg = _raw_window(**over)
    assert rc == -1 and msg.startswith("cflx_dbg_gemm_narrow_window: refused, ") and what in msg, (rc, msg)


def test_gemm_narrow_window_takes_odd_k_transposed():
    assert _raw_window(trans=1, K=6)[0] == 0


def _raw_diag(**over):
    a = dict(tri=0, lower=0, v=32, nb=8, rows=40, ld=40, row0=0, col0=0, ldn=4)
    a.update(over)
    share = np.zeros((max(a["rows"], 1), max(a["ld"], 1)))
    R = np.zeros((max(a["v"], 1), max(a["ldn"], 1)))
    Y = np.zeros_like(R)
    rc = cb.lib().cflx_dbg_diag_solve(a["tri"], a["lower"], a["v"], a["nb"], share.ctypes.data, a["rows"], a["ld"],
                                      a["row0"], a["col0"], a["ldn"], R.ctypes.data, Y.ctypes.data, None)
    return rc, cb.lib().cflx_last_error().decode()


@pytest.mark.parametrize("over,what,status", [
    (dict(tri=5), "tri outside 0 .. 4", -1), (dict(tri=-1), "tri outside 0 .. 4", -1),
    (dict(lower=2), "lower not 0 or 1", -1),
    (dict(lower=1, tri=1), "tri not one the solves use", -1), (dict(lower=1, tri=4), "tri not one the solves use", -1),
    (dict(tri=2), "tri not one the solves use", -1),
    (dict(nb=12, v=36), "nb not 4, 8, 16, 32, 64 or 128", -4), (dict(nb=256, v=256), "nb not 4", -4),
    (dict(v=36), "v not a positive multiple of nb", -1), (dict(v=0), "v not a positive multiple of nb", -1),
    (dict(ldn=0), "ldn < 1", -1), (dict(row0=-8), "negative tile offset", -1),
    (dict(ld=41), "odd ld or col0", -1), (dict(col0=3), "odd ld or col0", -1),
    (dict(row0=9), "tile outside the share", -1), (dict(col0=10), "tile outside the share", -1)])
def test_diag_solve_refusals(over, what, status):
    rc, msg = _raw_diag(**over)
    assert rc == status and msg.startswith("cflx_dbg_diag_solve: refused, ") and what in msg, (rc, msg)
