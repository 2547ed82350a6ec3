"""GPU: the LU path kernel by kernel and end to end, against the extended-precision references and the error bounds of
oracle/hp_ref.py, at the launch windows and run-time switches the factorisation uses.

Constants: every tolerance is one of the hp_ref bounds (gamma_n = n u / (1 - n u), u = 2^-53), or bit identity:
  * gemm_tn_kernel:                 |D^ - (beta C + alpha A^T B)| <= gamma_{K+1} (|beta| |C| + |alpha| |A|^T |B|), and the
                                    exact product bit for bit on integer inputs (K max|a| max|b| < 2^53)
  * the int8 update (ozaki.cu):     bit for bit against oracle/ozaki_ref.py on the same window
  * the TRSMs (inverted blocks):    ||X^ U - B||_F <= gamma_{v+1} (1 + 4 kappa_max) || |X^| |U| ||_F (and L Y = R)
  * the panel kernels:              |P A - L^ U^| <= gamma_v |L^| |U^|, |l| <= 1
  * the whole factorisation:        ||P A - L^ U^||_F <= gamma_{n+1} (1 + 4 kappa_max) || |L^| |U^| ||_F
Two switches are read once per process (CFLX_TRSM_NB in lu.cu, CFLX_GEMM_TILE in gemm.cu): their cases run in a child
interpreter that writes its results to a temporary directory."""
import hashlib
import json
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import hp_ref as hp, layout, ozaki_ref, restate
from tests._harness import n_gpus, run_ranks
from tests.golden import make_lu_golden

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = np.nan


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint64),
                                                 np.ascontiguousarray(b).view(np.uint64))


def _child(fn, arg, env, tmp_path):
    """fn(arg) of this module in a fresh interpreter with env added (switches read once per process); returns what it
    wrote to tmp_path as JSON.  Under the NCCL loopback the child runs its grids on one device as the parent does."""
    out = os.path.join(str(tmp_path), f"{fn}.json")
    code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import _loopback; _loopback.install_if_preloaded(); "
            f"import json; from tests import test_gpu_lu_edges as t; "
            f"json.dump(t.{fn}({arg!r}), open({out!r}, 'w'))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=dict(os.environ, **env), cwd=ROOT, timeout=900,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    with open(out) as f:
        return json.load(f)


# ----------------------------------------------------------------------------------------------- gemm_tn_kernel
def _seed(name, kind):
    return sum(map(ord, name)) * 7 + len(kind)


def _rup2(x):
    return x + (x & 1)


def _window_cases():
    """(name, dict) of the windows the factorisation launches: the trailing update's two parts (odd M, ldc = Nl,
    col_lo > 0, B offset w), both TRSM sweeps, K tails that wrap the 4-stage ring, and a narrow N = 2."""
    cases = []
    for v in (64, 128, 256):
        Nl, fnpr = 5 * v, v
        M = 4 * v - 1                                          # n_act; odd as on a multi-row grid
        ldu = Nl - v                                           # the U panel of step 0: ncols columns
        cases.append((f"update_part0_v{v}", dict(M=M, N=v, K=v, ldat=_rup2(M), at_rows=v + 4, at_off=(0, 0),
                                                 ldb=ldu + 2, b_rows=v + 4, b_off=(0, 0), c_rows=5 * v, ldc=Nl,
                                                 c_off=(fnpr, v), alpha=-1.0, beta=1.0, in_place=True)))
        cases.append((f"update_part1_v{v}", dict(M=M, N=ldu - v, K=v, ldat=_rup2(M), at_rows=v + 4, at_off=(0, 0),
                                                 ldb=ldu + 2, b_rows=v + 4, b_off=(0, v), c_rows=5 * v, ldc=Nl,
                                                 c_off=(fnpr, 2 * v), alpha=-1.0, beta=1.0, in_place=True)))
    for v, nb in ((256, 128), (512, 128), (96, 32)):
        n = 3 * v + 10
        ld = _rup2(n) + 2
        cases.append((f"trsm_block_v{v}_nb{nb}", dict(M=nb, N=_rup2(n), K=nb, ldat=nb, at_rows=nb + 4, at_off=(0, 0),
                                                      ldb=ld, b_rows=v + 4, b_off=(nb, 0), c_rows=v, ldc=ld,
                                                      c_off=(nb, 0), alpha=1.0, beta=0.0, in_place=False)))
        j = 0
        cases.append((f"trsm_update_v{v}_nb{nb}", dict(M=v - (j + 1) * nb, N=_rup2(n), K=nb, ldat=v, at_rows=v,
                                                       at_off=(j * nb, (j + 1) * nb), ldb=ld, b_rows=v, b_off=(j * nb, 0),
                                                       c_rows=v, ldc=ld, c_off=((j + 1) * nb, 0), alpha=-1.0, beta=1.0,
                                                       in_place=True)))
    for K in (68, 72, 76, 260):                                # K % 16 in {4, 8, 12}, past one trip around the ring
        cases.append((f"ktail_K{K}", dict(M=199, N=130, K=K, ldat=202, at_rows=K + 4, at_off=(0, 0), ldb=134,
                                          b_rows=K + 4, b_off=(0, 2), c_rows=210, ldc=140, c_off=(5, 4), alpha=-1.0,
                                          beta=1.0, in_place=True)))
    cases.append(("narrow_M37_N2", dict(M=37, N=2, K=12, ldat=40, at_rows=16, at_off=(0, 0), ldb=4, b_rows=16,
                                        b_off=(0, 0), c_rows=40, ldc=6, c_off=(1, 2), alpha=-1.0, beta=1.0,
                                        in_place=True)))
    return cases


def _window_buffers(c, kind, seed):
    """whole buffers with the operands in the window and NaN in every entry the kernel must not use (C outside the
    window, AT / B rows >= K and outside their blocks, B columns >= N, C in the window when beta == 0).  Column M of AT
    (odd M) is read by the producer, which copies an even width; only row M of D depends on it and it is not stored, so
    it holds NaN too."""
    rng = np.random.default_rng(seed)
    M, N, K = c["M"], c["N"], c["K"]
    AT = np.full((c["at_rows"], c["ldat"]), NAN)
    B = np.full((c["b_rows"], c["ldb"]), NAN)
    C = np.full((c["c_rows"], c["ldc"]), NAN)
    if kind == "int":
        a = rng.integers(-8, 9, (K, M)).astype(np.float64)
        b = rng.integers(-8, 9, (K, N)).astype(np.float64)
        cc = rng.integers(-64, 65, (M, N)).astype(np.float64)
    else:                                                      # multipliers 1, 1e-3, 1e-7; U rows over 2^+-30
        a = rng.uniform(-1, 1, (K, M)) * rng.choice([1.0, 1e-3, 1e-7], size=(K, M))
        b = rng.standard_normal((K, N)) * np.exp2(rng.integers(-30, 31, (K, 1)).astype(np.float64))
        cc = rng.standard_normal((M, N)) * np.exp2(rng.integers(-30, 31, (1, N)).astype(np.float64))
    (ar, ac), (br, bc), (cr, ccol) = c["at_off"], c["b_off"], c["c_off"]
    AT[ar:ar + K, ac:ac + M] = a
    B[br:br + K, bc:bc + N] = b
    if c["beta"] != 0:
        C[cr:cr + M, ccol:ccol + N] = cc
    return AT, B, C, a, b, cc


def _run_window(c, AT, B, C):
    return cb.dbg.gemm_tn_window(AT, B, C, c["M"], c["N"], c["K"], c["alpha"], c["beta"], at_off=c["at_off"],
                                 b_off=c["b_off"], c_off=c["c_off"], in_place=c["in_place"])


def _check_window(name, c, kind, seed):
    AT, B, C, a, b, cc = _window_buffers(c, kind, seed)
    D, Cafter, _ = _run_window(c, AT, B, C)
    M, N = c["M"], c["N"]
    cr, ccol = c["c_off"]
    win = np.zeros(C.shape, dtype=bool)
    win[cr:cr + M, ccol:ccol + N] = True
    Dw = D[win].reshape(M, N)
    assert np.all(np.isfinite(Dw)), name                                   # no canary reached the window
    assert _same_bits(D[~win], C[~win]), name                              # nothing outside it was written
    if not c["in_place"]:
        assert _same_bits(Cafter, C), name                                 # C is only read
    if kind == "int":
        exact = c["alpha"] * (a.T.astype(np.int64) @ b.astype(np.int64)).astype(np.float64)
        if c["beta"] != 0:
            exact = exact + c["beta"] * cc
        assert np.array_equal(Dw, exact), (name, np.argwhere(Dw != exact)[:5])
    else:
        assert hp.gemm_ok(a, b, cc, c["alpha"], c["beta"], Dw), name
    return Dw


@pytest.mark.parametrize("name,c", _window_cases(), ids=[n for n, _ in _window_cases()])
@pytest.mark.parametrize("kind", ["int", "graded"])
def test_gemm_tn_at_the_factorisations_windows(name, c, kind):
    _check_window(name, c, kind, _seed(name, kind))


def test_gemm_tn_epilogue_rounds_once():
    """D = fma(alpha, acc, fl(beta c)): with an exact integer accumulator and alpha, beta that are not powers of two,
    every entry is the correctly rounded value of alpha * acc + fl(beta c) (a separate rounding of alpha * acc differs)"""
    rng = np.random.default_rng(5)
    M, N, K = 70, 66, 68
    a = rng.integers(-8, 9, (K, M)).astype(np.float64)
    b = rng.integers(-8, 9, (K, N)).astype(np.float64)
    C = rng.integers(-999, 1000, (M, N)).astype(np.float64)
    alpha, beta = 0.1, 0.3
    D, _ = cb.dbg.gemm_tn(a, b, C, alpha, beta)
    acc = a.T.astype(np.int64) @ b.astype(np.int64)
    t = beta * C
    want = np.array([[float(Fraction(alpha) * int(acc[i, j]) + Fraction(float(t[i, j]))) for j in range(N)]
                     for i in range(M)])
    assert np.array_equal(D, want), np.argwhere(D != want)[:5]
    assert not np.array_equal(want, alpha * acc + t)                     # the two roundings do differ on this input


def test_gemm_tn_c2_first_step_exact():
    """the first trailing update of the benchmark configuration (16128 x 16128 x 256, in place), on integer inputs whose
    product is exact, so no longdouble reference is needed"""
    rng = np.random.default_rng(16128)
    M = N = 16128
    K = 256
    a = rng.integers(-8, 9, (K, M)).astype(np.float64)
    b = rng.integers(-8, 9, (K, N)).astype(np.float64)
    C = rng.integers(-64, 65, (M, N)).astype(np.float64)
    D, _, _ = cb.dbg.gemm_tn_window(a, b, C, M, N, K, -1.0, 1.0, in_place=True)
    assert np.array_equal(D, C - a.T @ b)                      # integer BLAS product: exact (|sum| < 2^53)


def gemm_window_digests(_):
    """sha256 of the window result of every case (run in a child under CFLX_GEMM_TILE=64)"""
    out = {}
    for name, c in _window_cases():
        for kind in ("int", "graded"):
            AT, B, C, *_ = _window_buffers(c, kind, _seed(name, kind))
            out[f"{name}_{kind}"] = _digest(_run_window(c, AT, B, C)[0])
    return out


def test_gemm_tn_64_tile_is_bit_identical_to_the_128_tile(tmp_path):
    """both tiles run the same k order per element on the same 64 x 32 warp tiles"""
    want = gemm_window_digests(None)
    got = _child("gemm_window_digests", None, {"CFLX_GEMM_TILE": "64"}, tmp_path)
    assert got == want


# ----------------------------------------------------------------------------------------------- ozaki_gemm_kernel
@pytest.mark.parametrize("M,N,K,row0,col0,max_ctas", [(1023, 768, 128, 0, 128, 100), (768, 512, 256, 0, 256, 7),
                                                       (600, 384, 256, 256, 512, 0), (255, 130, 128, 128, 128, 3)])
def test_ozaki_gemm_at_the_factorisations_windows(M, N, K, row0, col0, max_ctas):
    """the LU's part-1 update (col0 = w, CTAs capped for the concurrent pivot search) and the Cholesky's tile update
    (row0 > 0): bit for bit against the restatement on the same window"""
    rng = np.random.default_rng(M + N + K + row0)
    AT = rng.uniform(-1, 1, (K, row0 + M)) * rng.choice([1.0, 1e-3, 1e-7], size=(K, row0 + M))
    B = rng.standard_normal((K, col0 + N)) * np.exp2(rng.integers(-30, 31, (1, col0 + N)).astype(np.float64))
    C = rng.standard_normal((M, N))
    r = cb.dbg.ozaki_gemm(AT, B, C, row0=row0, col0=col0, max_ctas=max_ctas)
    ref, _ = ozaki_ref.gemm(AT[:, row0:], B[:, col0:], C)
    assert np.array_equal(r["D"], ref), (np.abs(r["D"] - ref).max(), np.argwhere(r["D"] != ref)[:5])


# ----------------------------------------------------------------------------------------------- TRSM
TRSM_CASES = [(v, nb) for v in (96, 128, 384, 512) for nb in (4, 8, 16, 32, 64, 128) if v % nb == 0]


def _trsm_triangles(v, kind, rng):
    Lo = np.tril(rng.uniform(-1, 1, (v, v)), -1) * (2.0 / np.sqrt(v))
    U = np.triu(rng.uniform(-1, 1, (v, v))) * (2.0 / np.sqrt(v)) + np.diag(1.0 + rng.random(v))
    if kind == "graded":
        U = np.logspace(-6, 6, v)[:, None] * U
    return Lo, U


@pytest.mark.parametrize("v,nb", TRSM_CASES)
@pytest.mark.parametrize("kind", ["random", "graded"])
def test_trsm_kappa_bound_at_every_block_size(v, nb, kind):
    rng = np.random.default_rng(v * 13 + nb)
    Lo, U = _trsm_triangles(v, kind, rng)
    n = 2 * v + 7                                             # odd: the padding column is read and must stay there
    B = rng.standard_normal((n, v))
    R = rng.standard_normal((v, n))
    if kind == "graded":
        R = np.exp2(rng.integers(-20, 21, (v, 1)).astype(np.float64)) * R
    X, Y = cb.dbg.trsm(Lo + U, B, R, nb=nb, ld=_rup2(n) + 6)
    L = Lo + np.eye(v)
    assert hp.trsm_upper_ok(U, B, X, hp.diag_block_kappa(U, nb)), (v, nb)
    assert hp.trsm_lower_unit_ok(L, R, Y, hp.diag_block_kappa(L, nb)), (v, nb)
    X2, Y2 = cb.dbg.trsm(Lo + U, B, R, nb=nb)                 # the leading dimension does not change a bit
    assert _same_bits(X, X2) and _same_bits(Y, Y2)


def _exact_unit_lower(v, nb, n, rng):
    """integer unit-lower L (entries in {-1, 0, 1}, sparse) and integer R such that the blocked solve with inverted
    diagonal blocks is exact in float64; shown here with exact integer arithmetic: every inverse entry, product and
    partial sum of the sweep stays below 2^53 in magnitude (bounded by the products of absolute values)"""
    L = np.eye(v, dtype=np.int64)
    mask = rng.random((v, v)) < 1.5 / v
    L += np.tril(rng.integers(-1, 2, (v, v)) * mask, -1)
    R = rng.integers(-4, 5, (v, n)).astype(np.int64)
    lim = 2.0 ** 53
    Rw = R.copy()
    Y = np.zeros_like(R)
    for j in range(0, v, nb):
        Ljj = L[j:j + nb, j:j + nb]
        W = np.eye(nb, dtype=np.int64)                       # inv(L_jj) by substitution, as diag_inverse_kernel runs it
        for r in range(nb):
            W[r] = np.eye(nb, dtype=np.int64)[r] - Ljj[r, :r] @ W[:r]
            assert (np.abs(Ljj[r, :r]) @ np.abs(W[:r])).max(initial=0) < lim
        assert (np.abs(W).astype(np.float64) @ np.abs(Rw[j:j + nb]).astype(np.float64)).max() < lim
        Y[j:j + nb] = W @ Rw[j:j + nb]
        bound = np.abs(L[j + nb:, j:j + nb]).astype(np.float64) @ np.abs(Y[j:j + nb]).astype(np.float64)
        assert (bound + np.abs(Rw[j + nb:])).max(initial=0) < lim
        Rw[j + nb:] -= L[j + nb:, j:j + nb] @ Y[j:j + nb]
    assert np.array_equal(L @ Y, R)                            # the exact solution
    return L.astype(np.float64), R.astype(np.float64), Y.astype(np.float64)


@pytest.mark.parametrize("v,nb", TRSM_CASES)
def test_trsm_exact_on_integer_unit_lower(v, nb):
    rng = np.random.default_rng(v + 7 * nb)
    n = 66
    L, R, Y0 = _exact_unit_lower(v, nb, n, rng)
    U = np.triu(np.ones((v, v)))                               # the upper part only feeds the U inverses
    _, Y = cb.dbg.trsm(np.tril(L, -1) + U, R=R, nb=nb, ld=n + 4)
    assert np.array_equal(Y, Y0), np.argwhere(Y != Y0)[:5]


# ----------------------------------------------------------------------------------------------- panel kernels
PANEL_SHAPES = [(8, 4), (64, 8), (200, 16), (300, 32), (1024, 32), (4096, 64), (1024, 512), (300, 12), (1000, 48),
                (800, 96), (3000, 96)]


def _panel_input(kind, n, v, rng):
    if kind == "random":
        return rng.standard_normal((n, v))
    if kind == "ties":
        return rng.integers(0, 4, size=(n, v)).astype(np.float64)
    return np.exp2(rng.integers(-30, 31, (n, 1)).astype(np.float64)) * rng.standard_normal((n, v))


@pytest.mark.parametrize("n,v", PANEL_SHAPES)
@pytest.mark.parametrize("stack", ["1", "0"])
def test_panel_kernels_componentwise_bound(n, v, stack, monkeypatch):
    monkeypatch.setenv("CFLX_STACK_KERNEL", stack)              # read per workspace: per dbg.panel call
    rng = np.random.default_rng(n * 3 + v)
    for kind in ("random", "ties", "graded"):
        P = _panel_input(kind, n, v, rng)
        perm, A00, LU, _ = cb.dbg.panel(P)
        full = np.concatenate([perm, np.setdiff1d(np.arange(n), perm)])
        assert sorted(full) == list(range(n)), kind
        LUp = LU[full].copy()
        LUp[:v] = A00                                           # the pivot rows' L\U (the row-owner kernel keeps it there)
        assert hp.lu_componentwise_ok(P, LUp, full), (kind, n, v)
        assert np.abs(np.tril(LUp, -1)).max(initial=0) <= 1.0, (kind, n, v)


# ----------------------------------------------------------------------------------------------- whole factorisation
LU_SHAPES = [(240, 12), (960, 48), (1000, 80), (1536, 96), (1536, 384), (2048, 512), (2048, 256)]


def _nb(v):
    return next(nb for nb in (128, 64, 32, 16, 8, 4) if v % nb == 0)


def _lu_input(kind, M, rng):
    if kind == "k1e12":                                        # U diag(logspace) V^T, kappa_2 = 1e12
        Q1, _ = np.linalg.qr(rng.standard_normal((M, M)))
        Q2, _ = np.linalg.qr(rng.standard_normal((M, M)))
        return (Q1 * np.logspace(0, -12, M)) @ Q2.T
    if kind == "graded":                                       # rows graded by powers of two over 2^+-20
        return np.exp2(rng.integers(-20, 21, (M, 1)).astype(np.float64)) * rng.standard_normal((M, M))
    raise ValueError(kind)


def _factor_grid(N, v, grid=(1, 1, 1), A=None):
    """one factorisation on a grid: (global A, global L\\U, perm, launch count of rank 0, uses the int8 update)"""
    import ctypes

    from conflux_b200 import _lib
    Px, Py, Pz = grid
    locs = layout.scatter(A, v, Px, Py, Pz) if A is not None else None

    def body(comm):
        gv = cb.lu_params(N, N, v, Px, Py, Pz, comm)
        if locs is not None:
            gv.data[...] = locs[gv.rank]
        cnt = ctypes.c_int64()
        _lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(cnt), 1)
        C = np.zeros((gv.Ml, gv.Nl))
        perm = np.zeros(gv.M, dtype=np.int32)
        cb.LU_rep(gv, C, perm)
        _lib.lib().cflx_lu_launch_count(gv._h, ctypes.byref(cnt), 1)
        r = dict(A=gv.data.copy(), C=C, perm=perm, launches=cnt.value, oz=_lib.lib().cflx_lu_uses_ozaki(gv._h))
        gv.free_comms()
        return r

    rs = run_ranks(Px * Py * Pz, body)
    return (layout.assemble([r["A"] for r in rs], N, v, Px, Py, Pz), layout.assemble([r["C"] for r in rs], N, v, Px, Py, Pz),
            rs[0]["perm"], rs[0]["launches"], rs[0]["oz"])


@pytest.mark.parametrize("N,v", LU_SHAPES)
def test_factor_generator_input(N, v):
    A, LU, perm, _, _ = _factor_grid(N, v)
    o = restate.lu([A], N, v)
    assert np.array_equal(perm, o["perm"])
    assert hp.lu_normwise_ok(A, LU, perm, hp.lu_kappa_max(LU, _nb(v)))


@pytest.mark.parametrize("N,v", LU_SHAPES)
@pytest.mark.parametrize("kind", ["k1e12", "graded"])
def test_factor_hard_inputs_and_column_scaling(N, v, kind):
    """kappa = 1e12 and row-graded inputs meet the bound (a near-tie may resolve differently than in another rounding,
    so perm only has to be a permutation); and for D = diag(2^k) the factor of A D is (L, U D) bit for bit with the same
    perm: power-of-two column scaling commutes with every rounding and with the pivot choice"""
    rng = np.random.default_rng(N + v + len(kind))
    M = layout.dims(N, v, 1, 1, 1)["M"]
    A = _lu_input(kind, M, rng)
    _, LU, perm, _, _ = _factor_grid(N, v, A=A)
    assert sorted(perm) == list(range(M))
    assert hp.lu_normwise_ok(A, LU, perm, hp.lu_kappa_max(LU, _nb(v)))
    d = np.exp2(rng.integers(-10, 11, M).astype(np.float64))
    _, LUd, permd, _, _ = _factor_grid(N, v, A=A * d[None, :])
    assert np.array_equal(permd, perm)
    want = np.tril(LU, -1) + np.triu(LU) * d[None, :]
    assert _same_bits(LUd, want)


@pytest.mark.parametrize("update,kind,N,v", [(u,) + c for u in make_lu_golden.UPDATES for c in make_lu_golden.update_cases(u)])
def test_default_path_factor_bits_are_pinned(update, kind, N, v, golden_dir):
    """the factor, the permutation and the launch count of each trailing-update kind are those recorded in
    tests/golden/lu_factor_bits.json (the default FP64 update) and update_factor_bits.json (int8, TF32, TF32x3), by
    tests/golden/make_lu_golden.py"""
    want = make_lu_golden.golden(update, golden_dir)[f"{kind}_{N}_{v}"]
    assert make_lu_golden.factor_bits(kind, N, v, update) == want


# ----------------------------------------------------------------------------------------------- run-time switches
SWITCH_SHAPES = [(2048, 256), (1536, 128)]
GRIDS = [(1, 1, 1), (2, 2, 1), (1, 1, 2)]


def _needs(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")


def _kappa(LU, v, grid):
    return hp.lu_kappa_max(LU, _nb(v), upper=grid[0] > 1)


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("N,v", SWITCH_SHAPES)
@pytest.mark.parametrize("env", [{"CFLX_LOOKAHEAD": "0"}, {"CFLX_PANEL_CTAS": "8"}, {"CFLX_PANEL_CTAS": "132"},
                                 {"CFLX_STACK_KERNEL": "0"}, {"CFLX_LOOKAHEAD_MULTI": "0"}],
                         ids=lambda e: "-".join(f"{k}={x}" for k, x in e.items()))
def test_switch_is_bit_identical(N, v, grid, env, monkeypatch):
    """switches that change where or on how many SMs work runs, never an operation order: same factor, same perm, and
    (LOOKAHEAD off: the same launches on one stream) the same launch count"""
    _needs(grid)
    if "CFLX_LOOKAHEAD_MULTI" in env and grid == (1, 1, 1):
        pytest.skip("one rank: CFLX_LOOKAHEAD_MULTI does not apply")
    _, LU0, p0, n0, _ = _factor_grid(N, v, grid)
    for k, x in env.items():
        monkeypatch.setenv(k, x)
    _, LU1, p1, n1, _ = _factor_grid(N, v, grid)
    assert np.array_equal(p1, p0)
    assert _same_bits(LU1, LU0)
    assert n1 == n0


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("N,v", SWITCH_SHAPES)
@pytest.mark.parametrize("lookahead", ["1", "0"])
def test_ozaki_update_meets_the_bound(N, v, grid, lookahead, monkeypatch):
    _needs(grid)
    A, LU0, p0, _, oz0 = _factor_grid(N, v, grid)
    monkeypatch.setenv("CFLX_GEMM", "ozaki")
    monkeypatch.setenv("CFLX_LOOKAHEAD", lookahead)
    _, LU, perm, _, oz = _factor_grid(N, v, grid)
    whole = (v // grid[2]) % 128 == 0                         # the layer's contraction is whole 128-element chunks
    assert (oz0, oz) == (0, int(whole)), "CFLX_GEMM=ozaki did not select the int8 update where it applies"
    assert np.array_equal(perm, p0)
    assert hp.lu_normwise_ok(A, LU, perm, _kappa(LU, v, grid))


def test_ozaki_update_falls_back_where_the_layer_is_not_whole_chunks(monkeypatch):
    N, v = 1536, 96
    _, LU0, p0, n0, _ = _factor_grid(N, v)
    monkeypatch.setenv("CFLX_GEMM", "ozaki")
    _, LU, perm, n1, oz = _factor_grid(N, v)
    assert oz == 0
    assert np.array_equal(perm, p0) and _same_bits(LU, LU0) and n1 == n0


def factor_digests(cases):
    """[(N, v, grid)] -> sha256 of the factor, the perm, and launch counts (run in a child under a per-process switch)"""
    out = []
    for N, v, grid in cases:
        A, LU, perm, launches, _ = _factor_grid(N, v, tuple(grid))
        out.append(dict(factor=_digest(LU), perm=_digest(perm), launches=launches,
                        ok=hp.lu_normwise_ok(A, LU, perm, _kappa(LU, v, grid))))
    return out


def _grid_cases():
    return [(N, v, g) for N, v in SWITCH_SHAPES for g in GRIDS if n_gpus() >= g[0] * g[1] * g[2]]


def test_gemm_tile_64_is_bit_identical(tmp_path):
    cases = _grid_cases()
    want = factor_digests(cases)
    got = _child("factor_digests", cases, {"CFLX_GEMM_TILE": "64"}, tmp_path)
    assert got == want


@pytest.mark.parametrize("nb", [4, 32])
def test_trsm_block_size_switch(nb, tmp_path):
    """CFLX_TRSM_NB caps the diagonal block size: the factor meets the bound with the same perm, and every U solve issues
    2 (v / nb) - 1 launches instead of 2 (v / 128) - 1 (one process row, one layer: 2 Nt - 3 U solves, the column
    windows split around the look-ahead fork)"""
    cases = _grid_cases()
    want = factor_digests(cases)
    got = _child("factor_digests", cases, {"CFLX_TRSM_NB": str(nb)}, tmp_path)
    for (N, v, grid), w, g in zip(cases, want, got):
        assert g["ok"], (N, v, grid)
        assert g["perm"] == w["perm"], (N, v, grid)
        if tuple(grid) == (1, 1, 1):
            Nt = layout.dims(N, v, 1, 1, 1)["Nt"]
            assert g["launches"] - w["launches"] == (2 * Nt - 3) * 2 * (v // nb - v // _nb(v)), (N, v)
