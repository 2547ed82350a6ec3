"""GPU: cflx_lu_det and cflx_chol_det (the determinant from the factors left on the device, as an exact-range pair).

  * the product kernel (cflx_dbg_det) equals oracle/det_ref.py bit for bit: mantissa, exponent, parity, first zero and
    the non-finite flag, on lengths around the CTA's 256 threads, extreme, subnormal, negative, zero and non-finite
    entries, and in the square and divisor modes;
  * on the device's own factors (cflx_lu_get_factors / cflx_chol_get_local) the results equal the restatement's bit for
    bit, log|det| within 4 ulp of it, and numpy's slogdet of the input within (kappa + |log det|) n u; where a plain
    product of the diagonal overflows, the pair is finite and right;
  * unscaled = 1 gives det of the input before equilibration, unscaled = 0 det of the scaled matrix, the same bits with
    equed = 'N';
  * an exactly zero pivot gives info = k (cflx_lu_inverse's), sign 0 and -inf;
  * two calls give the same bits; the factors, the permutation, the launch count and a later solve do not change; the
    state and argument rules are the solves';
  * on several GPUs every rank gets the same bits (skipped on fewer GPUs)."""
import ctypes
import math

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, det_ref, hp_ref, layout
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


def _bits(x):
    return np.float64(x).tobytes()


def _same_as_ref(dev, ref):
    assert _bits(dev["mantissa"]) == _bits(ref["mant"])
    assert (dev["exponent"], dev["neg"], dev["first_zero"], dev["nonfinite"]) == (ref["exp"], ref["neg"],
                                                                                   ref["first_zero"], ref["nonfinite"])


def _ulps(a, b, n):
    """|a - b| <= n ulp of the larger of the terms log(mant) and exp ln 2 that make up log|det|"""
    return abs(a - b) <= n * np.spacing(max(abs(a), abs(b), 1.0))


def _tol(A, logdet):
    """kappa n u for the factors, plus n u |log det| for the rounding of a sum of n logarithms"""
    return (np.linalg.cond(A, 1) + abs(logdet)) * A.shape[0] * U


# ----------------------------------------------------------------------------------------------- the product kernel
def _kernel_cases():
    rng = np.random.default_rng(7)
    for n in (1, 255, 256, 257, 16384):
        yield f"normal{n}", rng.standard_normal(n) * np.exp2(rng.integers(-40, 40, n)), None, None, False
    n = 1000
    yield "pow1000", np.exp2(rng.choice([-1000.0, 1000.0], n)) * rng.uniform(0.5, 2, n), None, None, False
    yield "subnormal", rng.choice([5e-324, 2.5e-310, -1e-315, 3.0, -7.0], n), None, None, False
    yield "negative", -rng.uniform(0.1, 10, 257), None, None, False
    for pos in (0, n // 2, n - 1):
        d = rng.standard_normal(n)
        d[pos] = 0.0
        yield f"zero{pos}", d, None, None, False
    d = rng.standard_normal(n)
    d[100], d[600] = np.inf, 0.0
    yield "inf_first", d, None, None, False
    d = rng.standard_normal(n)
    d[100], d[600] = 0.0, np.nan
    yield "zero_first", d, None, None, False
    d = rng.standard_normal(n)
    d[999] = -np.inf
    yield "neg_inf", d, None, None, False
    d = rng.standard_normal(16384) * 40
    s1, s2 = rng.uniform(1e-3, 1e3, 16384), np.exp2(rng.integers(-900, 900, 16384).astype(float))
    yield "square", d, None, None, True
    yield "div1", d, s1, None, False
    yield "div2", d, s1, s2, False
    yield "square_div1", d, s1, None, True
    yield "square_div2", d, -s1, s2, True
    s3 = s1.copy()
    s3[5] = 0.0
    yield "zero_divisor", d, s3, None, False
    s3[5] = 2.0 ** -1070
    yield "subnormal_divisor", d, s3, s2, False


@pytest.mark.parametrize("case", list(_kernel_cases()), ids=lambda c: c[0])
def test_kernel_matches_restatement(case):
    _, d, s1, s2, square = case
    _same_as_ref(cb.dbg.det(d, s1, s2, square), det_ref.product(d, s1, s2, square))


# ----------------------------------------------------------------------------------------------- LU
def _factors(gv):
    C, perm = np.zeros((gv.Ml, gv.Nl)), np.zeros(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "get_factors")
    return C, perm


def _check_lu(o, ref):
    assert _bits(o["mantissa"]) == _bits(ref["mantissa"]) and o["exponent"] == ref["exponent"]
    assert o["sign"] == ref["sign"] and o["info"] == ref["info"]
    assert _ulps(o["logabsdet"], ref["logabsdet"], 4)


@pytest.mark.parametrize("N,v", [(16, 4), (100, 16), (1024, 128), (4096, 256)])
@pytest.mark.parametrize("gen", ["normal", "default"])
def test_lu_det(N, v, gen):
    if gen == "default" and N != 4096:
        pytest.skip("the default generator is checked where its determinant overflows")
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    M = gv.M
    if gen == "normal":
        gv.data[...] = np.random.default_rng(N + v).standard_normal((M, M))
    A = gv.data.copy()                                               # 1x1x1: the share is the matrix
    cb.LU_rep(gv)
    o = cb.lu_det(gv)
    C, perm = _factors(gv)
    _check_lu(o, det_ref.lu_det([C], perm, N, v))
    s_np, l_np = np.linalg.slogdet(A)
    assert o["sign"] == s_np and o["info"] == 0
    assert abs(o["logabsdet"] - l_np) <= _tol(A, l_np)
    assert 0.5 <= o["mantissa"] < 1.0
    if gen == "default":
        with np.errstate(over="ignore"):
            assert not np.isfinite(np.prod(np.diag(C)))              # the plain product overflows
        assert o["exponent"] > 1024
        assert abs(math.log(o["mantissa"]) + o["exponent"] * math.log(2) - l_np) <= 1e-9 * abs(l_np)
    gv.free_comms()
    comm.close()


def _scaled(n, seed, kind):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    if kind == "plain":
        return A
    s, t = np.logspace(0, 12, n), np.logspace(0, 12, n)
    rng.shuffle(s)
    rng.shuffle(t)
    return A * s[:, None] * t[None, :]


def _host_scaled(A, e):
    r = e["r"] if e["equed"] in "RB" else np.ones(len(A))
    c = e["c"] if e["equed"] in "CB" else np.ones(len(A))
    return (c[None, :] * r[:, None]) * A, r, c


@pytest.mark.parametrize("kind", ["both", "plain"])
def test_lu_unscaled(kind):
    N, v = 100, 16
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    A = _scaled(gv.M, 3, kind)
    gv.data[...] = A
    e = cb.lu_equilibrate(gv)
    assert e["equed"] == ("B" if kind == "both" else "N")
    cb.LU_rep(gv, upload=False)
    o0, o1 = cb.lu_det(gv), cb.lu_det(gv, unscaled=True)
    As, r, c = _host_scaled(A, e)
    s_s, l_s = np.linalg.slogdet(As)
    tol = _tol(As, l_s)
    assert o0["sign"] == s_s and abs(o0["logabsdet"] - l_s) <= tol
    s_a, l_a = np.linalg.slogdet(A)
    assert o1["sign"] == s_a
    assert abs(o1["logabsdet"] - l_a) <= tol + 8 * gv.M * U * (abs(l_a) + abs(l_s))
    C, perm = _factors(gv)
    ref = det_ref.lu_det([C], perm, N, v, r=r if e["equed"] in "RB" else None, c=c if e["equed"] in "CB" else None)
    _check_lu(o1, ref)
    if kind == "plain":
        assert o0 == o1                                              # equed = 'N': the same bits
    gv.free_comms()
    comm.close()


def _launches(fn, h):
    n = ctypes.c_int64()
    cb.check(fn(h, ctypes.byref(n), 1), "launch_count")
    return n.value


def test_lu_zero_pivot_state_rules_and_side_effects():
    n, v = 64, 16
    rng = np.random.default_rng(12)
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_det(gv)                                                # no factorisation yet
    A = np.triu(rng.integers(1, 9, (n, n)).astype(float)) + np.diag(np.full(n, 50.0))
    A[20, 20] = 0.0                                                  # partial pivoting keeps every row: U(21, 21) = 0
    gv.data[...] = A
    cb.LU_rep(gv)
    o = cb.lu_det(gv)
    assert (o["info"], o["sign"], o["logabsdet"], o["mantissa"], o["exponent"]) == (21, 0.0, -math.inf, 0.0, 0)
    assert cb.lu_inverse(gv)[1] == o["info"]
    h = ctypes.c_double()
    assert cb.lib().cflx_lu_det(gv._h, 2, None, None, None, None, ctypes.byref(ctypes.c_int())) == -1
    assert cb.lib().cflx_lu_det(gv._h, 0, ctypes.byref(h), None, None, None, None) == -1      # NULL info_out
    info = ctypes.c_int()
    assert cb.lib().cflx_lu_det(gv._h, 0, None, None, None, None, ctypes.byref(info)) == 0 and info.value == 21
    a = np.ascontiguousarray(gv.data)
    cb.check(cb.lib().cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    with pytest.raises(cb.ConfluxError, match="status -5"):
        cb.lu_det(gv)                                                # new input, not factored yet
    gv.free_comms()

    N, v = 2048, 256
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    cb.LU_rep(gv)
    o1 = cb.lu_det(gv)                                               # cold: prepares the solve cache
    C0, perm0 = _factors(gv)
    B = rng.standard_normal((gv.M, 3))
    x0 = cb.lu_solve(gv, B)
    _launches(cb.lib().cflx_lu_launch_count, gv._h)
    o2 = cb.lu_det(gv)
    assert o1 == o2                                                  # two calls, cold and warm: the same bits
    assert _launches(cb.lib().cflx_lu_launch_count, gv._h) == 0
    assert np.array_equal(cb.lu_solve(gv, B), x0)
    C1, perm1 = _factors(gv)
    assert np.array_equal(C1, C0) and np.array_equal(perm1, perm0)
    gv.free_comms()
    comm.close()


# ----------------------------------------------------------------------------------------------- Cholesky
@pytest.mark.parametrize("N,v", [(16, 4), (100, 16), (1024, 128), (4096, 256)])
def test_chol_det(N, v):
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    Np = ch.N
    if N == 4096:                                                    # the library's generator: det overflows
        S = chol_ref.lower_sym(chol_ref.assemble([ch.data], N, v, 1, 1, 1))
    else:
        S = hp_ref.random_spd(Np, 1e3, np.random.default_rng(N + v))
        ch.data[...] = S
    ch.parallelCholesky()
    o = ch.det()
    L = ch.local_factor()
    ref = det_ref.chol_det([L], N, v)
    assert _bits(o["mantissa"]) == _bits(ref["mantissa"]) and o["exponent"] == ref["exponent"]
    assert _ulps(o["logdet"], ref["logabsdet"], 4)
    ld = 2 * math.fsum(np.log(np.diag(L)))
    assert abs(o["logdet"] - ld) <= 4 * Np * U * max(1.0, abs(ld))
    s_np, l_np = np.linalg.slogdet(S)
    assert s_np == 1.0 and abs(o["logdet"] - l_np) <= _tol(S, l_np)
    if N == 4096:
        with np.errstate(over="ignore"):
            assert not np.isfinite(np.prod(np.diag(L)) ** 2)
        assert o["exponent"] > 1024
    ch.finalize()
    comm.close()


def _spd(n, kind, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    A = G @ G.T / n + np.eye(n)
    if kind == "scaled":
        s = np.logspace(0, 6, n)
        rng.shuffle(s)
        A = A * s[:, None] * s[None, :]
    return A


@pytest.mark.parametrize("kind", ["scaled", "plain"])
def test_chol_unscaled(kind):
    N, v = 100, 16
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    A = _spd(ch.N, kind, 5)
    ch.data[...] = chol_solve_ref.scatter(A, ch.N, v, 1, 1, 1, upper=np.nan, pad=np.nan, layers=np.nan)[0]
    e = ch.equilibrate()
    assert e["equed"] == ("Y" if kind == "scaled" else "N")
    ch.parallelCholesky(upload=False)
    o0, o1 = ch.det(), ch.det(unscaled=True)
    s = e["s"] if e["equed"] == "Y" else np.ones(ch.N)
    As = (s[None, :] * s[:, None]) * A
    l_s, l_a = np.linalg.slogdet(As)[1], np.linalg.slogdet(A)[1]
    tol = _tol(As, l_s)
    assert abs(o0["logdet"] - l_s) <= tol
    assert abs(o1["logdet"] - l_a) <= tol + 8 * ch.N * U * (abs(l_a) + abs(l_s))
    ref = det_ref.chol_det([ch.local_factor()], N, v, s=e["s"] if e["equed"] == "Y" else None)
    assert _bits(o1["mantissa"]) == _bits(ref["mantissa"]) and o1["exponent"] == ref["exponent"]
    if kind == "plain":
        assert o0 == o1
    ch.finalize()
    comm.close()


def test_chol_state_rules_and_side_effects():
    N, v = 1024, 128
    rng = np.random.default_rng(1)
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.det()                                                     # no factorisation yet
    S = hp_ref.random_spd(N, 1e2, rng)
    ch.data[...] = S
    ch.parallelCholesky()
    L0 = ch.local_factor()
    B = rng.standard_normal((N, 3))
    x0 = ch.solve(B)
    n0 = _launches(cb.lib().cflx_chol_launch_count, ch._h)
    o1, o2 = ch.det(), ch.det()
    assert o1 == o2 and n0 > 0
    assert _launches(cb.lib().cflx_chol_launch_count, ch._h) == 0
    assert np.array_equal(ch.solve(B), x0) and np.array_equal(ch.local_factor(), L0)
    assert cb.lib().cflx_chol_det(ch._h, 2, None, None, None) == -1
    bad = S.copy()
    bad[N // 2, N // 2] = -1.0
    ch.data = bad
    with pytest.raises(cb.ConfluxError, match="positive definite"):
        ch.parallelCholesky()
    with pytest.raises(cb.ConfluxError, match="status -5"):
        ch.det()                                                     # the factorisation failed
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- multi-GPU
@pytest.mark.parametrize("grid", [(1, 1, 2), (2, 2, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_lu_det(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1024, 64
    M = layout.dims(N, v, *grid)["M"]
    A = np.random.default_rng(P).standard_normal((M, M))
    locs = layout.scatter(A, v, *grid)

    def body(comm):
        gv = cb.lu_params(N, N, v, *grid, comm)
        gv.data[...] = locs[gv.rank]
        cb.LU_rep(gv)
        o = cb.lu_det(gv)
        C, perm = _factors(gv)
        gv.free_comms()
        return o, C, perm

    rs = run_ranks(P, body)
    assert all(o == rs[0][0] for o, _, _ in rs)                      # every rank: the same bits
    _check_lu(rs[0][0], det_ref.lu_det([C for _, C, _ in rs], rs[0][2], N, v, *grid))
    s_np, l_np = np.linalg.slogdet(A)
    assert rs[0][0]["sign"] == s_np and abs(rs[0][0]["logabsdet"] - l_np) <= _tol(A, l_np)


@pytest.mark.parametrize("grid", [(1, 1, 2), (2, 2, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_chol_det(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1000, 48
    Np = chol_ref.dims(N, v, *grid)["N"]
    S = hp_ref.random_spd(Np, 1e2, np.random.default_rng(P))
    locs = chol_solve_ref.scatter(S, N, v, *grid)

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        res = ch.det(), ch.local_factor()
        ch.finalize()
        return res

    rs = run_ranks(P, body)
    assert all(o == rs[0][0] for o, _ in rs)
    ref = det_ref.chol_det([L for _, L in rs], N, v, *grid)
    assert _bits(rs[0][0]["mantissa"]) == _bits(ref["mantissa"]) and rs[0][0]["exponent"] == ref["exponent"]
