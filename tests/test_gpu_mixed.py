"""GPU: the mixed-precision drivers cflx_lu_sv_mixed / cflx_chol_sv_mixed and their TF32 trailing update.
  * the kernel (tf32.cu) against oracle/mixed_ref.py: the split terms and exponents bit for bit, the product within the
    stated FP32-accumulation bound, for one and three terms, K tails, M / N tails, row0 / col0 windows and rows scaled
    by 2^+-300; three terms clearly more accurate than one;
  * factorisations with the TF32 update: cflx_*_validate within the stated bound and above FP64 level (the TF32 path
    ran), launch counts those of the FP64 path plus the splits;
  * the drivers on the generator inputs (the LU's + N I) on 1x1x1 and on multi-rank grids (run on one device under the
    NCCL loopback): iter in [1, itmax], backward errors at FP64 level and no worse than the FP64 factor + solve;
  * the fallback on kappa = 1e12 and indefinite inputs, bit-identical to the FP64 factor + solve;
  * the state rule: after a converged run every call that needs FP64 factors refuses by name, until a plain factor."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import conflux_b200 as cb
from conflux_b200._lib import ConfluxError, lib
from oracle import layout, mixed_ref
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2.0 ** -53


def _operands(K, Ma, Nb, seed, scaled=False):
    rng = np.random.default_rng(seed)
    AT = rng.uniform(-1, 1, (K, Ma)) * rng.choice([1.0, 1e-3, 1e-7], size=(K, Ma))
    B = rng.standard_normal((K, Nb)) * 6.0
    if scaled:
        AT *= np.exp2(rng.choice([-300.0, 0.0, 300.0], size=(1, Ma)))
        B *= np.exp2(rng.choice([-300.0, 300.0], size=(1, Nb)))
        AT[:, 3] = 0.0                                                  # a zero row of each operand
        B[:, 1] = 0.0
    return AT, B


def _check_kernel(terms, K, M, N, row0, col0, scaled=False):
    AT, B = _operands(K, row0 + M, col0 + N, 31 * K + M + N + terms, scaled)
    C = np.random.default_rng(K).standard_normal((M, N))
    if scaled:
        C *= np.ldexp(1.0, 300)
    r = cb.dbg.gemm_tf32(terms, AT, B, C, row0=row0, col0=col0)
    D, bound, (hA, lA, ea, hB, lB, eb) = mixed_ref.gemm(AT, B, C, terms, row0, col0)
    assert np.array_equal(r["ea"], ea) and np.array_equal(r["eb"], eb)
    assert np.array_equal(r["hiA"].view(np.uint32), hA.view(np.uint32))
    assert np.array_equal(r["hiB"].view(np.uint32), hB.view(np.uint32))
    if terms == 3:
        assert np.array_equal(r["loA"].view(np.uint32), lA.view(np.uint32))
        assert np.array_equal(r["loB"].view(np.uint32), lB.view(np.uint32))
    err = np.abs(r["D"] - D)
    assert np.all(err <= bound), (err / bound).max()
    return r["D"], C - AT[:, row0:].T @ B[:, col0:]


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("K", [4, 12, 64, 128, 256, 512])
def test_kernel_vs_oracle(terms, K):
    _check_kernel(terms, K, 200, 130, 3, 5)


@pytest.mark.parametrize("terms", [1, 3])
@pytest.mark.parametrize("M,N,row0,col0", [(128, 128, 0, 0), (37, 3, 0, 0), (300, 257, 64, 130), (129, 1, 7, 9),
                                           (1000, 514, 256, 0)])
def test_kernel_tails_and_windows(terms, M, N, row0, col0):
    _check_kernel(terms, 256, M, N, row0, col0)


@pytest.mark.parametrize("terms", [1, 3])
def test_kernel_exponent_range(terms):
    _check_kernel(terms, 64, 150, 70, 2, 4, scaled=True)


def test_three_terms_clearly_more_accurate():
    err = {}
    for terms in (1, 3):
        D, exact = _check_kernel(terms, 256, 512, 384, 0, 0)
        err[terms] = np.abs(D - exact).max()
    assert err[3] < err[1] / 100, err


# ---------------------------------------------------------------------------------------------- the drivers, one GPU
def _dominant(gv):
    """the library's generator + N I (layer 0 holds the input)"""
    if gv.pk != 0:
        return
    r = np.arange(gv.Ml)
    c = np.arange(gv.Nl)
    grow = ((r // gv.v) * gv.Px + gv.pi) * gv.v + r % gv.v
    gcol = ((c // gv.v) * gv.Py + gv.pj) * gv.v + c % gv.v
    hit = (grow[:, None] == gcol[None, :]) & (grow[:, None] < gv.N)
    gv.data[hit] += gv.N


def _launches(fn, h):
    n = ctypes.c_int64()
    cb.check(fn(h, ctypes.byref(n), 1), "launch_count")
    return n.value


def _berr(A, B, X):
    B, X = B.reshape(A.shape[0], -1), X.reshape(A.shape[0], -1)
    return np.abs(B - A @ X).max(axis=0) / (np.abs(A).sum(axis=1).max() * np.abs(X).max(axis=0))


LU_REFUSE = ["lu_solve", "lu_solve_trans", "lu_solve_local", "lu_rcond", "lu_refine", "lu_refine_x", "lu_svx", "lu_svxx",
             "lu_inverse", "lu_det", "lu_rbt_solve"]


def _lu_refusals(gv, B):
    calls = {
        "lu_solve": lambda: cb.lu_solve(gv, B),
        "lu_solve_trans": lambda: cb.lu_solve(gv, B, trans=True),
        "lu_solve_local": lambda: lib().cflx_lu_solve_local(gv._h, 0, 1, np.zeros((gv.Ml, gv.v)).ctypes.data, gv.v, None, 0),
        "lu_rcond": lambda: cb.lu_rcond(gv),
        "lu_refine": lambda: cb.lu_refine(gv, B, B),
        "lu_refine_x": lambda: cb.lu_refine_x(gv, B, B),
        "lu_svx": lambda: cb.lu_svx(gv, B),
        "lu_svxx": lambda: lib().cflx_lu_svxx(gv._h, 0, 1, B.ctypes.data, 1, np.empty(gv.M).ctypes.data, 1,
                                              ctypes.byref(ctypes.c_double()), None, None,
                                              np.empty(3).ctypes.data, None, None, ctypes.byref(ctypes.c_int())),
        "lu_inverse": lambda: lib().cflx_lu_inverse(gv._h, None, ctypes.byref(ctypes.c_int())),
        "lu_det": lambda: lib().cflx_lu_det(gv._h, 0, None, None, None, None, ctypes.byref(ctypes.c_int())),
        "lu_rbt_solve": lambda: cb.lu_rbt_solve(gv, B),
    }
    for name in LU_REFUSE:
        try:
            rc = calls[name]()
        except ConfluxError as e:
            msg = str(e)
        else:
            assert rc != 0, name
            msg = lib().cflx_last_error().decode()
        assert f"cflx_{name}:" in msg and "mixed-precision" in msg, (name, msg)


@pytest.mark.parametrize("prec", ["tf32", "tf32x3"])
def test_lu_sv_mixed_one_gpu(prec):
    N, v = 1024, 256
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    _dominant(gv)
    A = gv.data.copy()
    rng = np.random.default_rng(11)
    B = rng.standard_normal((N, 3))
    cb.LU_rep(gv)
    n64 = _launches(lib().cflx_lu_launch_count, gv._h)
    _, rel64 = cb.validate(gv)
    X64 = cb.lu_solve(gv, B)
    _launches(lib().cflx_lu_launch_count, gv._h)
    X, it, berr = cb.lu_sv_mixed(gv, B, prec=prec, itmax=10)
    nmix = _launches(lib().cflx_lu_launch_count, gv._h)
    assert 1 <= it <= 10, it
    assert np.all(berr <= np.sqrt(N) * EPS), berr
    assert np.all(_berr(A, B, X) <= np.sqrt(N) * EPS)
    assert np.all(berr <= np.sqrt(N) * np.maximum(_berr(A, B, X64), EPS))
    # the low-precision factors: within the bound of the update's precision, and above FP64 level
    _, rel = cb.validate(gv)
    lim = 2.0 ** -8 if prec == "tf32" else 2.0 ** -16
    print(f"\n[{prec}] iter {it}  berr {berr.max():.2e}  validate {rel:.2e} (FP64 {rel64:.2e})  launches {nmix} vs {n64}")
    assert 1e3 * max(rel64, EPS) < rel < lim, (rel, rel64)
    Nt = N // v
    assert n64 < nmix <= n64 + 3 * Nt                                  # the FP64 path's launches plus the splits
    _lu_refusals(gv, B[:, 0].copy())
    C = np.zeros((gv.Ml, gv.Nl))
    perm = np.zeros(gv.M, dtype=np.int32)
    cb.check(lib().cflx_lu_get_factors(gv._h, C.ctypes.data, perm.ctypes.data), "lu_get_factors")
    assert np.isfinite(C).all()
    cb.LU_rep(gv, upload=False)                                       # a plain factorisation restores the calls
    assert np.array_equal(cb.lu_solve(gv, B), X64)
    cb.lu_rcond(gv)
    gv.free_comms()
    comm.close()


CHOL_REFUSE = ["chol_solve", "chol_solve_local", "chol_rcond", "chol_refine", "chol_refine_x", "chol_svx", "chol_svxx",
               "chol_inverse", "chol_det", "chol_rbt_solve"]


def _chol_refusals(ch, B):
    h = ch._h
    Y = np.empty(ch.N)
    d = ctypes.byref(ctypes.c_double())
    i = ctypes.byref(ctypes.c_int())
    calls = {
        "chol_solve": lambda: lib().cflx_chol_solve(h, 1, B.ctypes.data, 1, Y.ctypes.data, 1),
        "chol_solve_local": lambda: lib().cflx_chol_solve_local(h, 1, np.zeros((ch.Ml, ch.v)).ctypes.data, ch.v, None, 0),
        "chol_rcond": lambda: lib().cflx_chol_rcond(h, d, None),
        "chol_refine": lambda: lib().cflx_chol_refine(h, 1, B.ctypes.data, 1, Y.ctypes.data, 1, None, None),
        "chol_refine_x": lambda: lib().cflx_chol_refine_x(h, 1, B.ctypes.data, 1, Y.ctypes.data, 1, None, None,
                                                          np.empty(3).ctypes.data, None, i),
        "chol_svx": lambda: lib().cflx_chol_svx(h, 1, B.ctypes.data, 1, Y.ctypes.data, 1, d, None, None, None, i),
        "chol_svxx": lambda: lib().cflx_chol_svxx(h, 1, B.ctypes.data, 1, Y.ctypes.data, 1, d, None, None,
                                                  np.empty(3).ctypes.data, None, None, i),
        "chol_inverse": lambda: lib().cflx_chol_inverse(h, None),
        "chol_det": lambda: lib().cflx_chol_det(h, 0, None, None, None),
        "chol_rbt_solve": lambda: lib().cflx_chol_rbt_solve(h, 1, B.ctypes.data, 1, Y.ctypes.data, 1, 0, None, None),
    }
    for name in CHOL_REFUSE:
        rc = calls[name]()
        msg = lib().cflx_last_error().decode()
        assert rc != 0 and f"cflx_{name}:" in msg and "mixed-precision" in msg, (name, rc, msg)


@pytest.mark.parametrize("prec", ["tf32", "tf32x3"])
def test_chol_sv_mixed_one_gpu(prec):
    N, v = 1024, 256
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky(N, v, (1, 1, 1), comm)
    A = np.tril(ch.data) + np.tril(ch.data, -1).T
    rng = np.random.default_rng(12)
    B = rng.standard_normal((N, 2))
    ch.parallelCholesky()
    n64 = _launches(lib().cflx_chol_launch_count, ch._h)
    _, rel64 = ch.validate()
    X64 = ch.solve(B)
    _launches(lib().cflx_chol_launch_count, ch._h)
    X, it, berr = ch.sv_mixed(B, prec=prec, itmax=10)
    nmix = _launches(lib().cflx_chol_launch_count, ch._h)
    assert 1 <= it <= 10, it
    assert np.all(berr <= np.sqrt(N) * EPS), berr
    assert np.all(_berr(A, B, X) <= np.sqrt(N) * EPS)
    assert np.all(berr <= np.sqrt(N) * np.maximum(_berr(A, B, X64), EPS))
    _, rel = ch.validate()
    lim = 2.0 ** -8 if prec == "tf32" else 2.0 ** -16
    print(f"\n[{prec}] iter {it}  berr {berr.max():.2e}  validate {rel:.2e} (FP64 {rel64:.2e})  launches {nmix} vs {n64}")
    assert 1e3 * max(rel64, EPS) < rel < lim, (rel, rel64)
    assert nmix == n64 + 2 * (N // v - 1)                              # the FP64 path's launches plus two splits a step
    _chol_refusals(ch, B[:, 0].copy())
    assert np.isfinite(ch.local_factor()).all()
    ch.parallelCholesky(upload=False)
    assert np.array_equal(ch.solve(B), X64)
    ch.finalize()
    comm.close()


def _ill(n, seed, spd):
    """kappa = 1e12 from prescribed singular values (eigenvalues when spd)"""
    rng = np.random.default_rng(seed)
    Q1, _ = np.linalg.qr(rng.standard_normal((n, n)))
    Q2 = Q1 if spd else np.linalg.qr(rng.standard_normal((n, n)))[0]
    A = Q1 @ np.diag(np.logspace(0, -12, n)) @ Q2.T
    return (A + A.T) / 2 if spd else A


@pytest.mark.parametrize("prec", ["tf32", "tf32x3"])
def test_lu_fallback_is_the_fp64_solve(prec):
    N, v = 512, 128
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    gv.data[...] = _ill(N, 3, False)
    B = np.random.default_rng(13).standard_normal((N, 2))
    X, it, berr = cb.lu_sv_mixed(gv, B, prec=prec, itmax=5)
    assert it in (mixed_ref.NO_CONVERGENCE, mixed_ref.LOW_PREC_FAILED), it
    X2 = cb.lu_solve(gv, B)                                            # the handle holds FP64 factors again
    cb.LU_rep(gv)
    assert np.array_equal(X, cb.lu_solve(gv, B)) and np.array_equal(X, X2)
    gv.free_comms()
    comm.close()


@pytest.mark.parametrize("prec", ["tf32", "tf32x3"])
def test_chol_fallback_is_the_fp64_solve(prec):
    N, v = 512, 128
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky(N, v, (1, 1, 1), comm)
    ch.data[...] = _ill(N, 4, True)
    B = np.random.default_rng(14).standard_normal((N, 2))
    X, it, berr = ch.sv_mixed(B, prec=prec, itmax=5)
    assert it in (mixed_ref.NO_CONVERGENCE, mixed_ref.LOW_PREC_FAILED), it
    X2 = ch.solve(B)
    ch.parallelCholesky()
    assert np.array_equal(X, ch.solve(B)) and np.array_equal(X, X2)
    # indefinite: the low-precision factorisation fails, and the FP64 one refuses like cflx_chol_factor
    ch.data[...] = np.diag(np.r_[np.ones(N - 1), -1.0])
    with pytest.raises(ConfluxError, match="not positive definite"):
        ch.sv_mixed(B, prec=prec)
    ch.finalize()
    comm.close()


def test_argument_refusals():
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(256, 256, 128, 1, 1, 1, comm)
    B = np.ones(256)
    X = np.empty(256)
    it = ctypes.c_int()
    assert lib().cflx_lu_sv_mixed(gv._h, 1, 1, B.ctypes.data, 1, X.ctypes.data, 1, 0, ctypes.byref(it), None, None) != 0
    assert "cflx_lu_sv_mixed" in lib().cflx_last_error().decode()         # before any upload
    cb.check(lib().cflx_lu_set_local(gv._h, np.ascontiguousarray(gv.data).ctypes.data), "set_local")
    for prec, rhs in ((2, 1), (1, 0)):
        assert lib().cflx_lu_sv_mixed(gv._h, prec, rhs, B.ctypes.data, 1, X.ctypes.data, 1, 0, ctypes.byref(it), None,
                                      None) != 0
        assert "cflx_lu_sv_mixed" in lib().cflx_last_error().decode()
    with pytest.raises(ValueError):
        cb.lu_sv_mixed(gv, B, prec="bf16")
    gv.free_comms()
    comm.close()


# ---------------------------------------------------------------------------------------------- multi-rank grids
GRIDS = [(2, 1, 1), (1, 2, 1), (2, 2, 1), (2, 2, 2)]   # the LU path needs Px == Py: the Cholesky alone on the others


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_sv_mixed(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1024, 128
    B = np.random.default_rng(15).standard_normal((N, 2))

    lu = grid[0] == grid[1]

    def body(comm):
        out = {}
        if lu:
            gv = cb.lu_params(N, N, v, *grid, comm)
            _dominant(gv)
            out["X"], out["it"], out["berr"] = cb.lu_sv_mixed(gv, B, prec="tf32x3", itmax=10)
            cb.LU_rep(gv, upload=False)
            out["X64"], out["share"] = cb.lu_solve(gv, B), gv.data.copy()
            gv.free_comms()
        ch = cb.cholesky(N, v, grid, comm)
        out["Y"], out["cit"], out["cberr"] = ch.sv_mixed(B, prec="tf32", itmax=10)
        ch.parallelCholesky(upload=False)
        out["Y64"], out["cdata"] = ch.solve(B), ch.data.copy()
        ch.finalize()
        return out

    rs = run_ranks(P, body)
    from oracle import chol_ref
    S = chol_ref.lower_sym(chol_ref.assemble([r["cdata"] for r in rs], N, v, *grid))
    cases = [(S, "Y", "Y64", "cberr", "cit")]
    if lu:
        cases.append((layout.assemble([r["share"] for r in rs], N, v, *grid), "X", "X64", "berr", "it"))
    r = rs[0]
    for M, x, x64, be, it in cases:
        assert all(np.array_equal(q[x], r[x]) and q[it] == r[it] for q in rs)
        assert 1 <= r[it] <= 10, r[it]
        X, X64, berr = r[x], r[x64], r[be]
        assert np.all(berr <= np.sqrt(N) * EPS), berr
        assert np.all(_berr(M, B, X) <= np.sqrt(N) * EPS)
        assert np.all(berr <= np.sqrt(N) * np.maximum(_berr(M, B, X64), EPS))


def test_multi_rank_grids_on_one_device(tmp_path):
    """the grid cases above in a child pytest under the NCCL loopback, every rank a thread on device 0"""
    from tests import _loopback
    xml = tmp_path / "junit.xml"
    preload = " ".join(p for p in (_loopback.build(), os.environ.get("LD_PRELOAD")) if p)
    env = dict(os.environ, LD_PRELOAD=preload)
    flags = ["-s"] if sys.flags.no_user_site else []
    cmd = [sys.executable] + flags + ["-m", "pytest", "-p", "tests._loopback", "-p", "no:cacheprovider", "-q", "-rA",
                                      f"--junitxml={xml}", "tests/test_gpu_mixed.py::test_multi_gpu_sv_mixed"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-4000:]
    import xml.etree.ElementTree as ET
    cases = [[e.tag for e in c] for c in ET.parse(xml).iter("testcase")]
    assert len(cases) == len(GRIDS) and not any(t for t in cases), cases
