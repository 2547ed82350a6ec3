"""GPU: the distributed refinement and expert drivers, cflx_lu_refine_local, _refine_x_local, _svx_local, _svxx_local
and their Cholesky counterparts (B and X distributed like A, blocks of refine_block_cols columns through the replicated
cores).  For every block, X's bits and the per-column outputs equal the replicated driver's on those columns alone, and
rcond, rpvgrw and equed equal its bits (oracle/refine_local_ref.py states the block rule); info merges to the first
global column; host and device shares, in-place svx and NULL B off layer 0 give the same bits; the layers agree; nothing
else changes; and the argument and state rules hold, on one GPU and on the grids of the NCCL loopback.

Tolerance: ||B - A X||_F / (||A||_F ||X||_F + ||B||_F) <= 1e-13, the solve tests' bound."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, hp_ref, layout, solve_ref
from oracle import refine_local_ref as rl
from tests import _loopback
from tests._harness import n_gpus, run_ranks

pytestmark = pytest.mark.gpu
ETA_TOL = 1e-13
SENTINEL = -7777.0
ERR_ARG, ERR_STATE = -1, -5
OPS = ("refine", "refine_x", "svx", "svxx")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ptr(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _launches(fn, h):
    n = ctypes.c_int64()
    cb.check(fn(h, ctypes.byref(n), 1), "launch_count")
    return n.value


# ----------------------------------------------------------------------------------------------- the drivers, uniformly
def _norm(op, r):
    """(X, per-column outputs, matrix-level outputs, info) of any driver's Python result"""
    if op == "refine":
        X, fe, be = r
        return X, dict(ferr=fe, berr=be), {}, 0
    X, d = r
    cols = {k: d.get(k) for k in (("ferr", "berr") if op == "svx" else ("berr", "err_norm", "err_comp"))}
    mat = {k: d[k] for k in ("rcond", "rpvgrw", "equed") if k in d}
    return X, cols, mat, d["info"]


def _local(kind, h, op, B, X0, nrhs, trans=False, out=None):
    """the distributed driver on this rank's shares (X0: the solution on entry of refine / refine_x; out: svx's X)"""
    if kind == "lu":
        t = dict(trans=trans)
        r = {"refine": lambda: cb.lu_refine_local(h, B, X0, nrhs, **t),
             "refine_x": lambda: cb.lu_refine_x_local(h, B, X0, nrhs, **t),
             "svx": lambda: cb.lu_svx_local(h, B, nrhs, out=out, **t),
             "svxx": lambda: cb.lu_svxx_local(h, B, nrhs, out=out, **t)}[op]()
    else:
        r = {"refine": lambda: h.refine_local(B, X0, nrhs), "refine_x": lambda: h.refine_x_local(B, X0, nrhs),
             "svx": lambda: h.svx_local(B, nrhs, out=out), "svxx": lambda: h.svxx_local(B, nrhs, out=out)}[op]()
    return _norm(op, r)


def _replicated(kind, h, op, B, X0, trans=False):
    """the replicated driver on the columns B (and X0) alone"""
    if kind == "lu":
        r = {"refine": lambda: cb.lu_refine(h, B, X0, trans=trans), "refine_x": lambda: cb.lu_refine_x(h, B, X0, trans=trans),
             "svx": lambda: cb.lu_svx(h, B, trans=trans), "svxx": lambda: cb.lu_svxx(h, B, trans=trans)}[op]()
    else:
        r = {"refine": lambda: h.refine(B, X0), "refine_x": lambda: h.refine_x(B, X0), "svx": lambda: h.svx(B),
             "svxx": lambda: h.svxx(B)}[op]()
    return _norm(op, r)


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, str):
        return a == b
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _rank_body(kind, h, ops, trans, G, X0, B_share, X0_share, X_other, nrhs):
    """every driver of `ops` distributed (B_share, X0_share; X_other: the X share of a layer pk != 0, sentinel-filled)
    and replicated block by block on this rank"""
    out = {}
    for op in ops:
        xin = op.startswith("refine")
        Xs = (X0_share.copy() if X0_share is not None else X_other.copy()) if xin else None
        res = _local(kind, h, op, B_share, Xs, nrhs, trans, out=None if xin or X_other is None else X_other.copy())
        reps = [_replicated(kind, h, op, np.ascontiguousarray(G[:, c0:c0 + w]),
                            np.ascontiguousarray(X0[:, c0:c0 + w]), trans) for c0, w in rl.blocks(nrhs, h.v)]
        out[op] = res, reps
    return out


def _check(kind, op, res, reps, X, M, nrhs, v):
    """X: the collected M x nrhs result of the distributed call res; reps: the replicated driver block by block"""
    _, cols, mat, info = res
    infos = []
    for (c0, w), (Xb, cb_, mb, ib) in zip(rl.blocks(nrhs, v), reps):
        assert np.array_equal(X[:, c0:c0 + w], Xb), (op, c0)
        for name, val in cb_.items():
            assert _same(None if cols[name] is None else cols[name][c0:c0 + w], val), (op, name, c0)
        for name, val in mb.items():
            assert _same(mat[name], val), (op, name)                    # the matrix-level outputs: the same bits
        infos.append(((c0, w), ib))
    want = reps[0][3] if op == "svx" else rl.merge_info(infos, M)
    assert info == want, (op, info, want)
    return info


# ----------------------------------------------------------------------------------------------- handles
def _lu(N, v, A, grid=(1, 1, 1), comm=None, equilibrate=False):
    comm = comm or cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(N, N, v, *grid, comm)
    gv.data[...] = A
    if equilibrate:
        e = cb.lu_equilibrate(gv)
        assert e["equed"] == "B" and e["info"] == 0
    cb.LU_rep(gv, upload=not equilibrate)
    return gv, comm


def _chol(N, v, S_local, grid=(1, 1, 1), comm=None, equilibrate=False):
    comm = comm or cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, grid, comm)
    ch.data[...] = S_local
    if equilibrate:
        e = ch.equilibrate()
        assert e["equed"] == "Y" and e["info"] == 0
    ch.parallelCholesky(upload=not equilibrate)
    return ch, comm


def _badly_scaled(M, rng, sym=False):
    d = np.logspace(-3, 3, M)
    rng.shuffle(d)
    if sym:
        S = hp_ref.random_spd(M, 1e2, rng)
        return d[:, None] * S * d[None, :]
    e = np.logspace(-3, 3, M)
    rng.shuffle(e)
    return d[:, None] * rng.standard_normal((M, M)) * e[None, :]


# ----------------------------------------------------------------------------------------------- 1. one GPU, bit identity
@pytest.mark.parametrize("kind,trans", [("lu", False), ("lu", True), ("chol", False)], ids=["lu-N", "lu-T", "chol"])
@pytest.mark.parametrize("equilibrate", [False, True], ids=["plain", "equilibrated"])
def test_blocks_equal_replicated_driver_bits(kind, trans, equilibrate):
    N, v = 1024, 64
    rng = np.random.default_rng(7 + trans + 2 * equilibrate)
    nrhs = N + 70
    assert len(rl.blocks(nrhs, v)) >= 4
    if kind == "lu":
        A = _badly_scaled(N, rng) if equilibrate else rng.standard_normal((N, N))
        h, comm = _lu(N, v, A, equilibrate=equilibrate)
        M, Kappa, Aop = h.M, None, A.T if trans else A
        G = rng.standard_normal((M, nrhs))
        X0 = cb.lu_solve(h, G, trans=trans)
    else:
        A = _badly_scaled(N, rng, sym=True) if equilibrate else hp_ref.random_spd(N, 1e3, rng)
        h, comm = _chol(N, v, A, equilibrate=equilibrate)
        M, Kappa, Aop = h.N, h.Kappa, A
        G = rng.standard_normal((M, nrhs))
        X0 = h.solve(G)
    B = rl.distribute(kind, G, v, Kappa=Kappa)[0]
    Xs = rl.distribute(kind, X0, v, Kappa=Kappa)[0]
    rs = _rank_body(kind, h, OPS, trans, G, X0, B, Xs, np.full_like(B, SENTINEL), nrhs)
    for op in OPS:
        res, reps = rs[op]
        X = rl.collect(kind, [res[0]], M, nrhs, v, Kappa=Kappa)
        assert _check(kind, op, res, reps, X, M, nrhs, v) == 0
        if not equilibrate:                                             # the scaled case: the replicated bits suffice
            assert solve_ref.backward_error(Aop, X, G) <= ETA_TOL, op
        if op.startswith("svx"):
            assert res[2]["equed"] == ("N" if not equilibrate else "B" if kind == "lu" else "Y")
    h.free_comms() if kind == "lu" else h.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- 2. info
def test_lu_zero_pivot_leaves_x_and_outputs_unwritten():
    N, v = 1024, 64
    rng = np.random.default_rng(12)
    A = np.triu(rng.integers(1, 9, (N, N)).astype(float)) + np.diag(np.full(N, 50.0))
    A[600, 600] = 0.0                                                   # partial pivoting keeps U = A: U(601, 601) = 0
    gv, comm = _lu(N, v, A)
    nrhs = 300
    ncl = cb.rhs_local_cols(nrhs, v, 1)
    B = rng.standard_normal((N, ncl))
    lib = cb.lib()
    for name in ("refine_x", "svx", "svxx"):
        X = np.full((N, ncl), SENTINEL)
        outs = [np.full(3 * nrhs, SENTINEL) for _ in range(3)]
        rcond, rpvgrw, info, equed = ctypes.c_double(-1), ctypes.c_double(-1), ctypes.c_int(-1), ctypes.c_char(b"?")
        if name == "refine_x":
            rc = lib.cflx_lu_refine_x_local(gv._h, 0, nrhs, _ptr(B), ncl, _ptr(X), ncl, ctypes.byref(rcond),
                                            _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]), ctypes.byref(info))
        elif name == "svx":
            rc = lib.cflx_lu_svx_local(gv._h, 0, nrhs, _ptr(B), ncl, _ptr(X), ncl, ctypes.byref(rcond), _ptr(outs[0]),
                                       _ptr(outs[1]), ctypes.byref(rpvgrw), ctypes.byref(equed), ctypes.byref(info))
        else:
            rc = lib.cflx_lu_svxx_local(gv._h, 0, nrhs, _ptr(B), ncl, _ptr(X), ncl, ctypes.byref(rcond),
                                        ctypes.byref(rpvgrw), _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]),
                                        ctypes.byref(equed), ctypes.byref(info))
        assert rc == 0 and info.value == 601 and rcond.value == 0.0, name
        assert np.all(X == SENTINEL) and all(np.all(o == SENTINEL) for o in outs), name
        _, rep = cb.lu_svx(gv, B[:, :2]) if name == "svx" else cb.lu_svxx(gv, B[:, :2]) if name == "svxx" else (0, {})
        if name != "refine_x":
            assert rpvgrw.value == rep["rpvgrw"] and equed.value == b"N"
    gv.free_comms()
    comm.close()


def test_lu_singular_to_working_precision_gives_m_plus_1():
    N, v = 1024, 64
    rng = np.random.default_rng(13)
    Q1, _ = np.linalg.qr(rng.standard_normal((N, N)))
    Q2, _ = np.linalg.qr(rng.standard_normal((N, N)))
    gv, comm = _lu(N, v, (Q1 * np.logspace(0, -17, N)) @ Q2.T)
    nrhs = 300
    G = rng.standard_normal((N, nrhs))
    B = rl.distribute("lu", G, v)[0]
    X, res = cb.lu_svx_local(gv, B, nrhs)
    assert res["info"] == N + 1 and res["rcond"] < 2.0 ** -53 and X is not None
    for c0, w in rl.blocks(nrhs, v):
        Xb, rep = cb.lu_svx(gv, np.ascontiguousarray(G[:, c0:c0 + w]))
        assert rep["info"] == N + 1 and np.array_equal(X[:, c0:c0 + w], Xb) and rep["rcond"] == res["rcond"]
    gv.free_comms()
    comm.close()


@pytest.mark.parametrize("kind", ["lu", "chol"])
def test_ill_column_in_a_later_block_gives_its_global_column(kind):
    N, v = 1024, 64
    rng = np.random.default_rng(14)
    nrhs = N + 70
    Xt = rng.standard_normal((N, nrhs))
    jbad = 700                                                          # block 2 of 256-column blocks
    Xt[:, jbad] = 1.0
    Xt[3, jbad] = 1e-30                                                  # componentwise far out of reach
    if kind == "lu":
        A = rng.standard_normal((N, N))
        h, comm = _lu(N, v, A)
        G = A @ Xt
        X0 = cb.lu_solve(h, G)
        Kappa = None
    else:
        A = hp_ref.random_spd(N, 1e2, rng)
        h, comm = _chol(N, v, A)
        G = A @ Xt
        X0 = h.solve(G)
        Kappa = h.Kappa
    B = rl.distribute(kind, G, v, Kappa=Kappa)[0]
    Xs = rl.distribute(kind, X0, v, Kappa=Kappa)[0]
    rs = _rank_body(kind, h, ("refine_x", "svxx"), False, G, X0, B, Xs, None, nrhs)
    for op in ("refine_x", "svxx"):
        res, reps = rs[op]
        X = rl.collect(kind, [res[0]], N, nrhs, v, Kappa=Kappa)
        assert _check(kind, op, res, reps, X, N, nrhs, v) == N + jbad + 1, op
    h.free_comms() if kind == "lu" else h.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- 3. other factor kinds
def test_other_factor_kinds_match_replicated_bits():
    N, v, nrhs = 1024, 64, 300
    rng = np.random.default_rng(15)
    G = rng.standard_normal((N, nrhs))
    comm = cb.Comm(1, 0, None, 0)
    # the LU after the butterflies and the fixed-order factorisation
    gv = cb.lu_params(N, N, v, 1, 1, 1, comm)
    gv.data[...] = rng.standard_normal((N, N))
    cb.LU_rep_rbt(gv, depth=2, seed=3)
    X0 = cb.lu_solve(gv, G)
    rs = _rank_body("lu", gv, OPS, False, G, X0, rl.distribute("lu", G, v)[0], rl.distribute("lu", X0, v)[0],
                    np.full((N, cb.rhs_local_cols(nrhs, v, 1)), SENTINEL), nrhs)
    for op in OPS:
        res, reps = rs[op]
        _check("lu", op, res, reps, rl.collect("lu", [res[0]], N, nrhs, v), N, nrhs, v)
    gv.free_comms()
    # the Cholesky's signed factor of an indefinite matrix, without and with the butterfly
    Q, _ = np.linalg.qr(rng.standard_normal((N, N)))
    K = (Q * np.where(np.arange(N) % 3 == 0, -1.0, 1.0) * np.logspace(0, 2, N)) @ Q.T
    for rbt in (False, True):
        ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
        ch.data[...] = K
        if rbt:
            ch.rbt(depth=2, seed=5)
        _, _, info, _ = ch.factor_ldlt(upload=not rbt)
        assert info == 0
        X0 = ch.solve(G)
        Bs, Xs = rl.distribute("chol", G, v, Kappa=ch.Kappa)[0], rl.distribute("chol", X0, v, Kappa=ch.Kappa)[0]
        rs = _rank_body("chol", ch, OPS, False, G, X0, Bs, Xs, np.full_like(Bs, SENTINEL), nrhs)
        for op in OPS:
            res, reps = rs[op]
            _check("chol", op, res, reps, rl.collect("chol", [res[0]], N, nrhs, v, Kappa=ch.Kappa), N, nrhs, v)
        ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- 4, 5. memory, side effects
def test_lu_memory_kinds_in_place_and_side_effects():
    import torch
    N, v = 1024, 64
    rng = np.random.default_rng(16)
    A = rng.standard_normal((N, N))
    gv, comm = _lu(N, v, A)
    nrhs = 2 * 256 + 3                                                   # three blocks, padding in the last local tile
    G = rng.standard_normal((N, nrhs))
    X0 = cb.lu_solve(gv, G)
    B = rl.distribute("lu", G, v, pad=np.nan, ld_extra=5)[0]            # NaN in the padding and the ld padding
    Xs = rl.distribute("lu", X0, v, pad=np.nan, ld_extra=5)[0]
    B0 = B.copy()
    C0, perm0 = np.zeros((gv.Ml, gv.Nl)), np.empty(gv.M, dtype=np.int32)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C0.ctypes.data, perm0.ctypes.data), "get_factors")
    b1 = G[:, :5].copy()
    x1 = cb.lu_solve(gv, b1)
    r1 = cb.lu_refine(gv, b1, x1)
    _launches(cb.lib().cflx_lu_launch_count, gv._h)

    Xh, fe, be = cb.lu_refine_local(gv, B, Xs.copy(), nrhs)              # host in, host out
    assert np.array_equal(B, B0, equal_nan=True) and np.all(np.isnan(Xh[:, nrhs:]))
    tb, tx = torch.from_numpy(B).cuda(), torch.from_numpy(Xs).cuda()
    Xd, fe_d, be_d = cb.lu_refine_local(gv, tb, tx, nrhs)                # device in, device out
    assert Xd is tx and np.array_equal(tx.cpu().numpy(), Xh, equal_nan=True)
    assert np.array_equal(fe_d, fe) and np.array_equal(be_d, be)
    tx2 = torch.from_numpy(Xs).cuda()
    cb.lu_refine_local(gv, B, tx2, nrhs)                                 # host B, device X
    assert np.array_equal(tx2.cpu().numpy(), Xh, equal_nan=True)
    assert np.array_equal(tb.cpu().numpy(), B0, equal_nan=True)

    Xsv, res = cb.lu_svx_local(gv, B, nrhs, out=np.full_like(B, SENTINEL))
    assert np.all(Xsv[:, nrhs:] == SENTINEL)
    for how in ("device", "in place host", "in place device", "device in host out"):
        if how == "device":
            o = torch.full(B.shape, SENTINEL, dtype=torch.float64, device="cuda")
            X2, r2 = cb.lu_svx_local(gv, tb, nrhs, out=o)
        elif how == "in place host":
            o = B.copy()
            X2, r2 = cb.lu_svx_local(gv, o, nrhs, out=o)
        elif how == "in place device":
            o = torch.from_numpy(B).cuda()
            X2, r2 = cb.lu_svx_local(gv, o, nrhs, out=o)
        else:
            o = np.full_like(B, SENTINEL)
            X2, r2 = cb.lu_svx_local(gv, tb, nrhs, out=o)
        assert X2 is o, how
        got = o.cpu().numpy() if hasattr(o, "cpu") else o
        assert np.array_equal(got[:, :nrhs], Xsv[:, :nrhs]), how
        assert all(_same(r2[k], res[k]) for k in res), how
    Xxx, rxx = cb.lu_svxx_local(gv, tb, nrhs, out=torch.from_numpy(B).cuda())
    Xxh, rxh = cb.lu_svxx_local(gv, B, nrhs)
    assert np.array_equal(Xxx.cpu().numpy()[:, :nrhs], Xxh[:, :nrhs]) and all(_same(rxx[k], rxh[k]) for k in rxh)
    Xr, dr = cb.lu_refine_x_local(gv, tb, torch.from_numpy(Xs).cuda(), nrhs)
    Xrh, drh = cb.lu_refine_x_local(gv, B, Xs.copy(), nrhs)
    assert np.array_equal(Xr.cpu().numpy(), Xrh, equal_nan=True) and all(_same(dr[k], drh[k]) for k in drh)

    assert _launches(cb.lib().cflx_lu_launch_count, gv._h) == 0         # no factorisation launched
    assert np.array_equal(cb.lu_solve(gv, b1), x1)                      # a later solve and refine: the same bits
    r2 = cb.lu_refine(gv, b1, x1)
    assert all(np.array_equal(a, b) for a, b in zip(r1, r2))            # the input is unchanged
    C1, perm1 = np.zeros_like(C0), np.empty_like(perm0)
    cb.check(cb.lib().cflx_lu_get_factors(gv._h, C1.ctypes.data, perm1.ctypes.data), "get_factors")
    assert np.array_equal(C1, C0) and np.array_equal(perm1, perm0)
    gv.free_comms()
    comm.close()


def test_chol_memory_kinds_and_side_effects():
    import torch
    N, v = 1000, 48                                                      # Kappa = 21 tiles: rows beyond the real tiles
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    rng = np.random.default_rng(17)
    ch.data[...] = hp_ref.random_spd(ch.N, 1e2, rng)
    ch.parallelCholesky()
    A0, L0 = ch.local_input(), ch.local_factor()
    nrhs = 300
    G = rng.standard_normal((ch.N, nrhs))
    X0 = ch.solve(G)
    B = rl.distribute("chol", G, v, Kappa=ch.Kappa, ld_extra=3)[0]
    Xs = rl.distribute("chol", X0, v, Kappa=ch.Kappa, ld_extra=3)[0]
    b1 = G[:, :3].copy()
    x1 = ch.solve(b1)
    n0 = _launches(cb.lib().cflx_chol_launch_count, ch._h)
    Xh, fe, be = ch.refine_local(B, Xs.copy(), nrhs)
    Xd, fe_d, be_d = ch.refine_local(torch.from_numpy(B).cuda(), torch.from_numpy(Xs).cuda(), nrhs)
    assert np.array_equal(Xd.cpu().numpy(), Xh, equal_nan=True) and np.array_equal(fe, fe_d) and np.array_equal(be, be_d)
    Xv, rv = ch.svx_local(B, nrhs, out=np.full_like(B, SENTINEL))
    tb = torch.from_numpy(B).cuda()
    Xv2, rv2 = ch.svx_local(tb, nrhs, out=tb)                            # in place on the device
    assert np.array_equal(Xv2.cpu().numpy()[:, :nrhs], Xv[:, :nrhs]) and all(_same(rv[k], rv2[k]) for k in rv)
    assert np.all(Xv[:, nrhs:] == SENTINEL)
    Xx, rx = ch.svxx_local(B, nrhs)
    Xx2, rx2 = ch.svxx_local(torch.from_numpy(B).cuda(), nrhs, out=torch.zeros(B.shape, dtype=torch.float64, device="cuda"))
    assert np.array_equal(Xx2.cpu().numpy()[:, :nrhs], Xx[:, :nrhs]) and all(_same(rx[k], rx2[k]) for k in rx)
    assert _launches(cb.lib().cflx_chol_launch_count, ch._h) == 0 and n0 > 0
    assert np.array_equal(ch.solve(b1), x1)
    assert np.array_equal(ch.local_input(), A0) and np.array_equal(ch.local_factor(), L0)
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- 6. refusals
def _refused(rc, status, who, what):
    msg = cb.lib().cflx_last_error().decode()
    assert rc == status and who in msg and what in msg, (rc, msg)


def test_lu_refusals_and_state_rules():
    n, v = 256, 32
    comm = cb.Comm(1, 0, None, 0)
    gv = cb.lu_params(n, n, v, 1, 1, 1, comm)
    nrhs = 40
    ncl = cb.rhs_local_cols(nrhs, v, 1)
    B, X = np.ones((n, ncl)), np.zeros((n, ncl))
    e3, e = np.zeros(3 * nrhs), np.zeros(nrhs)
    d, i, c = ctypes.c_double(), ctypes.c_int(), ctypes.c_char()
    L = cb.lib()
    calls = {
        "cflx_lu_refine_local": lambda b, x, ldx=ncl, t=0: L.cflx_lu_refine_local(gv._h, t, nrhs, b, ncl, x, ldx, _ptr(e), _ptr(e)),
        "cflx_lu_refine_x_local": lambda b, x, ldx=ncl, t=0, r=ctypes.byref(d), en=_ptr(e3), inf=ctypes.byref(i):
            L.cflx_lu_refine_x_local(gv._h, t, nrhs, b, ncl, x, ldx, r, _ptr(e), en, _ptr(e3), inf),
        "cflx_lu_svx_local": lambda b, x, ldx=ncl, t=0, r=ctypes.byref(d), inf=ctypes.byref(i):
            L.cflx_lu_svx_local(gv._h, t, nrhs, b, ncl, x, ldx, r, _ptr(e), _ptr(e), ctypes.byref(d), ctypes.byref(c), inf),
        "cflx_lu_svxx_local": lambda b, x, ldx=ncl, t=0, r=ctypes.byref(d), en=_ptr(e3), inf=ctypes.byref(i):
            L.cflx_lu_svxx_local(gv._h, t, nrhs, b, ncl, x, ldx, r, ctypes.byref(d), _ptr(e), en, _ptr(e3), ctypes.byref(c), inf),
    }
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X)), ERR_STATE, who, "cflx_lu_factor")     # no factorisation yet
    gv.data[...] = np.random.default_rng(1).standard_normal((n, n)) + n * np.eye(n)
    cb.LU_rep(gv)
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X), t=2), ERR_ARG, who, "trans != 0 && trans != 1")
        _refused(f(None, _ptr(X)), ERR_ARG, who, "g.pk == 0 && !B")
        _refused(f(_ptr(B), _ptr(X), ldx=ncl - 1), ERR_ARG, who, "X && ldx < local_cols")
        if "refine" in who:
            _refused(f(_ptr(B), None), ERR_ARG, who, "g.pk == 0 && !X")
            _refused(f(_ptr(B), _ptr(B)), ERR_ARG, who, "X_local overlaps B_local")
            Bw = np.ones((n, 2 * ncl))
            _refused(f(ctypes.c_void_p(Bw.ctypes.data), ctypes.c_void_p(Bw.ctypes.data + 8 * (ncl - 1))), ERR_ARG, who,
                     "X_local overlaps B_local")                        # a partial overlap in each row
        else:
            assert f(_ptr(B), None) == 0                                # X output only: may be NULL
            Bw = np.ones((n, ncl + 8))
            _refused(f(_ptr(Bw), _ptr(Bw), ldx=ncl + 8), ERR_ARG, who, "X_local == B_local needs ldx == ldb")
        if who != "cflx_lu_refine_local":
            _refused(f(_ptr(B), _ptr(X), inf=None), ERR_ARG, who, "!info_out")
        if "svx" in who:
            _refused(f(_ptr(B), _ptr(X), r=None), ERR_ARG, who, "!rcond_out")
        if who.endswith(("refine_x_local", "svxx_local")):
            _refused(f(_ptr(B), _ptr(X), en=None), ERR_ARG, who, "!err_bnds_norm_out")
    # a queued next input: the refinement reads this input, which the queued upload overwrites
    mats = [cb.pinned_empty((gv.Ml, gv.Nl)) for _ in range(2)]
    for k, m in enumerate(mats):
        m[...] = np.random.default_rng(k).standard_normal((n, n)) + n * np.eye(n)
    gv.data = mats[0]
    cb.LU_rep(gv, next_data=mats[1])
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X)), ERR_STATE, who, "queued next matrix")
    cb.LU_rep(gv, upload=False)
    for who, f in calls.items():
        Xc = X.copy()
        assert f(_ptr(B), _ptr(Xc)) == 0, who
    gv.data = np.array(mats[1])
    for m in mats:
        cb.pinned_free(m)
    # the low-precision factors of a mixed-precision driver
    X_, it, _ = cb.lu_sv_mixed(gv, np.ones((n, 1)), prec="tf32x3")
    assert it >= 0
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X)), ERR_STATE, who, "mixed-precision")
    a = np.ascontiguousarray(gv.data)
    cb.check(L.cflx_lu_set_local(gv._h, a.ctypes.data), "set_local")
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X)), ERR_STATE, who, "cflx_lu_set_local")  # a new input, not factored yet
    gv.free_comms()
    comm.close()


def test_chol_refusals_and_state_rules():
    N, v = 256, 32
    comm = cb.Comm(1, 0, None, 0)
    ch = cb.cholesky.initialize(N, v, (1, 1, 1), comm)
    nrhs = 40
    ncl = cb.rhs_local_cols(nrhs, v, 1)
    B, X = np.ones((N, ncl)), np.zeros((N, ncl))
    e3, e = np.zeros(3 * nrhs), np.zeros(nrhs)
    d, i, c = ctypes.c_double(), ctypes.c_int(), ctypes.c_char()
    L = cb.lib()
    calls = {
        "cflx_chol_refine_local": lambda b, x, inf=None, r=None: L.cflx_chol_refine_local(ch._h, nrhs, b, ncl, x, ncl, _ptr(e), _ptr(e)),
        "cflx_chol_refine_x_local": lambda b, x, inf=ctypes.byref(i), r=None:
            L.cflx_chol_refine_x_local(ch._h, nrhs, b, ncl, x, ncl, None, _ptr(e), _ptr(e3), None, inf),
        "cflx_chol_svx_local": lambda b, x, inf=ctypes.byref(i), r=ctypes.byref(d):
            L.cflx_chol_svx_local(ch._h, nrhs, b, ncl, x, ncl, r, _ptr(e), _ptr(e), ctypes.byref(c), inf),
        "cflx_chol_svxx_local": lambda b, x, inf=ctypes.byref(i), r=ctypes.byref(d):
            L.cflx_chol_svxx_local(ch._h, nrhs, b, ncl, x, ncl, r, None, _ptr(e), _ptr(e3), None, None, inf),
    }
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X)), ERR_STATE, who, "cflx_chol_factor")
    S = hp_ref.random_spd(N, 1e2, np.random.default_rng(3))
    ch.data[...] = S
    ch.parallelCholesky()
    for who, f in calls.items():
        _refused(f(None, _ptr(X)), ERR_ARG, who, "g.pk == 0 && !B")
        if "refine" in who:
            _refused(f(_ptr(B), None), ERR_ARG, who, "g.pk == 0 && !X")
            _refused(f(_ptr(B), _ptr(B)), ERR_ARG, who, "X_local overlaps B_local")
        else:
            _refused(f(_ptr(B), _ptr(X), r=None), ERR_ARG, who, "!rcond_out")
        if who != "cflx_chol_refine_local":
            _refused(f(_ptr(B), _ptr(X), inf=None), ERR_ARG, who, "!info_out")
        Xc = X.copy()
        assert f(_ptr(B), _ptr(Xc)) == 0, who
    _, it, _ = ch.sv_mixed(np.ones((N, 1)), prec="tf32x3")
    assert it >= 0
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X)), ERR_STATE, who, "mixed-precision")
    a = np.ascontiguousarray(ch.data)
    cb.check(L.cflx_chol_set_local(ch._h, a.ctypes.data), "set_local")
    for who, f in calls.items():
        _refused(f(_ptr(B), _ptr(X)), ERR_STATE, who, "cflx_chol_set_local")
    ch.finalize()
    comm.close()


# ----------------------------------------------------------------------------------------------- 7. multi-rank grids
@pytest.mark.parametrize("grid", [(1, 1, 2), (2, 2, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_lu_refine_local(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1024, 64
    M = layout.dims(N, v, *grid)["M"]
    rng = np.random.default_rng(P)
    A = rng.standard_normal((M, M))
    locs = layout.scatter(A, v, *grid)
    nrhs = M + 70
    G = rng.standard_normal((M, nrhs))
    Bs = rl.distribute("lu", G, v, *grid)

    def body(comm):
        gv = cb.lu_params(N, N, v, *grid, comm)
        gv.data[...] = locs[gv.rank]
        cb.LU_rep(gv)
        out = {}
        for trans in (False, True):
            X0 = cb.lu_solve(gv, G, trans=trans)
            Xs = rl.distribute("lu", X0, v, *grid, pad=SENTINEL)[gv.rank]
            layer0 = gv.pk == 0
            out[trans] = _rank_body("lu", gv, OPS, trans, G, X0, Bs[gv.rank] if layer0 else None,  # B not read off layer 0
                                    Xs if layer0 else None, np.full_like(Xs, SENTINEL), nrhs)
        gv.free_comms()
        return out

    rs = run_ranks(P, body)
    for trans in (False, True):
        for op in OPS:
            for r in range(P):                                          # the layers agree bit for bit
                assert _same(rs[r][trans][op][0][0], rs[r - r % grid[2]][trans][op][0][0]), (op, r)
                assert all(_same(rs[r][trans][op][0][1][k], rs[0][trans][op][0][1][k]) for k in rs[0][trans][op][0][1])
            res, reps = rs[0][trans][op]
            X = rl.collect("lu", [x[trans][op][0][0] for x in rs], M, nrhs, v, *grid)
            _check("lu", op, res, reps, X, M, nrhs, v)
            assert solve_ref.backward_error(A.T if trans else A, X, G) <= ETA_TOL, (op, trans)


@pytest.mark.parametrize("grid", [(2, 1, 1), (2, 2, 2)], ids=lambda g: "%dx%dx%d" % g)
def test_multi_gpu_chol_refine_local(grid):
    P = grid[0] * grid[1] * grid[2]
    if n_gpus() < P:
        pytest.skip(f"needs {P} GPUs")
    N, v = 1024, 64
    d = chol_ref.dims(N, v, *grid)
    S = hp_ref.random_spd(d["N"], 1e2, np.random.default_rng(P))
    locs = chol_solve_ref.scatter(S, N, v, *grid)
    nrhs = d["N"] + 70
    G = np.random.default_rng(P + 1).standard_normal((d["N"], nrhs))
    Bs = rl.distribute("chol", G, v, *grid, Kappa=d["Kappa"])

    def body(comm):
        ch = cb.cholesky.initialize(N, v, grid, comm)
        ch.data[...] = locs[ch.rank]
        ch.parallelCholesky()
        X0 = ch.solve(G)
        Xs = rl.distribute("chol", X0, v, *grid, Kappa=d["Kappa"], pad=SENTINEL)[ch.rank]
        layer0 = ch.pz == 0
        out = _rank_body("chol", ch, OPS, False, G, X0, Bs[ch.rank] if layer0 else None, Xs if layer0 else None,
                         np.full_like(Xs, SENTINEL), nrhs)
        ch.finalize()
        return out

    rs = run_ranks(P, body)
    for op in OPS:
        for r in range(P):
            assert _same(rs[r][op][0][0], rs[r - r % grid[2]][op][0][0]), (op, r)
        res, reps = rs[0][op]
        X = rl.collect("chol", [x[op][0][0] for x in rs], d["N"], nrhs, v, *grid, Kappa=d["Kappa"])
        _check("chol", op, res, reps, X, d["N"], nrhs, v)
        assert solve_ref.backward_error(S, X, G) <= ETA_TOL, op


def test_multi_rank_grids_on_one_device(tmp_path):
    """the two grid tests above in a child pytest under the NCCL loopback, every grid on device 0"""
    if "LD_PRELOAD" in os.environ and "nccl_loopback" in os.environ["LD_PRELOAD"]:
        pytest.skip("already under the loopback")
    lib = _loopback.build()
    xml, stats_out = tmp_path / "junit.xml", tmp_path / "stats.json"
    preload = " ".join(p for p in (lib, os.environ.get("LD_PRELOAD")) if p)
    env = dict(os.environ, LD_PRELOAD=preload, **{_loopback.STATS_ENV: str(stats_out)})
    flags = ["-s"] if sys.flags.no_user_site else []
    f = "tests/test_gpu_refine_local.py"
    cmd = [sys.executable] + flags + ["-m", "pytest", "-p", "tests._loopback", "-p", "no:cacheprovider", "-q", "-rA",
                                      f"--junitxml={xml}", f"{f}::test_multi_gpu_lu_refine_local",
                                      f"{f}::test_multi_gpu_chol_refine_local"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-6000:] + "\n--- stderr ---\n" + r.stderr[-6000:]
    import xml.etree.ElementTree as ET
    cases = [[e.tag for e in c] for c in ET.parse(xml).iter("testcase")]
    assert len(cases) == 5 and not any(tags for tags in cases), r.stdout[-3000:]
