"""Every refusal of the C entry points explains itself: the status, then a message that starts with the function's own
name and names the condition that failed.  Each call follows an unrelated refusal, so that a refusal which sets no
text (and would show the previous one) is caught.

The CPU part passes NULL handles and the documented bad arguments of the host-only functions; the GPU part walks the
ARG and STATE cases the header documents for one LU and one Cholesky handle, through their states."""
import ctypes

import numpy as np
import pytest

import conflux_b200 as cb
from conflux_b200 import _lib

ARG, STATE, UNSUPPORTED = -1, -5, -4

LU_HANDLE = ["cflx_lu_info", "cflx_lu_set_local", "cflx_lu_queue_next_local", "cflx_lu_factor", "cflx_lu_factor_fixed",
             "cflx_lu_rbt", "cflx_lu_rbt_solve", "cflx_lu_rbt_apply_local", "cflx_lu_get_factors",
             "cflx_lu_get_permutation", "cflx_lu_residual", "cflx_lu_validate", "cflx_lu_solve", "cflx_lu_solve_trans",
             "cflx_lu_solve_local", "cflx_lu_rcond", "cflx_lu_refine", "cflx_lu_refine_x", "cflx_lu_equilibrate",
             "cflx_lu_svx", "cflx_lu_equilibrate_b", "cflx_lu_svxx", "cflx_lu_inverse", "cflx_lu_det",
             "cflx_lu_launch_count", "cflx_lu_set_profiling", "cflx_lu_phase_ms", "cflx_lu_timeline",
             "cflx_lu_set_kernel_timing", "cflx_lu_trailing_stats"]
CHOL_HANDLE = ["cflx_chol_info", "cflx_chol_set_local", "cflx_chol_factor", "cflx_chol_get_local", "cflx_chol_validate",
               "cflx_chol_solve", "cflx_chol_solve_local", "cflx_chol_rcond", "cflx_chol_refine", "cflx_chol_refine_x",
               "cflx_chol_equilibrate", "cflx_chol_svx", "cflx_chol_equilibrate_b", "cflx_chol_svxx",
               "cflx_chol_inverse", "cflx_chol_det", "cflx_chol_launch_count"]
COMM_HANDLE = ["cflx_comm_barrier", "cflx_lu_create", "cflx_chol_create"]


def _filler(t):
    """a harmless value of ctypes type t for the arguments after the one that is refused"""
    if t in (ctypes.c_double,):
        return 0.0
    if t in (ctypes.c_int, ctypes.c_int64, ctypes.c_uint64, ctypes.c_size_t):
        return 1
    return None


def _prime(L, name):
    """an unrelated refusal; returns its message"""
    n = ctypes.c_int()
    if name == "cflx_rhs_local_cols":
        assert L.cflx_auto_grid(0, 1, 1, None, None, None) == ARG
    else:
        assert L.cflx_rhs_local_cols(0, 1, 1, ctypes.byref(n)) == ARG
    return L.cflx_last_error().decode()


def call(L, name, args, status, cond, messages=True):
    """name(*args) after an unrelated refusal: (status it returned, its message, the message before it)"""
    prev = _prime(L, name)
    rc = getattr(L, name)(*args)
    msg = L.cflx_last_error().decode()
    if status == 0 or not messages:
        return rc == status, rc, msg
    ok = rc == status and msg != prev and msg.startswith(name + ":") and cond in msg
    return ok, rc, msg


def _check(L, rows):
    bad = []
    for name, args, status, cond in rows:
        ok, rc, msg = call(L, name, args, status, cond)
        if not ok:
            bad.append((name, status, cond, rc, msg))
    assert not bad, "\n".join(map(str, bad))


# ------------------------------------------------------------------------------------------------------ CPU
def test_null_handles_are_refused_by_name():
    L = _lib.lib()
    rows = []
    for name, cond in [(n, "!lu") for n in LU_HANDLE] + [(n, "!ch") for n in CHOL_HANDLE] + \
                      [(n, "!c") for n in COMM_HANDLE]:
        types = getattr(L, name).argtypes
        rows.append((name, [None] + [_filler(t) for t in types[1:]], ARG, f"refused, {cond}"))
    _check(L, rows)


def test_host_only_arguments_are_refused_by_name():
    L = _lib.lib()
    i3 = (ctypes.c_int * 3)()
    o8 = (ctypes.c_int * 8)()
    buf = np.zeros(64 * 64)
    p = buf.ctypes.data
    one = ctypes.c_int()
    vp = ctypes.c_void_p()
    rows = [
        ("cflx_auto_grid", (0, 8, 1, i3, i3, i3), ARG, "M <= 0"),
        ("cflx_auto_grid", (8, 0, 1, i3, i3, i3), ARG, "N <= 0"),
        ("cflx_auto_grid", (8, 8, 0, i3, i3, i3), ARG, "P <= 0"),
        ("cflx_chol_auto_grid", (0, 8, i3), ARG, "P <= 0"),
        ("cflx_chol_auto_grid", (1, 8, None), ARG, "!grid3"),
        ("cflx_rhs_local_cols", (0, 4, 1, ctypes.byref(one)), ARG, "nrhs < 1"),
        ("cflx_rhs_local_cols", (4, 0, 1, ctypes.byref(one)), ARG, "v < 1"),
        ("cflx_rhs_local_cols", (4, 4, 0, ctypes.byref(one)), ARG, "Py < 1"),
        ("cflx_rhs_local_cols", (4, 4, 1, None), ARG, "!cols_out"),
        ("cflx_rbt_multipliers", (64, 0, 0, p, None), ARG, "depth < 1"),
        ("cflx_rbt_multipliers", (64, 5, 0, p, None), ARG, "depth > 4"),
        ("cflx_rbt_multipliers", (0, 1, 0, p, None), ARG, "M < 1"),
        ("cflx_rbt_multipliers", (63, 1, 0, p, None), ARG, "M % (1 << depth) != 0"),
        ("cflx_rbt_multipliers", (64, 1, 0, None, None), ARG, "!u_out && !v_out"),
        ("cflx_host_alloc", (8, None), ARG, "!out"),
        ("cflx_comm_create", (1, 0, None, 0, None), ARG, "!out"),
        ("cflx_comm_create", (0, 0, None, 0, ctypes.byref(vp)), ARG, "world_size < 1"),
        ("cflx_comm_create", (2, -1, None, 0, ctypes.byref(vp)), ARG, "world_rank < 0"),
        ("cflx_comm_create", (2, 2, None, 0, ctypes.byref(vp)), ARG, "world_rank >= world_size"),
    ]
    lu_args = dict(M=16, N=16, v=4, Px=2, Py=2, Pz=1)
    for k in lu_args:
        a = dict(lu_args, **{k: 0})
        rows.append(("cflx_lu_dims", (*a.values(), o8), ARG, f"{k} <= 0"))
        rows.append(("cflx_init_matrix_host", (*a.values(), 0, 1, p), ARG, f"{k} <= 0"))
    rows += [("cflx_lu_dims", (*lu_args.values(), None), ARG, "!o"),
             ("cflx_init_matrix_host", (*lu_args.values(), -1, 1, p), ARG, "rank < 0"),
             ("cflx_init_matrix_host", (*lu_args.values(), 4, 1, p), ARG, "rank >= Px * Py * Pz"),
             ("cflx_init_matrix_host", (*lu_args.values(), 0, 1, None), ARG, "!out")]
    chol_args = dict(N=16, v=4, Px=2, Py=2, Pz=1)
    for k in chol_args:
        a = dict(chol_args, **{k: 0})
        rows.append(("cflx_chol_dims", (*a.values(), o8), ARG, f"{k} <= 0"))
        rows.append(("cflx_chol_init_matrix_host", (*a.values(), 0, p), ARG, f"{k} <= 0"))
    rows += [("cflx_chol_dims", (*chol_args.values(), None), ARG, "!o"),
             ("cflx_chol_init_matrix_host", (*chol_args.values(), -1, p), ARG, "rank < 0"),
             ("cflx_chol_init_matrix_host", (*chol_args.values(), 4, p), ARG, "rank >= Px * Py * Pz"),
             ("cflx_chol_init_matrix_host", (*chol_args.values(), 0, None), ARG, "!out")]
    _check(L, rows)


# ------------------------------------------------------------------------------------------------------ GPU
N, V, NRHS = 256, 32, 4
NO_LU = "before cflx_lu_factor"
NO_CH = "before a successful cflx_chol_factor"
QUEUED = "queued next matrix"
NO_RBT = "carry no random butterfly"


def _walk(L, messages=True):
    """Builds one LU and one Cholesky handle (N = 256, v = 32, 1 x 1 x 1), walks them through their states and calls
    every documented refusal in each; returns the rows that did not come out as the table says (all of them checked for
    the status, and with `messages` for the text too)."""
    bad = []

    def run(rows):
        for name, args, status, cond in rows:
            ok, rc, msg = call(L, name, args, status, cond, messages)
            if not ok:
                bad.append((name, status, cond, rc, msg))

    def ok(rc):
        assert rc == 0, L.cflx_last_error().decode()

    B = np.ones((N, NRHS))
    X = np.zeros((N, NRHS))
    Bl = np.ones((N, 32))                                   # the local share: rhs_local_cols(4, 32, 1) = 32 columns
    Xl = np.zeros((N, 32))
    b, x, bl, xl = B.ctypes.data, X.ctypes.data, Bl.ctypes.data, Xl.ctypes.data
    dbl = np.zeros(4 * N)
    d = dbl.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    ints = np.zeros(N, dtype=np.int32)
    i = ints.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    i64s = np.zeros(4, dtype=np.int64)
    i64 = i64s.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    ch_ = ctypes.create_string_buffer(4)
    full = np.zeros((N, N))
    f = full.ctypes.data
    A = np.zeros((N, N))
    ok(L.cflx_init_matrix_host(N, N, V, 1, 1, 1, 0, 7, A.ctypes.data))
    S = np.zeros((N, N))
    ok(L.cflx_chol_init_matrix_host(N, V, 1, 1, 1, 0, S.ctypes.data))
    A_scaled = A.copy()
    A_scaled[0] *= 1e-6                                     # rowcnd far below 0.1: dgeequ scales
    S_scaled = S.copy()
    S_scaled[0] *= 1e-3
    S_scaled[:, 0] *= 1e-3                                  # scond far below 0.1: dpoequ scales
    S_bad = S.copy()
    S_bad[5, 5] = -S_bad[5, 5]                              # not positive definite

    comm = ctypes.c_void_p()
    ok(L.cflx_comm_create(1, 0, None, 0, ctypes.byref(comm)))
    lu, ch = ctypes.c_void_p(), ctypes.c_void_p()
    run([("cflx_lu_create", (comm, N, N, 30, 1, 1, 1, ctypes.byref(lu)), UNSUPPORTED, "tile size v=30"),
         ("cflx_lu_create", (comm, N, N, V, 2, 2, 1, ctypes.byref(lu)), ARG, "does not match"),
         ("cflx_chol_create", (comm, N, 30, 1, 1, 1, ctypes.byref(ch)), UNSUPPORTED, "tile size v=30")])
    ok(L.cflx_lu_create(comm, N, N, V, 1, 1, 1, ctypes.byref(lu)))
    ok(L.cflx_chol_create(comm, N, V, 1, 1, 1, ctypes.byref(ch)))
    nxt = cb.pinned_empty((N, N))
    try:
        # the calls on the factors, with valid arguments: their state rules
        def on_lu_factors(own_only=False):
            rows = [("cflx_lu_validate", (lu, d, d), True), ("cflx_lu_residual", (lu, d), True),
                    ("cflx_lu_rcond", (lu, d, d), True),
                    ("cflx_lu_refine", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d), True),
                    ("cflx_lu_refine_x", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, d, d, i), True),
                    ("cflx_lu_svx", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, d, d, ch_, i), True),
                    ("cflx_lu_svxx", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, d, d, d, ch_, i), True),
                    ("cflx_lu_rbt_solve", (lu, 0, NRHS, b, NRHS, x, NRHS, 1, d, d), True),
                    ("cflx_lu_solve", (lu, NRHS, b, NRHS, x, NRHS), False),
                    ("cflx_lu_solve_trans", (lu, NRHS, b, NRHS, x, NRHS), False),
                    ("cflx_lu_solve_local", (lu, 0, NRHS, bl, 32, xl, 32), False),
                    ("cflx_lu_inverse", (lu, f, i), False),
                    ("cflx_lu_det", (lu, 0, d, d, d, i64, i), False),
                    ("cflx_lu_get_permutation", (lu, i), False), ("cflx_lu_get_factors", (lu, f, i), False),
                    ("cflx_lu_rbt_apply_local", (lu, 0, NRHS, bl, 32), False)]
            return [(n, a, STATE, QUEUED if own_only else NO_LU) for n, a, own in rows if own or not own_only]

        ch_factors = [("cflx_chol_get_local", (ch, f)), ("cflx_chol_validate", (ch, d, d)),
                      ("cflx_chol_solve", (ch, NRHS, b, NRHS, x, NRHS)),
                      ("cflx_chol_solve_local", (ch, NRHS, bl, 32, xl, 32)), ("cflx_chol_rcond", (ch, d, d)),
                      ("cflx_chol_refine", (ch, NRHS, b, NRHS, x, NRHS, d, d)),
                      ("cflx_chol_refine_x", (ch, NRHS, b, NRHS, x, NRHS, d, d, d, d, i)),
                      ("cflx_chol_svx", (ch, NRHS, b, NRHS, x, NRHS, d, d, d, ch_, i)),
                      ("cflx_chol_svxx", (ch, NRHS, b, NRHS, x, NRHS, d, d, d, d, d, ch_, i)),
                      ("cflx_chol_inverse", (ch, f)), ("cflx_chol_det", (ch, 0, d, d, i64))]
        ch_factors = [(n, a, STATE, NO_CH) for n, a in ch_factors]

        # ---- before set_local
        run([("cflx_lu_factor", (lu, d), STATE, "before cflx_lu_set_local"),
             ("cflx_lu_factor_fixed", (lu, None, 0.0, i, i, d), STATE, "before cflx_lu_set_local"),
             ("cflx_lu_rbt", (lu, 2, 0, None, None), STATE, "before cflx_lu_set_local"),
             ("cflx_lu_queue_next_local", (lu, nxt.ctypes.data), STATE, "before cflx_lu_set_local"),
             ("cflx_lu_equilibrate", (lu, 0, d, d, d, d, d, ch_, i), STATE, "before cflx_lu_set_local"),
             ("cflx_lu_equilibrate_b", (lu, 1, d, d, d, d, d, ch_, i), STATE, "before cflx_lu_set_local"),
             ("cflx_chol_factor", (ch, d), STATE, "before cflx_chol_set_local"),
             ("cflx_chol_equilibrate", (ch, 0, d, d, d, ch_, i), STATE, "before cflx_chol_set_local"),
             ("cflx_chol_equilibrate_b", (ch, 1, d, d, d, ch_, i), STATE, "before cflx_chol_set_local")]
            + on_lu_factors() + ch_factors)

        # ---- after set_local, before a factorisation
        ok(L.cflx_lu_set_local(lu, A.ctypes.data))
        ok(L.cflx_chol_set_local(ch, S.ctypes.data))
        run([("cflx_lu_factor_fixed", (lu, None, 0.0, i, i, d), STATE, "perm = NULL before any factorisation")]
            + on_lu_factors() + ch_factors)

        # ---- after a factorisation: the arguments
        ok(L.cflx_lu_factor(lu, d))
        ok(L.cflx_chol_factor(ch, d))
        s3 = NRHS - 1
        run([
            ("cflx_lu_info", (lu, None), ARG, "!o"),
            ("cflx_lu_set_local", (lu, None), ARG, "!host_local"),
            ("cflx_lu_queue_next_local", (lu, None), ARG, "!host_next"),
            ("cflx_lu_factor_fixed", (lu, None, -1.0, i, i, d), ARG, "!(tiny >= 0.0)"),
            ("cflx_lu_factor_fixed", (lu, None, float("nan"), i, i, d), ARG, "!(tiny >= 0.0)"),
            ("cflx_lu_factor_fixed", (lu, None, 0.0, i, None, d), ARG, "!info_out"),
            ("cflx_lu_factor_fixed", (lu, np.zeros(N, np.int32).ctypes.data, 0.0, i, i, d), ARG, "not a permutation"),
            ("cflx_lu_rbt", (lu, 0, 0, None, None), ARG, "depth < 1"),
            ("cflx_lu_rbt", (lu, 5, 0, None, None), ARG, "depth > 4"),
            ("cflx_lu_rbt_solve", (lu, 2, NRHS, b, NRHS, x, NRHS, 0, d, d), ARG, "trans != 0 && trans != 1"),
            ("cflx_lu_rbt_solve", (lu, 0, NRHS, b, NRHS, x, NRHS, 2, d, d), ARG, "refine != 0 && refine != 1"),
            ("cflx_lu_rbt_solve", (lu, 0, NRHS, b, NRHS, None, NRHS, 0, d, d), ARG, "x_required && !X"),
            ("cflx_lu_rbt_solve", (lu, 0, NRHS, b, s3, x, NRHS, 0, d, d), ARG, "ldb < nrhs"),
            ("cflx_lu_rbt_solve", (lu, 0, NRHS, b, NRHS, x, NRHS, 0, d, d), STATE, NO_RBT),
            ("cflx_lu_rbt_apply_local", (lu, -1, NRHS, bl, 32), ARG, "op < 0"),
            ("cflx_lu_rbt_apply_local", (lu, 4, NRHS, bl, 32), ARG, "op > 3"),
            ("cflx_lu_rbt_apply_local", (lu, 0, 0, bl, 32), ARG, "nrhs < 1"),
            ("cflx_lu_rbt_apply_local", (lu, 0, NRHS, None, 32), ARG, "!B_local"),
            ("cflx_lu_rbt_apply_local", (lu, 0, NRHS, bl, 31), ARG, "ldb < ncl"),
            ("cflx_lu_rbt_apply_local", (lu, 0, NRHS, bl, 32), STATE, NO_RBT),
            ("cflx_lu_get_permutation", (lu, None), ARG, "!perm_out"),
            ("cflx_lu_residual", (lu, None), ARG, "!rel_out"),
            ("cflx_lu_solve", (lu, 0, b, NRHS, x, NRHS), ARG, "nrhs < 1"),
            ("cflx_lu_solve", (lu, NRHS, None, NRHS, x, NRHS), ARG, "!B"),
            ("cflx_lu_solve", (lu, NRHS, b, s3, x, NRHS), ARG, "ldb < nrhs"),
            ("cflx_lu_solve", (lu, NRHS, b, NRHS, x, s3), ARG, "X && ldx < nrhs"),
            ("cflx_lu_solve", (lu, NRHS, b, NRHS, None, 0), 0, None),   # X NULL: ldx is not read
            ("cflx_lu_solve_trans", (lu, NRHS, b, s3, x, NRHS), ARG, "ldb < nrhs"),
            ("cflx_lu_solve_trans", (lu, NRHS, b, NRHS, x, s3), ARG, "X && ldx < nrhs"),
            ("cflx_lu_solve_trans", (lu, NRHS, b, NRHS, None, 0), 0, None),
            ("cflx_lu_solve_local", (lu, 2, NRHS, bl, 32, xl, 32), ARG, "trans != 0 && trans != 1"),
            ("cflx_lu_solve_local", (lu, 0, 0, bl, 32, xl, 32), ARG, "nrhs < 1"),
            ("cflx_lu_solve_local", (lu, 0, NRHS, None, 32, xl, 32), ARG, "!B"),
            ("cflx_lu_solve_local", (lu, 0, NRHS, bl, 31, xl, 32), ARG, "ldb < local_cols"),
            ("cflx_lu_solve_local", (lu, 0, NRHS, bl, 32, xl, 31), ARG, "ldx < local_cols"),
            ("cflx_lu_solve_local", (lu, 0, NRHS, bl, 32, bl, 33), ARG, "X_local == B_local needs ldx == ldb"),
            ("cflx_lu_rcond", (lu, None, d), ARG, "!rcond_out"),
            ("cflx_lu_refine", (lu, 2, NRHS, b, NRHS, x, NRHS, d, d), ARG, "trans != 0 && trans != 1"),
            ("cflx_lu_refine", (lu, 0, NRHS, b, NRHS, None, NRHS, d, d), ARG, "x_required && !X"),
            ("cflx_lu_refine", (lu, 0, NRHS, b, NRHS, x, s3, d, d), ARG, "X && ldx < nrhs"),
            ("cflx_lu_refine_x", (lu, -1, NRHS, b, NRHS, x, NRHS, d, d, d, d, i), ARG, "trans != 0 && trans != 1"),
            ("cflx_lu_refine_x", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, None, d, i), ARG, "!err_bnds_norm_out"),
            ("cflx_lu_refine_x", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, d, d, None), ARG, "!info_out"),
            ("cflx_lu_equilibrate", (lu, 2, d, d, d, d, d, ch_, i), ARG, "apply != 0 && apply != 1"),
            ("cflx_lu_equilibrate", (lu, 0, d, d, d, d, d, ch_, None), ARG, "!info_out"),
            ("cflx_lu_equilibrate_b", (lu, -1, d, d, d, d, d, ch_, i), ARG, "apply != 0 && apply != 1"),
            ("cflx_lu_svx", (lu, 2, NRHS, b, NRHS, x, NRHS, d, d, d, d, ch_, i), ARG, "trans != 0 && trans != 1"),
            ("cflx_lu_svx", (lu, 0, NRHS, b, s3, x, NRHS, d, d, d, d, ch_, i), ARG, "ldb < nrhs"),
            ("cflx_lu_svx", (lu, 0, NRHS, b, NRHS, x, NRHS, None, d, d, d, ch_, i), ARG, "!rcond_out"),
            ("cflx_lu_svx", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, d, d, ch_, None), ARG, "!info_out"),
            ("cflx_lu_svxx", (lu, 0, NRHS, b, NRHS, x, NRHS, None, d, d, d, d, ch_, i), ARG, "!rcond_out"),
            ("cflx_lu_svxx", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, d, None, d, ch_, i), ARG, "!err_bnds_norm_out"),
            ("cflx_lu_svxx", (lu, 0, NRHS, b, NRHS, x, NRHS, d, d, d, d, d, ch_, None), ARG, "!info_out"),
            ("cflx_lu_inverse", (lu, f, None), ARG, "!info_out"),
            ("cflx_lu_det", (lu, 2, d, d, d, i64, i), ARG, "unscaled != 0 && unscaled != 1"),
            ("cflx_lu_det", (lu, 0, d, d, d, i64, None), ARG, "!info_out"),
            ("cflx_lu_launch_count", (lu, None, 0), ARG, "!count_out"),
            ("cflx_lu_set_profiling", (lu, 3), ARG, "mode > 2"),
            ("cflx_lu_set_profiling", (lu, -1), ARG, "mode < 0"),
            ("cflx_lu_phase_ms", (lu, None), ARG, "!ms_out"),
            ("cflx_lu_trailing_stats", (lu, None, d), ARG, "!ms_out"),
            ("cflx_lu_trailing_stats", (lu, d, None), ARG, "!flops_out"),
            ("cflx_chol_info", (ch, None), ARG, "!o"),
            ("cflx_chol_set_local", (ch, None), ARG, "!host_local"),
            ("cflx_chol_get_local", (ch, None), ARG, "!L_host"),
            ("cflx_chol_solve", (ch, 0, b, NRHS, x, NRHS), ARG, "nrhs < 1"),
            ("cflx_chol_solve", (ch, NRHS, None, NRHS, x, NRHS), ARG, "!B"),
            ("cflx_chol_solve", (ch, NRHS, b, s3, x, NRHS), ARG, "ldb < nrhs"),
            ("cflx_chol_solve", (ch, NRHS, b, NRHS, x, s3), ARG, "X && ldx < nrhs"),
            ("cflx_chol_solve", (ch, NRHS, b, NRHS, None, 0), 0, None),
            ("cflx_chol_solve_local", (ch, 0, bl, 32, xl, 32), ARG, "nrhs < 1"),
            ("cflx_chol_solve_local", (ch, NRHS, bl, 31, xl, 32), ARG, "ldb < local_cols"),
            ("cflx_chol_solve_local", (ch, NRHS, bl, 32, xl, 31), ARG, "ldx < local_cols"),
            ("cflx_chol_rcond", (ch, None, d), ARG, "!rcond_out"),
            ("cflx_chol_refine", (ch, NRHS, b, NRHS, None, NRHS, d, d), ARG, "x_required && !X"),
            ("cflx_chol_refine", (ch, NRHS, b, NRHS, x, s3, d, d), ARG, "X && ldx < nrhs"),
            ("cflx_chol_refine_x", (ch, NRHS, b, NRHS, x, NRHS, d, d, None, d, i), ARG, "!err_bnds_norm_out"),
            ("cflx_chol_refine_x", (ch, NRHS, b, NRHS, x, NRHS, d, d, d, d, None), ARG, "!info_out"),
            ("cflx_chol_equilibrate", (ch, 2, d, d, d, ch_, i), ARG, "apply != 0 && apply != 1"),
            ("cflx_chol_equilibrate_b", (ch, 0, d, d, d, ch_, None), ARG, "!info_out"),
            ("cflx_chol_svx", (ch, NRHS, b, NRHS, x, NRHS, None, d, d, ch_, i), ARG, "!rcond_out"),
            ("cflx_chol_svx", (ch, NRHS, b, NRHS, x, NRHS, d, d, d, ch_, None), ARG, "!info_out"),
            ("cflx_chol_svxx", (ch, NRHS, b, NRHS, x, NRHS, None, d, d, d, d, ch_, i), ARG, "!rcond_out"),
            ("cflx_chol_svxx", (ch, NRHS, b, NRHS, x, NRHS, d, d, d, None, d, ch_, i), ARG, "!err_bnds_norm_out"),
            ("cflx_chol_svxx", (ch, NRHS, b, NRHS, x, NRHS, d, d, d, d, d, ch_, None), ARG, "!info_out"),
            ("cflx_chol_det", (ch, 2, d, d, i64), ARG, "unscaled != 0 && unscaled != 1"),
            ("cflx_chol_launch_count", (ch, None, 0), ARG, "!count_out"),
        ])

        # ---- after a factorisation that handed its input buffer to the queued next matrix
        nxt[...] = A
        ok(L.cflx_lu_queue_next_local(lu, nxt.ctypes.data))
        ok(L.cflx_lu_factor(lu, d))
        run(on_lu_factors(own_only=True))

        # ---- a scaled input, a transformed input
        ok(L.cflx_lu_set_local(lu, A_scaled.ctypes.data))
        ok(L.cflx_lu_equilibrate(lu, 1, d, d, d, d, d, ch_, i))
        assert ch_.value in (b"R", b"B")
        run([("cflx_lu_equilibrate", (lu, 1, d, d, d, d, d, ch_, i), STATE, "already scaled"),
             ("cflx_lu_equilibrate_b", (lu, 1, d, d, d, d, d, ch_, i), STATE, "already scaled"),
             ("cflx_lu_rbt", (lu, 2, 0, None, None), STATE, "scaled (equed")])
        ok(L.cflx_lu_set_local(lu, A.ctypes.data))
        ok(L.cflx_lu_rbt(lu, 2, 0, None, None))
        run([("cflx_lu_equilibrate", (lu, 1, d, d, d, d, d, ch_, i), STATE, "random butterfly transform"),
             ("cflx_lu_rbt", (lu, 2, 0, None, None), STATE, "already transformed")])
        ok(L.cflx_chol_set_local(ch, S_scaled.ctypes.data))
        ok(L.cflx_chol_equilibrate(ch, 1, d, d, d, ch_, i))
        assert ch_.value == b"Y"
        run([("cflx_chol_equilibrate", (ch, 1, d, d, d, ch_, i), STATE, "already scaled"),
             ("cflx_chol_equilibrate_b", (ch, 1, d, d, d, ch_, i), STATE, "already scaled")])

        # ---- a Cholesky factorisation that found a non-positive pivot
        ok(L.cflx_chol_set_local(ch, S_bad.ctypes.data))
        run([("cflx_chol_factor", (ch, d), STATE, "not positive definite")] + ch_factors)
    finally:
        L.cflx_lu_destroy(lu)
        L.cflx_chol_destroy(ch)
        L.cflx_comm_destroy(comm)
        cb.pinned_free(nxt)
    return bad


@pytest.mark.gpu
def test_documented_refusals_on_the_handles():
    L = _lib.lib()
    bad = _walk(L)
    assert not bad, "\n".join(map(str, bad))
