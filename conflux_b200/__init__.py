"""conflux_b200 -- H100-native (sm_90a) implementation of CONFLUX's LU hot path.

Python mirror of the reference's driver-facing interface for this path (same names, argument meaning and
error behaviour; reference file:line relative to eth-cscs/conflux):

    lu_params(M, N, v[, Px, Py, Pz], comm)   src/conflux/lu/lu_params.hpp:401-409   sizes, grid, InitMatrix, data
    LU_rep(params, C, permutation) -> ms      src/conflux/lu/conflux_opt.hpp:343-346 the factorisation

All arithmetic happens in libconflux_b200.so (hand-written CUDA, include/conflux_b200.h is the C ABI);
this package is a thin ctypes host layer and never falls back to a CPU path.
"""
import ctypes

import numpy as np

from ._lib import ConfluxError, LIB_PATH, SYMBOLS, ShareLayout, check, lib

__all__ = ["pinned_empty", "pinned_free", "Comm", "lu_params", "LU_rep", "LU_rep_fixed", "rbt_multipliers", "LU_rep_rbt", "lu_rbt_solve", "lu_rbt_apply_local", "residual", "validate", "lu_solve", "lu_rcond", "lu_refine", "lu_refine_x", "lu_equilibrate", "lu_svx", "lu_equilibrate_b", "lu_svxx", "lu_inverse", "lu_det", "rhs_local_cols", "lu_solve_local", "refine_block_cols", "lu_refine_local", "lu_refine_x_local", "lu_svx_local", "lu_svxx_local", "timeline", "auto_grid", "lu_dims", "init_matrix_host", "ConfluxError", "dbg", "cholesky", "chol_dims", "chol_auto_grid"]


def auto_grid(M, N, P):
    """lu_params::get_p_grid (lu_params.hpp:21-47)."""
    px, py, pz = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    check(lib().cflx_auto_grid(int(M), int(N), int(P), ctypes.byref(px), ctypes.byref(py), ctypes.byref(pz)), "auto_grid")
    return px.value, py.value, pz.value


def lu_dims(M, N, v, Px, Py, Pz):
    """Padded sizes exactly as lu_params::initialize (lu_params.hpp:67-82)."""
    o = (ctypes.c_int * 8)()
    check(lib().cflx_lu_dims(int(M), int(N), int(v), int(Px), int(Py), int(Pz), o), "lu_dims")
    return dict(M=o[0], N=o[1], Ml=o[2], Nl=o[3], Nt=o[4], nlayr=o[5], Mt=o[6], P=o[7])


def init_matrix_host(M, N, v, Px, Py, Pz, rank, seed=42, out=None):
    """lu_params::InitMatrix, random branch (lu_params.hpp:364-375) for one rank."""
    d = lu_dims(M, N, v, Px, Py, Pz)
    if out is None:
        out = np.empty((d["Ml"], d["Nl"]), dtype=np.float64)
    check(lib().cflx_init_matrix_host(int(M), int(N), int(v), int(Px), int(Py), int(Pz), int(rank), int(seed),
                                      out.ctypes.data), "init_matrix_host")
    return out


def pinned_empty(shape, dtype=np.float64):
    """numpy array backed by page-locked host memory (cudaHostAlloc) -- staging for LU_rep's host->device copy."""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = ctypes.c_void_p()
    check(lib().cflx_host_alloc(n, ctypes.byref(p)), "host_alloc")
    buf = (ctypes.c_char * n).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype).reshape(shape)
    _PINNED[arr.ctypes.data] = p
    return arr


_PINNED = {}


def pinned_free(arr):
    p = _PINNED.pop(arr.ctypes.data, None)
    if p is not None:
        lib().cflx_host_free(p)


class Comm:
    """Process-grid handle: the MPI_Comm of the reference.  One per rank (= per GPU)."""

    def __init__(self, world_size=1, rank=0, unique_id=None, device=0):
        self.world_size, self.rank, self.device = int(world_size), int(rank), int(device)
        self._h = ctypes.c_void_p()
        idbuf = None
        if unique_id is not None:
            idbuf = ctypes.create_string_buffer(bytes(unique_id), 128)
        check(lib().cflx_comm_create(self.world_size, self.rank, idbuf, self.device, ctypes.byref(self._h)), "comm_create")

    @staticmethod
    def unique_id():
        buf = ctypes.create_string_buffer(128)
        check(lib().cflx_get_unique_id(buf), "get_unique_id")
        return bytes(buf.raw)

    @classmethod
    def from_torch_distributed(cls, device=None):
        """Bootstrap over an initialised torch.distributed group (plumbing only): rank 0's NCCL id is broadcast."""
        import torch
        import torch.distributed as dist
        if not dist.is_initialized() or dist.get_world_size() == 1:
            return cls(1, 0, None, 0 if device is None else device)
        rank, world = dist.get_rank(), dist.get_world_size()
        obj = [cls.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(obj, src=0)
        if device is None:
            device = rank % max(1, torch.cuda.device_count())
        return cls(world, rank, obj[0], device)

    def barrier(self):
        check(lib().cflx_comm_barrier(self._h), "comm_barrier")

    def close(self):
        if self._h:
            lib().cflx_comm_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class lu_params:
    """Mirror of conflux::lu_params<double> (lu_params.hpp:8-459): public fields M, N, P, Ml, Nl, Px, Py, Pz, v,
    nlayr, Mt, Nt, pi, pj, pk, rank, seed, data (Ml x Nl numpy array owned by the object), InitMatrix(),
    free_comms().  `comm` is a conflux_b200.Comm instead of an MPI_Comm."""

    def __init__(self, M, N, v, *grid_and_comm):
        if len(grid_and_comm) == 1:
            (comm,) = grid_and_comm
            Px = Py = Pz = -1
        elif len(grid_and_comm) == 4:
            Px, Py, Pz, comm = grid_and_comm
        else:
            raise TypeError("lu_params(M, N, v, comm) or lu_params(M, N, v, Px, Py, Pz, comm)")
        self.lu_comm = comm
        self.seed = 42
        self._h = ctypes.c_void_p()
        check(lib().cflx_lu_create(comm._h, int(M), int(N), int(v), int(Px), int(Py), int(Pz), ctypes.byref(self._h)),
              "lu_create")
        info = (ctypes.c_int * 16)()
        check(lib().cflx_lu_info(self._h, info), "lu_info")
        (self.M, self.N, self.Ml, self.Nl, self.Nt, self.nlayr, self.P, self.Px, self.Py, self.Pz, self.pi, self.pj,
         self.pk, self.rank, self.v) = list(info)[:15]
        self.Mt = self.M // self.v
        self.tA11x, self.tA11y = self.Ml // self.v, self.Nl // self.v
        self.use_collectives = self.v > 1024
        self.data = np.zeros((self.Ml, self.Nl), dtype=np.float64)
        self.InitMatrix()

    def InitMatrix(self):
        init_matrix_host(self.M, self.N, self.v, self.Px, self.Py, self.Pz, self.rank, self.seed, out=self.data)

    def free_comms(self):
        if self._h:
            lib().cflx_lu_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.free_comms()
        except Exception:
            pass


def LU_rep(gv, C=None, permutation=None, upload=True, next_data=None):
    """conflux::LU_rep<double>(gv, C, permutation) (conflux_opt.hpp:343-346): collective over gv.lu_comm, does not
    modify gv.data, fills C (Ml x Nl, L\\U of PA in the conflux layout, layer 0) and permutation (M ints) when they
    are given, returns the time of the main loop in ms (device-timed).

    upload=True copies gv.data to the device first; upload=False factors the input that is already there (the previous
    one, or the matrix a previous call streamed in through next_data).  next_data (page-locked array of gv.data's shape):
    the input of the NEXT factorisation, uploaded on a copy stream while this one runs (cflx_lu_queue_next_local)."""
    if upload:
        a = np.ascontiguousarray(gv.data, dtype=np.float64)
        check(lib().cflx_lu_set_local(gv._h, a.ctypes.data), "lu_set_local")
    if next_data is not None:
        assert next_data.dtype == np.float64 and next_data.flags.c_contiguous and next_data.size == gv.Ml * gv.Nl
        check(lib().cflx_lu_queue_next_local(gv._h, next_data.ctypes.data), "lu_queue_next_local")
    ms = ctypes.c_double()
    check(lib().cflx_lu_factor(gv._h, ctypes.byref(ms)), "lu_factor")
    if C is not None:
        assert C.dtype == np.float64 and C.flags.c_contiguous and C.size >= gv.Ml * gv.Nl
        if permutation is None:
            permutation = np.empty(gv.M, dtype=np.int32)
        check(lib().cflx_lu_get_factors(gv._h, C.ctypes.data, permutation.ctypes.data), "lu_get_factors")
    elif permutation is not None:
        assert permutation.dtype == np.int32 and permutation.size >= gv.M
        check(lib().cflx_lu_get_permutation(gv._h, permutation.ctypes.data), "lu_get_permutation")
    return ms.value


def LU_rep_fixed(gv, perm=None, tiny=0.0, C=None, permutation=None, upload=True, next_data=None):
    """LU_rep with a prescribed row order instead of the pivot search (cflx_lu_factor_fixed): P A = L U with row q of
    P A = row perm[q] of A.  perm (M ints, the same on every rank) defaults to the permutation of the last completed
    factorisation of gv, so that a nearby matrix is factored with the pivots of the previous one.  tiny >= 0: pivots
    with |u| < tiny become copysign(tiny, u) (+tiny for +-0).  C, permutation, upload and next_data as LU_rep.
    COLLECTIVE.  Returns (ms, nrepl, info): the main loop's device time, the pivots replaced over the grid, and 1 + the
    global column of the first exactly zero pivot (0: none), identical on every rank."""
    if upload:
        a = np.ascontiguousarray(gv.data, dtype=np.float64)
        check(lib().cflx_lu_set_local(gv._h, a.ctypes.data), "lu_set_local")
    if next_data is not None:
        assert next_data.dtype == np.float64 and next_data.flags.c_contiguous and next_data.size == gv.Ml * gv.Nl
        check(lib().cflx_lu_queue_next_local(gv._h, next_data.ctypes.data), "lu_queue_next_local")
    p = None
    if perm is not None:
        p = np.ascontiguousarray(perm, dtype=np.int32)
        if p.shape != (gv.M,):
            raise ValueError(f"LU_rep_fixed: perm must have shape ({gv.M},), got {p.shape}")
    ms, nrepl, info = ctypes.c_double(), ctypes.c_int(), ctypes.c_int()
    check(lib().cflx_lu_factor_fixed(gv._h, _ptr(p), float(tiny), ctypes.byref(nrepl), ctypes.byref(info),
                                     ctypes.byref(ms)), "lu_factor_fixed")
    if C is not None:
        assert C.dtype == np.float64 and C.flags.c_contiguous and C.size >= gv.Ml * gv.Nl
        if permutation is None:
            permutation = np.empty(gv.M, dtype=np.int32)
        check(lib().cflx_lu_get_factors(gv._h, C.ctypes.data, permutation.ctypes.data), "lu_get_factors")
    elif permutation is not None:
        assert permutation.dtype == np.int32 and permutation.size >= gv.M
        check(lib().cflx_lu_get_permutation(gv._h, permutation.ctypes.data), "lu_get_permutation")
    return ms.value, nrepl.value, info.value


def rbt_multipliers(M, depth, seed):
    """The multipliers r of cflx_lu_rbt's butterflies U and V for an order-M matrix (cflx_rbt_multipliers, pure host):
    (u, v), two (depth, M) arrays, row l = level l, every r in [e^-0.05, e^0.05]."""
    u, v = np.empty((int(depth), int(M))), np.empty((int(depth), int(M)))
    check(lib().cflx_rbt_multipliers(int(M), int(depth), ctypes.c_uint64(int(seed)), u.ctypes.data, v.ctypes.data),
          "rbt_multipliers")
    return u, v


def LU_rep_rbt(gv, depth=2, seed=0, tiny=0.0, upload=True, C=None, permutation=None, u_out=None, v_out=None):
    """The LU of a random butterfly transform of the input, without the pivot search (MAGMA's dgesv_rbt): cflx_lu_rbt
    replaces the input A by W = U^T A V (U, V random recursive butterflies of `depth` levels from `seed`, the same on every
    rank), then cflx_lu_factor_fixed factors W in the identity order with the tiny rule of LU_rep_fixed.  Solve with
    lu_rbt_solve, or lu_rbt_apply_local around lu_solve_local.  Every other call on the factors (lu_solve, lu_rcond, lu_svx,
    validate, ...) refers to W.  gv.M must be a multiple of 2**depth * v * Px.  upload=True copies gv.data to the device
    first; upload=False transforms the input already there.  C and permutation as LU_rep; u_out / v_out ((depth, M)
    float64 arrays) receive the multipliers.  COLLECTIVE.  Returns (ms, nrepl, info) as LU_rep_fixed."""
    if upload:
        a = np.ascontiguousarray(gv.data, dtype=np.float64)
        check(lib().cflx_lu_set_local(gv._h, a.ctypes.data), "lu_set_local")
    for o in (u_out, v_out):
        if o is not None:
            assert o.dtype == np.float64 and o.flags.c_contiguous and o.size == depth * gv.M
    check(lib().cflx_lu_rbt(gv._h, int(depth), ctypes.c_uint64(int(seed)), _ptr(u_out), _ptr(v_out)), "lu_rbt")
    return LU_rep_fixed(gv, perm=np.arange(gv.M, dtype=np.int32), tiny=tiny, C=C, permutation=permutation, upload=False)


def lu_rbt_solve(gv, B, trans=False, refine=True):
    """Solves A X = B (A^T X = B when trans) with factors of a transformed input (LU_rep_rbt): X = V inv(W) U^T B, or
    U inv(W)^T V^T B.  refine=True refines the transformed system's solution as lu_refine does.  Returns (X, ferr, berr):
    X in B's shape, and with refine the forward and backward errors of the transformed system (None without).  B as
    lu_solve.  COLLECTIVE over gv.lu_comm; identical on every rank."""
    B, B2, nrhs = _rhs(gv.M, B, "lu_rbt_solve")
    X = np.empty_like(B2)
    fe, be = np.empty(nrhs), np.empty(nrhs)
    check(lib().cflx_lu_rbt_solve(gv._h, 1 if trans else 0, nrhs, B2.ctypes.data, nrhs, X.ctypes.data, nrhs,
                                  1 if refine else 0, fe.ctypes.data, be.ctypes.data), "lu_rbt_solve")
    return X.reshape(B.shape), (fe if refine else None), (be if refine else None)


def lu_rbt_apply_local(gv, op, B_share, nrhs):
    """One butterfly of the factors' transform (LU_rep_rbt) on the rows of this rank's right-hand side share, in place:
    op 0 U^T, 1 V, 2 V^T, 3 U.  B_share as lu_solve_local's (a NumPy array or a torch CUDA tensor, (gv.Ml, n >=
    rhs_local_cols(nrhs, gv.v, gv.Py)) float64 with contiguous rows).  A X = B distributed: lu_rbt_apply_local(gv, 0, B),
    lu_solve_local, lu_rbt_apply_local(gv, 1, X); A^T X = B: ops 2 and 3 around the transposed solve.  Not collective.
    Returns B_share."""
    ptr, out, ld = _share_out(B_share, gv.Ml, rhs_local_cols(nrhs, gv.v, gv.Py), "lu_rbt_apply_local", strided=True,
                              name="B_share")
    check(lib().cflx_lu_rbt_apply_local(gv._h, int(op), int(nrhs), ptr, ld), "lu_rbt_apply_local")
    return out


def timeline(gv):
    """Per-region device time of the last LU_rep run under cflx_lu_set_profiling(gv._h, 1 or 2): dict(main={region: (ms,
    count)}, side={...}); region names are the reference's semiprof regions."""
    import json
    n = lib().cflx_lu_timeline(gv._h, None, 0)
    buf = ctypes.create_string_buffer(max(n, 2))
    check(lib().cflx_lu_timeline(gv._h, buf, n), "lu_timeline")
    return json.loads(buf.value.decode())


def validate(gv):
    """The reference's validation (examples/conflux_miniapp.cpp:349-500) of the last LU_rep on the GPU grid.
    COLLECTIVE over gv.lu_comm.  Returns (||PA - LU||_F, ||PA - LU||_F / ||A||_F), identical on every rank."""
    a, r = ctypes.c_double(), ctypes.c_double()
    check(lib().cflx_lu_validate(gv._h, ctypes.byref(a), ctypes.byref(r)), "lu_validate")
    return a.value, r.value


def residual(gv):
    """||PA - LU||_F / ||A||_F of the last LU_rep, computed on the GPU grid (collective)."""
    return validate(gv)[1]


def _rhs(n, B, what):
    """B as float64, checked to be (n,) or (n, nrhs): (B, B as a C-contiguous n x nrhs array, nrhs)."""
    B = np.asarray(B, dtype=np.float64)
    if B.ndim not in (1, 2) or B.shape[0] != n:
        raise ValueError(f"{what}: B must have shape ({n},) or ({n}, nrhs), got {B.shape}")
    B2 = np.ascontiguousarray(B.reshape(n, -1))
    return B, B2, B2.shape[1]


def lu_solve(gv, B, trans=False):
    """Solves A X = B (A^T X = B when trans) with the factors of the last LU_rep (P A = L U) on the GPU grid, like
    LAPACK's getrs.  COLLECTIVE over gv.lu_comm; every rank passes the same B, (M,) or (M, nrhs) with M = gv.M (the padded
    size), and gets the same X in the same shape.  The factors and the input matrix are left as they are."""
    B, B2, nrhs = _rhs(gv.M, B, "lu_solve")
    X = np.empty_like(B2)
    fn = lib().cflx_lu_solve_trans if trans else lib().cflx_lu_solve
    check(fn(gv._h, nrhs, B2.ctypes.data, max(nrhs, 1), X.ctypes.data, max(nrhs, 1)), "lu_solve")
    return X.reshape(B.shape)


_PREC = {"tf32": 1, "tf32x3": 3}


def _sv_mixed(fn, what, h, n, B, prec, itmax):
    if prec not in _PREC:
        raise ValueError(f"{what}: prec must be one of {sorted(_PREC)}, got {prec!r}")
    B, B2, nrhs = _rhs(n, B, what)
    X = np.empty_like(B2)
    be = np.empty(nrhs)
    it, ms = ctypes.c_int(), ctypes.c_double()
    check(fn(h, _PREC[prec], nrhs, B2.ctypes.data, nrhs, X.ctypes.data, nrhs, int(itmax), ctypes.byref(it), be.ctypes.data,
             ctypes.byref(ms)), what)
    return X.reshape(B.shape), it.value, be


def lu_sv_mixed(gv, B, prec="tf32x3", itmax=0, upload=True):
    """LAPACK dsgesv on the GPU grid: factors the input (upload=True copies gv.data to the device first; upload=False
    takes the one already there) with the trailing update on the TF32 tensor cores (prec "tf32": one term, "tf32x3": three), then refines x in FP64 against
    that input until ||b - A x||_inf <= ||x||_inf ||A||_inf eps sqrt(M) for every column, at most itmax corrections (0:
    30).  Returns (X, iter, berr): X in B's shape; iter the corrections taken, -3 (a zero pivot) or -31 (no convergence),
    in which case X comes from an FP64 refactorisation exactly as LU_rep + lu_solve give it; berr per column ||r||_inf /
    (||A||_inf ||x||_inf).  After a converged run the handle holds the low-precision factors: lu_solve, lu_refine and the
    other calls that need FP64 factors refuse until the next LU_rep.  COLLECTIVE; identical on every rank."""
    if upload:
        a = np.ascontiguousarray(gv.data, dtype=np.float64)
        check(lib().cflx_lu_set_local(gv._h, a.ctypes.data), "lu_set_local")
    return _sv_mixed(lib().cflx_lu_sv_mixed, "lu_sv_mixed", gv._h, gv.M, B, prec, itmax)


def lu_rcond(gv):
    """LAPACK dgecon (1-norm) of the last LU_rep on the GPU grid: (rcond, anorm) with anorm = ||A||_1 of the padded input
    and rcond = 1 / (anorm * estimate of ||A^-1||_1), 0 for an exactly singular U.  COLLECTIVE; identical on every rank."""
    r, a = ctypes.c_double(), ctypes.c_double()
    check(lib().cflx_lu_rcond(gv._h, ctypes.byref(r), ctypes.byref(a)), "lu_rcond")
    return r.value, a.value


def _refine_args(n, B, X, what):
    B, B2, nrhs = _rhs(n, B, what)
    X = np.asarray(X, dtype=np.float64)
    if X.shape != B.shape:
        raise ValueError(f"{what}: X must have the shape of B, {B.shape}, got {X.shape}")
    X2 = np.array(X.reshape(n, -1), dtype=np.float64, order="C")
    return B.shape, B2, X2, nrhs, np.empty(nrhs), np.empty(nrhs)


def lu_refine(gv, B, X, trans=False, ferr=True):
    """LAPACK dgerfs with the factors of the last LU_rep on the GPU grid: refines X, a solution of A X = B (A^T X = B when
    trans), e.g. from lu_solve, and returns (X, ferr, berr) -- the refined X in B's shape, and per right-hand side the
    estimated forward error bound ||x - x_true||_inf / ||x||_inf and the componentwise backward error.  ferr=False skips
    the estimator (ferr is then None).  COLLECTIVE over gv.lu_comm; every rank passes the same B and X and gets the same
    results.  The factors, the input and later solves are left as they are."""
    shape, B2, X2, nrhs, fe, be = _refine_args(gv.M, B, X, "lu_refine")
    check(lib().cflx_lu_refine(gv._h, 1 if trans else 0, nrhs, B2.ctypes.data, nrhs, X2.ctypes.data, nrhs,
                               fe.ctypes.data if ferr else None, be.ctypes.data), "lu_refine")
    return X2.reshape(shape), (fe if ferr else None), be


def _refine_x(fn, n, B, X, cwise, what, *lead):
    shape, B2, X2, nrhs, be, _ = _refine_args(n, B, X, what)
    en, ec = np.zeros((nrhs, 3)), np.zeros((nrhs, 3))
    rcond, info = ctypes.c_double(), ctypes.c_int()
    check(fn(*lead, nrhs, B2.ctypes.data, nrhs, X2.ctypes.data, nrhs, ctypes.byref(rcond), be.ctypes.data, en.ctypes.data,
             ec.ctypes.data if cwise else None, ctypes.byref(info)), what)
    return X2.reshape(shape), dict(rcond=rcond.value, berr=be, err_norm=en, err_comp=ec if cwise else None,
                                   info=info.value)


def lu_refine_x(gv, B, X, trans=False, cwise=True):
    """LAPACK dgerfsx with the factors of the last LU_rep on the GPU grid: refines X, a solution of A X = B (A^T X = B
    when trans), with residuals in double-double, to full working accuracy whenever the problem is not too
    ill-conditioned.  Returns (X, dict(rcond, berr, err_norm, err_comp, info)): err_norm and err_comp are nrhs x 3 rows
    {trust, err, rcond} (LAPACK's ERR_BNDS) bounding the normwise and componentwise relative errors of the solution,
    trusted where trust is 1; cwise=False neither pursues nor estimates componentwise accuracy (err_comp is None).  info
    = k for an exactly zero U(k,k) (X returned as given), M + j when column j's bound was set to 1 because the problem is
    too ill-conditioned, else 0.  COLLECTIVE over gv.lu_comm; identical on every rank.  The factors, the input and
    later solves are left as they are."""
    return _refine_x(lib().cflx_lu_refine_x, gv.M, B, X, cwise, "lu_refine_x", gv._h, 1 if trans else 0)


def _lu_equilibrate(gv, apply, upload, fn, what):
    if upload:
        a = np.ascontiguousarray(gv.data, dtype=np.float64)
        check(lib().cflx_lu_set_local(gv._h, a.ctypes.data), "lu_set_local")
    r, c = np.zeros(gv.M), np.zeros(gv.M)
    rowcnd, colcnd, amax, equed, info = (ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_char(),
                                         ctypes.c_int())
    check(fn(gv._h, 1 if apply else 0, r.ctypes.data, c.ctypes.data, ctypes.byref(rowcnd), ctypes.byref(colcnd),
             ctypes.byref(amax), ctypes.byref(equed), ctypes.byref(info)), what)
    return dict(r=r, c=c, rowcnd=rowcnd.value, colcnd=colcnd.value, amax=amax.value, equed=equed.value.decode(),
                info=info.value)


def lu_equilibrate(gv, apply=True, upload=True):
    """LAPACK dgeequ (+ dlaqge when apply) on the padded input on the GPU grid.  upload=True first copies gv.data to the
    device (cflx_lu_set_local), so that LU_rep(gv, upload=False) then factors the scaled matrix As, whose factors carry
    the scaling to lu_svx.  Returns dict(r, c, rowcnd, colcnd, amax, equed, info) as dgeequ / dlaqge give them.
    COLLECTIVE over gv.lu_comm; identical on every rank."""
    return _lu_equilibrate(gv, apply, upload, lib().cflx_lu_equilibrate, "lu_equilibrate")


def lu_equilibrate_b(gv, apply=True, upload=True):
    """LAPACK dgeequb (+ dlaqge when apply): lu_equilibrate with the scales rounded to powers of two, so that scaling A
    and B and unscaling X are exact.  Arguments and result as lu_equilibrate; the factors carry the scaling to lu_svxx
    (or lu_svx).  COLLECTIVE over gv.lu_comm; identical on every rank."""
    return _lu_equilibrate(gv, apply, upload, lib().cflx_lu_equilibrate_b, "lu_equilibrate_b")


def _svxx(fn, n, B, cwise, what, *lead):
    B, B2, nrhs = _rhs(n, B, what)
    X = np.empty_like(B2)
    be, en, ec = np.empty(nrhs), np.zeros((nrhs, 3)), np.zeros((nrhs, 3))
    rcond, rpvgrw, equed, info = ctypes.c_double(), ctypes.c_double(), ctypes.c_char(), ctypes.c_int()
    check(fn(*lead, nrhs, B2.ctypes.data, nrhs, X.ctypes.data, nrhs, ctypes.byref(rcond), ctypes.byref(rpvgrw),
             be.ctypes.data, en.ctypes.data, ec.ctypes.data if cwise else None, ctypes.byref(equed), ctypes.byref(info)),
          what)
    k = info.value
    solved = not (0 < k <= n)
    return (X.reshape(B.shape) if solved else None), dict(rcond=rcond.value, rpvgrw=rpvgrw.value,
                                                          berr=be if solved else None, err_norm=en if solved else None,
                                                          err_comp=ec if solved and cwise else None,
                                                          equed=equed.value.decode(), info=k)


def lu_svxx(gv, B, trans=False, cwise=True):
    """LAPACK dgesvxx with the factors of the last LU_rep and the scaling they carry (lu_equilibrate_b or
    lu_equilibrate): solves A X = B (A^T X = B when trans) with extra-precise refinement.  Returns (X, dict(rcond,
    rpvgrw, berr, err_norm, err_comp, equed, info)): rpvgrw is dla_gerpvgrw's per-column reciprocal pivot growth, the
    rest as lu_refine_x returns it for the unscaled solution.  X (and berr, err_norm, err_comp) is None when U has an
    exactly zero pivot (info = k).  COLLECTIVE over gv.lu_comm; identical on every rank."""
    return _svxx(lib().cflx_lu_svxx, gv.M, B, cwise, "lu_svxx", gv._h, 1 if trans else 0)


def lu_svx(gv, B, trans=False):
    """LAPACK dgesvx with the factors of the last LU_rep and the scaling they carry (lu_equilibrate): solves A X = B (A^T
    X = B when trans) with refinement.  Returns (X, dict(rcond, ferr, berr, rpvgrw, equed, info)); X is None when U has
    an exactly zero pivot (info = k).  COLLECTIVE over gv.lu_comm; identical on every rank."""
    B, B2, nrhs = _rhs(gv.M, B, "lu_svx")
    X = np.empty_like(B2)
    fe, be = np.empty(nrhs), np.empty(nrhs)
    rcond, rpvgrw, equed, info = ctypes.c_double(), ctypes.c_double(), ctypes.c_char(), ctypes.c_int()
    check(lib().cflx_lu_svx(gv._h, 1 if trans else 0, nrhs, B2.ctypes.data, nrhs, X.ctypes.data, nrhs, ctypes.byref(rcond),
                            fe.ctypes.data, be.ctypes.data, ctypes.byref(rpvgrw), ctypes.byref(equed), ctypes.byref(info)),
          "lu_svx")
    k = info.value
    solved = not (0 < k <= gv.M)
    return (X.reshape(B.shape) if solved else None), dict(rcond=rcond.value, ferr=fe if solved else None,
                                                          berr=be if solved else None, rpvgrw=rpvgrw.value,
                                                          equed=equed.value.decode(), info=k)


def _share_out(out, Ml, Nl, what, strided=False, name="out"):
    """(pointer, array, ld) of the Ml x Nl float64 share an inverse or a distributed solve reads or writes: a new NumPy
    array when out is None, else out itself -- a NumPy array, or any object with __cuda_array_interface__ (a torch CUDA
    tensor).  The share must be C-contiguous (ld = Nl); with strided, any (Ml, n >= Nl) array whose rows are contiguous
    is accepted, ld being its row stride in elements."""
    if out is None:
        out = np.empty((Ml, Nl))
    if isinstance(out, np.ndarray):
        if strided:
            return out.ctypes.data, out, _rows_share(out.dtype == np.float64, out.shape, out.strides, Ml, Nl, what, name,
                                                     "array")
        if out.dtype != np.float64 or not out.flags.c_contiguous or out.shape != (Ml, Nl):
            raise ValueError(f"{what}: {name} must be a C-contiguous float64 array of shape ({Ml}, {Nl}), got {out.dtype} "
                             f"{out.shape}")
        return out.ctypes.data, out, Nl
    cai = getattr(out, "__cuda_array_interface__", None)
    if cai is None:
        raise ValueError(f"{what}: {name} must be a NumPy array or expose __cuda_array_interface__")
    shape, strides = tuple(cai["shape"]), cai.get("strides")
    if strided:
        if strides is None and len(shape) == 2:
            strides = (8 * shape[1], 8)
        return cai["data"][0], out, _rows_share(cai["typestr"] == "<f8", shape, strides, Ml, Nl, what, name,
                                                "device array")
    if cai["typestr"] != "<f8" or shape != (Ml, Nl) or strides not in (None, (8 * Nl, 8)):
        raise ValueError(f"{what}: {name} must be a C-contiguous float64 device array of shape ({Ml}, {Nl}), got "
                         f"{cai['typestr']} {shape} strides {strides}")
    return cai["data"][0], out, Nl


def _rows_share(f8, shape, strides, Ml, Nl, what, name, kind):
    """the row stride in elements of a float64 (Ml, n >= Nl) share with contiguous rows, else ValueError"""
    if (not f8 or len(shape) != 2 or shape[0] != Ml or shape[1] < Nl or strides is None or strides[1] != 8
            or strides[0] % 8 or strides[0] < 8 * shape[1]):
        raise ValueError(f"{what}: {name} must be a float64 {kind} of shape ({Ml}, n >= {Nl}) with contiguous rows, got "
                         f"shape {tuple(shape)} strides {strides}")
    return strides[0] // 8


def lu_inverse(gv, out=None):
    """inv(A) of the padded matrix of the last LU_rep (P A = L U) on the GPU grid, like LAPACK's dgetri: returns (share,
    info), this rank's Ml x Nl share of inv(A) in the conflux layout (layers pk != 0 get layer 0's bits).  info = k when
    U(k,k) is exactly zero (the first such k, counted from 1); the share is then None and out is left as it was.  out: the
    share to write into, a NumPy array or a torch CUDA tensor (float64, C-contiguous, (Ml, Nl)).  The columns are solves
    A X = I, so A X - I is the small residual.  COLLECTIVE over gv.lu_comm; the factors and later solves are left as they
    are."""
    ptr, arr, _ = _share_out(out, gv.Ml, gv.Nl, "lu_inverse")
    info = ctypes.c_int()
    check(lib().cflx_lu_inverse(gv._h, ptr, ctypes.byref(info)), "lu_inverse")
    return (None if info.value else arr), info.value


def rhs_local_cols(nrhs, v, Py):
    """The local columns of an M x nrhs right-hand side share on a grid with Py grid columns (lu_solve_local,
    cholesky.solve_local): v * ceil(ceil(nrhs / v) / Py), so nrhs = M gives the matrix's Nl."""
    n = ctypes.c_int()
    check(lib().cflx_rhs_local_cols(int(nrhs), int(v), int(Py), ctypes.byref(n)), "rhs_local_cols")
    return n.value


def refine_block_cols(v):
    """The block width of the distributed refinement and expert drivers (lu_refine_local ... cholesky.svxx_local) for
    tile size v: the whole number of tiles nearest 256 columns, at least one tile."""
    n = ctypes.c_int()
    check(lib().cflx_refine_block_cols(int(v), ctypes.byref(n)), "refine_block_cols")
    return n.value


def _local_args(what, Ml, v, Py, layer0, B_share, nrhs, X_share, x_in, x_name="out"):
    """(B pointer, ldb, X pointer, ldx, X) of a distributed call: B_share / X_share checked as (Ml, n >= rhs_local_cols)
    float64 shares with contiguous rows.  B_share None is allowed off layer 0 (it is not read there).  x_in: X_share is
    the solution on entry, required on layer 0 and None allowed elsewhere (not written); else X_share None is a new zeroed
    NumPy array."""
    ncl = rhs_local_cols(nrhs, v, Py)
    bptr, ldb = None, ncl
    if B_share is not None:
        bptr, _, ldb = _share_out(B_share, Ml, ncl, what, strided=True, name="B_share")
    elif layer0:
        raise ValueError(f"{what}: B_share is read on layer 0 and may not be None there")
    if X_share is None and x_in:
        if layer0:
            raise ValueError(f"{what}: {x_name} is read on layer 0 and may not be None there")
        return bptr, ldb, None, ncl, None
    if X_share is None:
        X_share = np.zeros((Ml, ncl))
    xptr, X_share, ldx = _share_out(X_share, Ml, ncl, what, strided=True, name=x_name)
    return bptr, ldb, xptr, ldx, X_share


def _solve_local(fn, what, Ml, v, Py, layer0, B_share, nrhs, out, *lead):
    """B_share / out checked as (Ml, n >= rhs_local_cols) float64 shares with contiguous rows; out None: a new zeroed NumPy
    array; B_share None is allowed off layer 0 (it is not read there)"""
    bptr, ldb, xptr, ldx, out = _local_args(what, Ml, v, Py, layer0, B_share, nrhs, out, False)
    check(fn(*lead, int(nrhs), bptr, ldb, xptr, ldx), what)
    return out


def _refine_local(fn, what, Ml, v, Py, layer0, B_share, X_share, nrhs, ferr, *lead):
    bptr, ldb, xptr, ldx, X = _local_args(what, Ml, v, Py, layer0, B_share, nrhs, X_share, True, "X_share")
    fe, be = np.empty(nrhs), np.empty(nrhs)
    check(fn(*lead, int(nrhs), bptr, ldb, xptr, ldx, fe.ctypes.data if ferr else None, be.ctypes.data), what)
    return X, (fe if ferr else None), be


def _refine_x_local(fn, what, Ml, v, Py, layer0, B_share, X_share, nrhs, cwise, *lead):
    bptr, ldb, xptr, ldx, X = _local_args(what, Ml, v, Py, layer0, B_share, nrhs, X_share, True, "X_share")
    be, en, ec = np.empty(nrhs), np.zeros((nrhs, 3)), np.zeros((nrhs, 3))
    rcond, info = ctypes.c_double(), ctypes.c_int()
    check(fn(*lead, int(nrhs), bptr, ldb, xptr, ldx, ctypes.byref(rcond), be.ctypes.data, en.ctypes.data,
             ec.ctypes.data if cwise else None, ctypes.byref(info)), what)
    return X, dict(rcond=rcond.value, berr=be, err_norm=en, err_comp=ec if cwise else None, info=info.value)


def _svx_local(fn, what, M, Ml, v, Py, layer0, B_share, nrhs, out, growth, *lead):
    """cflx_*_svx_local: (X or None when the factors have an exactly zero pivot, dict(rcond, ferr, berr, [rpvgrw,] equed,
    info)); growth: the LU's signature, with rpvgrw_out"""
    bptr, ldb, xptr, ldx, out = _local_args(what, Ml, v, Py, layer0, B_share, nrhs, out, False)
    fe, be = np.empty(nrhs), np.empty(nrhs)
    rcond, rpvgrw, equed, info = ctypes.c_double(), ctypes.c_double(), ctypes.c_char(), ctypes.c_int()
    mid = [ctypes.byref(rpvgrw)] if growth else []
    check(fn(*lead, int(nrhs), bptr, ldb, xptr, ldx, ctypes.byref(rcond), fe.ctypes.data, be.ctypes.data, *mid,
             ctypes.byref(equed), ctypes.byref(info)), what)
    k = info.value
    solved = not (0 < k <= M)
    res = dict(rcond=rcond.value, ferr=fe if solved else None, berr=be if solved else None, equed=equed.value.decode(),
               info=k)
    if growth:
        res["rpvgrw"] = rpvgrw.value
    return (out if solved else None), res


def _svxx_local(fn, what, M, Ml, v, Py, layer0, B_share, nrhs, out, cwise, *lead):
    bptr, ldb, xptr, ldx, out = _local_args(what, Ml, v, Py, layer0, B_share, nrhs, out, False)
    be, en, ec = np.empty(nrhs), np.zeros((nrhs, 3)), np.zeros((nrhs, 3))
    rcond, rpvgrw, equed, info = ctypes.c_double(), ctypes.c_double(), ctypes.c_char(), ctypes.c_int()
    check(fn(*lead, int(nrhs), bptr, ldb, xptr, ldx, ctypes.byref(rcond), ctypes.byref(rpvgrw), be.ctypes.data,
             en.ctypes.data, ec.ctypes.data if cwise else None, ctypes.byref(equed), ctypes.byref(info)), what)
    k = info.value
    solved = not (0 < k <= M)
    return (out if solved else None), dict(rcond=rcond.value, rpvgrw=rpvgrw.value, berr=be if solved else None,
                                           err_norm=en if solved else None, err_comp=ec if solved and cwise else None,
                                           equed=equed.value.decode(), info=k)


def lu_solve_local(gv, B_share, nrhs, trans=False, out=None):
    """Solves A X = B (A^T X = B when trans) with the factors of the last LU_rep, like ScaLAPACK's pdgetrs, with B and X
    distributed like A: M x nrhs matrices tiled v x v, global tile (I, J) on grid position (I % Px, J % Py) at local tile
    (I / Px, J / Py).  B_share: this rank's share, (gv.Ml, n >= rhs_local_cols(nrhs, gv.v, gv.Py)) float64 with
    contiguous rows, a NumPy array or any __cuda_array_interface__ object (a torch CUDA tensor on this rank's device);
    read on layer 0 only (None elsewhere).  out: X's share, the same kinds; a new zeroed NumPy array when None, and
    `out is B_share` solves in place.  Local columns whose global index is >= nrhs are neither read nor written.  Returns
    out; every layer gets layer 0's bits.  COLLECTIVE over gv.lu_comm; every rank passes the same nrhs and trans.  The
    factors, the input and later solves are left as they are."""
    return _solve_local(lib().cflx_lu_solve_local, "lu_solve_local", gv.Ml, gv.v, gv.Py, gv.pk == 0, B_share, nrhs, out,
                        gv._h, 1 if trans else 0)


def lu_refine_local(gv, B_share, X_share, nrhs, trans=False, ferr=True):
    """lu_refine with B and X distributed like A (cflx_lu_refine_local, ScaLAPACK's pdgerfs): B_share and X_share are
    this rank's shares in lu_solve_local's layout, NumPy arrays or torch CUDA tensors.  X_share holds the solution on
    entry (read on layer 0, where it is required; may be None elsewhere) and the refined one on return, every layer
    getting layer 0's bits; it must not overlap B_share.  Returns (X_share, ferr, berr) with ferr and berr per column,
    identical on every rank.  The columns go in blocks of refine_block_cols(gv.v), each with the bits lu_refine gives
    those columns alone.  COLLECTIVE over gv.lu_comm."""
    return _refine_local(lib().cflx_lu_refine_local, "lu_refine_local", gv.Ml, gv.v, gv.Py, gv.pk == 0, B_share, X_share,
                         nrhs, ferr, gv._h, 1 if trans else 0)


def lu_refine_x_local(gv, B_share, X_share, nrhs, trans=False, cwise=True):
    """lu_refine_x with B and X distributed like A (cflx_lu_refine_x_local): shares as lu_refine_local; returns
    (X_share, dict(rcond, berr, err_norm, err_comp, info)) as lu_refine_x, info = M + j with j the first global column
    whose bound was set to 1.  COLLECTIVE over gv.lu_comm."""
    return _refine_x_local(lib().cflx_lu_refine_x_local, "lu_refine_x_local", gv.Ml, gv.v, gv.Py, gv.pk == 0, B_share,
                           X_share, nrhs, cwise, gv._h, 1 if trans else 0)


def lu_svx_local(gv, B_share, nrhs, trans=False, out=None):
    """lu_svx with B and X distributed like A (cflx_lu_svx_local): B_share and out as lu_solve_local's (`out is B_share`
    solves in place).  Returns (out, dict(rcond, ferr, berr, rpvgrw, equed, info)); out is None (and left as it was) when
    U has an exactly zero pivot (info = k).  COLLECTIVE over gv.lu_comm; identical on every rank."""
    return _svx_local(lib().cflx_lu_svx_local, "lu_svx_local", gv.M, gv.Ml, gv.v, gv.Py, gv.pk == 0, B_share, nrhs, out,
                      True, gv._h, 1 if trans else 0)


def lu_svxx_local(gv, B_share, nrhs, trans=False, cwise=True, out=None):
    """lu_svxx with B and X distributed like A (cflx_lu_svxx_local): shares as lu_svx_local; returns (out, dict(rcond,
    rpvgrw, berr, err_norm, err_comp, equed, info)) as lu_svxx.  COLLECTIVE over gv.lu_comm; identical on every rank."""
    return _svxx_local(lib().cflx_lu_svxx_local, "lu_svxx_local", gv.M, gv.Ml, gv.v, gv.Py, gv.pk == 0, B_share, nrhs,
                       out, cwise, gv._h, 1 if trans else 0)


def lu_det(gv, unscaled=False):
    """det(A) of the padded matrix of the last LU_rep (P A = L U) on the GPU grid, as an exact-range pair that neither
    overflows nor underflows: returns dict(sign, logabsdet, mantissa, exponent, info) with det = sign * mantissa *
    2**exponent, mantissa in [0.5, 1) (0 when singular), logabsdet = log|det|.  info = k when U(k,k) is exactly zero (the
    first such k, counted from 1): sign 0, logabsdet -inf.  A non-finite U(k,k) before any zero gives NaN.  unscaled=True
    divides by the scales the factors carry (lu_equilibrate), giving det of the input before scaling.  COLLECTIVE over
    gv.lu_comm; identical on every rank.  The factors, the permutation and later solves are left as they are."""
    sign, lad, mant, exp, info = (ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_int64(),
                                  ctypes.c_int())
    check(lib().cflx_lu_det(gv._h, 1 if unscaled else 0, ctypes.byref(sign), ctypes.byref(lad), ctypes.byref(mant),
                            ctypes.byref(exp), ctypes.byref(info)), "lu_det")
    return dict(sign=sign.value, logabsdet=lad.value, mantissa=mant.value, exponent=exp.value, info=info.value)


class cholesky:
    """Mirror of the reference's CONFCHOX driver interface (src/conflux/cholesky/Cholesky.h:20-22):
        initialize(N, v, grid, comm) -> object;  obj.parallelCholesky() -> ms;  obj.finalize().
    grid = (0, 0, 0) and v = 0 select the reference's automatic choices (Cholesky.cpp:75-134).  `data` is this rank's share
    of the input (Ml x Nl, conflux tile layout), filled by the reference's generator (CholeskyIO.cpp:100-172)."""

    def __init__(self, N, v, grid, comm):
        self.comm = comm
        self._h = ctypes.c_void_p()
        g = tuple(int(x) for x in grid)
        check(lib().cflx_chol_create(comm._h, int(N), int(v), g[0], g[1], g[2], ctypes.byref(self._h)), "chol_create")
        info = (ctypes.c_int * 16)()
        check(lib().cflx_chol_info(self._h, info), "chol_info")
        (self.N, self.v, self.Kappa, self.Ml, self.Nl, self.l, self.P, self.PX, self.PY, self.PZ, self.px, self.py, self.pz,
         self.rank) = list(info)[:14]
        self.data = np.zeros((self.Ml, self.Nl))
        self.generateInputMatrixDistributed()

    @classmethod
    def initialize(cls, N, v, grid, comm):
        return cls(N, v, grid, comm)

    def generateInputMatrixDistributed(self):
        check(lib().cflx_chol_init_matrix_host(self.N, self.v, self.PX, self.PY, self.PZ, self.rank, self.data.ctypes.data),
              "chol_init_matrix_host")

    def parallelCholesky(self, upload=True):
        if upload:
            a = np.ascontiguousarray(self.data, dtype=np.float64)
            check(lib().cflx_chol_set_local(self._h, a.ctypes.data), "chol_set_local")
        ms = ctypes.c_double()
        check(lib().cflx_chol_factor(self._h, ctypes.byref(ms)), "chol_factor")
        return ms.value

    def factor_ldlt(self, tiny=0.0, upload=True):
        """The signed Cholesky A = R S R^T of the padded input without pivoting (cflx_chol_factor_ldlt), for symmetric
        indefinite matrices: R lower triangular with a positive diagonal (local_factor), S = diag(signs()).  tiny: pivots
        with |d| < tiny become copysign(tiny, d).  upload=True copies self.data to the device first.  Returns (nrepl,
        inertia, info, ms): the replaced pivots, (positive, negative, zero) pivots, 1 + the first exactly zero pivot's
        column (0: none) and the loop's device ms.  Every later call (solve, rcond, refine, svx, inverse, det, validate)
        refers to R S R^T.  COLLECTIVE; identical on every rank."""
        if upload:
            a = np.ascontiguousarray(self.data, dtype=np.float64)
            check(lib().cflx_chol_set_local(self._h, a.ctypes.data), "chol_set_local")
        nrepl, info, ms = ctypes.c_int(), ctypes.c_int(), ctypes.c_double()
        inertia = (ctypes.c_int64 * 3)()
        check(lib().cflx_chol_factor_ldlt(self._h, float(tiny), ctypes.byref(nrepl), inertia, ctypes.byref(info),
                                          ctypes.byref(ms)), "chol_factor_ldlt")
        return nrepl.value, tuple(inertia), info.value, ms.value

    def rbt(self, depth=2, seed=0, upload=True):
        """Symmetric random butterfly transform of the input (cflx_chol_rbt): A <- W = U^T A U, after the stored lower
        triangle is completed to the symmetric matrix.  Then factor_ldlt(upload=False) and rbt_solve.  N must be a
        multiple of 2**depth * v * lcm(PX, PY).  upload=True copies self.data to the device first.  Returns u, the
        (depth, N) multipliers of U (rbt_multipliers(N, depth, seed)[0]).  COLLECTIVE."""
        if upload:
            a = np.ascontiguousarray(self.data, dtype=np.float64)
            check(lib().cflx_chol_set_local(self._h, a.ctypes.data), "chol_set_local")
        u = np.empty((int(depth), self.N))
        check(lib().cflx_chol_rbt(self._h, int(depth), ctypes.c_uint64(int(seed)), u.ctypes.data), "chol_rbt")
        return u

    def rbt_solve(self, B, refine=True):
        """Solves A X = B with a factor of a transformed input (rbt, then factor_ldlt): X = U inv(W) U^T B; refine=True
        refines the transformed system's solution as refine does.  Returns (X, ferr, berr) as lu_rbt_solve.
        COLLECTIVE; identical on every rank."""
        B, B2, nrhs = _rhs(self.N, B, "cholesky.rbt_solve")
        X = np.empty_like(B2)
        fe, be = np.empty(nrhs), np.empty(nrhs)
        check(lib().cflx_chol_rbt_solve(self._h, nrhs, B2.ctypes.data, nrhs, X.ctypes.data, nrhs, 1 if refine else 0,
                                        fe.ctypes.data, be.ctypes.data), "chol_rbt_solve")
        return X.reshape(B.shape), (fe if refine else None), (be if refine else None)

    def rbt_apply_local(self, op, B_share, nrhs):
        """U^T (op 0) or U (op 1) of the factor's transform on the rows of this rank's right-hand side share, in place
        (cflx_chol_rbt_apply_local); B_share as solve_local's.  rbt_apply_local(0, B), solve_local, rbt_apply_local(1, X)
        solves A X = B distributed.  Not collective.  Returns B_share."""
        ptr, out, ld = _share_out(B_share, self.Ml, rhs_local_cols(nrhs, self.v, self.PY), "cholesky.rbt_apply_local",
                                  strided=True, name="B_share")
        check(lib().cflx_chol_rbt_apply_local(self._h, int(op), int(nrhs), ptr, ld), "chol_rbt_apply_local")
        return out

    def signs(self):
        """The signs S (N,) of the last factorisation: factor_ldlt's, all +1 after parallelCholesky."""
        s = np.empty(self.N)
        check(lib().cflx_chol_get_signs(self._h, s.ctypes.data), "chol_get_signs")
        return s

    def local_input(self):
        """This rank's share of the input as the factorisations read it (after equilibrate(apply) and rbt)."""
        A = np.empty((self.Ml, self.Nl))
        check(lib().cflx_chol_get_input(self._h, A.ctypes.data), "chol_get_input")
        return A

    def local_factor(self):
        L = np.empty((self.Ml, self.Nl))
        check(lib().cflx_chol_get_local(self._h, L.ctypes.data), "chol_get_local")
        return L

    def validate(self):
        a, r = ctypes.c_double(), ctypes.c_double()
        check(lib().cflx_chol_validate(self._h, ctypes.byref(a), ctypes.byref(r)), "chol_validate")
        return a.value, r.value

    def solve(self, B):
        """Solves A X = B with the factor of the last parallelCholesky (A = L L^T) on the GPU grid, like LAPACK's potrs.
        COLLECTIVE over the object's comm; every rank passes the same B, (N,) or (N, nrhs) with N = self.N (the padded
        size), and gets the same X in the same shape.  The factor and the input are left as they are."""
        B, B2, nrhs = _rhs(self.N, B, "cholesky.solve")
        X = np.empty_like(B2)
        check(lib().cflx_chol_solve(self._h, nrhs, B2.ctypes.data, max(nrhs, 1), X.ctypes.data, max(nrhs, 1)), "chol_solve")
        return X.reshape(B.shape)

    def sv_mixed(self, B, prec="tf32x3", itmax=0, upload=True):
        """LAPACK dsposv on the GPU grid: lu_sv_mixed's loop on the Cholesky path (upload=True copies self.data to the
        device first).  Returns (X, iter, berr) as lu_sv_mixed; iter -3 when the low-precision factorisation met a
        non-positive pivot.  Raises ConfluxError when the FP64 fallback finds the matrix not positive definite.
        COLLECTIVE; identical on every rank."""
        if upload:
            a = np.ascontiguousarray(self.data, dtype=np.float64)
            check(lib().cflx_chol_set_local(self._h, a.ctypes.data), "chol_set_local")
        return _sv_mixed(lib().cflx_chol_sv_mixed, "cholesky.sv_mixed", self._h, self.N, B, prec, itmax)

    def solve_local(self, B_share, nrhs, out=None):
        """Solves A X = B with the factor of the last parallelCholesky, like ScaLAPACK's pdpotrs, with B and X distributed
        like A; arguments and result as lu_solve_local's.  Only the rows of real tiles (global tile index < Kappa) are
        read or written.  COLLECTIVE; every rank passes the same nrhs."""
        return _solve_local(lib().cflx_chol_solve_local, "cholesky.solve_local", self.Ml, self.v, self.PY, self.pz == 0,
                            B_share, nrhs, out, self._h)

    def refine_local(self, B_share, X_share, nrhs, ferr=True):
        """refine with B and X distributed like A (cflx_chol_refine_local): arguments and results as lu_refine_local's;
        only the rows of real tiles are read and written.  COLLECTIVE."""
        return _refine_local(lib().cflx_chol_refine_local, "cholesky.refine_local", self.Ml, self.v, self.PY,
                             self.pz == 0, B_share, X_share, nrhs, ferr, self._h)

    def refine_x_local(self, B_share, X_share, nrhs, cwise=True):
        """refine_x with B and X distributed like A (cflx_chol_refine_x_local), as lu_refine_x_local.  COLLECTIVE."""
        return _refine_x_local(lib().cflx_chol_refine_x_local, "cholesky.refine_x_local", self.Ml, self.v, self.PY,
                               self.pz == 0, B_share, X_share, nrhs, cwise, self._h)

    def svx_local(self, B_share, nrhs, out=None):
        """svx with B and X distributed like A (cflx_chol_svx_local): (out, dict(rcond, ferr, berr, equed, info)), shares
        as lu_svx_local's.  COLLECTIVE."""
        return _svx_local(lib().cflx_chol_svx_local, "cholesky.svx_local", self.N, self.Ml, self.v, self.PY,
                          self.pz == 0, B_share, nrhs, out, False, self._h)

    def svxx_local(self, B_share, nrhs, cwise=True, out=None):
        """svxx with B and X distributed like A (cflx_chol_svxx_local), as lu_svxx_local.  COLLECTIVE."""
        return _svxx_local(lib().cflx_chol_svxx_local, "cholesky.svxx_local", self.N, self.Ml, self.v, self.PY,
                           self.pz == 0, B_share, nrhs, out, cwise, self._h)

    def rcond(self):
        """LAPACK dpocon of the last parallelCholesky on the GPU grid: (rcond, anorm) with anorm = ||A||_1 of the padded
        symmetric input and rcond = 1 / (anorm * estimate of ||A^-1||_1).  COLLECTIVE; identical on every rank."""
        r, a = ctypes.c_double(), ctypes.c_double()
        check(lib().cflx_chol_rcond(self._h, ctypes.byref(r), ctypes.byref(a)), "chol_rcond")
        return r.value, a.value

    def refine(self, B, X, ferr=True):
        """LAPACK dporfs with the factor of the last parallelCholesky on the GPU grid: refines X, a solution of A X = B (e.g.
        from solve), and returns (X, ferr, berr) as lu_refine does.  COLLECTIVE; identical on every rank."""
        shape, B2, X2, nrhs, fe, be = _refine_args(self.N, B, X, "cholesky.refine")
        check(lib().cflx_chol_refine(self._h, nrhs, B2.ctypes.data, nrhs, X2.ctypes.data, nrhs,
                                     fe.ctypes.data if ferr else None, be.ctypes.data), "chol_refine")
        return X2.reshape(shape), (fe if ferr else None), be

    def refine_x(self, B, X, cwise=True):
        """LAPACK dporfsx with the factor of the last parallelCholesky on the GPU grid: returns (X, dict(rcond, berr,
        err_norm, err_comp, info)) as lu_refine_x does.  COLLECTIVE; identical on every rank."""
        return _refine_x(lib().cflx_chol_refine_x, self.N, B, X, cwise, "cholesky.refine_x", self._h)

    def _equilibrate(self, apply, upload, fn, what):
        if upload:
            a = np.ascontiguousarray(self.data, dtype=np.float64)
            check(lib().cflx_chol_set_local(self._h, a.ctypes.data), "chol_set_local")
        s = np.zeros(self.N)
        scond, amax, equed, info = ctypes.c_double(), ctypes.c_double(), ctypes.c_char(), ctypes.c_int()
        check(fn(self._h, 1 if apply else 0, s.ctypes.data, ctypes.byref(scond), ctypes.byref(amax), ctypes.byref(equed),
                 ctypes.byref(info)), what)
        return dict(s=s, scond=scond.value, amax=amax.value, equed=equed.value.decode(), info=info.value)

    def equilibrate(self, apply=True, upload=True):
        """LAPACK dpoequ (+ dlaqsy, lower, when apply) on the padded input on the GPU grid.  upload=True first copies
        self.data to the device, so that parallelCholesky(upload=False) then factors the scaled matrix.  Returns dict(s,
        scond, amax, equed, info).  COLLECTIVE; identical on every rank."""
        return self._equilibrate(apply, upload, lib().cflx_chol_equilibrate, "chol_equilibrate")

    def equilibrate_b(self, apply=True, upload=True):
        """LAPACK dpoequb (+ dlaqsy, lower, when apply): equilibrate with the scales rounded to powers of two.
        Arguments and result as equilibrate.  COLLECTIVE; identical on every rank."""
        return self._equilibrate(apply, upload, lib().cflx_chol_equilibrate_b, "chol_equilibrate_b")

    def svxx(self, B, cwise=True):
        """LAPACK dposvxx with the factor of the last parallelCholesky and the scaling it carries (equilibrate_b or
        equilibrate): returns (X, dict(rcond, rpvgrw, berr, err_norm, err_comp, equed, info)) as lu_svxx does, rpvgrw
        being dla_porpvgrw's.  COLLECTIVE; identical on every rank."""
        return _svxx(lib().cflx_chol_svxx, self.N, B, cwise, "cholesky.svxx", self._h)

    def svx(self, B):
        """LAPACK dposvx with the factor of the last parallelCholesky and the scaling it carries (equilibrate): returns
        (X, dict(rcond, ferr, berr, equed, info)).  COLLECTIVE; identical on every rank."""
        B, B2, nrhs = _rhs(self.N, B, "cholesky.svx")
        X = np.empty_like(B2)
        fe, be = np.empty(nrhs), np.empty(nrhs)
        rcond, equed, info = ctypes.c_double(), ctypes.c_char(), ctypes.c_int()
        check(lib().cflx_chol_svx(self._h, nrhs, B2.ctypes.data, nrhs, X.ctypes.data, nrhs, ctypes.byref(rcond),
                                  fe.ctypes.data, be.ctypes.data, ctypes.byref(equed), ctypes.byref(info)), "chol_svx")
        return X.reshape(B.shape), dict(rcond=rcond.value, ferr=fe, berr=be, equed=equed.value.decode(), info=info.value)

    def inverse(self, out=None):
        """inv(A) from the factor of the last parallelCholesky on the GPU grid, like LAPACK's dpotri (lower): returns this
        rank's Ml x Nl share, whose real tiles on and below the diagonal hold inv(A); the tiles above the diagonal and
        those beyond Kappa are zero.  out as lu_inverse's.  COLLECTIVE; every layer gets layer 0's bits."""
        ptr, arr, _ = _share_out(out, self.Ml, self.Nl, "cholesky.inverse")
        check(lib().cflx_chol_inverse(self._h, ptr), "chol_inverse")
        return arr

    def det(self, unscaled=False):
        """det(A) = prod(l_ii)^2 of the padded matrix of the last parallelCholesky on the GPU grid: returns dict(logdet,
        mantissa, exponent) with det = mantissa * 2**exponent, mantissa in [0.5, 1), as lu_det's pair.  After factor_ldlt,
        det = prod(s_i r_ii^2): the mantissa carries its sign and logdet is log|det|.  unscaled=True
        divides by prod(s)^2 of the scaling the factor carries (equilibrate).  COLLECTIVE; identical on every rank."""
        ld, mant, exp = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
        check(lib().cflx_chol_det(self._h, 1 if unscaled else 0, ctypes.byref(ld), ctypes.byref(mant), ctypes.byref(exp)),
              "chol_det")
        return dict(logdet=ld.value, mantissa=mant.value, exponent=exp.value)

    def finalize(self, clean=True):
        if self._h:
            lib().cflx_chol_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.finalize()
        except Exception:
            pass


def chol_dims(N, v, Px, Py, Pz):
    o = (ctypes.c_int * 6)()
    check(lib().cflx_chol_dims(int(N), int(v), int(Px), int(Py), int(Pz), o), "chol_dims")
    return dict(N=o[0], Kappa=o[1], Ml=o[2], Nl=o[3], l=o[4], P=o[5])


def chol_auto_grid(P, N):
    g = (ctypes.c_int * 3)()
    check(lib().cflx_chol_auto_grid(int(P), int(N), g), "chol_auto_grid")
    return tuple(g)


def _ptr(a):
    return a.ctypes.data if a is not None else None


def _tiles(n, v):
    """whole tiles of v in n; v < 1 is left for the hook to refuse"""
    return int(n) // max(int(v), 1)


def _share(v, Ml, Nl, grid=(1, 1), pos=(0, 0), Kappa=None, M=None):
    """the cflx_share_layout of an Ml x Nl share at grid position pos of grid = (Px, Py); M defaults to the LU layout's
    (Ml / v) Px v, Kappa to no padding tiles"""
    Px, Py = (int(x) for x in grid)
    M = int(M) if M is not None else _tiles(Ml, v) * Px * int(v)
    return ShareLayout(M, int(v), int(Kappa if Kappa is not None else 1 << 30), int(Ml), int(Nl), Px, Py, int(pos[0]),
                       int(pos[1]))


class dbg:
    """Single-kernel hooks (tests and micro-benchmarks)."""

    @staticmethod
    def gemm_tn(AT, B, C=None, alpha=1.0, beta=0.0, reps=1):
        """D = beta*C + alpha * AT^T @ B on the trailing-update kernel (AT: K x M, B: K x N, C: M x N or None = zeros;
        K % 4 == 0), on contiguous out-of-place buffers with M and N padded to even.  Returns (D, mean ms of one
        launch)."""
        AT = np.asarray(AT, dtype=np.float64)
        B = np.asarray(B, dtype=np.float64)
        K, M = AT.shape
        N = B.shape[1]
        M2, N2 = M + (M & 1), N + (N & 1)
        ATp = np.zeros((K, M2))
        ATp[:, :M] = AT
        Bp = np.zeros((K, N2))
        Bp[:, :N] = B
        Cp = np.zeros((M, N2))
        if C is not None:
            Cp[:, :N] = C
        D, _, ms = dbg.gemm_tn_window(ATp, Bp, Cp, M, N2, K, alpha, beta, in_place=False, reps=reps)
        return D[:, :N], ms

    @staticmethod
    def gemm_tn_window(AT, B, C, M, N, K, alpha=1.0, beta=0.0, at_off=(0, 0), b_off=(0, 0), c_off=(0, 0), in_place=True,
                       reps=1):
        """The trailing-update kernel on a window of whole buffers, as the factorisation launches it: rows
        [c_off[0], +M) x columns [c_off[1], +N) of C become beta*C + alpha * AT'^T @ B', with AT' the K x M block of AT
        at (row, column) at_off and B' the K x N block of B at b_off.  in_place: D is C on the device (the trailing
        update); else D starts as a device copy of C.  Every entry outside those blocks may hold anything (NaN canaries):
        the kernel reads AT' with M rounded up to even, nothing else.  Returns (D, C, ms): the whole D and C buffers
        after the call (the same array in place) and the mean ms of one launch."""
        AT = np.ascontiguousarray(AT, dtype=np.float64)
        B = np.ascontiguousarray(B, dtype=np.float64)
        C = np.ascontiguousarray(C, dtype=np.float64)
        D = np.empty_like(C)
        Cout = D if in_place else np.empty_like(C)
        ms = ctypes.c_double()
        check(lib().cflx_dbg_gemm_tn(int(M), int(N), int(K), AT.ctypes.data, AT.shape[0], AT.shape[1],
                                     at_off[0] * AT.shape[1] + at_off[1], B.ctypes.data, B.shape[0], B.shape[1],
                                     b_off[0] * B.shape[1] + b_off[1], C.ctypes.data, C.shape[0], C.shape[1],
                                     int(c_off[0]), int(c_off[1]), float(alpha), float(beta), 1 if in_place else 0,
                                     D.ctypes.data, Cout.ctypes.data, int(reps), ctypes.byref(ms)), "dbg_gemm_tn")
        return D, Cout, ms.value

    @staticmethod
    def gemm_narrow(A, B, C=None, alpha=1.0, beta=0.0, reps=1, out=None):
        """D = beta*C + alpha * A @ B on the solve's narrow GEMM (K % 4 == 0).  Returns (D, mean ms of one launch).
        out: the array to write D into; passing C itself runs the kernel with D aliasing C."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        B = np.ascontiguousarray(B, dtype=np.float64)
        M, K = A.shape
        N = B.shape[1]
        Cp = None
        if C is not None:
            assert C.dtype == np.float64 and C.flags.c_contiguous and C.shape == (M, N)
            Cp = C.ctypes.data
        D = np.empty((M, N)) if out is None else out
        assert D.dtype == np.float64 and D.flags.c_contiguous and D.shape == (M, N)
        ms = ctypes.c_double()
        check(lib().cflx_dbg_gemm_narrow(M, N, K, A.ctypes.data, B.ctypes.data, Cp, float(alpha), float(beta), D.ctypes.data,
                                         int(reps), ctypes.byref(ms)), "dbg_gemm_narrow")
        return D, ms.value

    @staticmethod
    def gemm_narrow_tn(AT, B, C=None, alpha=1.0, beta=0.0, reps=1, out=None):
        """D = beta*C + alpha * AT^T @ B on the Cholesky solve's transposed narrow GEMM (AT is K x M, read in place; any
        K).  Returns (D, mean ms of one launch).  out: the array to write D into; passing C itself runs the kernel with D
        aliasing C."""
        AT = np.ascontiguousarray(AT, dtype=np.float64)
        B = np.ascontiguousarray(B, dtype=np.float64)
        K, M = AT.shape
        if B.ndim != 2 or B.shape[0] != K:
            raise ValueError(f"gemm_narrow_tn: B must have {K} rows, got shape {B.shape}")
        N = B.shape[1]
        Cp = None
        if C is not None:
            assert C.dtype == np.float64 and C.flags.c_contiguous and C.shape == (M, N)
            Cp = C.ctypes.data
        D = np.empty((M, N)) if out is None else out
        assert D.dtype == np.float64 and D.flags.c_contiguous and D.shape == (M, N)
        ms = ctypes.c_double()
        check(lib().cflx_dbg_gemm_narrow_tn(M, N, K, AT.ctypes.data, B.ctypes.data, Cp, float(alpha), float(beta),
                                            D.ctypes.data, int(reps), ctypes.byref(ms)), "dbg_gemm_narrow_tn")
        return D, ms.value

    @staticmethod
    def gemm_narrow_window(A, B, C, M, N, K, alpha=1.0, beta=0.0, a_off=(0, 0), b_off=(0, 0), c_off=(0, 0), trans=False,
                           in_place=True):
        """The solve's narrow GEMM on a window of whole buffers, as the solve engine launches it: rows [c_off[0], +M) x
        columns [c_off[1], +N) of C become beta*C + alpha * op(A') @ B', with A' the block of A at (row, column) a_off
        (M x K, or with trans K x M and op(A') = A'^T on the transposed kernel) and B' the K x N block of B at b_off.  C
        is read only when beta != 0.  in_place: D is C on the device; else D starts as a device copy of C.  Entries
        outside the blocks may hold anything (NaN canaries).  Returns (D, C): the whole buffers after the call (the same
        array in place)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        B = np.ascontiguousarray(B, dtype=np.float64)
        C = np.ascontiguousarray(C, dtype=np.float64)
        D = np.empty_like(C)
        Cout = D if in_place else np.empty_like(C)
        check(lib().cflx_dbg_gemm_narrow_window(
            1 if trans else 0, int(M), int(N), int(K), A.ctypes.data, A.shape[0], A.shape[1], int(a_off[0]),
            int(a_off[1]), B.ctypes.data, B.shape[0], B.shape[1], int(b_off[0]), int(b_off[1]), C.ctypes.data,
            C.shape[0], C.shape[1], int(c_off[0]), int(c_off[1]), float(alpha), float(beta), 1 if in_place else 0,
            D.ctypes.data, Cout.ctypes.data), "dbg_gemm_narrow_window")
        return D, Cout

    DIAG_SOLVE_MODES = {"lower": 0, "upper": 1, "lower_t": 2, "unit_lower_t": 3, "upper_t": 4}

    @staticmethod
    def diag_solve(mode, share, R, v, nb, pos=(0, 0), lower=False):
        """One diagonal tile of the solve engine: the v x v tile at (row, column) pos of share (lower: the Cholesky
        factor L, zeros above its diagonal; else the LU's L\\U), its nb x nb diagonal blocks inverted as the solves cache
        them, then Y = T^-1 R (R: v x ldn) by the solves' block sweep.  mode: "lower" (T = L), "upper" (U), "lower_t"
        (L^T of the Cholesky tile), "unit_lower_t" (L^T of the LU's unit L), "upper_t" (U^T).  Returns (Y, inv) with inv
        (2, v // nb, nb, nb): the forward blocks inv(L_jj), then the backward ones (inv(U_jj), or inv(L_jj)^T)."""
        share = np.ascontiguousarray(share, dtype=np.float64)
        R = np.ascontiguousarray(R, dtype=np.float64)
        if R.ndim != 2 or R.shape[0] != v:
            raise ValueError(f"diag_solve: R must have {v} rows, got shape {R.shape}")
        Y = np.empty_like(R)
        inv = np.empty((2, max(int(v) // max(int(nb), 1), 1), max(int(nb), 1), max(int(nb), 1)))
        tri = dbg.DIAG_SOLVE_MODES[mode] if isinstance(mode, str) else int(mode)
        check(lib().cflx_dbg_diag_solve(tri, 1 if lower else 0, int(v), int(nb), share.ctypes.data, share.shape[0],
                                        share.shape[1], int(pos[0]), int(pos[1]), R.shape[1], R.ctypes.data,
                                        Y.ctypes.data, inv.ctypes.data), "dbg_diag_solve")
        return Y, inv

    @staticmethod
    def residual(A, mode, v, Kappa=None, grid=(1, 1), pos=(0, 0), Xc=None, Xr=None, reps=1):
        """The residual kernels of lu_refine / cholesky.refine on one layer-0 share A (Ml x Nl, conflux layout of tile v at
        grid position pos of grid = (Px, Py)).  mode "nn": P = A @ Xc, Q = |A| @ |Xc| (Xc: Nl x nrhs, X by local column);
        "tn": P = A.T @ Xr, Q = |A|.T @ |Xr| (Xr: Ml x nrhs, X by local row); "sym": the stored lower triangle of the real
        tiles (global tile index < Kappa), rows [0, Ml) the NN product over global row >= column and rows [Ml, Ml + Nl)
        the TN product over global row > column.  Returns (P, Q, mean ms of one launch)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        Ml, Nl = A.shape
        m = {"nn": 0, "tn": 1, "sym": 2}[mode]
        cvt = lambda X: None if X is None else np.ascontiguousarray(np.asarray(X, dtype=np.float64).reshape(X.shape[0], -1))
        Xc, Xr = cvt(Xc), cvt(Xr)
        nrhs = (Xc if Xc is not None else Xr).shape[1]
        rows = (Ml, Nl, Ml + Nl)[m]
        P, Q = np.empty((rows, nrhs)), np.empty((rows, nrhs))
        ms = ctypes.c_double()
        check(lib().cflx_dbg_residual(m, _share(v, Ml, Nl, grid, pos, Kappa, M=0), A.ctypes.data, nrhs, _ptr(Xc),
                                      _ptr(Xr), P.ctypes.data, Q.ctypes.data, int(reps), ctypes.byref(ms)), "dbg_residual")
        return P, Q, ms.value

    @staticmethod
    def residual_x(A, mode, v, Kappa=None, grid=(1, 1), pos=(0, 0), Xc=None, Xr=None, Xc_tail=None, Xr_tail=None,
                   reps=1):
        """The double-double residual kernels of lu_refine_x / cholesky.refine_x, arguments and modes as residual's,
        with the tails of X (None: zero).  Returns (Hi, Lo, mean ms of one launch): Hi + Lo = op(A) (X + X_tail)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        Ml, Nl = A.shape
        m = {"nn": 0, "tn": 1, "sym": 2}[mode]
        cvt = lambda X: None if X is None else np.ascontiguousarray(np.asarray(X, dtype=np.float64).reshape(X.shape[0], -1))
        Xc, Xr, Xct, Xrt = cvt(Xc), cvt(Xr), cvt(Xc_tail), cvt(Xr_tail)
        nrhs = (Xc if Xc is not None else Xr).shape[1]
        rows = (Ml, Nl, Ml + Nl)[m]
        H, L = np.empty((rows, nrhs)), np.empty((rows, nrhs))
        ms = ctypes.c_double()
        check(lib().cflx_dbg_residual_x(m, _share(v, Ml, Nl, grid, pos, Kappa, M=0), A.ctypes.data, nrhs, _ptr(Xc),
                                        _ptr(Xct), _ptr(Xr), _ptr(Xrt), H.ctypes.data, L.ctypes.data, int(reps),
                                        ctypes.byref(ms)), "dbg_residual_x")
        return H, L, ms.value

    @staticmethod
    def equil(A, v, Kappa=None, grid=(1, 1), pos=(0, 0), M=None, r=None, c=None, equed="N", ncols=None):
        """The per-share kernels of lu_equilibrate / cholesky.equilibrate / lu_svx on one layer-0 share A (Ml x Nl,
        conflux layout of tile v at grid position pos of grid = (Px, Py)), over M global indices (default: the LU layout's
        (Ml / v) Px v).  r, c: M-vectors (r is also the Cholesky's s; default ones).  Returns dict(rowmax, colmax, diag,
        scaled, sym_scaled, growth, zero_pivot): the partial row maxima, the column maxima of |a| r, the diagonal of the
        real tiles (global tile index < Kappa), the share after dlaqge's scaling for equed and after dlaqsy's, (max |a|
        over global row <= column, max |a|) over the global columns < ncols (default M), and 1 + the first zero diagonal
        entry (0: none)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        sh = _share(v, *A.shape, grid, pos, Kappa, M)
        M = sh.M
        r = np.ascontiguousarray(np.ones(M) if r is None else r, dtype=np.float64)
        c = np.ascontiguousarray(np.ones(M) if c is None else c, dtype=np.float64)
        out = dict(rowmax=np.empty(M), colmax=np.empty(M), diag=np.empty(M), scaled=np.empty_like(A),
                   sym_scaled=np.empty_like(A), growth=np.empty(2))
        zp = ctypes.c_int()
        check(lib().cflx_dbg_equil(sh, A.ctypes.data, r.ctypes.data, c.ctypes.data, equed.encode(),
                                   int(ncols if ncols is not None else M), out["rowmax"].ctypes.data,
                                   out["colmax"].ctypes.data, out["diag"].ctypes.data, out["scaled"].ctypes.data,
                                   out["sym_scaled"].ctypes.data, out["growth"].ctypes.data, ctypes.byref(zp)), "dbg_equil")
        out["zero_pivot"] = zp.value
        return out

    @staticmethod
    def growth_cols(mode, F, A, v, Kappa=None, grid=(1, 1), pos=(0, 0), M=None, ncols=None):
        """The per-column pivot growth pass of lu_svxx (mode "lu") and cholesky.svxx (mode "chol") on one layer-0 share
        F (the factor) and A (the input), both Ml x Nl in dbg.equil's layout.  Returns (amax, fmax), M-vectors by global
        column j < ncols (default M), zeros elsewhere: "lu" max |a_ij| over every row and max |f_ij| over the rows
        i <= j; "chol" both over the real tiles' (global tile index < Kappa) rows j <= i < ncols."""
        F = np.ascontiguousarray(F, dtype=np.float64)
        A = np.ascontiguousarray(A, dtype=np.float64)
        sh = _share(v, *A.shape, grid, pos, Kappa, M)
        amax, fmax = np.empty(sh.M), np.empty(sh.M)
        check(lib().cflx_dbg_growth_cols({"lu": 0, "chol": 1}[mode], sh, int(ncols if ncols is not None else sh.M),
                                         F.ctypes.data, A.ctypes.data, amax.ctypes.data, fmax.ctypes.data),
              "dbg_growth_cols")
        return amax, fmax

    @staticmethod
    def inverse_share(mode, v, grid, pos, M, c0, nc, Ml, Nl, Kappa=None, rows=None, X=None, perm=None, share=None,
                      zero_fill=False):
        """The per-share kernels of lu_inverse (mode "lu") and cholesky.inverse (mode "chol") on one Ml x Nl share at grid
        position pos of grid = (Px, Py), for the block of nc columns from global column c0.  Returns (W, share): W (Ml x
        round_up(nc, 8)) is the seed of the first `rows` local rows (default Ml); share is a copy of `share` after the
        scatter of X (M x nc or wider, by global row) to global column perm[c0 + j] ("lu") or c0 + j ("chol": real tiles,
        global tile index < Kappa, on and below the diagonal), and with zero_fill ("chol") zeros on every entry the scatter
        never writes.  share is None when X or share is None."""
        m = {"lu": 0, "chol": 1}[mode]
        ldn = -(-int(nc) // 8) * 8
        W = np.empty((Ml, ldn))
        out = Xc = pm = None
        if X is not None and share is not None:
            Xc = np.ascontiguousarray(X, dtype=np.float64)
            out = np.array(share, dtype=np.float64, order="C")
            pm = np.ascontiguousarray(perm, dtype=np.int32) if perm is not None else None
        check(lib().cflx_dbg_inverse_share(m, _share(v, Ml, Nl, grid, pos, Kappa, M), int(c0), int(nc),
                                           int(rows if rows is not None else Ml), _ptr(Xc),
                                           Xc.shape[1] if Xc is not None else 0, _ptr(pm), W.ctypes.data, _ptr(out),
                                           1 if zero_fill else 0), "dbg_inverse_share")
        return W, out

    @staticmethod
    def solve_local_share(mode, v, grid, pos, M, nrhs, c0, w, Ml, Kappa=None, B=None, Xk=None, X=None):
        """The pack and scatter kernels of lu_solve_local (mode "lu") and cholesky.solve_local (mode "chol") on one
        right-hand side share of Ml rows at grid position pos of grid = (Px, Py), for the block of w columns from global
        column c0 of an M x nrhs matrix.  Returns (Bk, X): Bk (M x round_up(w, 8)) the pack of B (Ml x n >=
        rhs_local_cols, every local row for "lu", the real tiles' rows, global tile index < Kappa, for "chol"), and a copy
        of X after the scatter of Xk (M x round_up(w, 8), by global row) into it.  Either is None when its inputs are."""
        m = {"lu": 0, "chol": 1}[mode]
        sh = _share(v, Ml, rhs_local_cols(nrhs, v, grid[1]), grid, pos, Kappa, M)
        ldn = -(-int(w) // 8) * 8
        Bc = np.ascontiguousarray(B, dtype=np.float64) if B is not None else None
        Bk = np.empty((int(M), ldn)) if Bc is not None else None
        out = Xc = None
        if X is not None and Xk is not None:
            Xc = np.ascontiguousarray(Xk, dtype=np.float64)
            out = np.array(X, dtype=np.float64, order="C")
        check(lib().cflx_dbg_solve_local_share(m, sh, int(nrhs), int(c0), int(w), _ptr(Bc),
                                               Bc.shape[1] if Bc is not None else 0, _ptr(Bk), _ptr(Xc), _ptr(out),
                                               out.shape[1] if out is not None else 0), "dbg_solve_local_share")
        return Bk, out

    @staticmethod
    def rbt_share(op, X, v, depth, u=None, vv=None, grid=(1, 1), pos=(0, 0), M=None):
        """cflx_dbg_rbt_share: op 0 U^T, 1 V, 2 V^T, 3 U on the rows of the right-hand side share X (Ml x ncols), or 4 W =
        U^T X V on the matrix share X (Ml x Nl), with the r values u / vv ((depth, M) arrays, as rbt_multipliers gives
        them).  M defaults to the covered order.  Returns the transformed copy."""
        X = np.array(X, dtype=np.float64, order="C")
        Ml, n = X.shape
        lay = _share(v, Ml, n if op == 4 else 0, grid, pos, M=M)
        ua = None if u is None else np.ascontiguousarray(u, dtype=np.float64)
        va = None if vv is None else np.ascontiguousarray(vv, dtype=np.float64)
        check(lib().cflx_dbg_rbt_share(int(op), ctypes.byref(lay), int(depth), _ptr(ua), _ptr(va), n, X.ctypes.data, n),
              "dbg_rbt_share")
        return X

    def norm_share(mode, A, v, Kappa=None, grid=(1, 1), pos=(0, 0), M=None):
        """The per-share pass of lu_rcond / cholesky.rcond's 1-norm and of the infinity-norm on one layer-0 share A (Ml x
        Nl, dbg.equil's layout), before the sum over the grid.  mode "col": the column sums of |a| over every entry;
        "sym": the column sums of the symmetric matrix stored as the lower triangle of its real tiles (global tile index
        < Kappa); "row": the row sums.  Returns an M-vector (default M: (Ml / v) Px v) by global index, zero where the
        share holds nothing."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        sh = _share(v, *A.shape, grid, pos, Kappa, M)
        out = np.empty(sh.M)
        check(lib().cflx_dbg_norm_share({"col": 0, "sym": 1, "row": 2}[mode], sh, A.ctypes.data, out.ctypes.data),
              "dbg_norm_share")
        return out

    @staticmethod
    def chol_validate_share(A, v, Kappa, grid=(1, 1), pos=(0, 0), t=0):
        """cholesky.validate's per-share kernels on one layer-0 share A (Ml x Nl, dbg.equil's layout).  Returns (PT,
        sumsq): PT (v x (Ml rounded up to even, + 2)) the masked transposed panel of step t as the validation extracts it
        (NaN where nothing is written, all NaN off grid column t % Py), sumsq the sum of squares of the lower triangle of
        the real tiles (global row >= column, global row < Kappa v)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        Ml, Nl = A.shape
        M = max(_tiles(Ml, v) * int(grid[0]), _tiles(Nl, v) * int(grid[1])) * int(v)
        PT = np.empty((int(v), Ml + (Ml & 1) + 2))
        ss = ctypes.c_double()
        check(lib().cflx_dbg_chol_validate_share(_share(v, Ml, Nl, grid, pos, Kappa, M), A.ctypes.data, int(t),
                                                 PT.ctypes.data, ctypes.byref(ss)), "dbg_chol_validate_share")
        return PT, ss.value

    @staticmethod
    def lu_validate_share(C, v, grid=(1, 1), pos=(0, 0), t=0):
        """The two extract kernels of step t of lu_validate's sweep on one layer-0 share C of the packed factors (Ml x Nl,
        dbg.equil's layout), under the sweep's owner guards.  Returns (LT, U): LT (v x (Ml rounded up to even)) the
        transposed block of unit-lower L in tile column t by local row, U (v x Nl) the block of U in tile row t by local
        column; NaN where nothing is written."""
        C = np.ascontiguousarray(C, dtype=np.float64)
        Ml, Nl = C.shape
        LT, U = np.empty((int(v), Ml + (Ml & 1))), np.empty((int(v), Nl))
        sh = _share(v, Ml, Nl, grid, pos, _tiles(Ml, v) * int(grid[0]))           # Kappa = M / v
        check(lib().cflx_dbg_lu_validate_share(sh, C.ctypes.data, int(t),
                                               LT.ctypes.data, U.ctypes.data), "dbg_lu_validate_share")
        return LT, U

    @staticmethod
    def chol_gather_cols(pieces, v, Px, Py, pj, Ml, Nl, gfirst):
        """The Cholesky trailing update's column-operand gather on one Ml x Nl share at grid column pj of Px x Py, from
        the Px broadcast pieces of the transposed panel of the global tiles >= gfirst (a list: piece p is v x ld_p, ld_p
        = grid row p's rows from its first tile >= gfirst on, rounded up to even, >= 2).  Returns Bc (v x Nl): tile t
        the panel's rows of the global tile of local column tile lj0 + t (lj0: the first with a global index >=
        gfirst), NaN in the tiles after the last."""
        flat = np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.float64).ravel() for p in pieces]))
        Bc = np.empty((int(v), int(Nl)))
        check(lib().cflx_dbg_chol_gather_cols(_share(v, Ml, Nl, (Px, Py), (0, pj), Kappa=0, M=0), int(gfirst),
                                              flat.ctypes.data, Bc.ctypes.data), "dbg_chol_gather_cols")
        return Bc

    @staticmethod
    def refine_assemble(mode, all_chunks, B, grid, v, M, Ml, Nl, nn, tn, nrhs):
        """The refinement's assembly from the partials of the Px x Py x Pz ranks of grid: all_chunks (Px Py Pz chunks in
        rank order, each ((nn ? Ml : 0) + (tn ? Nl : 0)) x 2 ldn) and B (M x ldn).  mode "gerfs": (R, ratio, W) as
        lu_refine assembles them; "lin_berr": (R, ratio, Q) as refine_x's backward error; "x": R = b - the double-double
        sum of the (Hi, Lo) partials, rounded once.  Returns a dict of M x ldn arrays (NaN past column nrhs)."""
        m = {"gerfs": 0, "lin_berr": 1, "x": 2}[mode]
        Px, Py, Pz = (int(x) for x in grid)
        B = np.ascontiguousarray(B, dtype=np.float64)
        ldn = B.shape[1]
        flat = np.ascontiguousarray(np.asarray(all_chunks, dtype=np.float64).ravel())
        out = {k: np.empty((int(M), ldn)) for k in ("R", "ratio", "W", "Q")}
        check(lib().cflx_dbg_refine_assemble(m, Px, Py, Pz, int(v), int(M), int(Ml), int(Nl), int(bool(nn)), int(bool(tn)),
                                             int(nrhs), ldn, flat.ctypes.data, B.ctypes.data, out["R"].ctypes.data,
                                             out["ratio"].ctypes.data, out["W"].ctypes.data, out["Q"].ctypes.data),
              "dbg_refine_assemble")
        return out

    @staticmethod
    def refine_columns(A, D, sel, nrhs, d=None, T=None):
        """The refinement's per-column steps on M x ldn arrays A and D (first nrhs columns) with the per-column selector
        sel (ldn ints).  Returns dict(max, stats, select, add, Y, T): column maxima of A (NaN wins); nrhs x 5 statistics of
        y = A, dy = D, scales d (None: ones); A where sel, else 0; A + D where sel; and (Y, T) = (A, T) updated by D with
        how = sel (1 plain, 2 dla_wwaddw, 0 none; T default zeros)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        D = np.ascontiguousarray(D, dtype=np.float64)
        M, ldn = A.shape
        sel = np.ascontiguousarray(sel, dtype=np.int32)
        dd = np.ascontiguousarray(d, dtype=np.float64) if d is not None else None
        Tio = np.array(np.zeros_like(A) if T is None else T, dtype=np.float64, order="C")
        out = dict(max=np.empty(nrhs), stats=np.empty((nrhs, 5)), select=np.empty_like(A), add=np.empty_like(A),
                   Y=np.empty_like(A))
        check(lib().cflx_dbg_refine_columns(M, ldn, int(nrhs), A.ctypes.data, D.ctypes.data,
                                            dd.ctypes.data if dd is not None else None, sel.ctypes.data,
                                            out["max"].ctypes.data, out["stats"].ctypes.data, out["select"].ctypes.data,
                                            out["add"].ctypes.data, out["Y"].ctypes.data, Tio.ctypes.data),
              "dbg_refine_columns")
        out["T"] = Tio
        return out

    @staticmethod
    def det(d, s1=None, s2=None, square=False):
        """The product kernel of lu_det / cholesky.det on a host vector d (and divisors s1, s2 of its length): returns
        dict(mantissa, exponent, neg, first_zero, nonfinite) with mantissa * 2**exponent = |prod d| (squared when square)
        / |prod s1| / |prod s2|, neg the parity of the negative entries (0 when square), first_zero 1 + the first zero
        index of d (0: none), nonfinite 1 when a non-finite entry (or a zero divisor) comes before it."""
        d = np.ascontiguousarray(d, dtype=np.float64).ravel()
        n = d.size
        vec = lambda s: None if s is None else np.ascontiguousarray(s, dtype=np.float64).ravel()  # noqa: E731
        s1, s2 = vec(s1), vec(s2)
        for s in (s1, s2):
            if s is not None and s.size != n:
                raise ValueError(f"dbg.det: a divisor must have {n} entries, got {s.size}")
        mant, exp, neg, fz, nf = ctypes.c_double(), ctypes.c_int64(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        check(lib().cflx_dbg_det(n, d.ctypes.data, _ptr(s1), _ptr(s2), 1 if square else 0, ctypes.byref(mant),
                                 ctypes.byref(exp), ctypes.byref(neg), ctypes.byref(fz), ctypes.byref(nf)), "dbg_det")
        return dict(mantissa=mant.value, exponent=exp.value, neg=neg.value, first_zero=fz.value, nonfinite=nf.value)

    @staticmethod
    def panel(P, reps=1):
        P = np.ascontiguousarray(P, dtype=np.float64)
        n, v = P.shape
        perm = np.zeros(v, dtype=np.int32)
        A00 = np.zeros((v, v))
        LU = np.zeros((max(n, 1), v))
        ms = ctypes.c_double()
        check(lib().cflx_dbg_panel(n, v, P.ctypes.data, perm.ctypes.data, A00.ctypes.data, LU.ctypes.data, int(reps),
                                   ctypes.byref(ms)), "dbg_panel")
        return perm, A00, LU[:n], ms.value

    @staticmethod
    def trsm(A00, B=None, R=None, nb=0, ld=0):
        """X = B @ inv(U) and Y = inv(L) @ R (A00 = L\\U, L unit lower) on the factorisation's TRSMs, with diagonal blocks
        of nb (0 = the factorisation's default) and the device panels' leading dimension ld (0 = the minimum; the padding
        holds NaN).  Returns (X, Y), None where B / R is None."""
        A00 = np.ascontiguousarray(A00, dtype=np.float64)
        v = A00.shape[0]
        X = Y = None
        n = B.shape[0] if B is not None else R.shape[1]
        if B is not None:
            B = np.ascontiguousarray(B, dtype=np.float64)
            X = np.empty_like(B)
        if R is not None:
            R = np.ascontiguousarray(R, dtype=np.float64)
            Y = np.empty_like(R)
        check(lib().cflx_dbg_trsm(n, v, int(nb), int(ld), A00.ctypes.data, B.ctypes.data if B is not None else None,
                                  X.ctypes.data if X is not None else None, R.ctypes.data if R is not None else None,
                                  Y.ctypes.data if Y is not None else None), "dbg_trsm")
        return X, Y

    @staticmethod
    def diag_inverse(A00, nb):
        """Inverses of the nb x nb diagonal blocks of A00 = L\\U (v x v) on diag_inverse_kernel, as the TRSMs use them.
        Returns (Uinv, LinvT), each (v // nb, nb, nb): inv(U_jj) and inv(L_jj)^T with L unit lower."""
        A00 = np.ascontiguousarray(A00, dtype=np.float64)
        v = A00.shape[0]
        Uinv = np.empty((max(v // nb, 1), nb, nb))
        LinvT = np.empty_like(Uinv)
        check(lib().cflx_dbg_diag_inverse(v, int(nb), A00.ctypes.data, Uinv.ctypes.data, LinvT.ctypes.data), "dbg_diag_inverse")
        return Uinv, LinvT

    @staticmethod
    def potrf_tile(A, variant=0):
        """Cholesky of one v x v tile (lower triangle read) on the factorisation's kernels: variant 0 the one-CTA kernel,
        1 the 128 x 128 block kernel, 2 the 128-block tile driver.  Returns (L, L^T, info); info = 1 + the first
        non-positive pivot's column, 0 on success."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        v = A.shape[0]
        L = np.empty((v, v))
        LT = np.empty((v, v))
        info = ctypes.c_int()
        check(lib().cflx_dbg_potrf_tile(v, A.ctypes.data, L.ctypes.data, LT.ctypes.data, ctypes.byref(info), int(variant)),
              "dbg_potrf_tile")
        return L, LT, info.value

    @staticmethod
    def ldlt_tile(A, tiny=0.0, variant=0):
        """Signed Cholesky A = R S R^T of one v x v tile (lower triangle read) on factor_ldlt's kernels, variants as
        potrf_tile.  Returns dict(R, SRT, s, nrepl, inertia, info): SRT = S R^T, s the signs, inertia (positive,
        negative, zero) pivots, info = 1 + the first exactly zero pivot's column (0: none)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        v = A.shape[0]
        R, SRT, sg = np.empty((v, v)), np.empty((v, v)), np.empty(v)
        nrepl, info = ctypes.c_int(), ctypes.c_int()
        inertia = (ctypes.c_int * 3)()
        check(lib().cflx_dbg_ldlt_tile(v, A.ctypes.data, float(tiny), R.ctypes.data, SRT.ctypes.data, sg.ctypes.data,
                                       ctypes.byref(nrepl), inertia, ctypes.byref(info), int(variant)), "dbg_ldlt_tile")
        return dict(R=R, SRT=SRT, s=sg, nrepl=nrepl.value, inertia=tuple(inertia), info=info.value)

    @staticmethod
    def solve_signs(Z, sgn, v, grid=(1, 1), pos=(0, 0), M=None):
        """cflx_dbg_solve_signs: the sign pass of a signed Cholesky solve on the column-partial buffer Z (Nl x ldn) of
        the share at grid position pos; sgn: the M signs.  Returns the scaled copy."""
        Z = np.array(Z, dtype=np.float64, order="C")
        sg = np.ascontiguousarray(sgn, dtype=np.float64)
        Nl, ldn = Z.shape
        lay = _share(v, v, Nl, grid, pos, M=M if M is not None else len(sg))
        check(lib().cflx_dbg_solve_signs(ctypes.byref(lay), int(ldn), sg.ctypes.data, Z.ctypes.data), "dbg_solve_signs")
        return Z

    @staticmethod
    def getrf_nopiv_tile(A, tiny=0.0, variant=0):
        """Unpivoted LU of one v x v block as LU_rep_fixed runs it: variant 0 the one-CTA kernel on the whole block, 1 the
        128-block driver (v % 128 == 0, v >= 256; what the factorisation runs there).  Returns
        (LU, nrepl, info): L\\U with unit L, the pivots replaced by the tiny rule, 1 + the first exactly zero pivot's
        column (0: none)."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        v = A.shape[0]
        LU = np.empty((v, v))
        nrepl, info = ctypes.c_int(), ctypes.c_int()
        check(lib().cflx_dbg_getrf_nopiv_tile(v, A.ctypes.data, float(tiny), LU.ctypes.data, ctypes.byref(nrepl),
                                              ctypes.byref(info), int(variant)), "dbg_getrf_nopiv_tile")
        return LU, nrepl.value, info.value

    @staticmethod
    def ozaki_gemm(AT, B, C=None, reps=1, want_planes=False, row0=0, col0=0, max_ctas=0):
        """D = C - AT'^T @ B' on the int8 wgmma path, AT' = AT[:, row0:], B' = B[:, col0:] (the planes of all of AT and B
        are made, as the factorisation makes them), on at most max_ctas CTAs (0 = one per SM).  Returns dict(D, ms,
        split_ms[, pa, pb, ea, eb]) with the planes and exponents of all of AT and B."""
        AT = np.ascontiguousarray(AT, dtype=np.float64)
        B = np.ascontiguousarray(B, dtype=np.float64)
        K, Ma = AT.shape
        Nb = B.shape[1]
        M, N = Ma - row0, Nb - col0
        D = np.empty((M, N))
        Cp = np.ascontiguousarray(C, dtype=np.float64) if C is not None else None
        pa = np.zeros((8, Ma, K), dtype=np.int8) if want_planes else None
        pb = np.zeros((8, Nb, K), dtype=np.int8) if want_planes else None
        ea = np.zeros(Ma, dtype=np.int32) if want_planes else None
        eb = np.zeros(Nb, dtype=np.int32) if want_planes else None
        ms, sms = ctypes.c_double(), ctypes.c_double()
        check(lib().cflx_dbg_ozaki_gemm(M, N, K, int(row0), int(col0), int(max_ctas), AT.ctypes.data, B.ctypes.data,
                                        _ptr(Cp), D.ctypes.data, _ptr(pa), _ptr(pb), _ptr(ea), _ptr(eb), int(reps),
                                        ctypes.byref(ms), ctypes.byref(sms)), "dbg_ozaki_gemm")
        return dict(D=D, ms=ms.value, split_ms=sms.value, pa=pa, pb=pb, ea=ea, eb=eb)

    @staticmethod
    def gemm_tf32(terms, AT, B, C=None, reps=1, row0=0, col0=0, max_ctas=0):
        """D = C - AT[:, row0:]^T B[:, col0:] on the TF32 wgmma path (terms 1 or 3); AT (K, row0 + M), B (K, col0 + N).
        Returns dict(D, ms, split_ms, hiA, loA, hiB, loB, ea, eb): the split terms as float32 (rows, KP) arrays (lo None
        with one term) and the int32 exponents, exactly as the kernels produced them."""
        AT = np.ascontiguousarray(AT, dtype=np.float64)
        B = np.ascontiguousarray(B, dtype=np.float64)
        K, Ma = AT.shape
        Nb = B.shape[1]
        M, N = Ma - int(row0), Nb - int(col0)
        KP = (K + 7) // 8 * 8
        Cp = None if C is None else np.ascontiguousarray(C, dtype=np.float64)
        D = np.empty((M, N))
        hiA, hiB = np.empty((Ma, KP), np.float32), np.empty((Nb, KP), np.float32)
        loA, loB = (np.empty((Ma, KP), np.float32), np.empty((Nb, KP), np.float32)) if terms == 3 else (None, None)
        ea, eb = np.empty(Ma, np.int32), np.empty(Nb, np.int32)
        ms, sms = ctypes.c_double(), ctypes.c_double()
        check(lib().cflx_dbg_gemm_tf32(int(terms), M, N, K, int(row0), int(col0), int(max_ctas), AT.ctypes.data,
                                       B.ctypes.data, _ptr(Cp), D.ctypes.data, _ptr(hiA), _ptr(loA), _ptr(hiB), _ptr(loB),
                                       _ptr(ea), _ptr(eb), int(reps), ctypes.byref(ms), ctypes.byref(sms)), "dbg_gemm_tf32")
        return dict(D=D, ms=ms.value, split_ms=sms.value, hiA=hiA, loA=loA, hiB=hiB, loB=loB, ea=ea, eb=eb)

    @staticmethod
    def push_pivots(A, pivot_rows, fnpr):
        """plan_moves + push_phase1..3 + gri update on one rank; returns (A_new, new_row -> old_row, extracted rows)."""
        A = np.array(A, dtype=np.float64, order="C")
        piv = np.ascontiguousarray(pivot_rows, dtype=np.int32)
        gri = np.zeros(A.shape[0], dtype=np.int32)
        a01 = np.zeros((max(1, len(piv)), A.shape[1]))
        check(lib().cflx_dbg_push_pivots(A.shape[0], A.shape[1], A.ctypes.data, len(piv), piv.ctypes.data, int(fnpr),
                                         gri.ctypes.data, a01.ctypes.data), "dbg_push_pivots")
        return A, gri, a01[:len(piv)]

    @staticmethod
    def wgmma_peak(n):
        """tera-MACs/s of back-to-back int8 wgmma 64 x n x 32 (n = 64, 128, 192, 256)."""
        t = ctypes.c_double()
        check(lib().cflx_dbg_wgmma_peak(int(n), ctypes.byref(t)), "dbg_wgmma_peak")
        return t.value

    @staticmethod
    def fp64_peak_ex(which):
        """(burst, sustained) TFLOP/s of the FP64 pipes: 0 the MMA shape gemm_tn_kernel issues (m16n8k8), 1 DFMA,
        2 / 3 / 4 mma m16n8k4 / m16n8k8 / m16n8k16, 5 mma m8n8k4."""
        a, b = ctypes.c_double(), ctypes.c_double()
        check(lib().cflx_dbg_fp64_peak_ex(int(which), ctypes.byref(a), ctypes.byref(b)), "dbg_fp64_peak_ex")
        return a.value, b.value

    @staticmethod
    def fp64_peak(which):
        tf = ctypes.c_double()
        check(lib().cflx_dbg_fp64_peak(int(which), ctypes.byref(tf)), "dbg_fp64_peak")
        return tf.value
