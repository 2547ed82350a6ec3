"""ctypes binding of libconflux_b200.so (the C ABI declared in include/conflux_b200.h).

The product path fails loudly when the CUDA library is missing or no device is visible -- there is no CPU
fallback and nothing here imports oracle/."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libconflux_b200.so")
_lib = None

c_double_p = ctypes.POINTER(ctypes.c_double)
c_int_p = ctypes.POINTER(ctypes.c_int)


class ConfluxError(RuntimeError):
    pass


class ShareLayout(ctypes.Structure):
    """cflx_share_layout: one rank's Ml x Nl share of the block-cyclic matrix (see include/conflux_b200.h)"""
    _fields_ = [(f, ctypes.c_int) for f in ("M", "v", "Kappa", "Ml", "Nl", "Px", "Py", "pi", "pj")]


# every exported symbol of include/conflux_b200.h (checked by tests/test_abi.py)
SYMBOLS = [
    "cflx_last_error", "cflx_version", "cflx_device_count", "cflx_get_unique_id", "cflx_comm_create",
    "cflx_comm_barrier", "cflx_comm_destroy", "cflx_host_alloc", "cflx_host_free", "cflx_auto_grid", "cflx_lu_dims", "cflx_init_matrix_host",
    "cflx_lu_create", "cflx_lu_info", "cflx_lu_set_local", "cflx_lu_queue_next_local", "cflx_lu_factor", "cflx_lu_factor_fixed", "cflx_rbt_multipliers", "cflx_lu_rbt", "cflx_lu_rbt_solve", "cflx_lu_rbt_apply_local", "cflx_lu_get_factors",
    "cflx_lu_get_permutation", "cflx_lu_residual", "cflx_lu_validate", "cflx_lu_solve", "cflx_lu_solve_trans", "cflx_rhs_local_cols", "cflx_lu_solve_local", "cflx_lu_rcond", "cflx_lu_refine", "cflx_lu_refine_x", "cflx_lu_equilibrate", "cflx_lu_svx", "cflx_lu_equilibrate_b", "cflx_lu_svxx", "cflx_refine_block_cols", "cflx_lu_refine_local", "cflx_lu_refine_x_local", "cflx_lu_svx_local", "cflx_lu_svxx_local", "cflx_lu_sv_mixed", "cflx_lu_inverse", "cflx_lu_det", "cflx_lu_launch_count", "cflx_lu_uses_ozaki", "cflx_lu_set_profiling", "cflx_lu_phase_ms", "cflx_lu_timeline",
    "cflx_lu_set_kernel_timing", "cflx_lu_trailing_stats", "cflx_lu_destroy", "cflx_chol_auto_grid", "cflx_chol_auto_tile", "cflx_chol_dims", "cflx_chol_init_matrix_host",
    "cflx_chol_create", "cflx_chol_info", "cflx_chol_set_local", "cflx_chol_factor", "cflx_chol_factor_ldlt", "cflx_chol_rbt", "cflx_chol_rbt_solve", "cflx_chol_rbt_apply_local", "cflx_chol_get_signs", "cflx_chol_get_input", "cflx_chol_get_local", "cflx_chol_validate",
    "cflx_chol_solve", "cflx_chol_solve_local", "cflx_chol_rcond", "cflx_chol_refine", "cflx_chol_refine_x", "cflx_chol_equilibrate", "cflx_chol_svx", "cflx_chol_equilibrate_b", "cflx_chol_svxx", "cflx_chol_refine_local", "cflx_chol_refine_x_local", "cflx_chol_svx_local", "cflx_chol_svxx_local", "cflx_chol_sv_mixed", "cflx_chol_inverse", "cflx_chol_det", "cflx_chol_launch_count", "cflx_chol_destroy", "cflx_dbg_gemm_tn", "cflx_dbg_gemm_narrow", "cflx_dbg_gemm_narrow_tn", "cflx_dbg_gemm_narrow_window", "cflx_dbg_diag_solve", "cflx_dbg_residual", "cflx_dbg_residual_x", "cflx_dbg_equil", "cflx_dbg_growth_cols", "cflx_dbg_inverse_share", "cflx_dbg_solve_local_share", "cflx_dbg_norm_share", "cflx_dbg_rbt_share", "cflx_dbg_chol_validate_share", "cflx_dbg_lu_validate_share", "cflx_dbg_chol_gather_cols", "cflx_dbg_refine_assemble", "cflx_dbg_refine_columns", "cflx_dbg_det", "cflx_dbg_panel", "cflx_dbg_trsm", "cflx_dbg_diag_inverse", "cflx_dbg_potrf_tile", "cflx_dbg_ldlt_tile", "cflx_dbg_solve_signs", "cflx_dbg_getrf_nopiv_tile", "cflx_dbg_push_pivots", "cflx_dbg_ozaki_gemm", "cflx_dbg_gemm_tf32", "cflx_dbg_wgmma_peak", "cflx_dbg_fp64_peak", "cflx_dbg_fp64_peak_ex",
]


def _preload_nccl():
    """libconflux_b200.so needs `libnccl.so.2`.  PyTorch bundles a newer NCCL under the same soname; if ours were
    loaded first a later `import torch` would bind to the older system library and fail to resolve its symbols, so
    the bundled one (when present) is loaded first and shared by both."""
    import sys
    for d in sys.path:
        cand = os.path.join(d, "nvidia", "nccl", "lib", "libnccl.so.2")
        if os.path.exists(cand):
            try:
                ctypes.CDLL(cand, mode=ctypes.RTLD_GLOBAL)
                return cand
            except OSError:
                pass
    return None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ConfluxError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(conflux_b200 has no CPU fallback)")
        _preload_nccl()
        L = ctypes.CDLL(LIB_PATH)
        L.cflx_last_error.restype = ctypes.c_char_p
        L.cflx_version.restype = ctypes.c_char_p
        L.cflx_comm_destroy.restype = None
        L.cflx_lu_destroy.restype = None
        L.cflx_comm_destroy.argtypes = [ctypes.c_void_p]
        L.cflx_lu_destroy.argtypes = [ctypes.c_void_p]
        L.cflx_comm_barrier.argtypes = [ctypes.c_void_p]
        L.cflx_comm_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.POINTER(ctypes.c_void_p)]
        L.cflx_lu_create.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 6 + [ctypes.POINTER(ctypes.c_void_p)]
        L.cflx_host_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p)]
        L.cflx_host_free.argtypes = [ctypes.c_void_p]
        L.cflx_lu_info.argtypes = [ctypes.c_void_p, c_int_p]
        L.cflx_lu_set_local.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_queue_next_local.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_factor.argtypes = [ctypes.c_void_p, c_double_p]
        L.cflx_lu_factor_fixed.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_double] + [ctypes.c_void_p] * 3
        L.cflx_rbt_multipliers.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_rbt.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_rbt_solve.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_rbt_apply_local.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.cflx_lu_get_factors.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_get_permutation.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_residual.argtypes = [ctypes.c_void_p, c_double_p]
        L.cflx_lu_validate.argtypes = [ctypes.c_void_p, c_double_p, c_double_p]
        L.cflx_lu_solve.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.cflx_lu_solve_trans.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                          ctypes.c_int]
        L.cflx_rhs_local_cols.argtypes = [ctypes.c_int] * 3 + [c_int_p]
        L.cflx_lu_solve_local.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_int]
        L.cflx_lu_rcond.argtypes = [ctypes.c_void_p, c_double_p, c_double_p]
        L.cflx_lu_refine.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_lu_refine_x.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.cflx_lu_equilibrate.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7
        L.cflx_lu_svx.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                  ctypes.c_int] + [ctypes.c_void_p] * 6
        L.cflx_lu_equilibrate_b.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7
        L.cflx_lu_svxx.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                   ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7
        # the distributed refinement and expert drivers: the replicated argtypes with B / X as shares (device pointers too)
        L.cflx_refine_block_cols.argtypes = [ctypes.c_int, c_int_p]
        for name in ("refine", "refine_x", "svx", "svxx"):
            getattr(L, f"cflx_lu_{name}_local").argtypes = getattr(L, f"cflx_lu_{name}").argtypes
        _mixed = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                  c_int_p, ctypes.c_void_p, c_double_p]
        L.cflx_lu_sv_mixed.argtypes = [ctypes.c_void_p] + _mixed
        L.cflx_chol_sv_mixed.argtypes = [ctypes.c_void_p] + _mixed
        L.cflx_lu_inverse.argtypes = [ctypes.c_void_p, ctypes.c_void_p, c_int_p]
        L.cflx_lu_det.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.cflx_lu_uses_ozaki.argtypes = [ctypes.c_void_p]
        L.cflx_lu_launch_count.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64), ctypes.c_int]
        L.cflx_lu_set_profiling.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.cflx_lu_phase_ms.argtypes = [ctypes.c_void_p, c_double_p]
        L.cflx_lu_timeline.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
        L.cflx_lu_set_kernel_timing.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.cflx_lu_trailing_stats.argtypes = [ctypes.c_void_p, c_double_p, c_double_p]
        L.cflx_chol_destroy.restype = None
        L.cflx_chol_destroy.argtypes = [ctypes.c_void_p]
        L.cflx_chol_auto_grid.argtypes = [ctypes.c_int, ctypes.c_int, c_int_p]
        L.cflx_chol_auto_tile.argtypes = [ctypes.c_int] * 3
        L.cflx_chol_dims.argtypes = [ctypes.c_int] * 5 + [c_int_p]
        L.cflx_chol_init_matrix_host.argtypes = [ctypes.c_int] * 6 + [ctypes.c_void_p]
        L.cflx_chol_create.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_void_p)]
        L.cflx_chol_info.argtypes = [ctypes.c_void_p, c_int_p]
        L.cflx_chol_set_local.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_chol_factor.argtypes = [ctypes.c_void_p, c_double_p]
        L.cflx_chol_factor_ldlt.argtypes = [ctypes.c_void_p, ctypes.c_double] + [ctypes.c_void_p] * 4
        L.cflx_chol_rbt.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64, ctypes.c_void_p]
        L.cflx_chol_rbt_solve.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                          ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_chol_rbt_apply_local.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.cflx_chol_get_signs.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_chol_get_input.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_chol_get_local.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_chol_validate.argtypes = [ctypes.c_void_p, c_double_p, c_double_p]
        L.cflx_chol_solve.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.cflx_chol_solve_local.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_int]
        L.cflx_chol_rcond.argtypes = [ctypes.c_void_p, c_double_p, c_double_p]
        L.cflx_chol_refine.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_chol_refine_x.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.c_int] + [ctypes.c_void_p] * 5
        L.cflx_chol_equilibrate.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.cflx_chol_svx.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int
                                    ] + [ctypes.c_void_p] * 5
        L.cflx_chol_equilibrate_b.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
        L.cflx_chol_svxx.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_int] + [ctypes.c_void_p] * 7
        for name in ("refine", "refine_x", "svx", "svxx"):
            getattr(L, f"cflx_chol_{name}_local").argtypes = getattr(L, f"cflx_chol_{name}").argtypes
        L.cflx_chol_inverse.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_chol_det.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3
        L.cflx_chol_launch_count.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64), ctypes.c_int]
        L.cflx_init_matrix_host.argtypes = [ctypes.c_int] * 8 + [ctypes.c_void_p]
        _buf = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64]
        L.cflx_dbg_gemm_tn.argtypes = [ctypes.c_int] * 3 + _buf + [ctypes.c_int64] + _buf + [ctypes.c_int64] + _buf + [
            ctypes.c_int] * 2 + [ctypes.c_double] * 2 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                                          c_double_p]
        L.cflx_dbg_gemm_narrow.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_double] * 2 + [
            ctypes.c_void_p, ctypes.c_int, c_double_p]
        L.cflx_dbg_gemm_narrow_tn.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_double] * 2 + [
            ctypes.c_void_p, ctypes.c_int, c_double_p]
        _blk = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int]
        L.cflx_dbg_gemm_narrow_window.argtypes = [ctypes.c_int] * 4 + _blk * 3 + [ctypes.c_double] * 2 + [
            ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_dbg_diag_solve.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64] + [
            ctypes.c_int] * 3 + [ctypes.c_void_p] * 3
        share = ctypes.POINTER(ShareLayout)
        L.cflx_dbg_residual.argtypes = [ctypes.c_int, share, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 4 + [
            ctypes.c_int, c_double_p]
        L.cflx_dbg_residual_x.argtypes = [ctypes.c_int, share, ctypes.c_void_p, ctypes.c_int] + [
            ctypes.c_void_p] * 6 + [ctypes.c_int, c_double_p]
        L.cflx_dbg_equil.argtypes = [share] + [ctypes.c_void_p] * 3 + [ctypes.c_char, ctypes.c_int] + [
            ctypes.c_void_p] * 7
        L.cflx_dbg_growth_cols.argtypes = [ctypes.c_int, share, ctypes.c_int] + [ctypes.c_void_p] * 4
        L.cflx_dbg_inverse_share.argtypes = [ctypes.c_int, share] + [ctypes.c_int] * 3 + [
            ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int]
        L.cflx_dbg_solve_local_share.argtypes = [ctypes.c_int, share] + [ctypes.c_int] * 3 + [
            ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int]
        L.cflx_dbg_norm_share.argtypes = [ctypes.c_int, share] + [ctypes.c_void_p] * 2
        L.cflx_dbg_rbt_share.argtypes = [ctypes.c_int, share, ctypes.c_int] + [ctypes.c_void_p] * 2 + [
            ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.cflx_dbg_chol_validate_share.argtypes = [share, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 2
        L.cflx_dbg_lu_validate_share.argtypes = [share, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 2
        L.cflx_dbg_chol_gather_cols.argtypes = [share, ctypes.c_int] + [ctypes.c_void_p] * 2
        L.cflx_dbg_refine_assemble.argtypes = [ctypes.c_int] * 12 + [ctypes.c_void_p] * 6
        L.cflx_dbg_refine_columns.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 10
        L.cflx_dbg_det.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int] + [ctypes.c_void_p] * 5
        L.cflx_dbg_panel.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_int, c_double_p]
        L.cflx_dbg_trsm.argtypes = [ctypes.c_int] * 3 + [ctypes.c_int64] + [ctypes.c_void_p] * 5
        L.cflx_dbg_diag_inverse.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 3
        L.cflx_dbg_potrf_tile.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_int]
        L.cflx_dbg_solve_signs.argtypes = [share, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_dbg_ldlt_tile.argtypes = ([ctypes.c_int, ctypes.c_void_p, ctypes.c_double] + [ctypes.c_void_p] * 6 +
                                         [ctypes.c_int])
        L.cflx_dbg_getrf_nopiv_tile.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_double] + [ctypes.c_void_p] * 3 + [
            ctypes.c_int]
        L.cflx_dbg_push_pivots.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p]
        L.cflx_dbg_ozaki_gemm.argtypes = [ctypes.c_int] * 6 + [ctypes.c_void_p] * 8 + [ctypes.c_int, c_double_p, c_double_p]
        L.cflx_dbg_gemm_tf32.argtypes = [ctypes.c_int] * 7 + [ctypes.c_void_p] * 10 + [ctypes.c_int, c_double_p, c_double_p]
        L.cflx_dbg_wgmma_peak.argtypes = [ctypes.c_int, c_double_p]
        L.cflx_dbg_fp64_peak.argtypes = [ctypes.c_int, c_double_p]
        L.cflx_dbg_fp64_peak_ex.argtypes = [ctypes.c_int, c_double_p, c_double_p]
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().cflx_last_error().decode(errors="replace")
        raise ConfluxError(f"{what} failed with status {rc}: {msg}")
