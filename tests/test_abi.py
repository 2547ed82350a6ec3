"""CPU: the C-ABI library loads and exports every symbol include/conflux_b200.h declares; host-only entry points
work; device entry points refuse loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

import conflux_b200 as cb
from conflux_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_exported():
    hdr = open(os.path.join(ROOT, "include", "conflux_b200.h")).read()
    declared = set(re.findall(r"\b(cflx_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.SYMBOLS)
    L = ctypes.CDLL(_lib.LIB_PATH)
    for s in declared:
        assert hasattr(L, s), s


def test_auto_grid_matches_reference_rule():
    # lu_params.hpp:21-47: 1 -> 1x1x1, 2 -> 1x1x2, 4 -> 2x2x1, 8 -> 2x2x2, 9 -> 3x3x1, 16 -> 4x4x1, 18 -> 3x3x2
    for P, g in [(1, (1, 1, 1)), (2, (1, 1, 2)), (4, (2, 2, 1)), (8, (2, 2, 2)), (9, (3, 3, 1)), (16, (4, 4, 1)),
                 (18, (3, 3, 2))]:
        assert cb.auto_grid(4096, 4096, P) == g


def test_dims_match_reference_rule():
    d = cb.lu_dims(65536, 65536, 512, 2, 2, 2)
    assert (d["M"], d["Ml"], d["Nl"], d["Nt"], d["nlayr"]) == (65536, 32768, 32768, 128, 256)
    d = cb.lu_dims(1000, 1000, 256, 1, 1, 1)       # padding to a multiple of v*Px (lu_params.hpp:67-71)
    assert (d["M"], d["N"], d["Nt"]) == (1024, 1024, 4)
    d = cb.lu_dims(27, 27, 3, 3, 3, 1)
    assert (d["Ml"], d["Nl"], d["Nt"]) == (9, 9, 9)


def test_init_matrix_host_is_the_reference_generator():
    from oracle import restate
    for (N, v, g) in [(64, 8, (2, 2, 2)), (96, 16, (1, 1, 1)), (72, 4, (3, 3, 2))]:
        ref = restate.init_matrix(N, v, *g)
        for rank in range(g[0] * g[1] * g[2]):
            assert np.array_equal(cb.init_matrix_host(N, N, v, *g, rank), ref[rank])


def test_fixed_input_matrices_are_the_references(golden_dir):
    """lu_params.hpp:157-363: for (padded) M == N in {8, 9, 16, 20, 27, 32} InitMatrix fills a FIXED matrix.  The golden
    fixtures hold what the reference itself produced on several grids (tests/golden/make_golden.py)."""
    G = np.load(os.path.join(golden_dir, "lu_cases.npz"))
    seen = set()
    for i, (N, v, Px, Py, Pz) in enumerate(G["cases"]):
        if int(N) not in (16, 27, 32):
            continue
        for rank in range(int(Px * Py * Pz)):
            mine = cb.init_matrix_host(int(N), int(N), int(v), int(Px), int(Py), int(Pz), rank)
            assert np.array_equal(mine.reshape(-1), G[f"c{i}_A"][rank].reshape(-1)), (N, v, Px, Py, Pz, rank)
        seen.add(int(N))
    assert seen == {16, 27, 32}
    # padding reaches a fixed size too: N = 30, v = 4, Px = 2 is padded to 32 and takes the 32 x 32 table
    a = cb.init_matrix_host(30, 30, 4, 2, 2, 1, 0)
    b = cb.init_matrix_host(32, 32, 4, 2, 2, 1, 0)
    assert np.array_equal(a, b) and float(a.max()) <= 9.0


def test_cholesky_host_rules_match_the_reference():
    # Cholesky.cpp:75-111 grid choice; :113-134 tile choice; CholeskyProperties (Kappa = N / v tiles, 2-D cyclic A11)
    assert cb.chol_auto_grid(8, 32768) == (4, 2, 1) and cb.chol_auto_grid(8, 8192) == (2, 2, 2)
    assert cb.chol_auto_grid(4, 65536) == (2, 2, 1) and cb.chol_auto_grid(16, 4096) == (4, 4, 1)
    assert cb.chol_auto_grid(2, 4096) == (2, 1, 1) and cb.chol_auto_grid(1, 4096) == (1, 1, 1)
    assert _lib.lib().cflx_chol_auto_tile(32768, 8, 1) == 512 and _lib.lib().cflx_chol_auto_tile(2048, 4, 1) == 128
    d = cb.chol_dims(32768, 512, 4, 2, 1)
    assert (d["Kappa"], d["Ml"], d["Nl"]) == (64, 8192, 16384)
    d = cb.chol_dims(100, 16, 2, 2, 2)                      # padded to a multiple of v (CholeskyIO.cpp:196-203)
    assert (d["N"], d["Kappa"], d["Ml"], d["l"]) == (112, 7, 64, 8)


def test_cholesky_generator_matches_restatement():
    """CholeskyIO.cpp:100-172: every tile = lower(R^T R) from rand() after srand(1), strengthened global diagonal."""
    from oracle import chol_ref
    N, v, g = 96, 16, (2, 2, 2)
    A, T, mx = chol_ref.init_matrix(N, v)
    d = cb.chol_dims(N, v, *g)
    locs = []
    for rank in range(8):
        out = np.zeros((d["Ml"], d["Nl"]))
        assert _lib.lib().cflx_chol_init_matrix_host(N, v, *g, rank, out.ctypes.data) == 0
        locs.append(out)
        if rank % 2:
            assert not out.any()                            # layers pz != 0 start at zero
    G = chol_ref.assemble(locs, N, v, *g)
    assert np.allclose(np.tril(G), A, rtol=1e-14, atol=1e-14)
    assert np.array_equal(np.diag(G), np.diag(A)) or np.allclose(np.diag(G), np.diag(A), rtol=1e-15)


def test_device_entry_points_refuse_without_gpu():
    n = ctypes.c_int(-1)
    assert _lib.lib().cflx_device_count(ctypes.byref(n)) == 0
    if n.value > 0:
        pytest.skip("GPU present")
    with pytest.raises(cb.ConfluxError, match="no CPU fallback"):
        cb.Comm(1, 0, None, 0)
    with pytest.raises(cb.ConfluxError, match="no CPU fallback"):
        cb.dbg.gemm_tn(np.ones((4, 4)), np.ones((4, 4)))
    A = np.ones((8, 8))
    for call in (lambda: cb.dbg.norm_share("sym", A, 4, Kappa=2),
                 lambda: cb.dbg.chol_validate_share(A, 4, 2),
                 lambda: cb.dbg.lu_validate_share(A, 4),
                 lambda: cb.dbg.chol_gather_cols([np.ones((4, 8))], 4, 1, 1, 0, 8, 8, 0),
                 lambda: cb.dbg.refine_assemble("x", np.zeros((8, 16)), np.zeros((8, 8)), (1, 1, 1), 4, 8, 8, 8, 1, 0, 8),
                 lambda: cb.dbg.refine_columns(A, A, np.ones(8), 8),
                 lambda: cb.dbg.gemm_narrow_window(A, A, A, 4, 4, 4),
                 lambda: cb.dbg.diag_solve("lower", A, np.ones((8, 2)), 8, 4)):
        with pytest.raises(cb.ConfluxError, match="no CPU fallback"):
            call()
