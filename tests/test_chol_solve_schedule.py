"""CPU: the schedule of cflx_chol_solve (oracle/chol_solve_ref.py: per-rank partial right-hand sides by tile row and by
tile column, reduce / broadcast / update per tile, nb-block inverse sweeps, final all-reduce) solves A X = B with the
Cholesky factor, on every grid shape, without reading anything the device must not read; every member of each
communicator issues the same collectives in the same order; and the C++ facade's choleskySolve compiles."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.linalg

from oracle import chol_ref, chol_solve_ref, hp_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRIDS = [(1, 1, 1), (2, 1, 1), (1, 2, 1), (2, 2, 1), (4, 2, 1), (2, 2, 2), (3, 2, 1), (1, 3, 2)]
# (100, 16): Kappa = 7 (N padded to 112), not a multiple of 2, 3 or 4;  (96, 8): Kappa = 12, a multiple of every grid side
SIZES = [(100, 16), (96, 8)]


def _members(r_comm, Px, Py, Pz):
    """ranks of one communicator named in the log"""
    kind = r_comm[0]
    if kind == "world":
        return list(range(Px * Py * Pz))
    if kind == "row":
        return [(r_comm[1] * Py + pj) * Pz for pj in range(Py)]
    return [(pi * Py + r_comm[1]) * Pz for pi in range(Px)]


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: "%dx%dx%d" % g)
@pytest.mark.parametrize("N,v", SIZES)
@pytest.mark.parametrize("nrhs", [1, 3, 17])
def test_schedule_solves_the_system(grid, N, v, nrhs):
    Px, Py, Pz = grid
    d = chol_ref.dims(N, v, Px, Py, Pz)
    rng = np.random.default_rng(N + nrhs + 10 * Px + Py)
    S = hp_ref.random_spd(d["N"], 1e2, rng)
    L = np.linalg.cholesky(S)
    # NaN wherever the device must not read: tiles above the diagonal, tiles beyond Kappa, layers pk != 0
    L_locals = chol_solve_ref.scatter(L, N, v, Px, Py, Pz, upper=np.nan, pad=np.nan, layers=np.nan)
    B = rng.standard_normal((d["N"], nrhs))
    log = {}
    X = chol_solve_ref.solve(L_locals, B, N, v, Px, Py, Pz, log=log)
    assert X.shape == B.shape and np.all(np.isfinite(X))
    Xh = scipy.linalg.cho_solve((L, True), B)
    assert np.abs(X - Xh).max() <= 1e-10 * np.abs(Xh).max()
    assert chol_solve_ref.backward_error(S, X, B) <= 1e-13
    # the same sequence of collectives on every member of every communicator (the stand-in for "does not deadlock")
    comms = {c for calls in log.values() for (c, *_rest) in calls}
    for c in comms:
        seqs = [[x for x in log[r] if x[0] == c] for r in _members(c, Px, Py, Pz)]
        assert all(s == seqs[0] for s in seqs), c
        assert seqs[0]
    for r, calls in log.items():                                     # layers pk != 0 take part in the all-reduce only
        if r % Pz:
            assert [x[1] for x in calls] == ["allreduce"]
    if Px * Py * Pz == 1:
        assert log[0] == []                                          # 1x1x1 makes no collective call


def test_vector_and_padded_system():
    N, v = 100, 16
    d = chol_ref.dims(N, v, 1, 1, 1)
    assert d["N"] == 112
    rng = np.random.default_rng(5)
    S = hp_ref.random_spd(d["N"], 1e2, rng)
    b = rng.standard_normal(d["N"])
    x = chol_solve_ref.solve(chol_solve_ref.scatter(np.linalg.cholesky(S), N, v), b, N, v)
    assert x.shape == (d["N"],)
    assert chol_solve_ref.backward_error(S, x, b) <= 1e-13


def test_scatter_inverts_assemble():
    N, v, grid = 100, 16, (3, 2, 2)
    A = np.random.default_rng(1).standard_normal((112, 112))
    locs = chol_solve_ref.scatter(A, N, v, *grid)
    assert np.array_equal(chol_ref.assemble(locs, N, v, *grid), A)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")
def test_cpp_facade_choleskySolve_compiles(tmp_path):
    src = tmp_path / "use_solve.cpp"
    src.write_text('#include "conflux/cholesky/conflux_b200_cholesky.hpp"\n'
                   "void f(const double* B, double* X) { conflux::choleskySolve(3, B, 3, X, 3); }\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)], check=True)
