"""CPU: the schedule of cflx_lu_inverse and cflx_chol_inverse (oracle/inverse_ref.py: blocks of nc columns seeded with the
identity, the engine's sweeps over the tile ranges that skip each block's zero rows, the world all-reduce, the scatter
into every rank's share) gives numpy's inverse on every grid shape, without reading anything the device must not read;
every member of each communicator issues the same collectives in the same order; skipping changes no bit; the block
updates count LAPACK's flops; and the C++ facades compile."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import chol_ref, chol_solve_ref, hp_ref, inverse_ref, layout, restate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-10


def _members(c, Px, Py, Pz, every_layer):
    """ranks of one communicator named in the log (the LU's row / column communicators hold every layer)"""
    layers = range(Pz) if every_layer else range(1)
    if c[0] == "world":
        return list(range(Px * Py * Pz))
    if c[0] == "row":
        return [(c[1] * Py + pj) * Pz + pk for pj in range(Py) for pk in layers]
    return [(pi * Py + c[1]) * Pz + pk for pi in range(Px) for pk in layers]


def _check_log(log, grid, every_layer):
    Px, Py, Pz = grid
    comms = {c for calls in log.values() for (c, *_rest) in calls}
    for c in comms:
        seqs = [[x for x in log[r] if x[0] == c] for r in _members(c, Px, Py, Pz, every_layer)]
        assert all(s == seqs[0] for s in seqs), c
        assert seqs[0]
    if Px * Py * Pz == 1:
        assert log[0] == []
    if not every_layer:
        for r, calls in log.items():                                 # the Cholesky's layers pk != 0: the all-reduces only
            if r % Pz:
                assert {x[1] for x in calls} == {"allreduce"}


def _lu_case(N, v, grid, seed):
    d = layout.dims(N, v, *grid)
    A = np.random.default_rng(seed).standard_normal((d["M"], d["M"]))
    f = restate.lu(layout.scatter(A, v, *grid), N, v, *grid)
    C = [c.copy() for c in f["C"]]
    for r in range(len(C)):
        if r % grid[2]:
            C[r][:] = np.nan                                          # layers pk != 0 hold no factors
    return d, A, C, f["perm"]


LU_CASES = [((1, 1, 1), 96, 8), ((1, 1, 2), 96, 8), ((2, 2, 1), 96, 8), ((2, 2, 2), 96, 8), ((3, 3, 1), 96, 8),
            ((1, 1, 1), 100, 16)]


@pytest.mark.parametrize("grid,N,v", LU_CASES, ids=lambda x: "x".join(map(str, x)) if isinstance(x, tuple) else str(x))
@pytest.mark.parametrize("nc_tiles", [1, 5])
def test_lu_schedule_inverts(grid, N, v, nc_tiles):
    d, A, C, perm = _lu_case(N, v, grid, N + v + sum(grid))
    M, Nt = d["M"], d["Nt"]
    assert nc_tiles == 1 or Nt % nc_tiles                             # several tiles: a narrower last block
    log, launches = {}, []
    shares = inverse_ref.lu_inverse(C, perm, N, v, *grid, nc=nc_tiles * v, log=log, launches=launches)
    X = layout.assemble(shares, N, v, *grid)
    Xi = np.linalg.inv(A)
    assert np.abs(X - Xi).max() <= TOL * np.abs(Xi).max()
    for r, s in enumerate(shares):                                   # layers pk != 0 receive layer 0's bits
        assert np.array_equal(s, shares[r - r % grid[2]])
    _check_log(log, grid, True)
    full = inverse_ref.lu_inverse(C, perm, N, v, *grid, nc=nc_tiles * v, skip=False)
    for a, b in zip(shares, full):
        assert np.array_equal(a, b)                                  # skipping the zero tiles changes no bit


CHOL_GRIDS = [(1, 1, 1), (2, 1, 1), (1, 2, 1), (2, 2, 1), (4, 2, 1), (2, 2, 2), (3, 2, 1), (1, 3, 2)]


def _lower_tiles(X, v, K):
    """the entries of the real tiles on and below the diagonal (whole diagonal tiles)"""
    tr = np.arange(X.shape[0]) // v
    return (tr[:, None] >= tr[None, :]) & (tr[:, None] < K) & (tr[None, :] < K)


@pytest.mark.parametrize("grid", CHOL_GRIDS, ids=lambda g: "%dx%dx%d" % g)
@pytest.mark.parametrize("N,v", [(100, 16), (96, 8)])
@pytest.mark.parametrize("nc_tiles", [1, 5])
def test_chol_schedule_inverts(grid, N, v, nc_tiles):
    d = chol_ref.dims(N, v, *grid)
    Np, K = d["N"], d["Kappa"]
    rng = np.random.default_rng(N + v + 7 * grid[0] + grid[1])
    S = hp_ref.random_spd(Np, 1e2, rng)
    L = np.linalg.cholesky(S)
    # NaN wherever the device must not read: tiles above the diagonal, tiles beyond Kappa, layers pk != 0
    L_locals = chol_solve_ref.scatter(L, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan)
    log, launches = {}, []
    shares = inverse_ref.chol_inverse(L_locals, N, v, *grid, nc=nc_tiles * v, log=log, launches=launches)
    for s in shares:
        assert np.all(np.isfinite(s))
    X = chol_ref.assemble(shares, N, v, *grid)
    Si = np.linalg.inv(S)
    low = _lower_tiles(X, v, K)
    assert np.abs(np.where(low, X - Si, 0.0)).max() <= TOL * np.abs(Si).max()
    assert np.all(X[~low] == 0.0)
    for r, s in enumerate(shares):                                   # every layer receives layer 0's bits
        assert np.array_equal(s, shares[r - r % grid[2]])
    for r, s in enumerate(shares):                                   # the local tiles beyond Kappa are zero
        pi, pj = r // (grid[1] * grid[2]), (r // grid[2]) % grid[1]
        for lt in range(d["Ml"] // v):
            if lt * grid[0] + pi >= K:
                assert np.all(s[lt * v:(lt + 1) * v] == 0.0)
        for lt in range(d["Nl"] // v):
            if lt * grid[1] + pj >= K:
                assert np.all(s[:, lt * v:(lt + 1) * v] == 0.0)
    _check_log(log, grid, False)
    full = inverse_ref.chol_inverse(L_locals, N, v, *grid, nc=nc_tiles * v, skip=False)
    for a, b in zip(shares, full):
        assert np.array_equal(a, b)


def _flops(launches):
    return sum(2 * m * n * k for _, m, n, k in launches)


@pytest.mark.parametrize("nc_tiles", [1, 3])
def test_block_updates_count_lapack_flops(nc_tiles):
    """the update launches of the skipping schedule count 4/3 M^3 (LU) and 2/3 M^3 (Cholesky) flops up to M^2 nc-order
    terms; without the skipping both count 2 M^3"""
    N, v = 256, 16
    nc = nc_tiles * v
    d, _, C, perm = _lu_case(N, v, (1, 1, 1), 3)
    M = d["M"]
    la, lf = [], []
    inverse_ref.lu_inverse(C, perm, N, v, nc=nc, launches=la)
    inverse_ref.lu_inverse(C, perm, N, v, nc=nc, skip=False, launches=lf)
    assert abs(_flops(la) - 4 / 3 * M ** 3) <= 2 * M * M * (nc + v)
    assert abs(_flops(lf) - 2 * M ** 3) <= 2 * M * M * (nc + v)
    S = hp_ref.random_spd(M, 1e2, np.random.default_rng(4))
    Ll = chol_solve_ref.scatter(np.linalg.cholesky(S), N, v)
    la, lf = [], []
    inverse_ref.chol_inverse(Ll, N, v, nc=nc, launches=la)
    inverse_ref.chol_inverse(Ll, N, v, nc=nc, skip=False, launches=lf)
    assert abs(_flops(la) - 2 / 3 * M ** 3) <= 2 * M * M * (nc + v)
    assert abs(_flops(lf) - 2 * M ** 3) <= 2 * M * M * (nc + v)


def test_share_kernels_restated():
    """the per-share seed, scatter and zero pass the GPU hook is compared against, on a small hand-checked case"""
    v, Px, Py, pi, pj = 2, 2, 3, 1, 2
    W = inverse_ref.seed_share(6, v, Px, pi, 4, 2, 4)                 # local rows 0..3 hold global rows 2, 3, 6, 7
    assert W.shape == (6, 8)
    assert [tuple(x) for x in np.argwhere(W)] == [(0, 0), (1, 1)]
    M = 12
    X = np.arange(M * 4, dtype=np.float64).reshape(M, 4)
    share = np.full((6, 4), -1.0)
    inverse_ref.scatter_share("chol", X, 4, 4, None, share, v, Px, Py, pi, pj, Kappa=5)
    # global columns 4, 5 (tile 2) live at local columns 0, 1; local rows 0..5 are global rows 2, 3, 6, 7, 10, 11
    assert np.array_equal(share[:, 2:], np.full((6, 2), -1.0))
    assert np.all(share[:2, :2] == -1.0)                              # tile 1 is above the diagonal tile 2
    assert np.array_equal(share[2:4, :2], X[6:8, :2])
    assert np.all(share[4:, :2] == -1.0)                              # tile 5 >= Kappa
    inverse_ref.zero_share(share, v, Px, Py, pi, pj, 5)
    assert np.all(share[:2] == 0.0) and np.all(share[4:] == 0.0) and np.all(share[:, 2:] == 0.0)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")
def test_cpp_facades_compile(tmp_path):
    src = tmp_path / "use_inverse.cpp"
    src.write_text('#include "conflux/lu/conflux_b200.hpp"\n'
                   '#include "conflux/cholesky/conflux_b200_cholesky.hpp"\n'
                   "int f(conflux::lu_params<double>& g, double* a) { conflux::choleskyInverse(a);\n"
                   "  return conflux::LU_inverse(g, a); }\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)], check=True)
