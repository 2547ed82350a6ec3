"""CPU: the schedule of cflx_lu_solve_local and cflx_chol_solve_local (oracle/solve_local_ref.py: B and X distributed like
A, each block of columns packed from the layer-0 shares, summed with one contributor per element, solved and scattered
into every rank's share) gives the dense solve on every grid shape, reads no entry of B it must not read (NaN there never
leaks in) and writes no entry of X it must not write (a sentinel there survives); the column count of the library
matches the restatement; and the C++ facades compile."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.linalg

import conflux_b200 as cb
from oracle import chol_ref, chol_solve_ref, hp_ref, layout, solve_local_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = -7777.0
TOL = 1e-9


def test_rhs_local_cols_matches_restatement():
    for nrhs in (1, 2, 7, 8, 9, 63, 64, 65, 1000, 65536):
        for v in (1, 4, 8, 256, 512):
            for Py in (1, 2, 3, 4):
                assert cb.rhs_local_cols(nrhs, v, Py) == solve_local_ref.rhs_local_cols(nrhs, v, Py)
    for N, v, g in [(65536, 512, (2, 2, 2)), (1000, 256, (1, 1, 1)), (27, 3, (3, 3, 1)), (40, 8, (3, 3, 2)),
                    (100, 16, (2, 2, 1))]:                             # nrhs = M gives Nl on the LU grids
        d = cb.lu_dims(N, N, v, *g)
        assert cb.rhs_local_cols(d["M"], v, g[1]) == d["Nl"]
    for N, v, g in [(32768, 512, (4, 2, 1)), (44, 8, (4, 2, 1)), (100, 16, (2, 1, 1)), (100, 16, (2, 2, 2)),
                    (1000, 48, (1, 2, 1))]:                            # and on Cholesky grids, Px != Py among them
        d = cb.chol_dims(N, v, *g)
        assert cb.rhs_local_cols(d["N"], v, g[1]) == d["Nl"]
    with pytest.raises(cb.ConfluxError):
        cb.rhs_local_cols(0, 8, 1)


def _shares(kind, G, nrhs, v, grid, Kappa, fill, pad, ld_extra=3):
    """G (M x nrhs) -> every rank's share (Ml x rhs_local_cols + ld_extra): G's entries at the ones a solve reads and
    writes (layer 0 only when `fill` is None elsewhere), `pad` everywhere else"""
    Px, Py, Pz = grid
    M = G.shape[0]
    Ml = M // v // Px * v if kind == "lu" else -(-Kappa // Px) * v
    ncl = solve_local_ref.rhs_local_cols(nrhs, v, Py)
    out = []
    for r in range(Px * Py * Pz):
        pi, pj, pk = r // (Py * Pz), (r // Pz) % Py, r % Pz
        s = np.full((Ml, ncl + ld_extra), pad)
        if pk == 0 or fill:
            for lr in range(Ml):
                gr = ((lr // v) * Px + pi) * v + lr % v
                if kind == "chol" and gr // v >= Kappa:
                    continue
                for lc in range(ncl):
                    gc = ((lc // v) * Py + pj) * v + lc % v
                    if gc < nrhs:
                        s[lr, lc] = G[gr, gc]
        out.append(s)
    return out


def _problem(kind, grid, v):
    """(N, M, Kappa, factor shares, perm, A): a random well-conditioned matrix and its factors in the device's layout,
    with NaN wherever the device must not read the factors"""
    rng = np.random.default_rng(sum(grid) * 7 + v)
    if kind == "lu":
        N = 40
        M = layout.dims(N, v, *grid)["M"]
        A = rng.standard_normal((M, M)) + 4 * np.eye(M)
        P, L, U = scipy.linalg.lu(A)
        perm = np.argmax(P, axis=0).astype(np.int32)                   # (P^T A)[i] = A[perm[i]]
        return N, M, None, layout.scatter(np.tril(L, -1) + U, v, *grid), perm, A
    N = 44
    d = chol_ref.dims(N, v, *grid)
    M, Kappa = d["N"], d["Kappa"]
    S = hp_ref.random_spd(M, 1e2, rng)
    Lf = np.linalg.cholesky(S)
    return N, M, Kappa, chol_solve_ref.scatter(Lf, N, v, *grid, upper=np.nan, pad=np.nan, layers=np.nan), None, S


LU_GRIDS = [(1, 1, 1), (1, 1, 2), (2, 2, 1), (2, 2, 2), (3, 3, 1), (3, 3, 2)]
CHOL_GRIDS = [(2, 1, 1), (4, 2, 1), (2, 2, 2)]
V = 8


def _nrhs_ids(M):
    return [1, V - 1, V, V + 1, M, 2 * M + 5]


def _cases():
    for kind, grids in (("lu", LU_GRIDS), ("chol", CHOL_GRIDS)):
        for g in grids:
            for k in range(6):
                for trans in ((False, True) if kind == "lu" else (False,)):
                    yield pytest.param(kind, g, k, trans, id=f"{kind}-{'x'.join(map(str, g))}-n{k}{'-T' if trans else ''}")


@pytest.mark.parametrize("kind,grid,k,trans", list(_cases()))
def test_schedule_solves_and_respects_the_masks(kind, grid, k, trans):
    N, M, Kappa, F, perm, A = _problem(kind, grid, V)
    nrhs = _nrhs_ids(M)[k]
    if nrhs == 2 * M + 5:
        nc = solve_local_ref.block_cols(M, V)
        assert -(-nrhs // nc) == 3 and nrhs % nc                       # three blocks, the last one narrower
    G = np.random.default_rng(nrhs).standard_normal((M, nrhs))
    B = _shares(kind, G, nrhs, V, grid, Kappa, fill=False, pad=np.nan)  # NaN wherever B must not be read
    X = [np.full_like(b, SENTINEL) for b in B]
    B0 = [b.copy() for b in B]
    solve_local_ref.solve_local(kind, F, perm, B, X, nrhs, N, V, *grid, trans=trans)
    Pz = grid[2]
    for r in range(len(X)):
        assert np.array_equal(X[r], X[r - r % Pz])                     # every layer gets layer 0's bits
        assert np.array_equal(B[r], B0[r], equal_nan=True)             # B is not written
    mask = _shares(kind, np.ones((M, nrhs)), nrhs, V, grid, Kappa, fill=True, pad=0.0)
    for r in range(len(X)):
        assert np.all(X[r][mask[r] == 0.0] == SENTINEL)                # every sentinel survives
        assert np.all(np.isfinite(X[r][mask[r] == 1.0]))               # no NaN leaks in
    Xg = np.zeros((M, nrhs))
    got = _shares(kind, np.arange(M * nrhs, dtype=float).reshape(M, nrhs), nrhs, V, grid, Kappa, fill=True, pad=-1.0)
    for r in range(len(X)):                                            # assemble X from its shares
        sel = got[r] >= 0
        Xg.reshape(-1)[got[r][sel].astype(np.int64)] = X[r][sel]
    Am = A.T if trans else A
    Xd = np.linalg.solve(Am, G)
    assert np.abs(Xg - Xd).max() <= TOL * max(1.0, np.abs(Xd).max())


@pytest.mark.parametrize("kind,grid", [("lu", (2, 2, 2)), ("chol", (4, 2, 1))], ids=["lu-2x2x2", "chol-4x2x1"])
def test_schedule_in_place(kind, grid):
    """X = B: block j is packed before it is scattered, so the shares give the bits of a separate X"""
    N, M, Kappa, F, perm, _ = _problem(kind, grid, V)
    nrhs = 2 * M + 5
    G = np.random.default_rng(3).standard_normal((M, nrhs))
    B = _shares(kind, G, nrhs, V, grid, Kappa, fill=True, pad=np.nan)
    X = [np.full_like(b, SENTINEL) for b in B]
    solve_local_ref.solve_local(kind, F, perm, B, X, nrhs, N, V, *grid)
    solve_local_ref.solve_local(kind, F, perm, B, B, nrhs, N, V, *grid)
    mask = _shares(kind, np.ones((M, nrhs)), nrhs, V, grid, Kappa, fill=True, pad=0.0)
    for r in range(len(B)):
        assert np.array_equal(B[r][mask[r] == 1.0], X[r][mask[r] == 1.0])
        assert np.all(np.isnan(B[r][mask[r] == 0.0]))


def test_pack_and_scatter_of_one_share():
    """the per-share kernels at an off-origin position of a 2 x 3 grid against plain loops"""
    v, Px, Py, pos, M, nrhs = 8, 2, 3, (1, 2), 96, 61
    rng = np.random.default_rng(4)
    for kind, Kappa in (("lu", None), ("chol", 10)):
        Ml = M // v // Px * v
        ncl = solve_local_ref.rhs_local_cols(nrhs, v, Py)
        rows = solve_local_ref.local_rows(kind, Ml, v, Px, pos[0], Kappa)
        B = rng.standard_normal((Ml, ncl + 2))
        for c0, w in [(0, 1), (0, 24), (13, 40), (48, 13)]:
            Bk = solve_local_ref.pack_share(kind, B, M, v, Px, Py, *pos, nrhs, c0, w, Kappa)
            want = np.zeros_like(Bk)
            for lr in range(rows):
                for lc in range(ncl):
                    gc = ((lc // v) * Py + pos[1]) * v + lc % v
                    if c0 <= gc < c0 + w:
                        want[((lr // v) * Px + pos[0]) * v + lr % v, gc - c0] = B[lr, lc]
            assert np.array_equal(Bk, want)
            X = np.full_like(B, SENTINEL)
            solve_local_ref.scatter_share(kind, want, X, v, Px, Py, *pos, nrhs, c0, w, Kappa)
            back = np.where(X == SENTINEL, B, X)
            assert np.array_equal(solve_local_ref.pack_share(kind, back, M, v, Px, Py, *pos, nrhs, c0, w, Kappa), want)
            assert np.count_nonzero(X != SENTINEL) == np.count_nonzero(want)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")
def test_cpp_facades_compile(tmp_path):
    src = tmp_path / "use_solve_local.cpp"
    src.write_text('#include "conflux/lu/conflux_b200.hpp"\n'
                   '#include "conflux/cholesky/conflux_b200_cholesky.hpp"\n'
                   "void f(conflux::lu_params<double>& g, const double* b, double* x) {\n"
                   "  conflux::choleskySolveLocal(3, b, 8, x, 8);\n"
                   "  conflux::LU_solve_local(g, 3, b, 8, x, 8); conflux::LU_solve_local(g, 3, b, 8, x, 8, true); }\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)], check=True)
