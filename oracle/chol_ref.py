"""oracle/chol_ref.py -- TEST INFRASTRUCTURE: CPU oracle of the CONFCHOX path.
  * assemble(): local conflux-layout shares -> the global matrix (same tile map as the LU path, oracle/layout.py);
  * reference factor = numpy.linalg.cholesky (LAPACK dpotrf, lower) of the assembled input, which is exactly what the
    reference's own checker compares against (examples/cholesky_helper.cpp:183-217: LAPACKE_dpotrf(ROW_MAJOR, 'L'));
  * init_matrix(): restatement of CholeskyIO::generateInputMatrixDistributed (CholeskyIO.cpp:100-172) with glibc's rand()
    through ctypes (srand(1)), for checking the library's generator."""
import ctypes

import numpy as np


def dims(N, v, Px, Py, Pz):
    K = -(-N // v)
    return dict(N=K * v, Kappa=K, Ml=-(-K // Px) * v, Nl=-(-K // Py) * v, P=Px * Py * Pz)


def assemble(locals_, N, v, Px, Py, Pz):
    d = dims(N, v, Px, Py, Pz)
    A = np.zeros((d["N"], d["N"]))
    for r, loc in enumerate(locals_):
        if r % Pz or loc is None:
            continue
        pi, pj = r // (Py * Pz), (r // Pz) % Py
        loc = np.asarray(loc).reshape(d["Ml"], d["Nl"])
        for lti in range(d["Ml"] // v):
            for ltj in range(d["Nl"] // v):
                gi, gj = lti * Px + pi, ltj * Py + pj
                if gi < d["Kappa"] and gj < d["Kappa"]:
                    A[gi * v:(gi + 1) * v, gj * v:(gj + 1) * v] = loc[lti * v:(lti + 1) * v, ltj * v:(ltj + 1) * v]
    return A


def lower_sym(A):
    """the symmetric matrix whose lower triangle is the lower triangle of A"""
    L = np.tril(A)
    return L + np.tril(A, -1).T


def init_matrix(N, v):
    """global lower triangle as the reference generates it (every tile = lower(R^T R), strengthened diagonal)"""
    libc = ctypes.CDLL(None)
    libc.srand(1)
    libc.rand.restype = ctypes.c_int
    RAND_MAX = 2147483647
    R = np.array([libc.rand() / RAND_MAX * 2 - 1 for _ in range(v * v)]).reshape(v, v)
    T = np.tril(R.T @ R)
    K = -(-N // v)
    mx = np.abs(T).sum(axis=1).max() * K * 2
    A = np.zeros((K * v, K * v))
    for i in range(K):
        for j in range(i + 1):
            A[i * v:(i + 1) * v, j * v:(j + 1) * v] = T
        A[i * v:(i + 1) * v, i * v:(i + 1) * v][np.diag_indices(v)] = mx
    return A, T, mx


# fixed inputs whose default-path factors are pinned bit for bit by tests/golden/chol_factor_bits.json
# (tests/golden/make_chol_golden.py): the library's own generator, and integer matrices M M^T + N I, exact in any
# summation order, so the input is the same bits on every machine
BITS_CASES = [("gen", 100, 16), ("gen", 256, 32), ("gen", 512, 128), ("gen", 1024, 256), ("gen", 2048, 512),
              ("int", 480, 48), ("int", 800, 100), ("int", 1152, 384), ("int", 2048, 256)]


def bits_case_input(kind, N):
    """None = the library's generator; else the integer SPD matrix of the case (float64, exact)"""
    if kind == "gen":
        return None
    M = np.random.default_rng(N).integers(-8, 9, (N, N)).astype(np.float64)
    return M @ M.T + N * np.eye(N)       # every entry: N products of magnitude <= 64, exact in float64


def factor_digest(L):
    """sha256 of the lower triangle of a factor, as float64 bytes"""
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(np.tril(L), dtype=np.float64).tobytes()).hexdigest()
