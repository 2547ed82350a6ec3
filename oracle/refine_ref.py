"""oracle/refine_ref.py -- TEST INFRASTRUCTURE: numpy restatement of cflx_lu_refine / cflx_chol_refine (conflux_b200/
csrc/refine.cu).

  * gerfs / porfs: LAPACK's dgerfs / dporfs, column by column, with the solves passed in as callbacks and the forward-
    error estimator cond_ref.dlacn2 (kase 1 applies diag(w) inv(op A)^T, kase 2 inv(op A) diag(w));
  * partials_lu / partials_chol: the residual products op(A) X and |op(A)| |X| as the grid forms them: every layer-0 rank
    multiplies its own share, masked as the device masks it, and the partials are added in the device's order (for
    global row g of tile T: the NN partials of the ranks (T % Px, pj), pj ascending, then the TN partials of the ranks
    (pi, T % Py), pi ascending);
  * perm_to_ipiv: a permutation vector (row perm[i] of A is row i of P A) as LAPACK's 1-based swap sequence ipiv;
  * backward_error: the componentwise backward error max_i |b - op(A) x|_i / (|op(A)| |x| + |b|)_i in long double."""
import numpy as np

from . import chol_ref, cond_ref, layout

ITMAX = 5
EPS = 2.0 ** -53
SAFMIN = 2.0 ** -1022


def _rfs(A, B, X, solve, solve_t, op):
    """the loop of dgerfs / dporfs: A the matrix op applies, solve(x) = inv(op A) x, solve_t(x) = inv(op A)^T x"""
    n, nrhs = B.shape
    X = np.array(X, dtype=np.float64)
    nz = n + 1
    safe1 = nz * SAFMIN
    safe2 = safe1 / EPS
    ferr, berr = np.zeros(nrhs), np.zeros(nrhs)
    for j in range(nrhs):
        b = B[:, j]
        count, lstres = 1, 3.0
        while True:
            x = X[:, j]
            r = b - op(A) @ x
            s = np.abs(op(A)) @ np.abs(x) + np.abs(b)
            ratio = np.where(s > safe2, np.abs(r) / np.where(s > safe2, s, 1.0), (np.abs(r) + safe1) / (s + safe1))
            berr[j] = ratio.max()
            if berr[j] > EPS and 2.0 * berr[j] <= lstres and count <= ITMAX:
                X[:, j] = x + solve(r)
                lstres = berr[j]
                count += 1
                continue
            break
        w = np.where(s > safe2, np.abs(r) + nz * EPS * s, np.abs(r) + nz * EPS * s + safe1)

        def apply(kase, v):
            return w * solve_t(v) if kase == 1 else solve(w * v)
        est = cond_ref.dlacn2(n, apply)
        xmax = np.abs(X[:, j]).max()
        ferr[j] = est / xmax if xmax != 0 else est
    return X, ferr, berr


def gerfs(A, B, X, solve, solve_t, trans=False):
    """dgerfs: solve(x) = inv(op A) x and solve_t(x) = inv(op A)^T x with op(A) = A^T when trans.  Returns (X, ferr, berr)."""
    return _rfs(np.asarray(A), np.asarray(B), X, solve, solve_t, (lambda M: M.T) if trans else (lambda M: M))


def porfs(A, B, X, solve):
    """dporfs: A symmetric, solve(x) = inv(A) x.  Returns (X, ferr, berr)."""
    return _rfs(np.asarray(A), np.asarray(B), X, solve, solve, lambda M: M)


def lu_solvers(LU, perm, trans=False):
    """solve / solve_t of gerfs from packed L\\U of P A = L U (row perm[i] of A is row i of P A)"""
    from scipy.linalg import solve_triangular
    perm = np.asarray(perm)

    def plain(x):   # inv(A) x = inv(U) inv(L) P x
        return solve_triangular(LU, solve_triangular(LU, x[perm], lower=True, unit_diagonal=True))

    def transp(x):  # inv(A)^T x = P^T inv(L)^T inv(U)^T x
        y = solve_triangular(LU, solve_triangular(LU, x, trans="T"), trans="T", lower=True, unit_diagonal=True)
        out = np.empty_like(y)
        out[perm] = y
        return out
    return (transp, plain) if trans else (plain, transp)


def chol_solver(L):
    from scipy.linalg import solve_triangular
    return lambda x: solve_triangular(L, solve_triangular(L, x, lower=True), lower=True, trans="T")


def perm_to_ipiv(perm):
    """LAPACK's ipiv (1-based: row i swapped with row ipiv[i] - 1, i ascending) that takes A to A[perm]"""
    perm = np.asarray(perm)
    n = len(perm)
    cur = np.arange(n)          # cur[p] = original row now at position p
    pos = np.arange(n)          # pos[r] = position of original row r
    ipiv = np.empty(n, dtype=np.int32)
    for i in range(n):
        j = pos[perm[i]]
        ipiv[i] = j + 1
        ri, rj = cur[i], cur[j]
        cur[i], cur[j] = rj, ri
        pos[ri], pos[rj] = j, i
    return ipiv


def lapack_gesvx(A, LU, ipiv, B, trans=False):
    """scipy's dgesvx(fact='F', equed='N') on the given factors: (X, ferr, berr, info)"""
    from scipy.linalg import lapack
    out = lapack.dgesvx(A, B, fact="F", trans="T" if trans else "N", af=LU, ipiv=ipiv, equed="N")
    return out[7], out[9], out[10], out[11]


def lapack_posvx(A, L, B):
    """scipy's dposvx(fact='F', equed='N', lower=1) on the given factor: (X, ferr, berr, info)"""
    from scipy.linalg import lapack
    out = lapack.dposvx(A, B, fact="F", af=L, equed="N", lower=1)
    return out[5], out[7], out[8], out[9]


def backward_error(A, B, X, trans=False):
    """max_i |b - op(A) x|_i / (|op(A)| |x| + |b|)_i per column, every product and sum in long double (no slicing: the
    entries of X may span more exponents than a sliced product keeps)"""
    LD = np.longdouble
    Ao = (np.asarray(A).T if trans else np.asarray(A)).astype(LD)
    X = np.asarray(X).reshape(len(Ao), -1).astype(LD)
    B = np.asarray(B).reshape(len(Ao), -1).astype(LD)
    R = B - Ao @ X
    S = np.abs(Ao) @ np.abs(X) + np.abs(B)
    return np.asarray(np.max(np.abs(R) / np.where(S > 0, S, 1), axis=0), dtype=np.float64)


# ------------------------------------------------------------------------------------------------ the grid product
def _gidx(l, P, p, v):
    return ((l // v) * P + p) * v + l % v


def _assemble(nn, tn, n, v, Px, Py, Ml):
    """op(A) x and |op(A)| |x| from the per-rank partials nn[(pi, pj)] / tn[(pi, pj)] ((P, Q) pairs), device order"""
    nrhs = next(iter((nn or tn).values()))[0].shape[1]
    P, Q = np.zeros((n, nrhs)), np.zeros((n, nrhs))
    for g in range(n):
        T, e = divmod(g, v)
        if nn:
            for pj in range(Py):
                p, q = nn[(T % Px, pj)]
                P[g] += p[(T // Px) * v + e]
                Q[g] += q[(T // Px) * v + e]
        if tn:
            for pi in range(Px):
                p, q = tn[(pi, T % Py)]
                P[g] += p[(T // Py) * v + e]
                Q[g] += q[(T // Py) * v + e]
    return P, Q


def partials_lu(A_locals, X, N, v, Px=1, Py=1, Pz=1, trans=False):
    """(A X, |A| |X|) -- or (A^T X, |A^T| |X|) -- of the padded LU input from the layer-0 shares, as the grid forms it"""
    d = layout.dims(N, v, Px, Py, Pz)
    M, Ml, Nl = d["M"], d["Ml"], d["Nl"]
    X = np.asarray(X).reshape(M, -1)
    parts = {}
    for pi in range(Px):
        for pj in range(Py):
            A = np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(Ml, Nl)
            if trans:
                Xr = X[[_gidx(l, Px, pi, v) for l in range(Ml)]]
                parts[(pi, pj)] = (A.T @ Xr, np.abs(A).T @ np.abs(Xr))
            else:
                Xc = X[[_gidx(l, Py, pj, v) for l in range(Nl)]]
                parts[(pi, pj)] = (A @ Xc, np.abs(A) @ np.abs(Xc))
    return _assemble(None if trans else parts, parts if trans else None, M, v, Px, Py, Ml)


def sym_masks(Ml, Nl, v, Kappa, Px, Py, pi, pj):
    """the entries of a share the symmetric product reads: (NN: global row >= column, TN: row > column), real tiles only"""
    gr = np.array([_gidx(l, Px, pi, v) for l in range(Ml)])[:, None]
    gc = np.array([_gidx(l, Py, pj, v) for l in range(Nl)])[None, :]
    real = (gr // v < Kappa) & (gc // v < Kappa)
    return real & (gr >= gc), real & (gr > gc)


def partials_chol(A_locals, X, N, v, Px=1, Py=1, Pz=1):
    """(A X, |A| |X|) of the symmetric matrix whose lower triangle the layer-0 shares hold, as the grid forms it; reads
    nothing above the diagonal, beyond Kappa or on the layers pk != 0 (NaN there does not reach the result)"""
    d = chol_ref.dims(N, v, Px, Py, Pz)
    n, K, Ml, Nl = d["N"], d["Kappa"], d["Ml"], d["Nl"]
    X = np.asarray(X).reshape(n, -1)
    nn, tn = {}, {}
    for pi in range(Px):
        for pj in range(Py):
            A = np.asarray(A_locals[layout.rank_of(pi, pj, 0, Px, Py, Pz)]).reshape(Ml, Nl)
            mnn, mtn = sym_masks(Ml, Nl, v, K, Px, Py, pi, pj)
            rows = [min(_gidx(l, Px, pi, v), n - 1) for l in range(Ml)]
            cols = [min(_gidx(l, Py, pj, v), n - 1) for l in range(Nl)]
            Xc, Xr = X[cols], X[rows]
            An, At = np.where(mnn, A, 0.0), np.where(mtn, A, 0.0)
            nn[(pi, pj)] = (An @ Xc, np.abs(An) @ np.abs(Xc))
            tn[(pi, pj)] = (At.T @ Xr, np.abs(At).T @ np.abs(Xr))
    return _assemble(nn, tn, n, v, Px, Py, Ml)
