"""CPU: the communication schedule of cflx_lu_solve (oracle/solve_ref.py: per-rank partial right-hand sides, the reduce /
broadcast / update sequence per tile, nb-block inverse sweeps, final all-reduce) solves A X = B with the factors the
restatement oracle produces, on every grid shape the solve runs on."""
import numpy as np
import pytest

from oracle import layout, restate, solve_ref

CASES = [(64, 8, 1, 1, 1), (128, 16, 1, 1, 2), (64, 8, 2, 2, 1), (128, 8, 2, 2, 2), (96, 8, 3, 3, 1),
         (256, 64, 1, 1, 1), (100, 16, 1, 1, 1)]


@pytest.fixture(scope="module", params=CASES, ids=lambda c: "N%d_v%d_%dx%dx%d" % c)
def factored(request):
    N, v, Px, Py, Pz = request.param
    A_locals = restate.init_matrix(N, v, Px, Py, Pz)
    o = restate.lu(A_locals, N, v, Px, Py, Pz)
    A = layout.assemble(A_locals, N, v, Px, Py, Pz)
    LU = layout.assemble(o["C"], N, v, Px, Py, Pz)
    return dict(case=request.param, C=o["C"], perm=o["perm"], A=A, LU=LU)


@pytest.mark.parametrize("nrhs", [1, 3, 17])
def test_schedule_solves_the_system(factored, nrhs):
    N, v, Px, Py, Pz = factored["case"]
    M = factored["A"].shape[0]
    B = np.random.default_rng(nrhs + N).standard_normal((M, nrhs))
    X = solve_ref.solve(factored["C"], factored["perm"], B, N, v, Px, Py, Pz)
    Xh = solve_ref.host_solve(factored["LU"], factored["perm"], B)
    assert X.shape == B.shape
    assert np.abs(X - Xh).max() <= 1e-10 * np.abs(Xh).max()
    assert solve_ref.backward_error(factored["A"], X, B) <= 1e-13


def test_padded_case_solves_the_padded_system():
    N, v = 100, 16
    d = layout.dims(N, v, 1, 1, 1)
    assert d["M"] == 112
    A_locals = restate.init_matrix(N, v)
    o = restate.lu(A_locals, N, v)
    b = np.random.default_rng(5).standard_normal(d["M"])
    x = solve_ref.solve(o["C"], o["perm"], b, N, v)
    assert x.shape == (d["M"],)
    assert solve_ref.backward_error(A_locals[0], x[:, None], b[:, None]) <= 1e-13
