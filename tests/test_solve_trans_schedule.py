"""CPU: the schedule of cflx_lu_solve_trans (oracle/solve_trans_ref.py: column-partial right-hand sides, the reduce /
broadcast / update sequence per tile of both sweeps, nb-block sweeps read transposed, the final all-reduce and P^T) solves
A^T X = B with the factors the restatement oracle produces, on every grid shape the LU solve runs on."""
import numpy as np
import pytest

from oracle import layout, restate, solve_trans_ref
from tests.test_solve_schedule import CASES


@pytest.fixture(scope="module", params=CASES, ids=lambda c: "N%d_v%d_%dx%dx%d" % c)
def factored(request):
    N, v, Px, Py, Pz = request.param
    A_locals = restate.init_matrix(N, v, Px, Py, Pz)
    o = restate.lu(A_locals, N, v, Px, Py, Pz)
    A = layout.assemble(A_locals, N, v, Px, Py, Pz)
    LU = layout.assemble(o["C"], N, v, Px, Py, Pz)
    return dict(case=request.param, C=o["C"], perm=o["perm"], A=A, LU=LU)


@pytest.mark.parametrize("nrhs", [1, 3, 17])
def test_transposed_schedule_solves_the_system(factored, nrhs):
    N, v, Px, Py, Pz = factored["case"]
    M = factored["A"].shape[0]
    B = np.random.default_rng(nrhs + 7 * N).standard_normal((M, nrhs))
    log = {}
    X = solve_trans_ref.solve(factored["C"], factored["perm"], B, N, v, Px, Py, Pz, log=log)
    Xh = solve_trans_ref.host_solve(factored["LU"], factored["perm"], B)
    assert X.shape == B.shape
    assert np.abs(X - Xh).max() <= 1e-10 * np.abs(Xh).max()
    assert solve_trans_ref.backward_error(factored["A"].T, X, B) <= 1e-13
    # every member of a communicator issues the same collectives in the same order
    per_comm = {}
    for r, calls in log.items():
        for c in calls:
            per_comm.setdefault(c[0], {}).setdefault(r, []).append(c)
    for comm, by_rank in per_comm.items():
        seqs = list(by_rank.values())
        assert all(s == seqs[0] for s in seqs), comm
    if Px * Py * Pz > 1:
        assert ("world",) in per_comm and len(per_comm[("world",)]) == Px * Py * Pz


def test_pa_mode_solves_with_p_a(factored):
    """pa=True (the condition estimate's products) solves (P A)^T X = B: no final P^T"""
    N, v, Px, Py, Pz = factored["case"]
    M = factored["A"].shape[0]
    b = np.random.default_rng(N).standard_normal(M)
    x = solve_trans_ref.solve(factored["C"], factored["perm"], b, N, v, Px, Py, Pz, pa=True)
    PA = factored["A"][np.asarray(factored["perm"])]
    assert x.shape == (M,)
    assert solve_trans_ref.backward_error(PA.T, x, b) <= 1e-13
