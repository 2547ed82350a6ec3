"""CPU: the restatement oracle against what the reference itself computed (tests/golden/ref_cases.npz, written by
tests/golden/make_golden.py from oracle/_ref/libref_lu.so): the generator is bit-identical to lu_params::InitMatrix, the
pivot sequence is identical, the factors agree at sampled entries, and the oracle's own factors meet the residual bar."""
import hashlib
import os

import numpy as np
import pytest

from oracle import layout, restate

REF_CASES = [(48, 4, 1, 1, 1), (128, 16, 2, 2, 1), (128, 8, 2, 2, 2), (96, 16, 1, 1, 2), (72, 4, 3, 3, 2), (256, 32, 4, 4, 1)]
REF_SAMPLES = 1024


def ref_sample_index(n):
    """the sampled flat indices of the concatenated local factors (shared with tests/golden/make_golden.py)"""
    return np.sort(np.random.default_rng(11).choice(n, size=min(n, REF_SAMPLES), replace=False))


@pytest.fixture(scope="module")
def G(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_cases.npz"))


@pytest.mark.parametrize("case", REF_CASES)
def test_matches_live_reference(case, G):
    i = REF_CASES.index(case)
    assert tuple(int(x) for x in G["cases"][i]) == case
    N, v, Px, Py, Pz = case
    A0 = restate.init_matrix(N, v, Px, Py, Pz)
    for a, h in zip(A0, G[f"c{i}_A_sha256"]):
        assert hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest() == h.tobytes()   # generator is bit-identical
    o = restate.lu(A0, N, v, Px, Py, Pz)
    assert np.array_equal(o["perm"], G[f"c{i}_perm"])
    C = np.concatenate([x.reshape(-1) for x in o["C"]])
    assert np.abs(C[ref_sample_index(C.size)] - G[f"c{i}_C_sample"]).max() <= 1e-10 * 6.0
    A = layout.assemble(A0, N, v, Px, Py, Pz)
    assert layout.residual(A, layout.assemble(o["C"], N, v, Px, Py, Pz), o["perm"]) <= 1e-12
