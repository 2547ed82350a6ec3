"""GPU: the slot exchange of the row-owner pivot search (panel_getrf_kernel) across grid sizes.  CFLX_PANEL_CTAS sets the
SM budget of cb.dbg.panel as it does for the factorisation's look-ahead, so one panel runs on 8 to 132 CTAs: on grids of
<= 32 CTAs the gather warp runs the exchange, on larger grids every thread polls.  Pivots, L00\\U00 and the multipliers
must agree bit for bit between all of them, with the column-owner kernel, and across launches that share a workspace."""
import numpy as np
import pytest

import conflux_b200 as cb
from oracle import restate

pytestmark = pytest.mark.gpu
CAPS = ("8", "16", "32", "132")


def _factor(P, monkeypatch, cap, reps=1, stack="0"):
    monkeypatch.setenv("CFLX_PANEL_CTAS", cap)
    monkeypatch.setenv("CFLX_STACK_KERNEL", stack)
    perm, A00, LU, _ = cb.dbg.panel(P, reps=reps)
    return perm, A00, LU


def _same_bits(a, b, n, v):
    (perm_a, A_a, LU_a), (perm_b, A_b, LU_b) = a, b
    assert np.array_equal(perm_a, perm_b)
    rest = np.setdiff1d(np.arange(n), perm_a[:min(n, v)])
    assert np.array_equal(LU_a[rest], LU_b[rest])          # the multipliers of every row that was never a pivot
    if n >= v:
        assert np.array_equal(A_a, A_b)                    # L00\U00 of the winners, every bit
        low = np.tril_indices(v, -1)
        assert np.array_equal(LU_a[perm_a][low], LU_b[perm_b][low])


def _against_oracle(P, perm):
    n, v = P.shape
    cand = np.concatenate([np.zeros((n, 1)), P], axis=1)
    perm_ref, _ = restate.getrf_perm(cand, n, v)
    assert np.array_equal(perm, perm_ref[:v])


@pytest.mark.parametrize("n,v", [(16128, 256), (7936, 256), (3840, 256), (2048, 64), (1056, 256), (4099, 32), (2500, 128),
                                 (40, 64)])
def test_grid_size_does_not_change_a_bit(n, v, monkeypatch):
    rng = np.random.default_rng(n * 3 + v)
    P = rng.uniform(-1, 1, (n, v))
    ref = _factor(P, monkeypatch, "32")
    for cap in CAPS:
        if cap != "32":
            _same_bits(ref, _factor(P, monkeypatch, cap), n, v)
    if n <= 4099:
        _against_oracle(P, ref[0])


def test_integer_ties_across_ctas(monkeypatch):
    """Equal maxima in different CTAs: the LAPACK position decides through the exchange, on every grid size."""
    rng = np.random.default_rng(3)
    for (n, v) in [(5000, 64), (2100, 32), (9000, 16)]:
        P = rng.integers(0, 4, size=(n, v)).astype(np.float64)
        ref = _factor(P, monkeypatch, "32")
        _against_oracle(P, ref[0])
        for cap in CAPS:
            _same_bits(ref, _factor(P, monkeypatch, cap), n, v)


@pytest.mark.parametrize("cap", ["8", "32", "132"])
def test_row_owner_grid_matches_the_column_owner_kernel(cap, monkeypatch):
    rng = np.random.default_rng(11)
    for P in (rng.standard_normal((1024, 256)), rng.integers(-3, 4, size=(1024, 128)).astype(np.float64)):
        n, v = P.shape
        _same_bits(_factor(P, monkeypatch, cap, stack="1"), _factor(P, monkeypatch, cap, stack="0"), n, v)


@pytest.mark.parametrize("n,v", [(3000, 64), (3000, 33), (7680, 512)])
def test_epochs_carry_over_between_launches_on_one_workspace(n, v, monkeypatch):
    """reps launches reuse the slots of one workspace (odd v included: the epoch base stays even); v = 512 is the panel
    width of the multi-GPU configurations."""
    rng = np.random.default_rng(n + v)
    P = rng.uniform(-1, 1, (n, v))
    first = _factor(P, monkeypatch, "32", reps=1)
    _same_bits(first, _factor(P, monkeypatch, "32", reps=4), n, v)
    _same_bits(first, _factor(P, monkeypatch, "132", reps=3), n, v)
    if v <= 64:
        _against_oracle(P, first[0])
