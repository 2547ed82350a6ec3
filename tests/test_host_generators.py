"""The host-side input generators (no GPU): the same shares whether the ranks of a grid call them one after another or
as threads of one process at once, which is how tests/_harness.py and the loopback run a grid."""
import ctypes
import threading

import numpy as np

import conflux_b200 as cb
from oracle import chol_ref


def _chol_share(N, v, grid, rank):
    d = (ctypes.c_int * 6)()
    cb.check(cb.lib().cflx_chol_dims(N, v, *grid, d), "chol_dims")
    out = np.full((d[2], d[3]), np.nan)
    cb.check(cb.lib().cflx_chol_init_matrix_host(N, v, *grid, rank, out.ctypes.data), "chol_init_matrix_host")
    return out


def test_chol_generator_is_the_references():
    N, v = 200, 40
    A, _, _ = chol_ref.init_matrix(N, v)
    got = _chol_share(N, v, (1, 1, 1), 0)
    assert np.allclose(np.tril(got), A, rtol=1e-15, atol=1e-15)     # dsyrk summation order may differ in the last bit


def test_chol_generator_gives_every_thread_the_same_shares():
    """eight threads each generate all shares of a 2 x 2 x 2 grid three times: every copy has the bits of the one-thread
    run (a generator on the process-wide rand() state deals the threads interleaved draws)"""
    N, v, grid = 512, 64, (2, 2, 2)
    P = grid[0] * grid[1] * grid[2]
    want = [_chol_share(N, v, grid, r) for r in range(P)]
    got = [[] for _ in range(8)]
    go = threading.Barrier(8)

    def body(t):
        go.wait()
        for _ in range(3):
            got[t] += [_chol_share(N, v, grid, r) for r in range(P)]

    th = [threading.Thread(target=body, args=(t,)) for t in range(8)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    for t in range(8):
        assert len(got[t]) == 3 * P
        for i, share in enumerate(got[t]):
            assert np.array_equal(share, want[i % P]), (t, i % P)
