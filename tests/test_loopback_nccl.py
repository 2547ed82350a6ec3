"""The NCCL loopback (tests/loopback/nccl_loopback.cpp) against numpy, in its host-only build on threads of this process.
Every multi-rank GPU test that runs on one device through it (test_gpu_grids_one_device.py) is only as good as this
library, so its collectives, splits, grouped messages, schedule check and timeout are checked first, without a GPU."""
import ctypes
import threading
from functools import reduce

import numpy as np
import pytest

from tests import _loopback

SUCCESS, INVALID_ARGUMENT, INVALID_USAGE = 0, 4, 5
INT, UINT64, FLOAT, DOUBLE = 2, 5, 7, 8
SUM, PROD, MAX, MIN = 0, 1, 2, 3
NOCOLOR = -1
NP_TYPE = {INT: np.int32, UINT64: np.uint64, DOUBLE: np.float64}


class UniqueId(ctypes.Structure):
    _fields_ = [("internal", ctypes.c_char * 128)]


@pytest.fixture(scope="module")
def L():
    lib = ctypes.CDLL(_loopback.build(host_only=True))
    vp, sz, i = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.ncclGetUniqueId.argtypes = [ctypes.POINTER(UniqueId)]
    lib.ncclCommInitRank.argtypes = [ctypes.POINTER(vp), i, UniqueId, i]
    lib.ncclCommSplit.argtypes = [vp, i, i, ctypes.POINTER(vp), vp]
    lib.ncclCommCount.argtypes = [vp, ctypes.POINTER(i)]
    lib.ncclCommUserRank.argtypes = [vp, ctypes.POINTER(i)]
    lib.ncclCommDestroy.argtypes = [vp]
    lib.ncclAllReduce.argtypes = [vp, vp, sz, i, i, vp, vp]
    lib.ncclReduce.argtypes = [vp, vp, sz, i, i, i, vp, vp]
    lib.ncclBroadcast.argtypes = [vp, vp, sz, i, i, vp, vp]
    lib.ncclAllGather.argtypes = [vp, vp, sz, i, vp, vp]
    lib.ncclSend.argtypes = [vp, sz, i, i, vp, vp]
    lib.ncclRecv.argtypes = [vp, sz, i, i, vp, vp]
    lib.ncclBcast.argtypes = [vp, sz, i, i, vp, vp]
    return lib


def on_threads(P, fn):
    """fn(r) on P threads; the results in rank order"""
    out, err = [None] * P, [None] * P

    def body(r):
        try:
            out[r] = fn(r)
        except BaseException as e:  # noqa: BLE001
            err[r] = e

    th = [threading.Thread(target=body, args=(r,)) for r in range(P)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=60)
        assert not t.is_alive(), "a rank is still waiting"
    for e in err:
        if e is not None:
            raise e
    return out


def world(L, P):
    uid = UniqueId()
    assert L.ncclGetUniqueId(ctypes.byref(uid)) == SUCCESS
    comms = [ctypes.c_void_p() for _ in range(P)]
    assert on_threads(P, lambda r: L.ncclCommInitRank(ctypes.byref(comms[r]), P, uid, r)) == [SUCCESS] * P
    return [c.value for c in comms]


def close(L, comms):
    for c in comms:
        assert L.ncclCommDestroy(c) == SUCCESS


def ptr(a, off=0):
    return a.ctypes.data + off * a.itemsize


def inputs(dtype, P, n, seed):
    rng = np.random.default_rng(seed)
    if dtype == DOUBLE:
        return [rng.standard_normal(n) for _ in range(P)]
    if dtype == INT:                              # near the ends of the range: a sum wraps around
        return [rng.integers(-2**31, 2**31, n).astype(np.int32) for _ in range(P)]
    return [rng.integers(2**63, 2**64, n, dtype=np.uint64) for _ in range(P)]


def rank_order(xs, op):
    f = {SUM: np.add, MAX: np.maximum, MIN: np.minimum}[op]
    with np.errstate(over="ignore"):
        return reduce(lambda a, b: f(a, b), xs)


# ------------------------------------------------------------------------------------------------------ collectives
@pytest.mark.parametrize("inplace", [False, True], ids=["out-of-place", "in-place"])
@pytest.mark.parametrize("op", [SUM, MAX, MIN], ids=["sum", "max", "min"])
@pytest.mark.parametrize("dtype", [INT, UINT64, DOUBLE], ids=["int", "uint64", "double"])
def test_allreduce_every_type_and_op(L, dtype, op, inplace):
    P, n = 3, 37
    xs = inputs(dtype, P, n, seed=10 * dtype + op)
    want = rank_order(xs, op)
    if op == SUM and dtype != DOUBLE:             # the case solve_local and the candH reduce rely on
        assert (want < reduce(np.maximum, xs)).any(), "the sum did not wrap: the inputs test nothing"
    comms = world(L, P)
    send = [x.copy() for x in xs]
    recv = [send[r] if inplace else np.zeros(n, NP_TYPE[dtype]) for r in range(P)]
    rc = on_threads(P, lambda r: L.ncclAllReduce(ptr(send[r]), ptr(recv[r]), n, dtype, op, comms[r], None))
    close(L, comms)
    assert rc == [SUCCESS] * P
    for r in range(P):
        assert np.array_equal(recv[r].view(np.uint8), want.view(np.uint8)), r      # bit for bit, rank order
        if not inplace:
            assert np.array_equal(send[r], xs[r])


@pytest.mark.parametrize("root", [0, 1, 2])
def test_reduce_reaches_only_its_root(L, root):
    P, n = 3, 16
    xs = inputs(UINT64, P, n, seed=root)
    comms = world(L, P)
    recv = [np.full(n, 7, np.uint64) for _ in range(P)]
    rc = on_threads(P, lambda r: L.ncclReduce(ptr(xs[r]), ptr(recv[r]), n, UINT64, SUM, root, comms[r], None))
    close(L, comms)
    assert rc == [SUCCESS] * P
    for r in range(P):
        assert np.array_equal(recv[r], rank_order(xs, SUM) if r == root else np.full(n, 7, np.uint64)), r


@pytest.mark.parametrize("inplace", [False, True], ids=["out-of-place", "in-place"])
@pytest.mark.parametrize("root", [0, 1, 2, 3])
def test_broadcast_from_every_root(L, root, inplace):
    P, n = 4, 23
    xs = inputs(DOUBLE, P, n, seed=root)
    comms = world(L, P)
    recv = [xs[r] if inplace else np.zeros(n) for r in range(P)]
    rc = on_threads(P, lambda r: L.ncclBroadcast(ptr(xs[r]), ptr(recv[r]), n, DOUBLE, root, comms[r], None))
    close(L, comms)
    assert rc == [SUCCESS] * P
    want = inputs(DOUBLE, P, n, seed=root)[root]
    for r in range(P):
        assert np.array_equal(recv[r], want), r


def test_allgather_in_place(L):
    P, n = 3, 5
    bufs = [np.full(P * n, -1.0) for _ in range(P)]
    for r in range(P):
        bufs[r][r * n:(r + 1) * n] = np.arange(n) + 100 * r
    comms = world(L, P)
    rc = on_threads(P, lambda r: L.ncclAllGather(ptr(bufs[r], r * n), ptr(bufs[r]), n, DOUBLE, comms[r], None))
    close(L, comms)
    assert rc == [SUCCESS] * P
    want = np.concatenate([np.arange(n) + 100 * r for r in range(P)])
    for r in range(P):
        assert np.array_equal(bufs[r], want), r


# ----------------------------------------------------------------------------------------------------------- splits
def test_split_orders_by_key_then_parent_rank_and_drops_nocolor(L):
    colors = [0, 1, 0, NOCOLOR, 1, 0]
    keys = [3, 0, 3, 7, -1, 1]
    P = len(colors)
    comms = world(L, P)
    sub = [ctypes.c_void_p() for _ in range(P)]
    rc = on_threads(P, lambda r: L.ncclCommSplit(comms[r], colors[r], keys[r], ctypes.byref(sub[r]), None))
    assert rc == [SUCCESS] * P
    assert sub[3].value is None                                   # NCCL_SPLIT_NOCOLOR: no communicator
    # colour 0: keys 3, 3, 1 at parent ranks 0, 2, 5 -> 5, 0, 2 (the tie of 0 and 2 by parent rank); colour 1: 4, 1
    want = {5: (0, 3), 0: (1, 3), 2: (2, 3), 4: (0, 2), 1: (1, 2)}
    for r, (rank, size) in want.items():
        got_r, got_s = ctypes.c_int(), ctypes.c_int()
        assert L.ncclCommUserRank(sub[r], ctypes.byref(got_r)) == SUCCESS
        assert L.ncclCommCount(sub[r], ctypes.byref(got_s)) == SUCCESS
        assert (got_r.value, got_s.value) == (rank, size), r
    # the members really share one communicator: an all-gather lists them in their new order
    members = [r for r in range(P) if colors[r] != NOCOLOR]
    bufs = {r: np.zeros(want[r][1], np.int32) for r in members}
    mine = {r: np.array([r], np.int32) for r in members}
    rc = on_threads(len(members), lambda i: L.ncclAllGather(ptr(mine[members[i]]), ptr(bufs[members[i]]), 1, INT,
                                                            sub[members[i]], None))
    assert rc == [SUCCESS] * len(members)
    for r in members:
        assert list(bufs[r]) == ([5, 0, 2] if colors[r] == 0 else [4, 1]), r
    close(L, [sub[r].value for r in members])
    close(L, comms)


# -------------------------------------------------------------------------------------------- grouped send / recv
def _flipbit(x, b):
    return x ^ (1 << b)


def _butterfly_pair(pi, r, Px):                  # lu.cu butterfly_pair
    src = _flipbit(pi, r)
    if src >= Px:
        if r == 0:
            src = pi
        else:
            src = _flipbit(src, r - 1)
            if src >= Px:
                src = Px - 1
    return src


@pytest.mark.parametrize("Px", [2, 3, 4, 5])
def test_tournament_exchange_in_one_group(L, Px):
    """the pattern of lu.cu's tournament round: in one group, a double block and an int block to every rank that pairs
    with me (my own half to a mutual partner, the lower half to a one-sided requester), then both blocks from my
    partner unless I am paired with myself"""
    hv, v = 12, 4
    nr = max(1, (Px - 1).bit_length())
    for r in range(nr):
        comms = world(L, Px)
        mine = [np.arange(2 * hv, dtype=np.float64) + 1000 * p + 100 * r for p in range(Px)]   # both halves
        tags = [np.arange(2 * v, dtype=np.int32) + 1000 * p for p in range(Px)]
        recv = [np.full(hv, np.nan) for _ in range(Px)]
        recv_t = [np.full(v, -1, np.int32) for _ in range(Px)]

        def body(pi):
            src = _butterfly_pair(pi, r, Px)
            self_ = src == pi
            if not any(pp != pi and _butterfly_pair(pp, r, Px) == pi for pp in range(Px)) and self_:
                return SUCCESS
            rcs = [L.ncclGroupStart()]
            for pp in range(Px):
                if pp == pi or _butterfly_pair(pp, r, Px) != pi:
                    continue
                mutual = not self_ and pp == src
                rcs.append(L.ncclSend(ptr(mine[pi], 0 if mutual else hv), hv, DOUBLE, pp, comms[pi], None))
                rcs.append(L.ncclSend(ptr(tags[pi], 0 if mutual else v), v, INT, pp, comms[pi], None))
            if not self_:
                rcs.append(L.ncclRecv(ptr(recv[pi]), hv, DOUBLE, src, comms[pi], None))
                rcs.append(L.ncclRecv(ptr(recv_t[pi]), v, INT, src, comms[pi], None))
            rcs.append(L.ncclGroupEnd())
            return max(rcs)

        assert on_threads(Px, body) == [SUCCESS] * Px
        close(L, comms)
        for pi in range(Px):
            src = _butterfly_pair(pi, r, Px)
            if src == pi:
                continue
            mutual = _butterfly_pair(src, r, Px) == pi
            assert np.array_equal(recv[pi], mine[src][:hv] if mutual else mine[src][hv:]), (r, pi)
            assert np.array_equal(recv_t[pi], tags[src][:v] if mutual else tags[src][v:]), (r, pi)


# ------------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("what", ["count", "datatype", "root"])
def test_schedule_mismatch_is_refused_on_every_rank(L, what, capfd):
    P = 2
    comms = world(L, P)
    bufs = [np.zeros(8) for _ in range(P)]

    def body(r):
        if what == "count":
            return L.ncclAllReduce(ptr(bufs[r]), ptr(bufs[r]), 4 + r, DOUBLE, SUM, comms[r], None)
        if what == "datatype":
            return L.ncclAllReduce(ptr(bufs[r]), ptr(bufs[r]), 4, (DOUBLE, UINT64)[r], SUM, comms[r], None)
        return L.ncclBroadcast(ptr(bufs[r]), ptr(bufs[r]), 4, DOUBLE, r, comms[r], None)

    assert on_threads(P, body) == [INVALID_USAGE] * P
    err = capfd.readouterr().err
    line = next(ln for ln in err.splitlines() if "schedule mismatch" in ln)
    calls = {"count": ("count=4", "count=5"), "datatype": ("ncclDouble", "ncclUint64"),
             "root": ("root=0", "root=1")}[what]
    for c in calls:
        assert c in line, err
    # the communicator is poisoned: the next call fails at once on every rank instead of waiting
    assert on_threads(P, lambda r: L.ncclAllReduce(ptr(bufs[r]), ptr(bufs[r]), 1, DOUBLE, SUM, comms[r], None)) == [
        INVALID_USAGE] * P
    close(L, comms)


def test_message_count_mismatch_is_refused(L, capfd):
    comms = world(L, 2)
    a, b = np.zeros(4), np.zeros(4)
    rc = on_threads(2, lambda r: L.ncclSend(ptr(a), 4, DOUBLE, 1, comms[0], None) if r == 0 else
                    L.ncclRecv(ptr(b), 3, DOUBLE, 0, comms[1], None))
    close(L, comms)
    assert rc == [SUCCESS, INVALID_USAGE]
    assert "sent count=4 ncclDouble, received as count=3 ncclDouble" in capfd.readouterr().err


def test_a_rank_that_never_arrives_times_out(L, capfd, monkeypatch):
    monkeypatch.setenv("LOOPBACK_TIMEOUT_S", "0.5")
    comms = world(L, 3)
    buf = np.zeros(2)
    # ranks 0 and 1 reach an all-reduce that rank 2 never issues
    rc = on_threads(2, lambda r: L.ncclAllReduce(ptr(buf), ptr(buf), 2, DOUBLE, SUM, comms[r], None))
    close(L, comms)
    assert rc == [INVALID_USAGE] * 2
    err = capfd.readouterr().err
    assert "timeout after" in err
    assert "rank 0 waits in call #0 ncclAllReduce(count=2" in err
    assert "rank 2 has not arrived" in err


def test_unsupported_types_ops_and_entry_points_are_refused_by_name(L, capfd):
    comms = world(L, 1)
    x = np.zeros(2, np.float32)
    assert L.ncclAllReduce(ptr(x), ptr(x), 2, FLOAT, SUM, comms[0], None) == INVALID_ARGUMENT
    assert L.ncclAllReduce(ptr(x), ptr(x), 2, DOUBLE, PROD, comms[0], None) == INVALID_ARGUMENT
    assert L.ncclBcast(ptr(x), 2, DOUBLE, 0, comms[0], None) == INVALID_USAGE
    close(L, comms)
    err = capfd.readouterr().err
    assert "datatype 7 is not one of" in err and "reduction op 1 is not one of" in err
    assert "ncclBcast is not implemented by the loopback" in err


def test_calls_are_counted(L):
    before = _loopback.stats(L)
    comms = world(L, 2)
    x = [np.ones(3) for _ in range(2)]
    on_threads(2, lambda r: L.ncclAllReduce(ptr(x[r]), ptr(x[r]), 3, DOUBLE, SUM, comms[r], None))
    close(L, comms)
    after = _loopback.stats(L)
    assert after["ncclAllReduce"] - before["ncclAllReduce"] == 2
    assert after["ncclCommInitRank"] - before["ncclCommInitRank"] == 2
