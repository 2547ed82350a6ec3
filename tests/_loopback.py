"""The NCCL loopback for tests: builds tests/loopback/nccl_loopback.cpp, runs a P-rank grid as P threads on device 0,
and, loaded as a pytest plugin (`-p tests._loopback`, in a process started with LD_PRELOAD=<library>), rebinds
tests._harness.run_ranks and n_gpus before any test module imports them.  Every multi-rank test then runs on one GPU
against its own oracle (DESIGN.md section 6 says what such a run proves and what it does not)."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "loopback", "nccl_loopback.cpp")
BUILD = os.path.join(HERE, "loopback", "build")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
# n_gpus() under the loopback.  Ranks are threads, so no grid is out of reach; a test that drops a grid it has no
# devices for (the golden LU fixtures `continue` past them) must never drop one here.  64 is above every grid the suite
# asks for (the largest is the 3 x 3 x 1 golden LU case).
GRID_RANKS = 64
STATS_ENV = "LOOPBACK_STATS_OUT"


def lib_path(host_only=False):
    return os.path.join(BUILD, "libnccl_loopback_host.so" if host_only else "libnccl_loopback.so")


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def build(host_only=False):
    """compiles the library (g++, host code only: the device build reaches libcuda through dlopen) when it is older
    than its source or this file; returns its path"""
    out = lib_path(host_only)
    if not _stale(out, [SRC, os.path.abspath(__file__)]):
        return out
    os.makedirs(BUILD, exist_ok=True)
    fd, tmp = tempfile.mkstemp(suffix=".so", dir=BUILD)          # rename into place: a concurrent build never sees half
    os.close(fd)
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-shared", "-fPIC", f"-I{CUDA_HOME}/include"]
    cmd += ["-DLOOPBACK_HOST_ONLY"] if host_only else []
    cmd += [SRC, "-o", tmp, "-lpthread"] + ([] if host_only else ["-ldl"])
    try:
        subprocess.run(cmd, check=True, capture_output=True, text=True)
    except subprocess.CalledProcessError as e:
        os.unlink(tmp)
        raise RuntimeError(f"building the NCCL loopback failed:\n{e.stderr}") from None
    os.replace(tmp, out)
    return out


def stats(lib=None):
    """{entry point: calls so far} of the loopback loaded in this process (or of `lib`, a ctypes handle)"""
    L = lib if lib is not None else ctypes.CDLL(None)
    L.loopback_stat_name.restype = ctypes.c_char_p
    buf = (ctypes.c_ulonglong * 32)()
    n = L.loopback_stats(buf, 32)
    return {L.loopback_stat_name(k).decode(): int(buf[k]) for k in range(n)}


def n_gpus():
    return GRID_RANKS


def run_ranks(P, fn):
    """tests._harness.run_ranks with every rank on device 0: fn(comm) on P threads; the results in rank order; re-raises
    the first exception"""
    import conflux_b200 as cb
    uid = cb.Comm.unique_id() if P > 1 else None
    out, err = [None] * P, [None] * P

    def body(r):
        try:
            comm = cb.Comm(P, r, uid, 0)
            try:
                out[r] = fn(comm)
            finally:
                comm.close()
        except BaseException as e:  # noqa: BLE001
            err[r] = e
            import traceback
            sys.stderr.write(f"[rank {r}] failed: {e!r}\n")
            traceback.print_exc()
            sys.stderr.flush()

    th = [threading.Thread(target=body, args=(r,)) for r in range(P)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for e in err:
        if e is not None:
            raise e
    return out


def in_effect():
    """True when the NCCL entry points this process resolves are the loopback's (LD_PRELOAD put it first)"""
    glob = ctypes.CDLL(None)
    try:
        glob.loopback_stats
    except AttributeError:
        return False
    mine = ctypes.CDLL(lib_path())
    addr = lambda L: ctypes.cast(L.ncclGetUniqueId, ctypes.c_void_p).value  # noqa: E731
    return addr(glob) == addr(mine)


def install():
    """rebinds tests._harness.run_ranks and n_gpus to their one-device versions (before the test modules import them)"""
    from tests import _harness
    _harness.run_ranks = run_ranks
    _harness.n_gpus = n_gpus


def install_if_preloaded():
    """install() in a child interpreter of a loopback run (LD_PRELOAD is inherited, the plugin is not); else nothing"""
    if in_effect():
        install()


# ------------------------------------------------------------------------------------------------------ pytest plugin
def pytest_configure(config):
    if not in_effect():
        import pytest
        raise pytest.UsageError(f"-p tests._loopback needs LD_PRELOAD={lib_path()} (the NCCL loopback is not in effect)")
    install()


def pytest_unconfigure(config):
    path = os.environ.get(STATS_ENV)
    if path:
        with open(path, "w") as f:
            json.dump(stats(), f)
