"""CPU: the block rule of the distributed refinement and expert drivers (oracle/refine_local_ref.py).  The blocks cover
[0, nrhs) in whole tiles; the width and the workspace bound are the ones include/conflux_b200.h and
conflux_b200/csrc/lu_state.h state, and the library reports the same width; the bound does not grow with nrhs; info
merges to the first flagged global column; the rule applied to a dense core gives the core's result on every column;
and the C++ facades compile."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import conflux_b200 as cb
from oracle import refine_local_ref as rl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _read(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


@pytest.mark.parametrize("v", [1, 4, 16, 48, 64, 100, 128, 256, 300, 512, 1024])
@pytest.mark.parametrize("nrhs", [1, 7, 63, 64, 65, 255, 256, 257, 1094, 5000])
def test_blocks_cover_columns_in_whole_tiles(v, nrhs):
    bl = rl.blocks(nrhs, v)
    nc = rl.block_cols(v)
    assert nc % v == 0 and nc >= v
    assert abs(nc - rl.REFINE_NC) <= v // 2 or nc == v               # the whole number of tiles nearest 256 columns
    assert bl[0][0] == 0 and sum(w for _, w in bl) == nrhs
    for (c0, w), (c1, _) in zip(bl, bl[1:]):
        assert c1 == c0 + w and w == nc                               # contiguous, every block but the last full
    assert 0 < bl[-1][1] <= nc


def test_library_width_matches_restatement():
    for v in (1, 3, 4, 16, 48, 64, 100, 128, 170, 256, 300, 512, 1024, 4096):
        assert cb.refine_block_cols(v) == rl.block_cols(v)
    assert rl.block_cols(64) == 256 and rl.block_cols(256) == 256 and rl.block_cols(512) == 512
    assert len(rl.blocks(1024 + 70, 64)) == 5                         # the GPU tests' M + 70 at v = 64: several blocks
    with pytest.raises(cb.ConfluxError):
        cb.refine_block_cols(0)


def test_width_and_workspace_are_the_ones_documented():
    assert re.search(r"#define CFLX_REFINE_NC %d\b" % rl.REFINE_NC, _read("conflux_b200", "csrc", "lu_state.h"))
    hdr = " ".join(_read("include", "conflux_b200.h").split())
    assert "CFLX_REFINE_NC = %d columns" % rl.REFINE_NC in hdr
    assert "ldn (15 M + 2 v + (2 P + 5)(Ml + Nl)) + 2 M doubles" in hdr
    design = " ".join(_read("DESIGN.md").split())
    assert "ldn (15 M + 2 v + (2 P + 5)(Ml + Nl)) + 2 M" in design
    assert rl.workspace_doubles(1024, 64, 1024, 1024, 1, 256) == 256 * (15 * 1024 + 128 + 7 * 2048) + 2 * 1024


def test_workspace_is_bounded_independent_of_nrhs():
    # the 8-GPU configuration: M = 65536 on 2 x 2 x 2, v = 512
    M, v, P = 65536, 512, 8
    Ml = Nl = M // 2
    peak = max(rl.workspace_doubles(M, v, Ml, Nl, P, w) for _, w in rl.blocks(M, v))
    assert peak == rl.workspace_doubles(M, v, Ml, Nl, P, rl.block_cols(v))
    assert peak * 8 < 10 * 2 ** 30                                    # under 10 GiB, against 32 GiB for B alone
    assert rl.workspace_doubles(M, v, Ml, Nl, P, 1) < peak            # one column needs less, never more


def test_info_merges_to_first_global_column():
    M = 1024
    bl = rl.blocks(M + 70, 64)
    assert rl.merge_info([(b, 0) for b in bl], M) == 0
    ks = [0, 0, M + 3, M + 1, 0]                                      # columns 3 of block 2 and 1 of block 3 flagged
    assert rl.merge_info(list(zip(bl, ks)), M) == M + 2 * 256 + 3
    assert rl.merge_info(list(zip(bl, [0, 0, 0, 0, M + 70])), M) == M + 4 * 256 + 70
    assert rl.merge_info(list(zip(bl, [M + 1, 0, M + 5, 0, 0])), M) == M + 1


def test_rule_with_a_dense_core_gives_the_core_on_every_column():
    rng = np.random.default_rng(0)
    M, v, nrhs = 96, 16, 230
    A = rng.standard_normal((M, M)) + M * np.eye(M)
    B = rng.standard_normal((M, nrhs))
    X0 = np.linalg.solve(A, B)

    def core(c0, Bk, Xk):
        Xr = Xk + np.linalg.solve(A, Bk - A @ Xk)                     # one correction, column by column independent
        berr = np.abs(Bk - A @ Xr).max(axis=0)
        flagged = np.flatnonzero(np.arange(c0, c0 + Bk.shape[1]) == 200)
        return Xr, dict(berr=berr, ferr=None), M + 1 + flagged[0] if flagged.size else 0

    X, out, info = rl.run(core, B, X0, nrhs, v)
    assert len(rl.blocks(nrhs, v)) == 1 or X.shape == (M, nrhs)
    Xw = X0 + np.linalg.solve(A, B - A @ X0)
    assert np.allclose(X, Xw, rtol=0, atol=1e-12) and out["berr"].shape == (nrhs,) and "ferr" not in out
    assert info == M + 201


@pytest.mark.parametrize("kind,grid,Kappa", [("lu", (1, 1, 1), None), ("lu", (2, 3, 2), None), ("chol", (2, 1, 1), 5)])
def test_distribute_collect_round_trip(kind, grid, Kappa):
    v, nrhs = 8, 70
    M = 48 if kind == "lu" else Kappa * v
    G = np.random.default_rng(1).standard_normal((M, nrhs))
    shares = rl.distribute(kind, G, v, *grid, Kappa=Kappa)
    assert np.array_equal(rl.collect(kind, shares, M, nrhs, v, *grid, Kappa=Kappa), G)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")
def test_cpp_facades_compile(tmp_path):
    src = tmp_path / "use_refine_local.cpp"
    src.write_text('#include "conflux/lu/conflux_b200.hpp"\n'
                   '#include "conflux/cholesky/conflux_b200_cholesky.hpp"\n'
                   "void f(conflux::lu_params<double>& g, const double* b, double* x, double* e, char* q) {\n"
                   "  conflux::LU_refine_local(g, 3, b, 8, x, 8, e, e, true);\n"
                   "  (void)conflux::LU_refine_x_local(g, 3, b, 8, x, 8, e, e, e, e);\n"
                   "  (void)conflux::LU_svx_local(g, 3, b, 8, x, 8, e, e, e, e, q, true);\n"
                   "  (void)conflux::LU_svxx_local(g, 3, b, 8, x, 8, e, e, e, e, e, q);\n"
                   "  conflux::choleskyRefineLocal(3, b, 8, x, 8, e, e);\n"
                   "  (void)conflux::choleskyRefineXLocal(3, b, 8, x, 8, e, e, e, e);\n"
                   "  (void)conflux::choleskySvxLocal(3, b, 8, x, 8, e, e, e, q);\n"
                   "  (void)conflux::choleskySvxxLocal(3, b, 8, x, 8, e, e, e, e, e, q); }\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)], check=True)
