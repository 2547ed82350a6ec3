"""CPU: conflux::conflux_layout of this repo's facade, both overloads, both orderings, several grids, produces exactly the
COSTA descriptors the REFERENCE's conflux_layout / lu_params::matrix produce (layout.cpp:30-135): row and column splits,
block owners, and every local block's position, stride and shape.  The reference side is stored in
tests/golden/layout_ref.txt (tests/golden/make_golden.py, tests/cpp/layout_dump_ref.cpp)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_layout_descriptors_match_costa(tmp_path, golden_dir):
    ref = open(os.path.join(golden_dir, "layout_ref.txt")).read()
    keys = [ln for ln in ref.splitlines() if ln.startswith(("bc ", "cart "))]
    assert len(keys) == 63                                   # 36 block-cyclic + 27 on the 3-D grid
    exe = tmp_path / "layout_dump_mine"
    subprocess.check_call(["g++", "-O1", "-std=c++17", f"-I{ROOT}/include", f"{ROOT}/tests/cpp/layout_dump_mine.cpp", "-o", str(exe)])
    out = subprocess.run([str(exe)], input="\n".join(keys) + "\n", capture_output=True, text=True, check=True).stdout
    assert out == ref
