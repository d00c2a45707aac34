"""Instruction footprint of the Newton iteration in the 32-warp Fetch step kernel (no GPU needed: nvcc cross-compiles, nvdisasm
reads the cubin).

`fetch_kernel<32, 21>` (the FetchPickAndPlace headline batch) runs 32 warps per SM under block-wide barriers, and every Newton
iteration streams the code of build_H, the direction solve and the move through the instruction caches.  Most of that code is
straight-line code that runs once per call, so its size is paid on every iteration (DESIGN.md 3, "Footprint of the Newton iteration").
The bounds pin the instruction counts of the stages of the loop; the counts include the divergent-warp copies that ptxas
emits after each function's return for the shuffles.
"""
import os
import subprocess

import pytest

from tests.test_local_memory import TOOLS, _tool, sass_by_function

pytestmark = pytest.mark.skipif(any(_tool(t) is None for t in TOOLS), reason="needs nvcc and nvdisasm (CUDA toolkit)")

# before: newton_move 3516, newton_begin 1809, spd_solve 2581, build_H 758; the iteration window 7663 instructions (120 KB)
BOUNDS = {"newton_move": 1650, "newton_begin": 450, "spd_solve": 2600, "build_H": 560}
WINDOW = ("newton_move", "spd_solve", "build_H", "mulM", "rows_from_vec", "newton_direction")
WINDOW_BOUND = 5500


@pytest.fixture(scope="module")
def funcs(tmp_path_factory):
    from gymnasium_robotics_b200 import _lib

    cubin = str(tmp_path_factory.mktemp("newton_footprint") / "b200sim.cubin")
    flags = [f for f in _lib.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    src = os.path.join(os.path.dirname(_lib.__file__), "csrc", "b200sim.cu")
    subprocess.check_call([_tool("nvcc")] + flags + ["-cubin", "-o", cubin, src])
    text = subprocess.run([_tool("nvdisasm"), "-c", cubin], check=True, capture_output=True, text=True).stdout
    f = sass_by_function(text)
    print("\nfunction             instructions     KB")
    for name in sorted(set(BOUNDS) | set(WINDOW)):
        print(f"{name:20s} {len(f.get(name, [])):12d} {16 * len(f.get(name, [])) / 1024:6.1f}")
    return f


@pytest.mark.parametrize("name", sorted(BOUNDS))
def test_stage_footprint(funcs, name):
    assert name in funcs, f"{name} is not a function of its own in fetch_kernel<32, 21>"
    assert len(funcs[name]) <= BOUNDS[name]


def test_newton_iteration_window(funcs):
    assert all(n in funcs for n in WINDOW)
    assert sum(len(funcs[n]) for n in WINDOW) <= WINDOW_BOUND
