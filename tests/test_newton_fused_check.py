"""The Newton convergence check ends the stage that moves the solver (sim_core.cuh `newton_begin`, `newton_move`).

The contact update of the move parks each contact's base-row forces and edge activity from the values it has just written, and the
move then runs the rest of the check (J^T f, gradient, norms, tests) before it returns: there is no `newton_check` or `pass_F`
call of its own.  This pins the SASS of `fetch_kernel<32, 21>` (no GPU needed): the fused move stays off local memory and the
entry function issues fewer stage calls.
"""
import os
import subprocess

import pytest

from tests.test_local_memory import TOOLS, _tool, count, sass_by_function

pytestmark = pytest.mark.skipif(any(_tool(t) is None for t in TOOLS), reason="needs nvcc and nvdisasm (CUDA toolkit)")


def test_newton_check_is_fused_into_the_move(tmp_path):
    from gymnasium_robotics_b200 import _lib

    cubin = str(tmp_path / "b200sim.cubin")
    flags = [f for f in _lib.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    src = os.path.join(os.path.dirname(_lib.__file__), "csrc", "b200sim.cu")
    subprocess.check_call([_tool("nvcc")] + flags + ["-cubin", "-o", cubin, src])
    text = subprocess.run([_tool("nvdisasm"), "-c", cubin], check=True, capture_output=True, text=True).stdout
    funcs = sass_by_function(text)
    assert not any(n in funcs for n in ("newton_check", "pass_F")), "the convergence check is a call again"
    mv, begin, entry = funcs["newton_move"], funcs["newton_begin"], funcs["ENTRY"]
    print(f"\nnewton_move: {len(mv)} instructions, LDL {count(mv, 'LDL')}  STL {count(mv, 'STL')}  CALL {count(mv, 'CALL')}"
          f"\nnewton_begin: {len(begin)} instructions, CALL {count(begin, 'CALL')}\nentry: CALL {count(entry, 'CALL')}")
    # before: newton_move 1 STL (the cost improvement, into the driver's variable), no LDL
    assert count(mv, "LDL") == 0
    assert count(mv, "STL") == 0
    # the check's gradient floor (gnorm < 2e-6 fnorm) is in both stages: the check was not compiled away
    floor = "1.9999999949504854158e-06"
    assert any(floor in l for l in mv) and any(floor in l for l in begin)
    # before: 28 CALLs in the entry function, one newton_check call in each of its two inlined copies of forward()
    assert count(entry, "CALL") <= 26
