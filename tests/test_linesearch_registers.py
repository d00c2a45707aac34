"""The Newton line search keeps the env's constraint edges in registers (sim_core.cuh `linesearch`, inlined into `newton_move`).

Lane l builds edge slots l + 32 j once per Newton move, and each cost evaluation (`ls_eval`) reads them from registers and returns
its three sums by value; the whole search is inlined into the Newton move.  Before, the edges went through a shared-memory list and
every evaluation was a call that returned its results through a stack array, which a 32-warp block keeps in L2 (beside a 231 KB shared-memory carve-out only ~25 KB of L1 are
left).  The first test pins the SASS of `fetch_kernel<32, 21>` (no GPU needed); the second replays a contact-heavy FetchPickAndPlace
rollout on the 32-lane emulation and requires the results of the previous sources bit for bit (tests/golden/make_linesearch_fixture.py).
"""
import os

import numpy as np
import pytest

from tests.test_local_memory import _tool, count, sass_by_function

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "linesearch_fetch_warp.npz")


@pytest.mark.skipif(_tool("nvcc") is None or _tool("nvdisasm") is None, reason="needs nvcc and nvdisasm (CUDA toolkit)")
def test_line_search_has_no_local_memory_and_no_calls(tmp_path):
    import subprocess

    from gymnasium_robotics_b200 import _lib

    cubin = str(tmp_path / "b200sim.cubin")
    flags = [f for f in _lib.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    src = os.path.join(os.path.dirname(_lib.__file__), "csrc", "b200sim.cu")
    subprocess.check_call([_tool("nvcc")] + flags + ["-cubin", "-o", cubin, src])
    text = subprocess.run([_tool("nvdisasm"), "-c", cubin], check=True, capture_output=True, text=True).stdout
    funcs = sass_by_function(text)
    # the line search is inlined into newton_move (before: a function of its own, with 4 LDL / 2 STL -- the results of every
    # evaluation went through a stack array -- and 3 CALLs: ls_edges and two ls_eval)
    assert not any(n in funcs for n in ("linesearch", "ls_eval", "ls_edges")), "the line search is a call again"
    mv = funcs["newton_move"]
    print(f"\nnewton_move: LDL {count(mv, 'LDL')}  STL {count(mv, 'STL')}  CALL {count(mv, 'CALL')}")
    assert count(mv, "LDL") == 0
    assert count(mv, "STL") <= 1   # the one store of the move's cost improvement into the driver's variable
    assert count(mv, "CALL") == 2  # mulM and rows_from_vec


def test_contact_heavy_rollout_is_bitwise_unchanged():
    from tests.golden.make_linesearch_fixture import ACTIONS, rollout

    want = np.load(GOLDEN)
    assert np.array_equal(want["actions"], np.asarray(ACTIONS, dtype=np.float32))
    assert int(want["counters"][:, 0].max()) == 16   # the contact table full: 16 contacts of 6 pyramid edges, 4 edge slots per lane
    got = rollout()
    for k in ("packed", "state", "info", "counters"):
        assert np.array_equal(got[k], want[k]), (k, np.argwhere(got[k] != want[k])[:5])
