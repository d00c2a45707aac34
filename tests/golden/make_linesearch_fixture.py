"""Writes tests/golden/linesearch_fetch_warp.npz: a FetchPickAndPlace rollout on the 32-lane emulation of the kernel source (the lane-parallel
code nvcc compiles, tests/hostsim flavor "warp"), from a seeded reset through steps that press the closed gripper onto the table and the
object and then drag it, so that every sub-step's Newton moves run line searches over contact, weld and joint-limit edges.  Per step:
the packed output row, the state record, the info word and the solver counters, stored as int32 bit patterns.
tests/test_linesearch_registers.py replays the rollout and compares bit for bit.  Run from the repository root:
    PYTHONPATH=. python tests/golden/make_linesearch_fixture.py"""
import os

import numpy as np
import torch

from tests.hostsim_backend import HostSimBackend

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "linesearch_fetch_warp.npz")
ACTIONS = [[0.0, 0.0, -1.0, -1.0]] * 8 + [[0.6, -0.4, -1.0, -1.0]] * 2 + [[-0.5, 0.5, 0.3, -1.0]] * 2


class W32(HostSimBackend):
    FLAVOR = "warp"


def rollout():
    from gymnasium_robotics_b200.fetch import FetchVectorEnv

    env = FetchVectorEnv("FetchPickAndPlace", num_envs=1, backend_factory=W32, rng_mode="numpy")
    env.reset(seed=0)
    b = env.backend
    out = b.new_outputs()
    packed, state, info, counters = [], [], [], []
    for a in ACTIONS:
        b.step(torch.tensor([a], dtype=torch.float32), out)
        packed.append(out["packed"][0].numpy().view(np.int32).copy())
        state.append(b.state[0].numpy().view(np.int32).copy())
        info.append(b.info.numpy().copy())
        counters.append(np.asarray(b.sim.counters(), dtype=np.int64).astype(np.int32))
    return dict(packed=np.stack(packed), state=np.stack(state), info=np.stack(info), counters=np.stack(counters))


if __name__ == "__main__":
    np.savez(OUT, actions=np.asarray(ACTIONS, dtype=np.float32), **rollout())
    print("wrote", OUT)
