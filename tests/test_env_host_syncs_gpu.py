"""Host-device synchronisations of `reset` and of ordinary `step`s, per env class (run with -m gpu on an H100).

DESIGN.md section 6 promises that a step synchronises only when the autoreset state machine has to read the device: when the
host-side bound on the step counters says an env may be due, or when an env can terminate.  Each case runs 64 envs with
device-resident actions and `max_episode_steps=4`, so the 10 steps cross two and a half episodes, and counts the synchronising
calls that `torch.cuda.set_sync_debug_mode("warn")` reports in a second seeded `reset` and in each `step`.  The tables were recorded on an
NVIDIA H100 80GB HBM3.  A change to the state machine or to a reset path that adds a device read fails here.
"""
import json
import os
import sys
import warnings

import pytest
import torch

import gymnasium_robotics_b200 as pkg

pytestmark = pytest.mark.gpu

N, T, STEPS, SEED = 64, 4, 10, 3
IDS = {
    "fetch_reach": ("FetchReach-v4", {}),
    "hand_rotate_z": ("HandManipulateBlockRotateZ-v1", {}),
    "hand_reach": ("HandReach-v3", {}),
    "adroit_door": ("AdroitHandDoor-v2", {}),
    "adroit_pen": ("AdroitHandPen-v2", {}),
    "antmaze_continuing": ("AntMaze_UMaze-v5", {"continuing_task": True}),
    "antmaze_terminating": ("AntMaze_UMaze-v5", {"continuing_task": False}),
    "pointmaze": ("PointMaze_UMaze-v3", {}),
    "kitchen": ("FrankaKitchen-v1", {}),
}
CASES = [(name, mode, rng) for name in IDS for mode in ("next_step", "same_step")
         for rng in (("torch",) if name == "kitchen" else ("torch", "device"))]

# (name, autoreset mode, rng_mode) -> (syncs in reset, [syncs in each of the 10 steps])
EXPECTED = {
    ("fetch_reach", "next_step", "torch"): (2, [0, 0, 0, 0, 1, 0, 0, 0, 0, 1]),
    ("fetch_reach", "next_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("fetch_reach", "same_step", "torch"): (1, [0, 0, 0, 1, 0, 0, 0, 1, 0, 0]),
    ("fetch_reach", "same_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("hand_rotate_z", "next_step", "torch"): (6, [0, 0, 0, 0, 6, 0, 0, 0, 0, 6]),
    ("hand_rotate_z", "next_step", "device"): (2, [0, 0, 0, 0, 2, 0, 0, 0, 0, 2]),
    ("hand_rotate_z", "same_step", "torch"): (6, [0, 0, 0, 6, 0, 0, 0, 6, 0, 0]),
    ("hand_rotate_z", "same_step", "device"): (2, [0, 0, 0, 2, 0, 0, 0, 2, 0, 0]),
    ("hand_reach", "next_step", "torch"): (5, [0, 0, 0, 0, 5, 0, 0, 0, 0, 5]),
    ("hand_reach", "next_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("hand_reach", "same_step", "torch"): (5, [0, 0, 0, 5, 0, 0, 0, 5, 0, 0]),
    ("hand_reach", "same_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("adroit_door", "next_step", "torch"): (1, [0, 0, 0, 0, 1, 0, 0, 0, 0, 1]),
    ("adroit_door", "next_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("adroit_door", "same_step", "torch"): (1, [0, 0, 0, 1, 0, 0, 0, 1, 0, 0]),
    ("adroit_door", "same_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("adroit_pen", "next_step", "torch"): (3, [0, 0, 0, 0, 3, 0, 0, 0, 0, 3]),
    ("adroit_pen", "next_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("adroit_pen", "same_step", "torch"): (3, [0, 0, 0, 3, 0, 0, 0, 3, 0, 0]),
    ("adroit_pen", "same_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("antmaze_continuing", "next_step", "torch"): (11, [0, 0, 0, 0, 8, 0, 0, 0, 0, 8]),
    ("antmaze_continuing", "next_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("antmaze_continuing", "same_step", "torch"): (11, [0, 0, 0, 8, 0, 0, 0, 8, 0, 0]),
    ("antmaze_continuing", "same_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("antmaze_terminating", "next_step", "torch"): (11, [1, 1, 1, 1, 10, 1, 1, 1, 1, 10]),
    ("antmaze_terminating", "next_step", "device"): (0, [1, 1, 1, 1, 1, 1, 1, 1, 1, 1]),
    ("antmaze_terminating", "same_step", "torch"): (11, [1, 1, 1, 10, 1, 1, 1, 10, 1, 1]),
    ("antmaze_terminating", "same_step", "device"): (0, [1, 1, 1, 1, 1, 1, 1, 1, 1, 1]),
    ("pointmaze", "next_step", "torch"): (11, [0, 0, 0, 0, 8, 0, 0, 0, 0, 8]),
    ("pointmaze", "next_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("pointmaze", "same_step", "torch"): (11, [0, 0, 0, 8, 0, 0, 0, 8, 0, 0]),
    ("pointmaze", "same_step", "device"): (0, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0]),
    ("kitchen", "next_step", "torch"): (3, [1, 1, 1, 1, 5, 1, 1, 1, 1, 5]),
    ("kitchen", "same_step", "torch"): (3, [1, 1, 1, 5, 1, 1, 1, 5, 1, 1]),
}


def _count(fn):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in caught)


def observe(name, mode, rng):
    env_id, kw = IDS[name]
    env = pkg.make_vec(env_id, num_envs=N, device="cuda:0", rng_mode=rng, autoreset_mode=mode, max_episode_steps=T, **kw)
    gen = torch.Generator(device="cuda:0")
    gen.manual_seed(SEED)
    nact = env.single_action_space.shape[0]
    actions = [torch.rand((N, nact), generator=gen, device="cuda:0") * 2 - 1 for _ in range(STEPS)]
    env.reset(seed=SEED)   # first calls build lazy tables and initialise the process's CUDA state: not counted
    torch.cuda.synchronize()
    on_reset = _count(lambda: env.reset(seed=SEED))
    on_step = [_count(lambda a=a: env.step(a)) for a in actions]
    torch.cuda.synchronize()
    env.close()
    return on_reset, on_step


@pytest.mark.parametrize("name,mode,rng", CASES, ids=["-".join(c) for c in CASES])
def test_host_syncs_per_call(name, mode, rng):
    on_reset, on_step = observe(name, mode, rng)
    assert (on_reset, on_step) == EXPECTED[(name, mode, rng)]


if __name__ == "__main__":   # print the table in the form of EXPECTED
    table = {"|".join(c): observe(*c) for c in CASES}
    text = json.dumps(table, indent=1)
    print(text)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(sys.argv[1]) or ".", exist_ok=True)
        with open(sys.argv[1], "w") as f:
            f.write(text)
