"""Partial resets through the CUDA library (run with -m gpu on an H100): the rule of tests/test_reset_mask.py for every family at 64
envs, and at the bench sizes of Fetch (4096) and the Kitchen (2048), with masks that hit the first and last env of a block and
fill part of one; and the synchronising calls of a partial reset in rng_mode="device" with a device mask."""
import ctypes
import json
import os
import subprocess
import sys
import warnings

import pytest
import torch

import gymnasium_robotics_b200 as pkg
from tests.test_reset_mask import check_autoreset_twin, check_reseed_rule

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDS = {
    "fetch": ("FetchPickAndPlace-v4", {}),
    "hand": ("HandManipulateBlockRotateZ-v1", {}),
    "hand_reach": ("HandReach-v3", {}),
    "adroit": ("AdroitHandHammer-v2", {}),
    "antmaze": ("AntMaze_UMaze-v5", {"continuing_task": True}),
    "antmaze_v3": ("AntMaze_UMaze-v3", {}),
    "pointmaze_reset_target": ("PointMaze_UMaze-v3", {"reset_target": True}),
    "kitchen": ("FrankaKitchen-v1", {}),
}


def _make(name, n, rng_mode, **kw):
    env_id, base = IDS[name]
    kw = dict(base, **kw)
    kw.setdefault("max_episode_steps", 50)
    kw.setdefault("autoreset_mode", "disabled")
    return pkg.make_vec(env_id, num_envs=n, device="cuda:0", rng_mode=rng_mode, **kw)


def _envs_per_block(env):
    wpb = ctypes.c_int()
    env.backend.L.b200sim_launch_config(env.backend.h, None, ctypes.byref(wpb), None)
    return wpb.value


def edge_mask(n, wpb):
    """Every 5th env, the first and last env of the step kernel's blocks and of the 128-thread draw blocks, the last env, and the first
    half of the block in the middle of the batch."""
    m = torch.arange(n) % 5 == 0
    for b in (wpb, 128):
        m[b - 1::b] = True
        m[b::b] = True
    m[-1] = True
    mid = (n // 2 // wpb) * wpb
    m[mid:mid + max(wpb // 2, 1)] = True
    m[mid + max(wpb // 2, 1):mid + wpb] = False
    return m.to("cuda:0")


def _mask_for(name, n, rng_mode):
    env = _make(name, n, rng_mode)
    m = edge_mask(n, _envs_per_block(env))
    env.close()
    return m


# (FrankaKitchen's numpy mode draws its noise on the host: the CPU suite covers it)
CASES = [(name, 64, rng) for name in IDS for rng in ("device", "numpy") if (name, rng) != ("kitchen", "numpy")] + \
    [("fetch", 4096, "device"), ("kitchen", 2048, "device")]


@pytest.mark.parametrize("name,n,rng_mode", CASES, ids=[f"{a}-{b}-{c}" for a, b, c in CASES])
def test_partial_reseed_equals_a_full_reset_and_leaves_the_others(name, n, rng_mode):
    check_reseed_rule(lambda: _make(name, n, rng_mode), _mask_for(name, n, rng_mode))


@pytest.mark.parametrize("name,n,rng_mode", CASES, ids=[f"{a}-{b}-{c}" for a, b, c in CASES])
def test_partial_reset_without_seed_is_an_autoreset_of_the_masked_envs(name, n, rng_mode):
    from tests.test_reset_mask import K

    check_autoreset_twin(lambda mode: _make(name, n, rng_mode, max_episode_steps=K, autoreset_mode=mode), _mask_for(name, n, rng_mode))


# ------------------------------------------------------------------ synchronising calls
def _sync_messages(fn):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in caught)


def partial_reset_syncs():
    """name -> (syncs of a partial reset with seed=None, with seed=9), 64 envs in rng_mode="device", a device mask."""
    res = {}
    _sync_messages(lambda: None)   # torch's one notice about the sync debug mode, printed the first time it is switched on
    for name in IDS:
        env = _make(name, 64, "device")
        mask = edge_mask(64, _envs_per_block(env))
        env.reset(seed=3)
        env.reset(seed=3, options={"reset_mask": mask})   # first calls: not counted
        torch.cuda.synchronize()
        res[name] = [_sync_messages(lambda s=s: env.reset(seed=s, options={"reset_mask": mask})) for s in (None, 9)]
        torch.cuda.synchronize()
        env.close()
    return res


# the Hand's settle loop reads `pending.any()` once per attempt, as in tests/test_env_host_syncs_gpu.py's reset table; the mazes keep
# per-env numpy streams for explicit `options` cells in every rng mode, so a reseeding partial reset reads the mask to reseed them
EXPECTED = {"fetch": [0, 0], "hand": [2, 2], "hand_reach": [0, 0], "adroit": [0, 0], "antmaze": [0, 1], "antmaze_v3": [0, 1],
            "pointmaze_reset_target": [0, 1], "kitchen": [0, 0]}


def test_device_partial_reset_makes_no_synchronising_call():
    # In a process of its own: torch prints its notice about the sync debug mode once per process, the first time the mode is
    # switched on, and tests/test_env_host_syncs_gpu.py counts that notice in the first reset it observes.
    code = "import json; from tests.test_reset_mask_gpu import partial_reset_syncs; print(json.dumps(partial_reset_syncs()))"
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-4000:]
    assert json.loads(res.stdout.strip().splitlines()[-1]) == EXPECTED
