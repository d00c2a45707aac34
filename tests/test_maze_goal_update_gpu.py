"""The goal update of continuing maze tasks (`reset_target=True`) on the GPU: the update kernel that b200sim_step launches after the
step kernel in rng_mode="device" (b200sim_set_goal_update) against the restatement in tests/test_maze_goal_update.py, its
invariance to batch shape, block size and sharding, the rest of the step left bit for bit alone, oracle parity in the numpy
mode, and steps that make no synchronising call.  Models come from the committed blobs."""
import warnings

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.maze import MAPS, NOISE, SUCCESS_RADIUS
from tests.parity_util import check_envelope, inject_records
from tests.test_gpu_parity import ENVELOPE
from tests.test_maze_goal_update import GoalOracleAntMaze, _dist_device, py_goal_update

pytestmark = pytest.mark.gpu

# two goal cells and one reset cell, in a map of its own
CUSTOM = [[1, 1, 1, 1, 1, 1], [1, "g", 0, 0, "g", 1], [1, 0, 1, 0, 0, 1], [1, 0, 0, "r", 0, 1], [1, 1, 1, 1, 1, 1]]
CASES = {"antmaze_large": ("AntMaze_Large-v5", 1024, {}), "pointmaze_large": ("PointMaze_Large-v3", 4096, {}),
         "pointmaze_custom": ("PointMaze_UMaze-v3", 512, {"maze_map": CUSTOM})}
f32 = np.float32


def _make(name, n=None, **kw):
    env_id, size, extra = CASES[name]
    kw = {**extra, "rng_mode": "device", "reset_target": True, "device": "cuda:0", **kw}
    return pkg.make_vec(env_id, num_envs=n or size, **kw)


def _goals(env):
    return env.backend.state[:, env._sl["goal"]].clone()


def _place_on_goals(env, shift=None):
    """Every agent onto its goal (+ shift [N, 2]), at rest, keeping the step counters."""
    st, el = env.get_state()
    q = env._sl["qpos"].start
    st[:, q:q + 2] = st[:, env._sl["goal"]] + (0 if shift is None else shift)
    st[:, env._sl["qvel"]] = 0
    env.set_state(st, el)


def _zeros(env):
    return torch.zeros((env.num_envs, env.single_action_space.shape[0]), device="cuda:0")


def _shift(n):
    """Every third env 0.6 m off its goal, outside the success radius (an ant whose legs land in a wall may be pushed back in)."""
    s = torch.zeros((n, 2), device="cuda:0")
    s[::3, 0] = 0.6
    return s


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_goal_update_equals_the_restatement(name):
    seed = 31
    env = _make(name, env_offset=7)
    env.reset(seed=seed)
    gl = env._goal_loc.cpu().numpy()
    for step in range(1, 3):
        _place_on_goals(env, _shift(env.num_envs))
        old = _goals(env).cpu().numpy()
        o, r, te, tr, info = env.step(_zeros(env))
        new, ach = _goals(env).cpu().numpy(), o["achieved_goal"].cpu().numpy()
        succ = info["success"].cpu().numpy()
        assert np.array_equal(o["desired_goal"].cpu().numpy(), old)        # the step's observation carries the old goal
        assert succ.sum() > env.num_envs // 2 and (~succ).sum() > env.num_envs // 6
        changed = (new != old).any(axis=1)
        assert np.array_equal(changed, succ)                                 # fires exactly for the success column
        for i in np.flatnonzero(succ):
            want, k = py_goal_update(gl, env.scaling, NOISE, SUCCESS_RADIUS, seed, 7 + i, 1, step, ach[i], old[i], dist=_dist_device)
            assert k > 0 and np.array_equal(new[i], want), (step, i)
            assert (np.abs(gl - new[i]).max(axis=1) <= NOISE * env.scaling + 1e-5).any()
            assert np.linalg.norm(ach[i].astype(np.float64) - new[i]) > SUCCESS_RADIUS - 1e-6
    env.close()


@pytest.mark.parametrize("name", ["antmaze_large", "pointmaze_large"])
def test_device_goals_are_invariant_to_batch_block_size_and_sharding(name, monkeypatch):
    seed, steps = 5, 3

    def run(n, offset=0, wpb=None):
        if wpb is None:
            monkeypatch.delenv("B200SIM_WPB", raising=False)
        else:
            monkeypatch.setenv("B200SIM_WPB", str(wpb))
        env = _make(name, n=n, env_offset=offset)
        monkeypatch.delenv("B200SIM_WPB", raising=False)
        env.reset(seed=seed)
        out = []
        for _ in range(steps):
            _place_on_goals(env)
            env.step(_zeros(env))
            out.append(_goals(env).cpu())
        env.close()
        return out

    n = CASES[name][1]
    full = run(n)
    for wpb in (7, 16):
        assert all(torch.equal(a, b) for a, b in zip(full, run(n, wpb=wpb)))
    assert all(torch.equal(a[:n // 4], b) for a, b in zip(full, run(n // 4)))
    # the second half in two shards (env_offset)
    for k in range(2):
        o = n // 2 + k * (n // 4)
        assert all(torch.equal(a[o:o + n // 4], b) for a, b in zip(full, run(n // 4, offset=o)))


@pytest.mark.parametrize("name", ["antmaze_large", "pointmaze_large"])
def test_the_rest_of_the_step_is_untouched(name):
    """The same seeded step with the update on and off: packed rows, flags and every record word but the goal slots are identical."""
    res = []
    for reset_target in (True, False):
        env = _make(name, reset_target=reset_target)
        env.reset(seed=9)
        _place_on_goals(env, _shift(env.num_envs))
        out = env.backend.new_outputs()
        env.backend.step(_zeros(env), out)
        st = env.backend.state.clone()
        g = env._sl["goal"]
        res.append((out["packed"].clone(), out["flags"].clone(), torch.cat([st[:, :g.start], st[:, g.stop:]], 1), st[:, g]))
        env.close()
    on, off = res
    for a, b in zip(on[:3], off[:3]):
        assert torch.equal(a, b)
    assert not torch.equal(on[3], off[3])


def test_antmaze_oracle_parity_with_reset_target():
    """AntMaze_Large-v5 in the numpy mode with reset_target=True against the oracle env with update_goal, from the oracle's state at
    every step; half the agents sit on their goals so that goals are redrawn.  Inside the stated antmaze/* envelopes."""
    n, seed = 8, 12
    env = pkg.make_vec("AntMaze_Large-v5", num_envs=n, device="cuda:0", rng_mode="numpy", reset_target=True)
    obs, _ = env.reset(seed=seed)
    oracles = [GoalOracleAntMaze(MAPS["Large"], model=env.model, include_cfrc_ext_in_observation=True, reset_target=True) for _ in range(n)]
    for i, o in enumerate(oracles):
        oo, _ = o.reset(seed=seed + i)
        np.testing.assert_allclose(obs["desired_goal"][i].double().cpu().numpy(), oo["desired_goal"], rtol=1e-6, atol=2e-6)
    rng = np.random.default_rng(2)
    epos, evel, ecf, updates = [], [], [], 0
    for step in range(6):
        for i, o in enumerate(oracles):
            if (i + step) % 2 == 0:
                o.sim.qpos[:2] = o.goal
                o.sim.forward()
        env.set_state(inject_records(env, oracles, lambda i, o, rec, lay: rec.__setitem__(slice(lay["goal"], lay["goal"] + 2), o.goal)))
        a = rng.uniform(-1, 1, (n, 8)).astype(np.float32)
        o_, r, te, tr, info = env.step(torch.as_tensor(a))
        goals = _goals(env).cpu().numpy()
        for i, orc in enumerate(oracles):
            before = orc.goal.copy()
            oo, orr, ote, otr, oi = orc.step(a[i].astype(np.float64))
            d = np.abs(o_["observation"][i].double().cpu().numpy() - oo["observation"])
            epos.append(d[:13].max()); evel.append(d[13:27].max()); ecf.append(d[27:].max())
            assert bool(info["success"][i]) == oi["success"] and float(r[i]) == float(orr)
            np.testing.assert_array_equal(goals[i], orc.goal.astype(f32))
            updates += int(not np.array_equal(before, orc.goal))
    assert updates >= 10
    check_envelope("antmaze/pos", epos, *ENVELOPE["antmaze/pos"])
    check_envelope("antmaze/vel", evel, *ENVELOPE["antmaze/vel"])
    check_envelope("antmaze/cfrc", ecf, *ENVELOPE["antmaze/cfrc"])
    env.close()


def _sync_messages(fn):
    """The synchronising calls torch.cuda.set_sync_debug_mode("warn") reports while fn runs (as tests/test_env_host_syncs_gpu.py
    counts them), without the notice that torch gives once per process when the mode is first switched on."""
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return [str(w.message) for w in caught if "synchroniz" in str(w.message) and "prototype feature" not in str(w.message)]


@pytest.mark.parametrize("env_id", ["AntMaze_UMaze-v5", "PointMaze_UMaze-v3"])
def test_device_mode_steps_with_goal_updates_make_no_synchronising_call(env_id):
    n = 64
    env = pkg.make_vec(env_id, num_envs=n, device="cuda:0", rng_mode="device", reset_target=True)
    env.reset(seed=3)
    gen = torch.Generator(device="cuda:0").manual_seed(3)
    nact = env.single_action_space.shape[0]
    actions = [torch.rand((n, nact), generator=gen, device="cuda:0") * 2 - 1 for _ in range(9)]
    env.step(actions[0])                 # first calls of this env: not counted
    _place_on_goals(env)                 # (set_state reads the step counters: not counted)
    g0 = _goals(env)
    torch.cuda.synchronize()
    syncs = [_sync_messages(lambda a=a: env.step(a)) for a in actions[1:]]
    torch.cuda.synchronize()
    assert syncs == [[]] * len(actions[1:])
    assert not torch.equal(_goals(env), g0)     # goals were redrawn on the way
    env.close()
