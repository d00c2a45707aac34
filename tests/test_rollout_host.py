"""SURVEY.md 8f row 4 on CPU (host emulation backend): EzPickle-style pickling of the vector envs and the trajectory dump."""
import pickle

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.rollout import RolloutRecorder, load_rollout
from tests.hostsim_backend import HostSimBackend


def fetch(n=3, **kw):
    return pkg.make_vec("FetchReach-v4", num_envs=n, backend_factory=HostSimBackend, rng_mode="numpy", **kw)


def test_pickle_round_trip_rebuilds_from_constructor_arguments():
    """EzPickle semantics (fetch/reach.py:125-147): the unpickled env is a fresh env built from the recorded ctor call."""
    env = fetch(2, max_episode_steps=7, reward_type="dense")
    env2 = pickle.loads(pickle.dumps(env))
    assert type(env2) is type(env) and env2.num_envs == 2 and env2.max_episode_steps == 7 and env2.reward_type == "dense"
    o1, _ = env.reset(seed=5)
    o2, _ = env2.reset(seed=5)
    a = np.full((2, 4), 0.25, dtype=np.float32)
    s1, s2 = env.step(a), env2.step(a)
    assert torch.equal(s1[0]["observation"], s2[0]["observation"]) and torch.equal(s1[1], s2[1])
    maze = pkg.make_vec("AntMaze_UMaze-v5", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    maze2 = pickle.loads(pickle.dumps(maze))
    assert maze2.maze_name == "UMaze" and maze2.max_episode_steps == maze.max_episode_steps


def _check_episode_chain(ep):
    L = len(ep["actions"])
    assert ep["observations"]["observation"].shape[0] == L + 1
    assert ep["rewards"].shape == (L,) and ep["terminations"].shape == (L,)
    assert not (ep["terminations"][:-1] | ep["truncations"][:-1]).any()


@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_recorder_cuts_episodes_at_time_limits(mode, tmp_path):
    n, T = 3, 5
    env = fetch(n, max_episode_steps=T, autoreset_mode=mode)
    rec = RolloutRecorder(env, capacity_steps=32, env_id="FetchReach-v4")
    obs0, _ = rec.reset(seed=11)
    rng = np.random.default_rng(0)
    calls = 14
    for _ in range(calls):
        rec.step(rng.uniform(-1, 1, size=(n, 4)).astype(np.float32))
    eps = rec.episodes()
    per_env = {i: [e for e in eps if e["env_index"] == i] for i in range(n)}
    for i in range(n):
        full = [e for e in per_env[i] if e["truncations"][-1]]
        # next_step spends one call per episode on the reset: 14 calls = 5 + (1 + 5) + (1 + 2); same_step: 5 + 5 + 4
        assert [len(e["actions"]) for e in per_env[i]] == ([5, 5, 2] if mode == "next_step" else [5, 5, 4])
        assert len(full) == 2
        for e in per_env[i]:
            _check_episode_chain(e)
        # first observation of the first episode is the reset observation, and consecutive rows chain
        assert np.array_equal(per_env[i][0]["observations"]["observation"][0], obs0["observation"][i].numpy())
        # the final observation of a finished episode is not the next episode's reset observation
        assert not np.array_equal(per_env[i][0]["observations"]["observation"][-1], per_env[i][1]["observations"]["observation"][0])
        # every episode of an env starts from that env's rest pose region: gripper velocity entries are ~0 at reset
        for e in per_env[i]:
            assert np.abs(e["observations"]["observation"][0][5:]).max() < 1e-2
    # the GoalEnv invariant holds on the stored data (core.py:61-62): reward == compute_reward(achieved, desired)
    e = per_env[0][0]
    r = env.compute_reward(e["observations"]["achieved_goal"][1:], e["observations"]["desired_goal"][1:], {})
    assert np.array_equal(r, e["rewards"])
    meta = rec.save(str(tmp_path / "roll"))
    assert meta["total_episodes"] == len(eps) and meta["total_steps"] == sum(len(e["actions"]) for e in eps)
    meta2, eps2 = load_rollout(str(tmp_path / "roll"))
    assert meta2["env_id"] == "FetchReach-v4" and meta2["autoreset_mode"] == mode and len(eps2) == len(eps)
    for a, b in zip(eps, eps2):
        assert a["env_index"] == b["env_index"] and np.array_equal(a["actions"], b["actions"])
        for k in a["observations"]:
            assert np.array_equal(a["observations"][k], b["observations"][k])
        assert np.array_equal(a["infos"]["is_success"], b["infos"]["is_success"])


def test_recorder_matches_a_plain_rollout():
    """Recording does not change what the env returns, and the stored rows are the returned tensors."""
    n = 2
    env_a, env_b = fetch(n, max_episode_steps=50), fetch(n, max_episode_steps=50)
    rec = RolloutRecorder(env_b, capacity_steps=8)
    env_a.reset(seed=3); rec.reset(seed=3)
    rng = np.random.default_rng(1)
    outs = []
    for _ in range(4):
        a = rng.uniform(-1, 1, size=(n, 4)).astype(np.float32)
        oa = env_a.step(a); ob = rec.step(a)
        assert torch.equal(oa[0]["observation"], ob[0]["observation"]) and torch.equal(oa[1], ob[1])
        outs.append(oa)
    ep = [e for e in rec.episodes() if e["env_index"] == 1][0]
    assert len(ep["actions"]) == 4
    for k, o in enumerate(outs):
        assert np.array_equal(ep["observations"]["observation"][k + 1], o[0]["observation"][1].numpy())
        assert ep["rewards"][k] == float(o[1][1])
    with pytest.raises(RuntimeError, match="full"):
        for _ in range(5):
            rec.step(np.zeros((n, 4), dtype=np.float32))


def test_recorder_on_flat_observations():
    """Adroit envs return a flat observation tensor and `info["success"]` (adroit_hammer.py:291-357)."""
    env = pkg.make_vec("AdroitHandHammer-v2", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy", max_episode_steps=3)
    rec = RolloutRecorder(env, capacity_steps=8)
    rec.reset(seed=0)
    for _ in range(5):
        rec.step(np.zeros((1, 26), dtype=np.float32))
    eps = rec.episodes()
    assert [len(e["actions"]) for e in eps] == [3, 1]
    assert eps[0]["observations"].shape == (4, 46) and "success" in eps[0]["infos"]


def test_recorder_on_nested_goal_dicts():
    """FrankaKitchen-v1: achieved / desired goals are dicts task -> array (kitchen_env.py:371-397); keys are flattened as a/b."""
    from gymnasium_robotics_b200.kitchen import KitchenVectorEnv

    from tests.test_kitchen_host import KitchenHostBackend      # module-level class: picklable by reference

    env = KitchenVectorEnv(num_envs=2, backend_factory=KitchenHostBackend, device="cpu", rng_mode="numpy",
                           tasks_to_complete=["microwave", "kettle"], max_episode_steps=3)
    rec = RolloutRecorder(env, capacity_steps=8, env_id="FrankaKitchen-v1")
    rec.reset(seed=2)
    for _ in range(5):
        rec.step(np.zeros((2, 9), dtype=np.float32))
    eps = [e for e in rec.episodes() if e["env_index"] == 0]
    assert [len(e["actions"]) for e in eps] == [3, 1]
    ob = eps[0]["observations"]
    assert ob["observation"].shape == (4, 59) and ob["achieved_goal/microwave"].shape == (4, 1) and ob["desired_goal/kettle"].shape == (4, 7)
    env2 = pickle.loads(pickle.dumps(env))
    assert env2.tasks == ["microwave", "kettle"] and env2.max_episode_steps == 3


def test_vector_env_attribute_surface():
    """What gymnasium.vector wrappers touch besides reset / step: unwrapped, spec, render_mode, metadata, closed, context manager."""
    with fetch(2) as env:
        assert env.unwrapped is env and env.spec is None and env.render_mode is None and env.render() is None
        assert env.metadata["autoreset_mode"] == "next_step" and env.num_envs == 2 and not env.closed
        assert len(env.np_random) == 2        # rng_mode="numpy": one PCG64 generator per env, as N reference envs would have
        env.reset(seed=0)
    assert env.closed


def test_float64_observations_on_request():
    """The spaces declare float64 (robot_env.py:87-100); obs_dtype=torch.float64 casts the returned observations, the default stays float32."""
    e32, e64 = fetch(2), fetch(2, obs_dtype=torch.float64)
    o32, _ = e32.reset(seed=1)
    o64, _ = e64.reset(seed=1)
    assert o32["observation"].dtype == torch.float32 and all(v.dtype == torch.float64 for v in o64.values())
    assert torch.equal(o32["observation"].double(), o64["observation"])
    a = np.full((2, 4), 0.1, dtype=np.float32)
    s32, s64 = e32.step(a), e64.step(a)
    assert s64[0]["achieved_goal"].dtype == torch.float64 and torch.equal(s32[0]["achieved_goal"].double(), s64[0]["achieved_goal"])
    assert e64.single_observation_space["observation"].dtype == np.float64
