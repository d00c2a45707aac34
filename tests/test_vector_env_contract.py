"""The gymnasium vector-env contract of every env class, on the host emulation: the three autoreset modes (NEXT_STEP, SAME_STEP,
disabled) of the one state machine in vector.py, the info keys each family reports, and the construction checks every family
shares (rng_mode, auto_recover, obs_dtype)."""
import numpy as np
import pytest
import torch

from tests.test_api_conformance import _leaves, _make

T = 2   # max_episode_steps: the second step truncates
CLASSES = {
    "FetchReach-v4": {},
    "HandManipulateBlockRotateZ-v1": {},
    "HandReach-v3": {},
    "AdroitHandDoor-v2": {},
    "AdroitHandPen-v2": {},
    "AntMaze_UMaze-v5/continuing": {"continuing_task": True},
    "AntMaze_UMaze-v5/terminating": {"continuing_task": False},
    "PointMaze_UMaze-v3": {},
    "FrankaKitchen-v1": {},
}
KITCHEN_INFO = {"tasks_to_complete", "step_task_completions", "episode_task_completions"}


def _env(case, n=2, **kw):
    return _make(case.split("/")[0], n, max_episode_steps=T, **CLASSES[case], **kw)


def _family(case):
    return "kitchen" if case.startswith("Franka") else "maze" if "Maze" in case else "adroit" if case.startswith("Adroit") else "robot"


# family -> (reset info keys, step info keys, final_info keys or None)
INFO_KEYS = {
    "robot": (set(), {"is_success", "_is_success", "solver_info"}, {"is_success", "_is_success"}),
    "adroit": (set(), {"success", "_success", "solver_info"}, {"success", "_success"}),
    "maze": ({"success"}, {"success", "solver_info"}, {"success", "_success"}),
    "kitchen": (KITCHEN_INFO, KITCHEN_INFO, None),
}
FINAL = {"final_obs", "_final_obs", "final_info", "_final_info"}


def _actions(env, k):
    rng = np.random.default_rng(100 + k)
    return torch.as_tensor(rng.uniform(-1, 1, (env.num_envs, env.single_action_space.shape[0])).astype(np.float32))


def _success(case, info):
    fam = _family(case)
    if fam == "kitchen":
        return info["step_task_completions"].any(dim=1)
    return info["is_success" if fam == "robot" else "success"] != 0


def _run(case, mode, steps):
    env = _env(case, autoreset_mode=mode)
    out = [env.reset(seed=4)]
    out += [env.step(_actions(env, k)) for k in range(steps)]
    return env, out


@pytest.mark.parametrize("case", CLASSES)
def test_next_step_resets_on_the_call_after_the_episode_ends(case):
    env, out = _run(case, "next_step", T + 1)
    reset_keys, step_keys, _ = INFO_KEYS[_family(case)]
    assert set(out[0][1]) == reset_keys
    _, r, te, tr, info = out[T]
    assert bool(tr.all()) and set(info) == step_keys            # the TimeLimit ends every episode on step T
    _, r, te, tr, info = out[T + 1]                             # this call resets them: its action is ignored
    assert set(info) == step_keys
    assert torch.equal(r, torch.zeros_like(r)) and not bool(te.any()) and not bool(tr.any())
    assert not bool(_success(case, info).any()) and torch.equal(env._elapsed, torch.zeros_like(env._elapsed))
    env.close()


@pytest.mark.parametrize("case", CLASSES)
def test_same_step_returns_the_final_observation_and_resets(case):
    env, out = _run(case, "same_step", T)
    _, step_keys, final_keys = INFO_KEYS[_family(case)]
    assert set(out[1][4]) == step_keys
    _, r, te, tr, info = out[T]
    assert bool(tr.all()) and set(info) == step_keys | (FINAL if final_keys else {"final_obs", "_final_obs"})
    assert bool(info["_final_obs"].all())
    if final_keys:
        assert set(info["final_info"]) == final_keys and bool(info["_final_info"].all())
    assert torch.equal(env._elapsed, torch.zeros_like(env._elapsed))
    env.close()


@pytest.mark.parametrize("case", [c for c in CLASSES if not c.startswith("Franka")])
def test_same_step_and_next_step_twins_see_the_same_episodes(case):
    """Same seed, same actions: SAME_STEP's final observation is NEXT_STEP's step-T observation, and SAME_STEP's step-T
    observation (the reset one) is NEXT_STEP's step-(T + 1) observation.  (The kitchen draws its step noise before the reset
    noise, so its two modes consume the stream in different orders.)"""
    _, same = _run(case, "same_step", T)
    _, nxt = _run(case, "next_step", T + 1)
    final = dict(_leaves(same[T][4]["final_obs"]))
    assert final.keys() == dict(_leaves(nxt[T][0])).keys()
    for (k, a), (_, b) in zip(_leaves(same[T][4]["final_obs"]), _leaves(nxt[T][0])):
        assert torch.equal(a, b), k
    for (k, a), (_, b) in zip(_leaves(same[T][0]), _leaves(nxt[T + 1][0])):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("case", CLASSES)
def test_disabled_autoreset_never_resets(case):
    env, out = _run(case, "disabled", T + 1)
    _, step_keys, _ = INFO_KEYS[_family(case)]
    assert all(set(o[4]) == step_keys for o in out[1:])
    assert bool(out[T + 1][3].all())                             # still past the TimeLimit: nothing was reset
    assert torch.equal(env._elapsed, torch.full_like(env._elapsed, T + 1))
    env.close()


@pytest.mark.parametrize("case", CLASSES)
def test_unknown_rng_mode_is_refused(case):
    with pytest.raises(ValueError, match="rng_mode"):
        _env(case, rng_mode="philox")


def test_kitchen_has_no_device_rng():
    with pytest.raises(NotImplementedError, match="rng_mode='device'"):
        _env("FrankaKitchen-v1", rng_mode="device")


@pytest.mark.parametrize("case", ["AntMaze_UMaze-v5/continuing", "PointMaze_UMaze-v3", "FrankaKitchen-v1"])
def test_auto_recover_is_refused_where_there_is_no_recovery(case):
    with pytest.raises(NotImplementedError, match="auto_recover"):
        _env(case, auto_recover=True)


def test_kitchen_applies_obs_dtype():
    env = _env("FrankaKitchen-v1", obs_dtype=torch.float64)
    obs, _ = env.reset(seed=1)
    step_obs = env.step(_actions(env, 0))[0]
    for o in (obs, step_obs):
        leaves = list(_leaves(o))
        assert {k.split("/")[1] for k, _ in leaves} == {"observation", "achieved_goal", "desired_goal"}
        assert all(v.dtype == torch.float64 for _, v in leaves)
    env.close()
