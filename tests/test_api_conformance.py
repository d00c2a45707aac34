"""API conformance of the vector envs, one id per env class / variant -- the local counterpart of the reference's
`tests/test_envs.py:39-53` (`gymnasium.utils.env_checker.check_env`), `:62-117` (same-seed determinism of a rollout), `:158-172`
(pickle round trip) and of the `GoalEnv` contract `reward == compute_reward(achieved_goal, desired_goal, info)`
(`gymnasium_robotics/core.py:45-62`).  Runs on the host emulation of the kernel source (no GPU); the CUDA path runs the same env
classes with another backend."""
import pickle

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from tests.hostsim_backend import HostSimBackend


class KitchenHostBackend(HostSimBackend):     # (module-level class: the pickled constructor call names its backend factory)
    FLAVOR = "kitchen"


def _factory(env_id):
    return KitchenHostBackend if env_id.startswith("Franka") else HostSimBackend


# (id, goal-env?, action dim, observation dim)
CASES = [
    ("FetchReach-v4", True, 4, 10), ("FetchPushDense-v4", True, 4, 25), ("FetchSlide-v4", True, 4, 25), ("FetchPickAndPlace-v4", True, 4, 25),
    ("HandReach-v3", True, 20, 63), ("HandReachDense-v3", True, 20, 63), ("HandManipulateBlockRotateZ-v1", True, 20, 61),
    ("HandManipulateBlockRotateXYZ_ContinuousTouchSensors-v1", True, 20, 153), ("HandManipulateEggFull-v1", True, 20, 61),
    ("HandManipulatePenRotateDense-v1", True, 20, 61),
    ("AdroitHandHammer-v2", False, 26, 46), ("AdroitHandRelocateSparse-v2", False, 30, 39), ("AdroitHandPen-v2", False, 24, 45),
    ("AdroitHandDoor-v2", False, 28, 39),
    ("AntMaze_UMaze-v5", True, 8, 105), ("AntMaze_Medium_Diverse_GR-v4", True, 8, 27), ("PointMaze_OpenDense-v3", True, 2, 4),
    ("FrankaKitchen-v1", True, 9, 59),
]


def _make(env_id, n=2, **kw):
    kw.setdefault("rng_mode", "numpy")
    if env_id.startswith("Franka"):
        kw.setdefault("device", "cpu")
    kw.setdefault("backend_factory", _factory(env_id))
    return pkg.make_vec(env_id, num_envs=n, **kw)


def _leaves(x, prefix=""):
    if isinstance(x, dict):
        for k in sorted(x):
            yield from _leaves(x[k], f"{prefix}/{k}")
    elif torch.is_tensor(x):
        yield prefix, x
    elif isinstance(x, np.ndarray):
        yield prefix, torch.as_tensor(x)


def _same(a, b):
    la, lb = list(_leaves(a)), list(_leaves(b))
    assert [k for k, _ in la] == [k for k, _ in lb]
    for (k, x), (_, y) in zip(la, lb):
        assert x.shape == y.shape and x.dtype == y.dtype, k
        assert torch.equal(x, y), k


@pytest.mark.parametrize("env_id,goal_env,nact,nobs", CASES, ids=[c[0] for c in CASES])
def test_api_conformance(env_id, goal_env, nact, nobs):
    n = 2
    env = _make(env_id, n)
    # ---- spaces (check_env: the spaces exist, are batched, and reset / step outputs live in them)
    assert env.num_envs == n
    assert env.single_action_space.shape == (nact,) and env.action_space.shape == (n, nact)
    assert float(env.single_action_space.low.min()) == -1.0 and float(env.single_action_space.high.max()) == 1.0
    osp = env.single_observation_space
    obs_shape = osp["observation"].shape if hasattr(osp, "spaces") else osp.shape
    assert obs_shape == (nobs,)
    obs, info = env.reset(seed=11)
    assert isinstance(info, dict)

    def check_obs(o):
        if goal_env:
            assert set(o) == {"observation", "achieved_goal", "desired_goal"}
            assert tuple(o["observation"].shape) == (n, nobs) and o["observation"].dtype == torch.float32
            for (ka, va), (kd, vd) in zip(_leaves(o["achieved_goal"]), _leaves(o["desired_goal"])):
                assert va.shape == vd.shape and va.shape[0] == n, (ka, kd)
        else:
            assert tuple(o.shape) == (n, nobs) and o.dtype == torch.float32
        for k, v in _leaves(o):
            assert bool(torch.isfinite(v).all()), k

    check_obs(obs)
    rng = np.random.default_rng(3)
    for t in range(3):
        a = torch.as_tensor(rng.uniform(-1, 1, (n, nact)).astype(np.float32))
        o, r, te, tr, inf = env.step(a)
        check_obs(o)
        assert tuple(r.shape) == (n,) and r.dtype == torch.float32 and bool(torch.isfinite(r).all())
        assert tuple(te.shape) == (n,) and te.dtype == torch.bool and tuple(tr.shape) == (n,) and tr.dtype == torch.bool
        assert isinstance(inf, dict)
        # the reference's info keys: robot_env.py:139-141 `is_success`; adroit_hammer.py:319 / maze_v4.py:401 `success`;
        # kitchen_env.py:399-423 the three task-bookkeeping entries
        want = ("is_success",) if env_id.startswith(("Fetch", "Hand")) else (("success",) if not env_id.startswith("Franka") else
                ("tasks_to_complete", "step_task_completions", "episode_task_completions"))
        assert all(k in inf for k in want), sorted(inf)
        if goal_env and not env_id.startswith("Franka"):
            # GoalEnv contract (core.py:45-62): the reward is a function of the goals in the observation
            rr = torch.as_tensor(env.compute_reward(o["achieved_goal"], o["desired_goal"], inf), dtype=torch.float32).reshape(n)
            if "Dense" in env_id:   # (the emulation backend's reward routine is a numpy twin of the kernel's: last-digit differences in acos)
                assert torch.allclose(rr, r, rtol=2e-6, atol=2e-6)
            else:
                assert torch.equal(rr, r)
        elif env_id.startswith("Franka"):
            assert torch.equal(env.compute_reward(o["achieved_goal"], o["desired_goal"], inf).reshape(n) >= r, torch.ones(n, dtype=torch.bool))
    # ---- wrong action shape is an error, not a broadcast
    with pytest.raises((ValueError, AssertionError, RuntimeError)):
        env.step(torch.zeros((n, nact + 1)))
    env.close()


@pytest.mark.parametrize("env_id", ["FetchPickAndPlace-v4", "HandManipulateBlockRotateXYZ-v1", "AdroitHandDoor-v2", "AntMaze_UMaze-v5",
                                    "PointMaze_UMaze-v3", "FrankaKitchen-v1"])
def test_same_seed_rollouts_are_bit_identical_and_pickle_round_trips(env_id):
    """tests/test_envs.py:62-117 (two instances, same seed, random steps: identical obs / reward / flags / info) and :158-172 (a pickled
    env behaves as the original)."""
    n = 2
    e1, e2 = _make(env_id, n), _make(env_id, n)
    e3 = pickle.loads(pickle.dumps(e1))     # EzPickle-style: the constructor call is replayed (backend factory included)
    nact = e1.single_action_space.shape[0]
    outs = [e.reset(seed=5) for e in (e1, e2, e3)]
    _same(outs[0][0], outs[1][0])
    _same(outs[0][0], outs[2][0])
    rng = np.random.default_rng(9)
    for t in range(4):
        a = torch.as_tensor(rng.uniform(-1, 1, (n, nact)).astype(np.float32))
        s1, s2, s3 = e1.step(a.clone()), e2.step(a.clone()), e3.step(a.clone())
        for x, y in ((s1, s2), (s1, s3)):
            _same(x[0], y[0])
            assert torch.equal(x[1], y[1]) and torch.equal(x[2], y[2]) and torch.equal(x[3], y[3])
            _same({k: v for k, v in x[4].items() if not k.startswith("solver")}, {k: v for k, v in y[4].items() if not k.startswith("solver")})
    # a different seed gives a different episode
    o4, _ = e2.reset(seed=6)
    o1, _ = e1.reset(seed=5)
    la, lb = dict(_leaves(o1)), dict(_leaves(o4))
    assert any(not torch.equal(la[k], lb[k]) for k in la)
    for e in (e1, e2, e3):
        e.close()


@pytest.mark.parametrize("env_id", ["FetchReach-v4", "FetchPush-v4", "FetchSlide-v4", "FetchPickAndPlace-v4", "HandReach-v3"])
def test_robot_env_reset_state(env_id):
    """tests/test_envs.py:175-231 `test_robot_env_reset`: after reset, qpos == initial_qpos (the object's xy, qpos[-7:-5], excluded for
    the tasks that draw it) and qvel == initial_qvel, for two seeds."""
    n = 3
    env = _make(env_id, n)
    sl = env._sl
    for seed in (24, 10):
        env.reset(seed=seed)
        st = env.backend.state
        qpos, qvel = st[:, sl["qpos"]].clone(), st[:, sl["qvel"]].clone()
        iq, iv = env.initial_qpos.clone().expand(n, -1), env.initial_qvel.clone().expand(n, -1)
        if any(t in env_id for t in ("FetchPush", "FetchPickAndPlace", "FetchSlide")):
            keep = [i for i in range(qpos.shape[1]) if i not in (qpos.shape[1] - 7, qpos.shape[1] - 6)]
            qpos, iq = qpos[:, keep], iq[:, keep]
        assert torch.equal(qpos, iq) and torch.equal(qvel, iv)
    env.close()
