"""FrankaKitchen-v1 vector env (gymnasium_robotics_b200/kitchen.py) on the kitchen-flavor host emulation of the kernel source
(-DB200_KITCHEN, WARP_W == 1) against the oracle env (oracle/kitchen_env.py): same seeds, same actions, observation /
reward / bookkeeping compared step by step.  The CUDA build of the same source is b200sim_kitchen.cu (GPU validation pending,
DESIGN.md section 7)."""
import numpy as np
import pytest
import torch

from gymnasium_robotics_b200.kitchen import KitchenVectorEnv
from gymnasium_robotics_b200.models import load_model
from oracle.kitchen_env import OracleKitchenEnv
from tests.hostsim_backend import HostSimBackend


class KitchenHostBackend(HostSimBackend):
    FLAVOR = "kitchen"


@pytest.fixture(scope="module")
def model():
    return load_model("franka_kitchen")


def _make(model, n, **kw):
    return KitchenVectorEnv(num_envs=n, backend_factory=KitchenHostBackend, device="cpu", rng_mode="numpy", model=model, **kw)


def test_reset_and_steps_track_the_oracle_env(model):
    n, seed = 2, 11
    env = _make(model, n)
    obs, info = env.reset(seed=seed)
    orcs = [OracleKitchenEnv(model) for _ in range(n)]
    oobs = [o.reset(seed=seed + i)[0] for i, o in enumerate(orcs)]
    assert obs["observation"].shape == (n, 59) and info["tasks_to_complete"].all()
    for i in range(n):
        assert np.abs(obs["observation"][i].numpy() - oobs[i]["observation"]).max() < 1e-5
    rng = np.random.default_rng(0)
    for k in range(4):
        a = rng.uniform(-1, 1, size=(n, 9))
        obs, rew, term, trunc, info = env.step(a)
        for i, o in enumerate(orcs):
            ob, r, te, tr, inf = o.step(a[i])
            e = np.abs(obs["observation"][i].numpy() - ob["observation"])
            assert e[:9].max() < 2e-4 and e[18:39].max() < 2e-4, (k, i, e.max())      # positions
            assert e[9:18].max() < 2e-2 and e[39:].max() < 2e-2, (k, i, e.max())      # velocities (fp32 vs fp64, 40 sub-steps)
            assert float(rew[i]) == r and bool(term[i]) == te
            for t in env.tasks:
                assert np.abs(obs["achieved_goal"][t][i].numpy() - ob["achieved_goal"][t]).max() < 2e-4
                assert np.allclose(obs["desired_goal"][t][i].numpy(), ob["desired_goal"][t])
            todo = {t for j, t in enumerate(env.tasks) if bool(info["tasks_to_complete"][i, j])}
            assert todo == set(inf["tasks_to_complete"])
    assert getattr(env.backend, "overflow_bits", 0) == 0


def test_task_bookkeeping_and_termination(model):
    """Put the microwave and the slide cabinet at their goals by editing qpos: both complete in the same step, are removed
    from `tasks_to_complete`, and the episode terminates once every listed task has been completed (kitchen_env.py:399-423)."""
    env = _make(model, 2, tasks_to_complete=["microwave", "slide cabinet"])
    env.reset(seed=3)
    q = env._sl["qpos"]
    env.backend.state[1, q.start + 22] = -0.75
    env.backend.state[1, q.start + 19] = 0.37
    obs, rew, term, trunc, info = env.step(np.zeros((2, 9)))
    assert rew.tolist() == [0.0, 2.0] and term.tolist() == [False, True] and not trunc.any()
    assert info["step_task_completions"].tolist() == [[False, False], [True, True]]
    assert info["tasks_to_complete"].tolist() == [[True, True], [False, False]]
    # NEXT_STEP autoreset: env 1 is reset on the following call, its bookkeeping starts over
    obs, rew, term, trunc, info = env.step(np.zeros((2, 9)))
    assert info["tasks_to_complete"].tolist() == [[True, True], [True, True]] and rew.tolist() == [0.0, 0.0] and not term.any()
    assert abs(float(obs["achieved_goal"]["microwave"][1, 0])) < 0.01


def test_time_limit_and_unknown_task(model):
    env = _make(model, 1, max_episode_steps=2, frame_skip=40)
    env.reset(seed=0)
    _, _, _, tr, _ = env.step(np.zeros((1, 9)))
    assert not tr.any()
    _, _, _, tr, _ = env.step(np.zeros((1, 9)))
    assert tr.all()
    with pytest.raises(ValueError):
        _make(model, 1, tasks_to_complete=["dishwasher"])


def test_same_step_autoreset_and_device_rng(model):
    """The configuration bench.py runs (same_step autoreset, device RNG): finished envs are reset inside the call, the
    returned observation is the reset one and `final_obs` carries the last observation of the finished episode."""
    env = KitchenVectorEnv(num_envs=3, backend_factory=KitchenHostBackend, device="cpu", rng_mode="torch", model=model,
                           autoreset_mode="same_step", max_episode_steps=2)
    obs, _ = env.reset(seed=5)
    a = torch.zeros((3, 9))
    obs, r, te, tr, info = env.step(a)
    assert not tr.any() and "final_obs" not in info
    obs, r, te, tr, info = env.step(a)
    assert tr.all() and info["_final_obs"].all() and info["final_obs"]["observation"].shape == (3, 59)
    assert (env._elapsed == 0).all() and torch.isfinite(obs["observation"]).all()
    # reset observation: INIT_QPOS plus noise
    assert float((obs["observation"][:, :9] - env.init_qpos[:9]).abs().max()) < 0.02
    obs, r, te, tr, info = env.step(a)
    assert not tr.any()
