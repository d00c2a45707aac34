"""GPU tests of the Franka-Kitchen kernel builds (csrc/b200sim_kitchen.cu: flat broad-phase scan; csrc/b200sim_kitchen_groups.cu:
two-level broad phase, the default), task kind 8.  They guard, among others, the out-of-bounds read of an empty eq_data override that once turned every env into NaN."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _backend(n):
    from gymnasium_robotics_b200.fetch import CudaBackend
    from gymnasium_robotics_b200.kitchen import make_kitchen_task
    from gymnasium_robotics_b200.models import load_model

    m = load_model("franka_kitchen")
    return m, CudaBackend(m, np.zeros((0, 11)), make_kitchen_task(m), n, "cuda:0")


from tests.parity_util import check_envelope

# stated envelope (p50, p99, max) of max |obs_gpu - obs_oracle| per (env, env-step) sample; measured on an H100 next to each limit
KITCHEN_ENVELOPE = {
    "kitchen/pos": (4e-6, 7e-6, 7e-6),      # 7.4e-7 / 1.3e-6 / 1.3e-6
    "kitchen/vel": (2.5e-5, 8e-5, 8e-5),    # 4.5e-6 / 1.6e-5 / 1.6e-5
    # mesh_collision="hull" (support-map narrow phase, csrc/b200sim_kitchen_hull.cu): free motion, then an arm link's hull on the kitchen
    "kitchen_hull/pos": (5e-6, 2.2e-5, 2.5e-5),     # 9.9e-7 / 5.2e-6 / 5.3e-6
    "kitchen_hull/vel": (9e-5, 3e-4, 4e-4),         # 1.8e-5 / 5.6e-5 / 7.2e-5  (the host emulation of the same source reaches 2.1e-4)
}


def test_kitchen_fixture_through_the_c_abi():
    """tests/golden/kitchen_quick.npz (fp32 host emulation of the same kernel source): refresh + 3 env-steps of 8 envs."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "kitchen_quick.npz"))
    state0, ctrls, exp = g["state0"], g["ctrls"], g["obs"]
    m, be = _backend(state0.shape[0])
    assert be.layout["stride"] == int(g["stride"])
    be.state.copy_(torch.as_tensor(state0))
    out = be.new_outputs()
    be.refresh(None, out)
    assert float((out["obs"].cpu() - torch.as_tensor(exp[0])).abs().max()) < 1e-5
    info = torch.zeros(state0.shape[0], dtype=torch.int32, device="cuda:0")
    pos_cols = list(range(9)) + list(range(18, 18 + m.nq - 9))
    for k in range(ctrls.shape[0]):
        be.step(torch.as_tensor(ctrls[k]).cuda().contiguous(), out, info)
        err = (out["obs"].cpu() - torch.as_tensor(exp[k + 1])).abs()
        assert float(err[:, pos_cols].max()) < 5e-4 and float(err.max()) < 5e-2
        assert int((info >> 16).max()) == 0      # no capacity overflow
    be.close()


def test_kitchen_env_tracks_the_oracle_env():
    from gymnasium_robotics_b200 import make_vec
    from oracle.kitchen_env import OracleKitchenEnv

    n, seed = 4, 21
    env = make_vec("FrankaKitchen-v1", num_envs=n, rng_mode="numpy")
    obs, info = env.reset(seed=seed)
    orcs = [OracleKitchenEnv(env.model) for _ in range(n)]
    for i, o in enumerate(orcs):
        ob, _ = o.reset(seed=seed + i)
        assert np.abs(obs["observation"][i].cpu().numpy() - ob["observation"]).max() < 1e-5
    rng = np.random.default_rng(2)
    pos_err, vel_err = [], []
    for k in range(4):
        a = rng.uniform(-1, 1, size=(n, 9))
        obs, rew, term, trunc, info = env.step(a)
        for i, o in enumerate(orcs):
            ob, r, te, tr, inf = o.step(a[i])
            e = np.abs(obs["observation"][i].cpu().numpy() - ob["observation"])
            pos_err.append(max(e[:9].max(), e[18:39].max()))      # robot qpos | object qpos
            vel_err.append(max(e[9:18].max(), e[39:].max()))      # robot qvel | object qvel
            assert float(rew[i]) == r and bool(term[i]) == te and bool(trunc[i]) == tr
    # free-running (the env is not re-injected: 4 env-steps x 40 sub-steps of accumulated fp32 / fp64 difference), every obs entry
    check_envelope("kitchen/pos", pos_err, *KITCHEN_ENVELOPE["kitchen/pos"])
    check_envelope("kitchen/vel", vel_err, *KITCHEN_ENVELOPE["kitchen/vel"])
    env.close()


def test_kitchen_groups_build_matches_the_flat_build():
    """The build with the two-level broad phase (csrc/b200sim_kitchen_groups.cu, broadphase="groups") against the validated flat
    build on the same states and actions: positions to 1e-4 (the contact numbering differs, not the candidate set), no overflow."""
    from gymnasium_robotics_b200 import make_vec

    def run(bp):
        env = make_vec("FrankaKitchen-v1", num_envs=16, rng_mode="numpy", robot_noise_ratio=0.0, object_noise_ratio=0.0,
                       broadphase=bp)
        env.reset(seed=5)
        rng = np.random.default_rng(1)
        obs = []
        for k in range(4):
            a = rng.uniform(-1, 1, size=(16, 9))
            if k >= 2:
                a[:, :7] = np.sign(a[:, :7])
            o, *_ = env.step(a)
            obs.append(o["observation"].cpu().clone())
        env.close()
        return torch.stack(obs)

    flat, groups = run("flat"), run("groups")
    assert torch.isfinite(groups).all()
    e = (flat - groups).abs()
    assert float(e[..., :9].max()) < 1e-4 and float(e[..., 18:39].max()) < 1e-4


def test_kitchen_timelimit_and_bookkeeping_on_gpu():
    """280-step TimeLimit from the kernel's flags (franka: max_episode_steps = 280, __init__.py:1117-1121), NEXT_STEP autoreset,
    finite observations under random actions, no capacity overflow in the first episode."""
    from gymnasium_robotics_b200 import make_vec

    n = 64
    env = make_vec("FrankaKitchen-v1", num_envs=n, rng_mode="torch", max_episode_steps=6)
    env.reset(seed=3)
    g = torch.Generator(device="cuda").manual_seed(9)
    for k in range(6):
        obs, rew, term, trunc, info = env.step(torch.rand((n, 9), generator=g, device="cuda") * 2 - 1)
        assert torch.isfinite(obs["observation"]).all()
        assert bool(trunc.all()) == (k == 5) and not bool(term.any())
    obs, rew, term, trunc, info = env.step(torch.zeros((n, 9), device="cuda"))    # the reset step of NEXT_STEP
    assert not bool(trunc.any()) and int(env._elapsed.max()) == 0
    assert float((obs["observation"][:, :9] - env.init_qpos[:9]).abs().max()) < 2e-3   # noisy initial robot pose
    assert int(env.backend.overflow_counter[0]) == 0
    env.close()


def test_kitchen_hull_build_tracks_the_oracle_env():
    """FrankaKitchen-v1 with mesh_collision="hull": the nine Franka collision meshes collide through their reduced convex hulls (kernels
    fetch_kernel_hull<W, 31>).  Env 0..2: random actions; env 3: the constant action that presses a link's hull onto the kitchen from
    env-step 7 on (tests/test_mesh_hull.py) -- the oracle env on the same hull model, same seeds and actions."""
    from gymnasium_robotics_b200 import make_vec
    from oracle.kitchen_env import OracleKitchenEnv

    n, seed = 4, 41
    env = make_vec("FrankaKitchen-v1", num_envs=n, rng_mode="numpy", mesh_collision="hull")
    assert int((np.asarray(env.model.geom_type) == 7).sum()) == 9
    obs, info = env.reset(seed=seed)
    orcs = [OracleKitchenEnv(env.model) for _ in range(n)]
    for i, o in enumerate(orcs):
        ob, _ = o.reset(seed=seed + i)
        assert np.abs(obs["observation"][i].cpu().numpy() - ob["observation"]).max() < 1e-5
    rng = np.random.default_rng(6)
    press = np.array([1.0, 1.0, 1.0, -1.0, -1.0, 1.0, -1.0, 0.0, 0.0])
    pos_err, vel_err, mesh_hits = [], [], 0
    for k in range(12):
        a = rng.uniform(-1, 1, size=(n, 9))
        a[3] = press
        obs, rew, term, trunc, info = env.step(a)
        for i, o in enumerate(orcs):
            ob, r, te, tr, inf = o.step(a[i])
            e = np.abs(obs["observation"][i].cpu().numpy() - ob["observation"])
            pos_err.append(max(e[:9].max(), e[18:39].max()))
            vel_err.append(max(e[9:18].max(), e[39:].max()))
            assert float(rew[i]) == r and bool(term[i]) == te and bool(trunc[i]) == tr
        gt = env.model.geom_type
        mesh_hits += int(any(gt[int(c["geom1"])] == 7 or (int(c["geom2"]) >= 0 and gt[int(c["geom2"])] == 7) for c in orcs[3].sim.contacts()))
    assert mesh_hits >= 3, "no hull geom in contact: the test would not exercise the hull narrow phase"
    check_envelope("kitchen_hull/pos", pos_err, *KITCHEN_ENVELOPE["kitchen_hull/pos"])
    check_envelope("kitchen_hull/vel", vel_err, *KITCHEN_ENVELOPE["kitchen_hull/vel"])
    env.close()
