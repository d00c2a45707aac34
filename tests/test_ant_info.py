"""AntMaze's Ant keywords and `ant_info=True` on the host emulation of the ant kernel build, against the fp64 oracle restatement
(tests/ant_info_oracle.py) from injected states, and the vector conventions of the new info keys."""
import functools
import pickle

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.maze import ANT_INFO_COLUMNS, MAPS
from tests.ant_info_oracle import OracleAntInfoEnv
from tests.hostsim_backend import HostSimBackend

V5_KEYS = set(ANT_INFO_COLUMNS)
V4_KEYS = (V5_KEYS - {"reward_contact"}) | {"forward_reward"}
# host emulation (fp32) vs oracle (fp64), one step from one injected state of a landed ant: the contact solve differs in the last
# bits and the ant's legs amplify that, so positions agree to ~2e-3 and the velocities (over dt = 0.05) to ~5e-2 (measured maxima
# 2e-3 / 4.8e-2 / contact cost 3e-3 over 18 env-steps; the envelopes are ~3x that).  The ctrl cost is the action's alone.
TOL = dict(x_position=6e-3, y_position=6e-3, distance_from_origin=1e-2, x_velocity=0.15, y_velocity=0.15, reward_forward=0.15,
           forward_reward=0.15, reward_ctrl=1e-5, reward_contact=1e-2, reward_survive=0.0)


class NoHooks(HostSimBackend):
    """A backend without the handle's optional hooks."""
    set_goal_update = set_goal_redraw = set_ant_info = set_obs_noise = None


def mk(env_id, n=3, **kw):
    return pkg.make_vec(env_id, num_envs=n, backend_factory=HostSimBackend, rng_mode="numpy", **kw)


def inject(env, oracles):
    lay = env.backend.layout
    rec = np.zeros((len(oracles), lay["stride"]))
    for i, o in enumerate(oracles):
        rec[i, lay["qpos"]:lay["qpos"] + 15] = o.sim.qpos
        rec[i, lay["qvel"]:lay["qvel"] + 14] = o.sim.qvel
        rec[i, lay["warm"]:lay["warm"] + 14] = o.sim.qacc_warmstart
        rec[i, lay["goal"]:lay["goal"] + 2] = o.goal
    env.set_state(torch.as_tensor(rec, dtype=torch.float32))
    for o in oracles:
        o.set_state(o.sim.qpos.copy(), o.sim.qvel.copy(), o.goal)


def settled_oracles(env, n, seed, **kw):
    oracles = [OracleAntInfoEnv(MAPS[env.maze_name], env.model, ant_version=env.ant.version,
                                include_cfrc_ext_in_observation=env.include_cfrc, **kw) for _ in range(n)]
    for i, o in enumerate(oracles):
        o.reset(seed=seed + i)
        for _ in range(10):     # the ant is dropped from z = 0.75: let it land, so that contacts and costs are not zero
            o.step(np.zeros(8))
    return oracles


@pytest.mark.parametrize("env_id,kw", [("AntMaze_Large-v5", {}), ("AntMaze_Large-v4", dict(use_contact_forces=True)),
                                       ("AntMaze_UMaze-v5", dict(contact_force_range=(-50.0, 50.0), ctrl_cost_weight=0.3,
                                                                 forward_reward_weight=2.0, healthy_z_range=(0.3, 0.9)))])
def test_every_key_matches_the_oracle(env_id, kw):
    n = 3
    env = mk(env_id, n, ant_info=True, **kw)
    env.reset(seed=4)
    oracles = settled_oracles(env, n, 4, **kw)
    keys = V5_KEYS if env.ant.version == 5 else V4_KEYS
    scale = dict(reward_forward=kw.get("forward_reward_weight", 1.0))
    tols = dict(TOL, reward_ctrl=TOL["reward_contact"]) if kw.get("use_contact_forces") else TOL   # Ant-v4: reward_ctrl = -contact_cost
    rng = np.random.default_rng(0)
    contact = 0.0
    for trial in range(6):
        inject(env, oracles)
        a = rng.uniform(-1, 1, (n, 8)).astype(np.float32)
        _, _, _, _, info = env.step(a)
        assert keys <= set(info) and all(info["_" + k].all() for k in keys)
        assert not (set(ANT_INFO_COLUMNS) | {"forward_reward"}) - keys & set(info)
        for i, orc in enumerate(oracles):
            _, _, _, _, oi = orc.step(a[i])
            for k in keys:
                want, got = float(oi[k]), float(info[k][i])
                tol = tols[k] * scale.get(k, 1.0) * (max(1.0, abs(want)) if k in ("reward_contact", "reward_ctrl") else 1.0)
                assert abs(got - want) <= tol, (k, i, got, want)
            contact = max(contact, abs(oi.get("reward_contact", oi["reward_ctrl"])))
    assert contact > 0     # the compared steps had contacts


def test_velocity_is_the_stale_torso_xpos():
    """x_velocity / y_velocity are the change of the torso's xpos of the last forward pass (the last RK4 stage), not of qpos: airborne
    ants (no contact, so the emulation follows the oracle to ~1e-5) with random velocities and actions, where the two differ by
    more than the tolerance."""
    n, tol = 3, 6e-5
    env = mk("AntMaze_Large-v5", n, ant_info=True)
    env.reset(seed=4)
    oracles = [OracleAntInfoEnv(MAPS["Large"], env.model, 5, True) for _ in range(n)]
    for i, o in enumerate(oracles):
        o.reset(seed=4 + i)
    rng = np.random.default_rng(1)
    apart = 0.0
    for trial in range(3):
        for o in oracles:
            o.sim.qvel[:] = rng.uniform(-3, 3, 14)
            o.sim.qpos[2] = 2.0
        inject(env, oracles)
        a = rng.uniform(-1, 1, (n, 8)).astype(np.float32)
        before = [o.sim.qpos[:2].copy() for o in oracles]
        _, _, _, _, info = env.step(a)
        for i, o in enumerate(oracles):
            _, _, _, _, oi = o.step(a[i])
            for k, c in (("x_velocity", 0), ("y_velocity", 1)):
                assert abs(float(info[k][i]) - oi[k]) <= tol, (k, float(info[k][i]), oi[k])
                apart = max(apart, abs((o.sim.qpos[c] - before[i][c]) / o.dt - oi[k]))
    assert apart > 2 * tol, apart


def test_reset_info_per_version():
    env = mk("AntMaze_Medium-v5", ant_info=True)
    obs, info = env.reset(seed=1)
    orcs = [OracleAntInfoEnv(MAPS["Medium"], env.model, 5, True) for _ in range(3)]
    for i, o in enumerate(orcs):
        _, oi = o.reset(seed=1 + i)
        for k in ("x_position", "y_position", "distance_from_origin"):
            assert abs(float(info[k][i]) - oi[k]) < 1e-5 and bool(info["_" + k][i])
    assert set(info) == {"success", "x_position", "y_position", "distance_from_origin", "_x_position", "_y_position", "_distance_from_origin"}
    _, info4 = mk("AntMaze_Medium-v4", ant_info=True).reset(seed=1)
    assert set(info4) == {"success"}


def test_contact_force_range_on_observation_and_cost():
    """contact_force_range replaces the +-1 clip of the (105,) observation and clips the contact cost's forces."""
    n = 2
    env = mk("AntMaze_UMaze-v5", n, contact_force_range=(-3.0, 3.0), ant_info=True)
    env.reset(seed=8)
    oracles = settled_oracles(env, n, 8, contact_force_range=(-3.0, 3.0))
    inject(env, oracles)
    o, _, _, _, info = env.step(np.zeros((n, 8), np.float32))
    seen = 0.0
    for i, orc in enumerate(oracles):
        oo, _, _, _, oi = orc.step(np.zeros(8))
        cf = o["observation"][i, 27:].double().numpy()
        assert np.abs(cf).max() <= 3.0
        np.testing.assert_allclose(cf, oo["observation"][27:], atol=5e-2)
        seen = max(seen, float(np.abs(cf).max()))
        assert abs(float(info["reward_contact"][i]) - oi["reward_contact"]) <= 2e-2 * max(1.0, abs(oi["reward_contact"]))
    assert seen > 1.0     # beyond the default range: the range reached the kernel


def test_v4_use_contact_forces_observation():
    env = mk("AntMaze_UMaze-v4", 2, use_contact_forces=True)
    assert env.single_observation_space["observation"].shape == (111,)
    env.reset(seed=3)
    for _ in range(25):      # dropped from z = 0.75, the ant has landed by now
        o, *_ = env.step(np.zeros((2, 8), np.float32))
    assert o["observation"].shape == (2, 111)
    assert float(o["observation"][:, 27:33].abs().max()) == 0.0      # cfrc_ext[0], the world row
    assert float(o["observation"][:, 33:].abs().max()) > 0.0
    assert mk("AntMaze_UMaze-v4", 2).single_observation_space["observation"].shape == (27,)


def test_frame_skip_10_is_two_frame_skip_5_steps():
    a = np.random.default_rng(5).uniform(-1, 1, (2, 8)).astype(np.float32)
    e10 = pkg.make_vec("AntMaze_UMaze-v5", num_envs=2, backend_factory=HostSimBackend, rng_mode="numpy", frame_skip=10)
    e5 = pkg.make_vec("AntMaze_UMaze-v5", num_envs=2, backend_factory=HostSimBackend, rng_mode="numpy")
    assert e10.dt == 2 * e5.dt and e10.backend.task.n_substeps == 10 and e10.metadata["render_fps"] == 10
    e10.reset(seed=2)
    e5.reset(seed=2)
    e10.step(a)
    e5.step(a)
    e5.step(a)
    assert torch.equal(e10.backend.state[:, :53], e5.backend.state[:, :53])
    with pytest.raises(ValueError):
        mk("AntMaze_UMaze-v5", frame_skip=0)


@pytest.mark.parametrize("env_id,kw,exc", [
    ("AntMaze_UMaze-v5", dict(reset_noise_scale=0.1), TypeError),
    ("AntMaze_UMaze-v4", dict(exclude_current_positions_from_observation=True), TypeError),
    ("AntMaze_UMaze-v4", dict(frame_skip=10), TypeError),
    ("AntMaze_UMaze-v4", dict(forward_reward_weight=2.0), TypeError),
    ("AntMaze_UMaze-v4", dict(main_body=1), TypeError),
    ("AntMaze_UMaze-v4", dict(include_cfrc_ext_in_observation=True), TypeError),
    ("AntMaze_UMaze-v4", dict(xml_file="ant.xml"), TypeError),
    ("AntMaze_UMaze-v5", dict(use_contact_forces=True), TypeError),
    ("AntMaze_UMaze-v5", dict(xml_file="ant.xml"), NotImplementedError),
    ("AntMaze_UMaze-v5", dict(main_body="leg"), NotImplementedError),
    ("AntMaze_UMaze-v5", dict(main_body=2), NotImplementedError),
])
def test_refusals(env_id, kw, exc):
    with pytest.raises(exc):
        mk(env_id, 1, **kw)


def test_main_body_torso_accepted():
    mk("AntMaze_UMaze-v5", 1, main_body="torso")
    mk("AntMaze_UMaze-v5", 1, main_body=1)


def _run_until_done(env, steps):
    rng = np.random.default_rng(0)
    out = []
    for _ in range(steps):
        out.append(env.step(rng.uniform(-1, 1, (env.num_envs, 8)).astype(np.float32)))
    return out


def test_next_step_convention():
    env = mk("AntMaze_UMaze-v5", 2, ant_info=True, max_episode_steps=2)
    env.reset(seed=0)
    res = _run_until_done(env, 3)
    info = res[2][4]     # the third call resets both envs (their episodes ended on the second) instead of stepping them
    for k in ANT_INFO_COLUMNS[3:]:
        assert not info["_" + k].any() and float(info[k].abs().max()) == 0.0
    obs = res[2][0]
    for k, c in (("x_position", 0), ("y_position", 1)):
        assert info["_" + k].all() and torch.equal(info[k], obs["achieved_goal"][:, c])
    assert info["_distance_from_origin"].all() and float(info["distance_from_origin"].abs().max()) == 0.0
    assert all(res[1][4]["_" + k].all() for k in ANT_INFO_COLUMNS)
    # the info of one step stays valid after the next
    assert float(res[1][4]["reward_survive"].min()) == 1.0


def test_same_step_and_disabled_conventions():
    env = mk("AntMaze_UMaze-v5", 2, ant_info=True, max_episode_steps=2, autoreset_mode="same_step")
    env.reset(seed=0)
    res = _run_until_done(env, 2)
    info = res[1][4]
    fi = info["final_info"]
    for k in ANT_INFO_COLUMNS:
        assert fi["_" + k].all() and k in fi
    assert float(fi["reward_survive"].min()) == 1.0 and float(fi["x_velocity"].abs().max()) > 0
    for k in ANT_INFO_COLUMNS[3:]:
        assert not info["_" + k].any()
    assert torch.equal(info["x_position"], res[1][0]["achieved_goal"][:, 0])      # the reset info of the new episodes
    env = mk("AntMaze_UMaze-v5", 2, ant_info=True, max_episode_steps=2, autoreset_mode="disabled")
    env.reset(seed=0)
    info = _run_until_done(env, 3)[2][4]
    assert all(info["_" + k].all() for k in ANT_INFO_COLUMNS) and "final_info" not in info


def test_pickle_round_trip():
    env = mk("AntMaze_UMaze-v4", 2, ant_info=True, use_contact_forces=True, healthy_reward=2.0)
    env2 = pickle.loads(pickle.dumps(env))
    assert env2.ant_info and env2.ant.version == 4 and env2.ant.kw["healthy_reward"] == 2.0
    assert env2.single_observation_space["observation"].shape == (111,)
    env2.reset(seed=0)
    _, _, _, _, info = env2.step(np.zeros((2, 8), np.float32))
    assert "forward_reward" in info and "reward_contact" not in info


@pytest.mark.parametrize("env_id", ["AntMaze_UMaze-v5", "AntMaze_UMaze-v4"])
def test_ant_info_off_keeps_todays_keys(env_id):
    env = pkg.make_vec(env_id, num_envs=2, backend_factory=HostSimBackend, rng_mode="numpy")
    _, info = env.reset(seed=0)
    assert set(info) == {"success"}
    _, _, _, _, info = env.step(np.zeros((2, 8), np.float32))
    assert set(info) == {"success", "solver_info"}
    assert env.backend.task.touch_mode == (1 if env_id.endswith("v5") else 0)


def test_set_ant_info_refused_on_plain_build():
    env = pkg.make_vec("AntMaze_UMaze-v5", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.backend.task.touch_mode == 1
    with pytest.raises(RuntimeError):
        env.backend.set_ant_info(env.ant.params(), None, None)
    with pytest.raises(NotImplementedError):
        pkg.make_vec("AntMaze_UMaze-v5", num_envs=1, backend_factory=functools.partial(NoHooks, flavor=False), rng_mode="numpy", ant_info=True)
