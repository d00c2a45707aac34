"""The AntMaze_*-v3 ids on the host emulation: envs/maze/maze.py's task logic on Gymnasium's Ant-v4 (ant_maze_v3.py).

  * registry, observation shapes, refusals, pickling and seeded determinism;
  * the start draw: farther than 0.5 from the goal (not half a cell) in the numpy mode, against the restatement on the same PCG64
    streams, and in the host build of csrc/reset_sample.cuh (b200sim_maze_reset_t.separation) against a Python Philox restatement;
  * the goal redraw inside the step (maze.py:283-302): one candidate, the reward of the new goal, the old goal in the observation --
    in rng_mode="device" (b200sim_set_goal_redraw, emulated), "numpy" (against the v3 oracle env) and "torch";
  * the Ant-v4 info with no `success` key, {} at reset, under the three autoreset modes."""
import ctypes
import pickle

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200._lib import MazeResetC
from gymnasium_robotics_b200.maze import MAPS, NOISE, SUCCESS_RADIUS, MazeCells, MazeVectorEnv
from tests import hostsim
from tests.antmaze_v3_oracle import MazeResetLogicV3, OracleAntMazeV3Env
from tests.hostsim import goal_redraw
from tests.hostsim_backend import HostSimBackend
from tests.test_ant_info import V4_KEYS
from tests.test_reset_device import M32, philox4x32_10, py_maze_draw, u01

f32 = np.float32
V3_IDS = [f"AntMaze_{m}{s}-v3" for m in ("UMaze", "Open", "Open_Diverse_G", "Open_Diverse_GR", "Medium", "Medium_Diverse_G",
                                          "Medium_Diverse_GR", "Large", "Large_Diverse_G", "Large_Diverse_GR") for s in ("", "Dense")]
STEP_KEYS = V4_KEYS | {"_" + k for k in V4_KEYS} | {"solver_info"}


def mk(env_id="AntMaze_Large-v3", n=3, **kw):
    kw.setdefault("rng_mode", "numpy")
    return pkg.make_vec(env_id, num_envs=n, backend_factory=HostSimBackend, **kw)


def _goals(env):
    return env.backend.state[:, env._sl["goal"]].clone()


def _place(env, xy):
    """Every ant to xy [N, 2] (float32), at rest, keeping the step counters."""
    st, el = env.get_state()
    q = env._sl["qpos"].start
    st[:, q:q + 2] = torch.as_tensor(np.asarray(xy, dtype=f32))
    st[:, env._sl["qvel"]] = 0
    return env.set_state(st, el)


def _toward_centre(env, goal):
    """An offset of 0.6 per axis from `goal` toward its cell's centre: 0.85 off the goal, outside the success radius, and the ant's
    legs stay clear of the walls."""
    centre = env.cells.cell_rowcol_to_xy(env.cells.cell_xy_to_rowcol(goal))
    return -0.6 * np.sign(goal - centre)


def _zeros(env):
    return np.zeros((env.num_envs, 8), dtype=f32)


# ---------------------------------------------------------------------------------------------- registry and constructor
def test_registry_and_every_id_builds():
    assert len(V3_IDS) == 20 and len(pkg.ENV_IDS) == 165
    assert pkg.ENV_IDS["AntMaze_Large-v3"] == dict(maze="Large", reward_type="sparse", max_episode_steps=1000, maze_version=3)
    for env_id in V3_IDS:
        env = mk(env_id, n=1)
        assert env.max_episode_steps == pkg.ENV_IDS[env_id.replace("-v3", "-v4")]["max_episode_steps"]
        assert env.ant.version == 4 and env.ant_info and env.reward_type == ("dense" if "Dense" in env_id else "sparse")
        obs, info = env.reset(seed=1)
        assert obs["observation"].shape == (1, 27) and info == {}
        o, r, te, tr, info = env.step(_zeros(env))
        assert set(info) == STEP_KEYS, env_id
        env.close()
    env = mk("AntMaze_UMaze-v3", n=1, use_contact_forces=True)
    obs, _ = env.reset(seed=0)
    assert obs["observation"].shape == (1, 111) and env.single_observation_space["observation"].shape == (111,)
    env.close()
    # ant_info is honoured when given; -v4 / -v5 keep it off by default
    env = mk("AntMaze_UMaze-v3", n=1, ant_info=False)
    env.reset(seed=0)
    assert set(env.step(_zeros(env))[4]) == {"solver_info"}
    env.close()
    assert not pkg.make_vec("AntMaze_UMaze-v4", num_envs=1, backend_factory=HostSimBackend).ant_info


@pytest.mark.parametrize("kw,exc", [(dict(reset_target=True), TypeError), (dict(reset_target=False), TypeError),
                                    (dict(forward_reward_weight=2.0), TypeError), (dict(main_body=1), TypeError),
                                    (dict(include_cfrc_ext_in_observation=True), TypeError), (dict(reset_noise_scale=0.1), TypeError),
                                    (dict(xml_file="ant.xml"), TypeError), (dict(frame_skip=10), TypeError)])
def test_refused_keywords(kw, exc):
    with pytest.raises(exc):
        mk("AntMaze_UMaze-v3", n=1, **kw)


def test_v3_is_the_ant_agents_and_v4_stays_the_default():
    with pytest.raises(ValueError):
        MazeVectorEnv("UMaze", agent="point", maze_version=3, backend_factory=HostSimBackend)
    with pytest.raises(ValueError):
        MazeVectorEnv("UMaze", maze_version=5, backend_factory=HostSimBackend)
    with pytest.raises(ValueError):
        MazeVectorEnv("UMaze", maze_version=3, ant_version=5, backend_factory=HostSimBackend)
    env = mk("AntMaze_UMaze-v4", n=1)
    assert env.maze_version == 4 and env.separation == 2.0 and not env.ant_info
    env.close()


def test_keywords_pickling_and_seeded_determinism():
    env = mk("AntMaze_MediumDense-v3", n=2, ctrl_cost_weight=0.1, healthy_reward=2.0, continuing_task=False)
    assert env.ant.kw["ctrl_cost_weight"] == 0.1 and not env.continuing_task
    clone = pickle.loads(pickle.dumps(env))
    runs = []
    for e in (env, clone):
        obs, _ = e.reset(seed=7)
        seq = [obs["observation"].clone()]
        for k in range(3):
            o, r, *_ = e.step(np.full((2, 8), 0.1 * k, dtype=f32))
            seq += [o["observation"].clone(), r.clone()]
        runs.append(seq)
        e.close()
    assert all(torch.equal(a, b) for a, b in zip(*runs))


@pytest.mark.parametrize("layout", [[[1, 1, 1, 1, 1], [1, "g", 0, "g", 1], [1, 1, 1, 1, 1]],
                                    [[1, 1, 1, 1, 1], [1, "r", 0, 0, 1], [1, 1, 1, 1, 1]]])
def test_layouts_without_reset_or_goal_cells_are_refused(layout):
    """v4 falls back to the empty cells (maze_v4.py:223-230); v3 has no fallback, so the reference cannot draw from such a layout."""
    with pytest.raises(ValueError, match="no (reset|goal) location"):
        mk("AntMaze_UMaze-v3", n=1, maze_map=layout)
    mk("AntMaze_UMaze-v4", n=1, maze_map=layout).close()
    env = mk("AntMaze_UMaze-v3", n=1, maze_map=[[1, 1, 1, 1], [1, 0, 0, 1], [1, 1, 1, 1]])   # unlabelled: every free cell, as in v3
    assert len(env.cells.goal_locations) == len(env.cells.reset_locations) == 2
    env.close()


# ---------------------------------------------------------------------------------------------- the start draw
def test_numpy_resets_match_the_restatement_and_can_start_in_the_goal_cell():
    n, in_goal_cell = 8, 0
    env = mk("AntMaze_Open-v3", n=n)
    for seed in range(0, 120, n):
        obs, _ = env.reset(seed=seed)
        st, _ = env.get_state()
        for i in range(n):
            logic = MazeResetLogicV3(MAPS["Open"], maze_size_scaling=4.0)
            goal, pos = logic.reset(seed=seed + i)
            assert np.array_equal(obs["desired_goal"][i].numpy(), goal.astype(f32))
            assert np.array_equal(st[i, :2].numpy(), pos.astype(f32))
            cell = env.cells.cell_xy_to_rowcol
            in_goal_cell += int(np.array_equal(cell(goal), cell(pos)))
    assert in_goal_cell >= 3          # the v4 draw never starts in the goal's cell (half a cell apart, cell centres 4 apart)
    env.close()


def _c_maze_draw(goal_xy, reset_xy, scaling, separation, seed, env, episode):
    L = hostsim.lib()
    p = MazeResetC()
    p.n_goal, p.n_reset, p.scaling, p.noise, p.separation = len(goal_xy), len(reset_xy), scaling, NOISE, separation
    g, r = np.ascontiguousarray(goal_xy, dtype=f32), np.ascontiguousarray(reset_xy, dtype=f32)
    rest, rec = np.zeros(8, dtype=f32), np.zeros(8, dtype=f32)
    L.hostsim_maze_reset_record(ctypes.byref(p), g.ctypes.data, r.ctypes.data, seed, env, episode, rest.ctypes.data, 8, 0, 4, rec.ctypes.data)
    return rec[4:6].copy(), rec[0:2].copy()


def py_maze_draw_sep(goal_xy, reset_xy, scaling, noise, separation, seed, env, episode):
    """rs_maze_reset_draw on the generator's numbers with an explicit start separation (float32 like the kernel)."""
    key = (seed & M32, (seed >> 32) & M32)
    amp = f32(noise) * f32(scaling)
    r = philox4x32_10((env, episode, 0, 0x3A2E), key)
    gi = (r[0] * len(goal_xy)) >> 32
    goal = np.array([goal_xy[gi][0] + (f32(2) * u01(r[1]) - f32(1)) * amp, goal_xy[gi][1] + (f32(2) * u01(r[2]) - f32(1)) * amp], dtype=f32)
    pos = goal.copy()
    for b in range(1, 33):
        r = philox4x32_10((env, episode, b, 0x3A2E), key)
        hit = [np.array(reset_xy[(w * len(reset_xy)) >> 32], dtype=f32) for w in r]
        ok = [p for p in hit if not np.sqrt((p[0] - goal[0]) ** 2 + (p[1] - goal[1]) ** 2) <= f32(separation)]
        if ok:
            pos = ok[0]
            break
        pos = hit[-1]
    r = philox4x32_10((env, episode, 33, 0x3A2E), key)
    return goal, np.array([pos[0] + (f32(2) * u01(r[0]) - f32(1)) * amp, pos[1] + (f32(2) * u01(r[1]) - f32(1)) * amp], dtype=f32)


def test_host_reset_draw_with_separation_known_answers():
    c = MazeCells(MAPS["Open"], 4.0)
    gl, rl = c.goal_locations.astype(f32), c.reset_locations.astype(f32)
    rng = np.random.default_rng(5)
    keys = [(0, 0, 0), (2 ** 64 - 1, 2 ** 31 - 1, 2 ** 32 - 1)] + [tuple(int(x) for x in rng.integers(0, 2 ** 32, 3)) for _ in range(60)]
    same_cell = 0
    for seed, env, ep in keys:
        got = _c_maze_draw(gl, rl, 4.0, 0.5, seed, env, ep)
        want = py_maze_draw_sep(gl, rl, 4.0, NOISE, 0.5, seed, env, ep)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (seed, env, ep)
        # separation 0 is v4's half cell, bit for bit
        v4 = _c_maze_draw(gl, rl, 4.0, 0.0, seed, env, ep)
        w4 = py_maze_draw(gl, rl, 4.0, NOISE, seed, env, ep)
        assert np.array_equal(v4[0], w4[0]) and np.array_equal(v4[1], w4[1])
        same_cell += int(np.array_equal(c.cell_xy_to_rowcol(got[0]), c.cell_xy_to_rowcol(got[1])))
    assert same_cell >= 1


def test_device_mode_resets_use_the_v3_separation():
    env = mk("AntMaze_Open-v3", n=16, rng_mode="device")
    obs, _ = env.reset(seed=3)
    st, _ = env.get_state()
    gl, rl = env._goal_loc.numpy(), env._reset_loc.numpy()
    for i in range(16):
        g, p = py_maze_draw_sep(gl, rl, 4.0, NOISE, 0.5, 3, i, 0)
        assert np.array_equal(obs["desired_goal"][i].numpy(), g) and np.array_equal(st[i, :2].numpy(), p)
    env.close()


# ---------------------------------------------------------------------------------------------- the redraw
def py_redraw(goal_xy, scaling, seed, env, episode, step):
    """Candidate 0 of rs_maze_goal_update (counter (env, episode, step, 0x60A1)), each product and sum rounded to float32."""
    r = philox4x32_10((int(env), int(episode), int(step), 0x60A1), (seed & M32, (seed >> 32) & M32))
    gi = (r[0] * len(goal_xy)) >> 32
    amp = f32(NOISE) * f32(scaling)
    return np.array([f32(goal_xy[gi][0]) + (f32(2) * u01(r[1]) - f32(1)) * amp,
                     f32(goal_xy[gi][1]) + (f32(2) * u01(r[2]) - f32(1)) * amp], dtype=f32)


def test_redraw_draws_exactly_one_candidate_even_within_the_radius():
    two = np.array([[0.0, 0.0], [4.0, 0.0]], dtype=f32)
    kept_inside = 0
    for step in range(400):
        for dense in (0, 1):
            new, r = goal_redraw(two, 4.0, NOISE, SUCCESS_RADIUS, dense, 99, 5, 1, step, [0.0, 0.0], [0.1, 0.0])
            assert np.array_equal(new, py_redraw(two, 4.0, 99, 5, 1, step)) and r is not None
            d = np.sqrt(f32(new[0] * new[0]) + f32(new[1] * new[1]))
            assert r == (np.exp(-d) if dense else f32(d <= f32(SUCCESS_RADIUS))) or dense
            kept_inside += int(d <= SUCCESS_RADIUS and not dense)
    assert kept_inside >= 2          # candidates within 0.45 are kept: v3 has no rejection loop
    new, r = goal_redraw(two, 4.0, NOISE, SUCCESS_RADIUS, 0, 99, 5, 1, 0, [0.0, 0.0], [0.46, 0.0])
    assert r is None and np.array_equal(new, f32([0.46, 0.0]))


@pytest.mark.parametrize("reward_type", ["sparse", "dense"])
def test_device_mode_redraw_rewrites_the_reward(reward_type):
    n, seed = 6, 11
    env = mk("AntMaze_Large-v3" if reward_type == "sparse" else "AntMaze_LargeDense-v3", n=n, rng_mode="device")
    env.reset(seed=seed)
    for step in range(1, 3):
        g0 = _goals(env).numpy()
        _place(env, g0 + np.array([[0.0, 0.0] if i % 2 == 0 else _toward_centre(env, g0[i]) for i in range(n)], dtype=f32))   # odd: off goal
        o, r, te, tr, info = env.step(_zeros(env))
        new, ach = _goals(env).numpy(), o["achieved_goal"].numpy()
        assert "success" not in info and set(info) == STEP_KEYS
        assert np.array_equal(o["desired_goal"].numpy(), g0)            # the observation was copied before the redraw
        for i in range(n):
            if i % 2:
                assert np.array_equal(new[i], g0[i])
                continue
            assert np.array_equal(new[i], py_redraw(env._goal_loc.numpy(), 4.0, seed, i, 1, step)), (step, i)
        want = env.compute_reward(o["achieved_goal"], _goals(env))
        assert torch.equal(r, want)                                        # the reward of the new goal, bit for bit
        assert not te.any()
    env.close()


def test_torch_mode_redraw_applies_one_candidate_where_the_success_column_is_1():
    n = 6
    env = mk("AntMaze_LargeDense-v3", n=n, rng_mode="torch")
    env.reset(seed=4)
    g0 = _goals(env).numpy()
    _place(env, g0 + np.array([[0.0, 0.0] if i % 2 == 0 else _toward_centre(env, g0[i]) for i in range(n)], dtype=f32))
    o, r, te, tr, info = env.step(_zeros(env))
    new = _goals(env).numpy()
    moved = (new != g0).any(axis=1)
    assert moved.tolist() == [True, False] * (n // 2)
    assert (np.abs(env.cells.goal_locations[None] - new[:, None]).max(axis=2) <= NOISE * 4.0 + 1e-5).any(axis=1).all()
    assert np.array_equal(o["desired_goal"].numpy(), g0)
    assert torch.equal(r, env.compute_reward(o["achieved_goal"], _goals(env)))
    env.close()


def test_no_redraw_in_an_episodic_task_or_with_one_goal_location():
    for kw in (dict(continuing_task=False), dict(maze_map=[[1, 1, 1, 1, 1], [1, "g", 0, "r", 1], [1, 1, 1, 1, 1]])):
        env = mk("AntMaze_UMaze-v3", n=2, rng_mode="device", **kw)
        env.reset(seed=2)
        assert env.backend.goal_args is None
        g0 = _goals(env)
        _place(env, g0.numpy())
        o, r, te, tr, info = env.step(_zeros(env))
        assert torch.equal(_goals(env), g0)
        assert te.all() == (not env.continuing_task)
        env.close()


# ---------------------------------------------------------------------------------------------- the numpy mode against the oracle
@pytest.mark.parametrize("mode", ["next_step", "same_step", "disabled"])
def test_numpy_mode_tracks_the_v3_oracle(mode):
    """Three envs over two 3-step episodes; envs 0 and 2 sit on their goals before every step, so goals are redrawn; the oracles
    take the same states.  Observation, reward, terminated and the info keys; the finished episodes' Ant keys in final_info."""
    n, seed, reward_type = 3, 14, "sparse"
    env = mk("AntMaze_Medium-v3", n=n, autoreset_mode=mode, max_episode_steps=3)
    obs, info = env.reset(seed=seed)
    assert info == {}
    oracles = [OracleAntMazeV3Env(MAPS["Medium"], env.model, reward_type=reward_type) for _ in range(n)]
    for i, o in enumerate(oracles):
        oo, oi = o.reset(seed=seed + i)
        assert oi == {} and np.array_equal(obs["desired_goal"][i].numpy(), oo["desired_goal"].astype(f32))
    redraws, t = 0, 0
    for step in range(7):
        if mode == "disabled" and t == 3:
            obs, info = env.reset()
            assert info == {}
            for i, o in enumerate(oracles):
                oo, _ = o.reset()
                assert np.array_equal(obs["desired_goal"][i].numpy(), oo["desired_goal"].astype(f32))
            t = 0
        if mode == "next_step" and t == 3:       # this call resets instead of stepping
            o_, r, te, tr, info = env.step(_zeros(env))
            for i, o in enumerate(oracles):
                oo, _ = o.reset()
                assert np.array_equal(o_["desired_goal"][i].numpy(), oo["desired_goal"].astype(f32))
                np.testing.assert_allclose(o_["achieved_goal"][i].numpy(), oo["achieved_goal"], atol=1e-5)
            assert not r.any() and not info["_x_position"].any()
            t = 0
            continue
        g = _goals(env).numpy()
        _place(env, g + np.array([[0.0, 0.0], _toward_centre(env, g[1]), [0.05, -0.05]], dtype=f32))
        st = env.backend.state.numpy()
        for i, o in enumerate(oracles):
            o.set_state(st[i, env._sl["qpos"]].astype(np.float64), st[i, env._sl["qvel"]].astype(np.float64), o.goal)
        o_, r, te, tr, info = env.step(_zeros(env))
        t += 1
        assert "success" not in info and set(V4_KEYS) <= set(info)
        for i, o in enumerate(oracles):
            before = o.goal.copy()
            oo, orr, ote, otr, oi = o.step(np.zeros(8))
            assert "success" not in oi and set(oi) == set(V4_KEYS)
            fin = info["final_obs"] if mode == "same_step" and t == 3 else o_
            assert np.array_equal(fin["desired_goal"][i].numpy(), oo["desired_goal"].astype(f32))
            np.testing.assert_allclose(fin["observation"][i].numpy(), oo["observation"], atol=5e-3, err_msg=f"{step} {t} {i}")
            assert float(r[i]) == orr and bool(te[i]) == ote
            for k in ("x_position", "y_position"):
                src = info["final_info"] if mode == "same_step" and t == 3 else info
                assert abs(float(src[k][i]) - oi[k]) < 6e-3
            if not (mode == "same_step" and t == 3):
                assert np.array_equal(_goals(env)[i].numpy(), o.goal.astype(f32)), (step, i)
            redraws += int(not np.array_equal(before, o.goal))
        if mode == "same_step" and t == 3:
            assert set(info["final_info"]) == STEP_KEYS - {"solver_info"}
            assert bool(tr.all())
            for i, o in enumerate(oracles):
                oo, _ = o.reset()
                assert np.array_equal(o_["desired_goal"][i].numpy(), oo["desired_goal"].astype(f32))
            t = 0
    assert redraws >= 6
    env.close()
