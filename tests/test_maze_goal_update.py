"""The goal update of continuing maze tasks (`reset_target=True`, maze_v4.py:400-418 update_goal) on the host emulation.

In rng_mode="device" the step launch redraws the goal of every env that succeeded (b200sim_set_goal_update, csrc/reset_sample.cuh
rs_maze_goal_update): Philox4x32-10 over (seed; global env index, episode, step after the step, 0x60A1 | candidate << 16), bit for
bit the restatement below.  The numpy mode keeps the reference's per-env streams and order, value-equal to the oracle env with
update_goal; the torch mode draws from the same streams."""
import numpy as np
import pytest
import torch
from scipy import stats

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.maze import NOISE, SUCCESS_RADIUS
from oracle.ant_maze_env import OracleAntMazeEnv
from oracle.maze import MazeResetLogic
from oracle.point_maze_env import OraclePointMazeEnv
from tests.hostsim import maze_goal
from tests.hostsim.maze_goal import GoalUpdateHostBackend
from tests.hostsim_backend import HostSimBackend
from tests.test_reset_device import M32, philox4x32_10, py_maze_draw, u01

TAG, CANDIDATES = 0x60A1, 64
f32 = np.float32


def _dist_host(ach, goal):
    """antmaze_observe's distance as the host build rounds it: round(dx^2) + round(dy^2), then sqrt."""
    dx, dy = f32(ach[0]) - f32(goal[0]), f32(ach[1]) - f32(goal[1])
    return np.sqrt(f32(dx * dx) + f32(dy * dy))


def _dist_device(ach, goal):
    """The device branch: sqrtf(fmaf(dy, dy, round(dx^2))).  The fused sum is formed in float64 (dy^2 is exact there) and rounded to
    float32; the two roundings differ from one only when the float64 sum lands on a float32 tie.  (The device's sqrtf is the fast
    approximation: a candidate within an ulp of the radius could be decided the other way.)"""
    dx, dy = f32(ach[0]) - f32(goal[0]), f32(ach[1]) - f32(goal[1])
    return np.sqrt(f32(float(dy) * float(dy) + float(f32(dx * dx))))


def py_goal_update(goal_xy, scaling, noise, radius, seed, env, episode, step, ach, goal, dist=_dist_host):
    """update_goal (maze_v4.py:400-418) on the generator's numbers: (new goal float32 [2], candidates drawn)."""
    goal = np.asarray(goal, dtype=f32).copy()
    if not dist(ach, goal) <= f32(radius):
        return goal, 0
    seed = int(seed)
    key = (seed & M32, (seed >> 32) & M32)
    amp = f32(noise) * f32(scaling)
    for c in range(CANDIDATES):
        r = philox4x32_10((int(env), int(episode), int(step), TAG | c << 16), key)
        gi = (r[0] * len(goal_xy)) >> 32
        goal = np.array([f32(goal_xy[gi][0]) + (f32(2) * u01(r[1]) - f32(1)) * amp,
                         f32(goal_xy[gi][1]) + (f32(2) * u01(r[2]) - f32(1)) * amp], dtype=f32)
        if not dist(ach, goal) <= f32(radius):
            break
    return goal, c + 1


# ---------------------------------------------------------------------------------------------- the oracle with update_goal
def oracle_update_goal(logic: MazeResetLogic, achieved_goal, goal, continuing_task=True, reset_target=True):
    """MazeEnv.update_goal (maze_v4.py:400-418) on the oracle's reset logic: its np_random, the reference's draw order."""
    if (continuing_task and reset_target and bool(np.linalg.norm(achieved_goal - goal) <= 0.45)
            and len(logic.maze.unique_goal_locations) > 1):
        while np.linalg.norm(achieved_goal - goal) <= 0.45:
            goal = logic.add_xy_position_noise(logic.generate_target_goal())
    return goal


class _UpdateGoal:
    """step() then update_goal, as AntMazeEnv.step (ant_maze_v5.py:295-310) and PointMazeEnv.step (point_maze.py:389-404) do: the
    returned observation carries the old goal."""

    def step(self, action):
        res = super().step(action)
        self.goal = oracle_update_goal(self.logic, res[0]["achieved_goal"], self.goal, self.continuing_task, self.reset_target)
        return res


class GoalOracleAntMaze(_UpdateGoal, OracleAntMazeEnv):
    pass


class GoalOraclePointMaze(_UpdateGoal, OraclePointMazeEnv):
    def __init__(self, maze_map, model, reward_type="sparse", continuing_task=True, reset_target=False):
        super().__init__(maze_map, model, reward_type, continuing_task)
        self.reset_target = reset_target


# ---------------------------------------------------------------------------------------------- helpers
def _make(env_id="PointMaze_Large-v3", n=4, backend=GoalUpdateHostBackend, **kw):
    kw.setdefault("rng_mode", "device")
    kw.setdefault("reset_target", True)
    return pkg.make_vec(env_id, num_envs=n, backend_factory=backend, **kw)


def _goals(env):
    return env.backend.state[:, env._sl["goal"]].clone()


def _place(env, xy):
    """Put every env's agent at xy [N, 2] (float32), at rest, keeping the step counters; returns the refreshed observation."""
    st, el = env.get_state()
    q = env._sl["qpos"].start
    st[:, q:q + 2] = torch.as_tensor(np.asarray(xy, dtype=np.float32))
    st[:, env._sl["qvel"]] = 0
    return env.set_state(st, el)


def _zeros(env):
    return np.zeros((env.num_envs, env.single_action_space.shape[0]), dtype=np.float32)


def _in_noise_box(env, g):
    return bool((np.abs(env.cells.goal_locations - np.asarray(g, dtype=np.float64)).max(axis=1) <= NOISE * env.scaling + 1e-6).any())


# ---------------------------------------------------------------------------------------------- the draw
def test_known_answers_and_edge_keys():
    goal_xy = np.array([[0.5, 1.5], [2.5, -1.5], [-3.5, 0.5], [1.5, 1.5], [-0.5, -2.5]], dtype=f32)
    keys = [(0, 0, 0, 1), (7, 3, 1, 5), (2 ** 64 - 1, 1 << 20, 12345, 2 ** 31 - 1), (2 ** 63 + 11, 2 ** 32 - 1, 2 ** 32 - 1, 2 ** 32 - 1),
            (123456789, 1 << 20, 999, 1000000)]
    rng = np.random.default_rng(4)
    for seed, env, ep, step in keys + [tuple(int(x) for x in rng.integers(0, 2 ** 32, 4)) for _ in range(40)]:
        for scaling in (1.0, 4.0):
            for ach in ([0.5, 1.5], [0.7, 1.6], [10.0, 10.0]):
                goal = np.asarray(ach, dtype=f32) + f32(0.2)
                want = py_goal_update(goal_xy * f32(scaling), scaling, NOISE, SUCCESS_RADIUS, seed, env, ep, step, ach, goal)
                got = maze_goal.goal_update(goal_xy * f32(scaling), scaling, NOISE, SUCCESS_RADIUS, seed, env, ep, step, ach, goal)
                assert got[1] == want[1] >= 1 and np.array_equal(got[0], want[0]), (seed, env, ep, step, scaling, ach)
    # no update when the achieved position is outside the radius
    g, n = maze_goal.goal_update(goal_xy, 1.0, NOISE, SUCCESS_RADIUS, 1, 2, 3, 4, [0.0, 0.0], [0.46, 0.0])
    assert n == 0 and np.array_equal(g, f32([0.46, 0.0]))
    # a key whose first candidates are rejected: the agent sits on one of two goal cells (scaling 1: its noise box lies in the disc)
    two = np.array([[0.0, 0.0], [3.0, 0.0]], dtype=f32)
    found = 0
    for step in range(200):
        want = py_goal_update(two, 1.0, NOISE, SUCCESS_RADIUS, 99, 5, 1, step, [0.0, 0.0], [0.0, 0.0])
        got = maze_goal.goal_update(two, 1.0, NOISE, SUCCESS_RADIUS, 99, 5, 1, step, [0.0, 0.0], [0.0, 0.0])
        assert got[1] == want[1] and np.array_equal(got[0], want[0])
        assert abs(float(got[0][0]) - 3.0) <= 0.25 and _dist_host([0, 0], got[0]) > f32(SUCCESS_RADIUS)
        found = max(found, got[1])
    assert found >= 4


def test_candidates_are_uniform_over_cells_and_noise():
    """Candidate 0 of many keys (the agent far from every cell, so it is accepted): chi-square on the cell index, KS on the noise."""
    goal_xy = np.array([[4.0 * k, 0.0] for k in range(7)], dtype=f32)
    far = [-100.0, -100.0]
    cells, noise = [], []
    for k in range(14000):
        g, n = maze_goal.goal_update(goal_xy, 4.0, NOISE, SUCCESS_RADIUS, 2024, k % 500, k // 500, 17, far, far)
        assert n == 1
        c = int(np.rint(g[0] / 4.0))
        cells.append(c)
        noise.extend([(float(g[0]) - 4.0 * c) / (NOISE * 4.0), float(g[1]) / (NOISE * 4.0)])
    counts = np.bincount(cells, minlength=7)
    assert stats.chisquare(counts).pvalue > 1e-3
    assert stats.kstest(noise, stats.uniform(loc=-1, scale=2).cdf).pvalue > 1e-3
    assert min(noise) >= -1 and max(noise) < 1


# ---------------------------------------------------------------------------------------------- the env in rng_mode="device"
def test_update_fires_exactly_when_success_and_draws_the_restated_goal():
    n, seed = 8, 11
    env = _make(n=n)
    obs, _ = env.reset(seed=seed)
    g0 = obs["desired_goal"].numpy().copy()
    # inside, outside, and within a few ulp of the radius on either side
    off = [0.0, 0.3, 1.0, 2.0, 0.45, 0.45, 0.45, 0.45]
    ulps = [0, 0, 0, 0, -2, -1, 1, 2]
    xy = g0.copy()
    for i in range(n):
        x = f32(g0[i, 0] + off[i])
        for _ in range(abs(ulps[i])):
            x = np.nextafter(x, f32(np.inf) if ulps[i] > 0 else f32(-np.inf))
        xy[i, 0] = x
    _place(env, xy)
    o, r, te, tr, info = env.step(_zeros(env))
    new = _goals(env).numpy()
    succ = info["success"].numpy()
    assert succ[:2].all() and not succ[2:4].any()
    assert np.array_equal(o["desired_goal"].numpy(), g0)                 # the step's observation carries the old goal
    ach = o["achieved_goal"].numpy()
    for i in range(n):
        changed = not np.array_equal(new[i], g0[i])
        assert changed == bool(succ[i]), i
        want, k = py_goal_update(env._goal_loc.numpy(), env.scaling, NOISE, SUCCESS_RADIUS, seed, i, 1, 1, ach[i], g0[i])
        assert np.array_equal(new[i], want) and (k > 0) == bool(succ[i])
        if changed:
            assert _dist_host(ach[i], new[i]) > f32(SUCCESS_RADIUS) and _in_noise_box(env, new[i])
    # the next step's reward and success use the new goal
    o2, r2, *_ = env.step(_zeros(env))
    assert np.array_equal(o2["desired_goal"].numpy(), new)
    d = np.array([_dist_host(a, g) for a, g in zip(o2["achieved_goal"].numpy(), new)])
    assert np.array_equal(r2.numpy(), (d <= f32(SUCCESS_RADIUS)).astype(np.float32))
    env.close()


@pytest.mark.parametrize("mode", ["same_step", "next_step"])
def test_autoreset_starts_from_the_reset_draw(mode):
    """An env that succeeds on its last step: under SAME_STEP its final_obs has the old goal; in both modes the next episode starts
    with the reset draw of its next episode number, untouched by the update."""
    n, seed = 4, 3
    env = _make(n=n, max_episode_steps=2, autoreset_mode=mode)
    obs, _ = env.reset(seed=seed)
    env.step(_zeros(env))
    g = _goals(env).numpy().copy()
    _place(env, g)                                       # every env succeeds on step 2, the truncating step
    o, r, te, tr, info = env.step(_zeros(env))
    assert tr.all() and info["success"].all()
    gl, rl = env._goal_loc.numpy(), env._reset_loc.numpy()
    if mode == "same_step":
        assert np.array_equal(info["final_obs"]["desired_goal"].numpy(), g)
        st = o
    else:
        st, *_ = env.step(_zeros(env))                   # the reset step
    for i in range(n):
        want, _ = py_maze_draw(gl, rl, env.scaling, NOISE, seed, i, 1)
        assert np.array_equal(st["desired_goal"][i].numpy(), want)
        assert np.array_equal(_goals(env)[i].numpy(), want)
    env.close()


@pytest.mark.parametrize("case", ["reset_target_false", "not_continuing", "one_goal_cell", "numpy_mode"])
def test_gates_leave_goals_and_launches_as_today(case):
    kw, env_id = {}, "PointMaze_Large-v3"
    if case == "reset_target_false":
        kw["reset_target"] = False
    elif case == "not_continuing":
        kw["continuing_task"] = False
    elif case == "one_goal_cell":
        kw["maze_map"] = [[1, 1, 1, 1, 1], [1, "g", 0, "r", 1], [1, 0, 0, 0, 1], [1, 1, 1, 1, 1]]
        env_id = "PointMaze_UMaze-v3"
    elif case == "numpy_mode":
        kw["rng_mode"] = "numpy"
    counts = []
    for backend in (GoalUpdateHostBackend, HostSimBackend):
        env = _make(env_id, n=3, backend=backend, **kw)
        obs, _ = env.reset(seed=8)
        g0 = _goals(env).clone()
        _place(env, g0.numpy())
        o, r, te, tr, info = env.step(_zeros(env))
        assert info["success"].all()
        if case != "numpy_mode":
            assert torch.equal(_goals(env), g0)          # no update in any mode
        assert env.backend.goal_args is None if backend is GoalUpdateHostBackend else True
        counts.append(env.backend.launches)
        env.close()
    assert counts[0] == counts[1]


def test_device_goals_are_invariant_to_batch_and_sharding_and_checkpointed():
    seed = 21

    def run(n, offset, steps=3):
        env = _make(n=n, env_offset=offset)
        env.reset(seed=seed)
        out = []
        for _ in range(steps):
            _place(env, _goals(env).numpy())
            env.step(_zeros(env))
            out.append(_goals(env).clone())
        env.close()
        return out

    full = run(4, 0)
    assert all(not torch.equal(a, b) for a, b in zip(full, full[1:]))
    for a, b, c in zip(full, run(2, 0), run(2, 2)):
        assert torch.equal(a[:2], b) and torch.equal(a[2:], c)
    # a checkpoint inside an episode replays the same updates
    env = _make(n=3)
    env.reset(seed=seed)
    env.step(_zeros(env))
    saved = env.get_state()
    runs = []
    for _ in range(2):
        env.set_state(*saved)
        gs = []
        for _ in range(3):
            _place(env, _goals(env).numpy())
            env.step(_zeros(env))
            gs.append(_goals(env).clone())
        runs.append(gs)
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    env.close()


def test_options_resets_advance_the_episode_of_the_update_stream():
    env = _make(n=2)
    opts = {"goal_cell": np.array([1, 1]), "reset_cell": np.array([1, 2])}
    env.reset(seed=5, options=opts)
    assert env._episode.tolist() == [1, 1]
    got = []
    for _ in range(2):
        _place(env, _goals(env).numpy())
        env.step(_zeros(env))
        got.append(_goals(env).clone())
        env.reset(options=opts)                          # unseeded: the device key stays, the episode moves on
    assert env._episode.tolist() == [3, 3]
    assert not torch.equal(got[0], got[1])
    env.close()


def test_backend_without_the_update_is_refused_in_device_mode():
    with pytest.raises(NotImplementedError):
        _make(n=2, backend=HostSimBackend)
    _make(n=2, backend=HostSimBackend, reset_target=False).close()


# ---------------------------------------------------------------------------------------------- numpy mode against the oracle
@pytest.mark.parametrize("agent", ["ant", "point"])
def test_numpy_mode_matches_the_oracle_with_update_goal(agent):
    n, seed = 3, 14
    env_id, maze = ("AntMaze_Medium-v5", "Medium") if agent == "ant" else ("PointMaze_Medium-v3", "Medium")
    env = _make(env_id, n=n, backend=HostSimBackend, rng_mode="numpy")
    obs, _ = env.reset(seed=seed)
    if agent == "ant":
        oracles = [GoalOracleAntMaze(pkg.maze.MAPS[maze], model=env.model, include_cfrc_ext_in_observation=True, reset_target=True)
                   for _ in range(n)]
    else:
        oracles = [GoalOraclePointMaze(pkg.maze.MAPS[maze], env.model, reset_target=True) for _ in range(n)]
    for i, o in enumerate(oracles):
        oo, _ = o.reset(seed=seed + i)
        assert np.array_equal(obs["desired_goal"][i].numpy(), oo["desired_goal"].astype(f32))
    for step in range(3):
        # envs 0 and 2 succeed (agent on the goal), env 1 does not; the oracles take the same states
        g = _goals(env).numpy()
        xy = g + np.array([[0.0, 0.0], [3.0 * env.scaling, 0.0], [0.1, -0.1]], dtype=f32)
        _place(env, xy)
        st = env.backend.state.numpy()
        q, v = env._sl["qpos"], env._sl["qvel"]
        for i, o in enumerate(oracles):
            o.sim.reset_data()
            o.sim.qpos[:] = st[i, q].astype(np.float64)
            o.sim.qvel[:] = st[i, v].astype(np.float64)
            o.sim.forward()
        o_, r, te, tr, info = env.step(_zeros(env))
        for i, o in enumerate(oracles):
            oo, orr, *_, oi = o.step(np.zeros(env.single_action_space.shape[0]))
            assert bool(info["success"][i]) == oi["success"] == (i != 1)
            assert np.array_equal(o_["desired_goal"][i].numpy(), oo["desired_goal"].astype(f32))
            assert np.array_equal(_goals(env)[i].numpy(), o.goal.astype(f32)), (step, i)
    env.close()


def test_numpy_and_torch_modes_draw_from_the_per_env_streams():
    """With reset_target=True the numpy and torch modes redraw from the per-env numpy streams in the reference's order, the
    succeeding envs only, and write float32(goal)."""
    for mode in ("numpy", "torch"):
        env = _make(n=4, backend=HostSimBackend, rng_mode=mode)
        env.reset(seed=2)
        rngs = [np.random.Generator(np.random.PCG64()) for _ in range(4)]
        for a, b in zip(rngs, env._np_rngs):
            a.bit_generator.state = b.bit_generator.state
        for _ in range(2):
            g = _goals(env).numpy()
            _place(env, g + np.array([[0.0, 0.0], [2.0, 0.0], [0.0, 0.0], [0.0, 0.1]], dtype=f32))
            o, r, te, tr, info = env.step(_zeros(env))
            assert info["success"].tolist() == [True, False, True, True]
            ach = o["achieved_goal"].double().numpy()
            for i in range(4):
                goal = g[i].astype(np.float64)
                while np.linalg.norm(ach[i] - goal) <= SUCCESS_RADIUS:
                    goal = env._noise_np(rngs[i], env.cells.goal_locations[rngs[i].integers(0, len(env.cells.goal_locations))].copy())
                assert np.array_equal(_goals(env)[i].numpy(), goal.astype(f32))
        env.close()
