"""Custom maze layouts (`maze_map=`) on the GPU, on layouts the named maps never reach: non-square, more than 32 columns (the
kernel's wall-bitmap rows straddle 32-bit words) and an open edge with no border wall.  Step parity against the fp64 oracle env
built on the same model, walls that hold, the reset draws of every rng_mode and the reference's known answers."""
import json
import os

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.maze import SUCCESS_RADIUS
from oracle.ant_maze_env import OracleAntMazeEnv
from oracle.point_maze_env import OraclePointMazeEnv
from tests.parity_util import check_envelope, inject_records
from tests.test_gpu_parity import ENVELOPE

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _wide():
    """5 x 35: interior walls in the middle of the map and beyond its 32nd column."""
    mp = [[1] * 35] + [[1] + [0] * 33 + [1] for _ in range(3)] + [[1] * 35]
    mp[1][18] = mp[2][16] = mp[2][20] = mp[2][31] = mp[2][32] = mp[1][33] = 1
    mp[1][1], mp[3][1], mp[1][30], mp[3][20], mp[3][33] = "r", "r", "g", "g", "c"
    return mp


WIDE = _wide()
# the top row and the left end of row 1 have no wall: outside the map there is nothing to collide with
OPEN_EDGE = [[0, 0, 0, 0, 0, 0],
             [0, "c", 0, 1, "c", 1],
             [1, 0, 0, 1, 0, 1],
             [1, 0, 0, 0, 0, 1],
             [1, 1, 1, 1, 1, 1]]
LAYOUTS = {"wide": WIDE, "open_edge": OPEN_EDGE}
# free cells next to a wall, and the direction (x, y) of that wall: the parity tests start agents there so that they hit it.
# The ant's wide-map cells lie within 12 m of the origin: the fp32 kernel's error against the fp64 oracle grows with the
# distance of the world coordinates from the origin (about 7e-5 in the ant's joint angles at 60 m, on no wall), and the stated
# antmaze/* envelopes are those of the named layouts, which reach 22 m
NEAR_WALL = {"wide": [((1, 17), (1, 0)), ((1, 19), (-1, 0)), ((2, 17), (-1, 0)), ((2, 15), (1, 0)), ((1, 16), (0, -1)),
                      ((2, 19), (1, 0)), ((3, 20), (0, 1)), ((1, 20), (0, -1))],
             "open_edge": [((1, 2), (1, 0)), ((1, 4), (-1, 0)), ((2, 2), (1, 0)), ((3, 4), (0, -1)), ((1, 1), (0, 1)),
                           ((2, 4), (1, 0)), ((1, 0), (0, 1)), ((3, 1), (-1, 0))]}
# the point (one metre cells) also starts next to the walls beyond the 32nd column of the wide map
BEYOND_32 = [((1, 32), (1, 0)), ((1, 32), (0, -1)), ((2, 30), (1, 0)), ((3, 32), (0, 1)), ((3, 33), (1, 0)), ((1, 31), (0, -1))]


def _place(env, oracles, places, offset):
    """Move each oracle's agent `offset` (in cells) from the centre of its cell in `places` towards that cell's wall."""
    for o, (cell, d) in zip(oracles, places):
        xy = env.cells.cell_rowcol_to_xy(cell) + offset * env.scaling * np.array(d, dtype=np.float64)
        o.sim.qpos[:2] = xy
        o.sim.forward()


def _wall_contacts(orc):
    names = orc.model.names["geom"]
    return sum(1 for c in orc.sim.contacts() if names[c["geom1"]].startswith("block_") or names[c["geom2"]].startswith("block_"))


def _in_wall(cells, xy):
    """Per row of `xy`: the point lies in a wall cell of the layout (points outside the map are in none)."""
    i = np.floor((cells.y_center - xy[:, 1]) / cells.scaling).astype(int)
    j = np.floor((xy[:, 0] + cells.x_center) / cells.scaling).astype(int)
    inside = (i >= 0) & (i < cells.length) & (j >= 0) & (j < cells.width)
    return np.array([bool(k) and cells.maze_map[a][b] == 1 for k, a, b in zip(inside, i, j)])


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_antmaze_custom_layout_step_parity_from_identical_state(layout):
    """AntMaze-v5 on a custom layout against the oracle env on the same model, from injected states next to walls, inside the
    stated antmaze/* envelopes of the named-layout test."""
    n = 8
    env = pkg.make_vec("AntMaze_UMaze-v5", num_envs=n, device="cuda:0", rng_mode="numpy", maze_map=LAYOUTS[layout])
    obs, _ = env.reset(seed=30)
    oracles = [OracleAntMazeEnv(LAYOUTS[layout], model=env.model, include_cfrc_ext_in_observation=True) for _ in range(n)]
    for i, o in enumerate(oracles):
        oo, _ = o.reset(seed=30 + i)
        # the same PCG64 stream; the goal is a float32 of up to 70 m here
        np.testing.assert_allclose(obs["desired_goal"][i].double().cpu().numpy(), oo["desired_goal"], rtol=1e-6, atol=2e-6)
    _place(env, oracles, NEAR_WALL[layout], 0.4)     # the legs reach into the wall at the first step
    rng = np.random.default_rng(5)
    epos, evel, ecf, touched = [], [], [], 0
    for step in range(12):
        env.set_state(inject_records(env, oracles, lambda i, o, rec, lay: rec.__setitem__(slice(lay["goal"], lay["goal"] + 2), o.goal)))
        a = rng.uniform(-1, 1, (n, 8)).astype(np.float32)
        o, r, te, tr, info = env.step(torch.as_tensor(a))
        for i, orc in enumerate(oracles):
            oo, orr, ote, otr, oi = orc.step(a[i].astype(np.float64))
            touched += _wall_contacts(orc)
            got = o["observation"][i].double().cpu().numpy()
            assert np.isfinite(got).all()
            d = np.abs(got - oo["observation"])
            epos.append(d[:13].max())
            evel.append(d[13:27].max())
            ecf.append(d[27:].max())
            assert float(r[i]) == float(orr) and bool(info["success"][i]) == oi["success"]
            assert bool(te[i]) == bool(ote) and bool(tr[i]) == bool(otr)
    assert touched > 0, "no ant touched a wall: the test did not exercise the custom walls"
    check_envelope("antmaze/pos", epos, *ENVELOPE["antmaze/pos"])
    check_envelope("antmaze/vel", evel, *ENVELOPE["antmaze/vel"])
    check_envelope("antmaze/cfrc", ecf, *ENVELOPE["antmaze/cfrc"])
    env.close()


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_pointmaze_custom_layout_step_parity_from_identical_state(layout):
    places = NEAR_WALL[layout] + (BEYOND_32 if layout == "wide" else [])
    n = len(places)
    env = pkg.make_vec("PointMaze_UMaze-v3", num_envs=n, device="cuda:0", rng_mode="numpy", maze_map=LAYOUTS[layout])
    env.reset(seed=40)
    oracles = [OraclePointMazeEnv(LAYOUTS[layout], env.model) for _ in range(n)]
    for i, o in enumerate(oracles):
        o.reset(seed=40 + i)
    _place(env, oracles, places, 0.3)
    rng = np.random.default_rng(6)
    worst, touched = 0.0, 0
    for _ in range(200):
        # from the oracle's state at every step: free-running, a contact that switches on at its margin one step earlier in
        # one of the two (fp32 against fp64) sets the velocities 0.1 m/s apart
        env.set_state(inject_records(env, oracles, lambda i, o, rec, lay: rec.__setitem__(slice(lay["goal"], lay["goal"] + 2), o.goal)))
        a = rng.uniform(-1.5, 1.5, (n, 2)).astype(np.float32)
        o, r, te, tr, info = env.step(torch.as_tensor(a))
        for i, orc in enumerate(oracles):
            oo, orr, *_ = orc.step(a[i].astype(np.float64))
            touched += _wall_contacts(orc)
            worst = max(worst, np.abs(o["observation"][i].double().cpu().numpy() - oo["observation"]).max())
            d = np.linalg.norm(oo["achieved_goal"] - oo["desired_goal"])
            if abs(d - SUCCESS_RADIUS) > 1e-3:
                assert float(r[i]) == float(orr) and bool(info["success"][i]) == (d <= SUCCESS_RADIUS)
    print(f"PointMaze {layout} 200 steps from injected states: worst {worst:.2e}, wall contacts {touched}")
    assert touched > 0 and worst < 2e-4
    env.close()


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_ant_never_enters_a_wall_cell(layout):
    n = 1024
    env = pkg.make_vec("AntMaze_UMaze-v5", num_envs=n, device="cuda:0", rng_mode="torch", maze_map=LAYOUTS[layout])
    env.reset(seed=0)
    g = torch.Generator(device="cuda").manual_seed(3)
    for t in range(40):
        a = torch.rand((n, 8), generator=g, device="cuda") * 2 - 1
        o, r, te, tr, info = env.step(a)
        assert torch.isfinite(o["observation"]).all()
        assert not _in_wall(env.cells, o["achieved_goal"].double().cpu().numpy()).any()
    env.close()


@pytest.mark.parametrize("rng_mode", ["device", "torch"])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("env_id", ["AntMaze_UMaze-v5", "PointMaze_UMaze-v3"])
def test_resets_draw_from_the_layout_cells(env_id, layout, rng_mode):
    """Goals within noise of a goal location (g / c cells), starts within noise of a reset location (r / c cells) whose centre
    is farther than half a cell from the goal, neither in a wall cell."""
    n = 2048
    env = pkg.make_vec(env_id, num_envs=n, device="cuda:0", rng_mode=rng_mode, maze_map=LAYOUTS[layout])
    cells, s = env.cells, env.scaling
    for seed in (1, 2):
        obs, info = env.reset(seed=seed)
        goal, start = obs["desired_goal"].double().cpu().numpy(), obs["achieved_goal"].double().cpu().numpy()
        dg = np.abs(goal[:, None, :] - cells.goal_locations[None]).max(axis=2)
        ds = np.abs(start[:, None, :] - cells.reset_locations[None]).max(axis=2)
        assert (dg.min(axis=1) <= 0.25 * s + 1e-4).all() and (ds.min(axis=1) <= 0.25 * s + 1e-4).all()
        centre = cells.reset_locations[ds.argmin(axis=1)]
        assert (np.linalg.norm(centre - goal, axis=1) > 0.5 * s).all()
        assert not _in_wall(cells, goal).any() and not _in_wall(cells, start).any()
        assert not bool(info["success"].any())
        # every goal and reset location is drawn
        assert len(set(dg.argmin(axis=1).tolist())) == len(cells.goal_locations)
        assert len(set(ds.argmin(axis=1).tolist())) == len(cells.reset_locations)
    env.close()


def test_pointmaze_reference_known_answers_through_maze_map():
    """The reference's known answers (tests/envs/maze/test_point_maze.py:20-45) with the layout given as `maze_map=`, no model."""
    for c in json.load(open(os.path.join(HERE, "golden", "maze_known_answers.json"))):
        env = pkg.make_vec("PointMaze_UMaze-v3", num_envs=3, device="cuda:0", rng_mode="numpy", maze_map=c["maze_map"])
        obs, info = env.reset(seed=[c["seed"]] * 3, options=c["options"])
        if "reset_pos" in c["expect"]:
            np.testing.assert_almost_equal(np.array(c["expect"]["reset_pos"] + [0, 0]), obs["observation"][0].double().cpu().numpy(),
                                           decimal=c["decimal"])
        if "goal" in c["expect"]:
            np.testing.assert_almost_equal(np.array(c["expect"]["goal"]), obs["desired_goal"][2].double().cpu().numpy(), decimal=c["decimal"])
        env.close()
