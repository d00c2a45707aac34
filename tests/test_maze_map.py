"""Custom maze layouts (`maze_map=`) for AntMaze and PointMaze on the CPU: the model builder against the committed blobs, the
public constructors, the layout checks, pickling and a rollout on the emulated kernel against the oracle env."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200 import models
from gymnasium_robotics_b200.maze import AGENTS, MAPS, AntMazeVectorEnv, MazeVectorEnv, PointMazeVectorEnv
from gymnasium_robotics_b200.mjcf import replace_maze_walls
from oracle.point_maze_env import OraclePointMazeEnv
from tests.hostsim_backend import HostSimBackend

HERE = os.path.dirname(os.path.abspath(__file__))
LAYOUTS = ("Open", "UMaze", "Medium", "Large")
# non-square, goal / reset / combined cells, an interior wall
CUSTOM = [[1, 1, 1, 1, 1, 1, 1],
          [1, "r", 0, 0, 1, "g", 1],
          [1, 0, 1, 0, 0, 0, 1],
          [1, "c", 0, 0, 1, "g", 1],
          [1, 1, 1, 1, 1, 1, 1]]


@pytest.fixture
def no_reference_assets(monkeypatch):
    monkeypatch.delenv("B200SIM_REFERENCE_ASSETS", raising=False)
    monkeypatch.setattr(models, "REFERENCE_ASSETS", "")


@pytest.mark.parametrize("agent", ["ant", "point"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_rebuilt_layout_is_byte_identical_to_the_committed_blob(agent, layout, no_reference_assets):
    """Every committed maze blob is reproduced from another committed blob of the same agent."""
    base = LAYOUTS[(LAYOUTS.index(layout) + 1) % len(LAYOUTS)]
    cfg = AGENTS[agent]
    m = replace_maze_walls(models.load_model(f"{agent}maze_{base.lower()}"), MAPS[layout], cfg["scaling"], cfg["height"])
    with open(os.path.join(models.MODEL_DIR, f"{agent}maze_{layout.lower()}.b200m"), "rb") as f:
        assert m.to_blob() == f.read()
    assert models.build_maze_model(agent, MAPS[layout]).to_blob() == m.to_blob()


@pytest.mark.skipif(not os.path.isdir(models.REFERENCE_ASSETS), reason="B200SIM_REFERENCE_ASSETS does not name the reference's assets")
@pytest.mark.parametrize("agent", ["ant", "point"])
def test_builder_matches_the_compiler_on_custom_layouts(agent):
    wide = [[1] * 35] + [[1] + [0] * 33 + [1] for _ in range(3)] + [[1] * 35]
    wide[2][16] = wide[2][32] = wide[1][33] = 1
    open_edge = [[0, 0, 0, 0, 0, 0], [1, "c", 0, 1, "c", 1], [1, 0, 0, 0, 0, 1], [1, 1, 1, 1, 1, 1]]
    for mp in (CUSTOM, wide, open_edge):
        assert models.build_maze_model(agent, mp).to_blob() == models.compile_maze_model(agent, mp).to_blob()


def test_custom_layout_model_places_the_walls_of_the_map(no_reference_assets):
    m = models.build_maze_model("point", CUSTOM)
    assert m.grid_dims.tolist() == [5, 7]
    assert m.grid_walls.tolist() == [int(c == 1) for row in CUSTOM for c in row]
    nwall = sum(c == 1 for row in CUSTOM for c in row)
    walls = [n for n in m.names["geom"] if n.startswith("block_")]
    assert len(walls) == nwall and walls[-1] == "block_4_6" and m.ngeom == 2 + nwall
    assert m.npair == 1 + nwall and int(m.pair_grid.sum()) == nwall     # ground-particle, particle-wall pairs
    i = m.names["geom"].index("block_2_2")
    assert m.geom_pos[i].tolist() == [-1.0, 0.0, 0.2] and m.geom_size[i].tolist() == [0.5, 0.5, 0.2]


def test_make_vec_honours_maze_map(no_reference_assets):
    env = pkg.make_vec("PointMaze_UMaze-v3", num_envs=2, maze_map=CUSTOM, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.cells.maze_map == CUSTOM and env.model.grid_dims.tolist() == [5, 7]
    assert env.max_episode_steps == 300 and env.reward_type == "sparse"     # the id's registry entry
    dense = pkg.make_vec("PointMaze_LargeDense-v3", num_envs=1, maze_map=CUSTOM, backend_factory=HostSimBackend)
    assert dense.max_episode_steps == 800 and dense.reward_type == "dense" and dense.cells.maze_map == CUSTOM
    for version, nobs in (("v5", 105), ("v4", 27)):
        ant = pkg.make_vec(f"AntMaze_Medium-{version}", num_envs=1, maze_map=CUSTOM, backend_factory=HostSimBackend)
        assert ant.cells.maze_map == CUSTOM and ant.model.grid_dims.tolist() == [5, 7] and ant.max_episode_steps == 1000
        assert ant.single_observation_space["observation"].shape == (nobs,)


def test_constructors_and_vector_entry_point_honour_maze_map(no_reference_assets):
    for cls, agent in ((AntMazeVectorEnv, "ant"), (PointMazeVectorEnv, "point")):
        env = cls(maze_map=CUSTOM, num_envs=1, backend_factory=HostSimBackend)
        assert env.cells.maze_map == CUSTOM and env.model.to_blob() == models.build_maze_model(agent, CUSTOM).to_blob()
    env = MazeVectorEnv(maze_map=CUSTOM, agent="point", num_envs=1, backend_factory=HostSimBackend)
    assert env.cells.maze_map == CUSTOM
    # what gymnasium.make_vec(id, maze_map=M, vectorization_mode="vector_entry_point") calls: the registered kwargs + the user's
    env = MazeVectorEnv(**pkg.ENV_IDS["PointMaze_Open-v3"], num_envs=1, maze_map=CUSTOM, backend_factory=HostSimBackend)
    assert env.cells.maze_map == CUSTOM and env.max_episode_steps == 300


def test_named_layouts_and_explicit_models_are_unchanged(no_reference_assets):
    env = pkg.make_vec("AntMaze_UMaze-v5", num_envs=1, backend_factory=HostSimBackend)
    assert env.model.to_blob() == models.load_model("antmaze_umaze").to_blob() and env.cells.maze_map == MAPS["UMaze"]
    model = models.load_model("pointmaze_medium")
    env = PointMazeVectorEnv(maze_map=CUSTOM, model=model, num_envs=1, backend_factory=HostSimBackend)
    assert env.model is model and env.cells.maze_map == CUSTOM
    with pytest.raises(ValueError):
        PointMazeVectorEnv(CUSTOM, maze_map=CUSTOM, model=model, num_envs=1, backend_factory=HostSimBackend)


def test_reference_known_answers_through_maze_map(no_reference_assets):
    """tests/envs/maze/test_point_maze.py:20-45 of the reference, with the layout given as `maze_map=` and no model."""
    for c in json.load(open(os.path.join(HERE, "golden", "maze_known_answers.json"))):
        env = PointMazeVectorEnv(maze_map=c["maze_map"], num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
        obs, info = env.reset(seed=c["seed"], options=c["options"])
        if "reset_pos" in c["expect"]:
            np.testing.assert_almost_equal(np.array(c["expect"]["reset_pos"] + [0, 0]), obs["observation"][0].double().numpy(),
                                           decimal=c["decimal"])
        if "goal" in c["expect"]:
            np.testing.assert_almost_equal(np.array(c["expect"]["goal"]), obs["desired_goal"][0].double().numpy(), decimal=c["decimal"])


@pytest.mark.parametrize("bad, reason", [
    ([], "empty"),
    ([[]], "empty"),
    ([[1, 1, 1], [1, 0]], "not rectangular"),
    ([[1, 1, 1], [1, 2, 1]], "a cell is"),
    ([[1, 1, 1], [1, "x", 1]], "a cell is"),
    ([[1, 1, 1], [1, 0.0, 1]], "a cell is"),
    ([[1, 1], [1, 1]], "no goal"),
    ([[1, 1, 1], [1, "g", 1], [1, "g", 1]], "no reset"),
    ([[1, 1, 1], [1, "c", 1]], "no reset location in another cell"),
    ([[1, 1, 1, 1], [1, "g", "r", 1], [1, "g", 1, 1]], None),
    ([[1, "r", 1], [1, "g", 1], [1, "g", 1]], None),
    (5, "list of rows"),
])
def test_invalid_layouts_raise_value_error(bad, reason, no_reference_assets):
    if reason is None:      # valid: every goal cell has a reset location in another cell
        PointMazeVectorEnv(maze_map=bad, num_envs=1, backend_factory=HostSimBackend)
        return
    with pytest.raises(ValueError, match=reason):
        PointMazeVectorEnv(maze_map=bad, num_envs=1, backend_factory=HostSimBackend)
    with pytest.raises(ValueError, match=reason):
        pkg.make_vec("AntMaze_UMaze-v5", num_envs=1, maze_map=bad, backend_factory=HostSimBackend)


def test_pickle_round_trip_keeps_the_layout(no_reference_assets):
    env = pkg.make_vec("PointMaze_UMaze-v3", num_envs=2, maze_map=CUSTOM, backend_factory=HostSimBackend, rng_mode="numpy")
    env2 = pickle.loads(pickle.dumps(env))
    assert env2.cells.maze_map == CUSTOM and env2.model.to_blob() == env.model.to_blob()
    assert env2.max_episode_steps == env.max_episode_steps
    o1, _ = env.reset(seed=3)
    o2, _ = env2.reset(seed=3)
    assert torch.equal(o1["desired_goal"], o2["desired_goal"]) and torch.equal(o1["observation"], o2["observation"])


def test_custom_layout_step_tracks_oracle_and_never_resets_into_success(no_reference_assets):
    env = PointMazeVectorEnv(maze_map=CUSTOM, num_envs=3, backend_factory=HostSimBackend, rng_mode="numpy")
    goals = {tuple(g) for g in env.cells.goal_locations.tolist()}
    for s in range(30):
        obs, info = env.reset(seed=200 + 3 * s)
        assert not bool(info["success"].any())
        assert bool((torch.linalg.norm(obs["achieved_goal"] - obs["desired_goal"], dim=1) > 0.45).all())
        for g in obs["desired_goal"].double().numpy():        # a g or c cell centre, plus noise of at most a quarter cell
            assert min(np.abs(g - np.array(c)).max() for c in goals) <= 0.25 + 1e-6
    obs, _ = env.reset(seed=7)
    oracles = [OraclePointMazeEnv(CUSTOM, env.model) for _ in range(3)]
    for i, o in enumerate(oracles):
        oo, _ = o.reset(seed=7 + i)
        assert np.allclose(obs["observation"][i].double().numpy(), oo["observation"], atol=1e-6)
    rng = np.random.default_rng(0)
    worst = 0
    for _ in range(150):
        a = rng.uniform(-1.5, 1.5, (3, 2)).astype(np.float32)
        o, r, te, tr, info = env.step(a)
        for i, orc in enumerate(oracles):
            oo, orr, *_ = orc.step(a[i].astype(np.float64))
            worst = max(worst, np.abs(o["observation"][i].double().numpy() - oo["observation"]).max())
            assert float(r[i]) == float(orr)
    assert worst < 5e-4, worst
