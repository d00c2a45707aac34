"""Batched AntMaze (v5) and PointMaze (v3) environments on the b200sim CUDA path.

Host-side mirror of the reference's maze stack, batched over `num_envs`:
  * map tables               envs/maze/maps.py:52-135 (data), ids/kwargs/max_episode_steps __init__.py:839-958
  * Maze grid math           envs/maze/maze_v4.py:135-146 (cell<->xy), :148-242 (goal/reset cell collection)
  * MazeEnv.reset / noise / update_goal     envs/maze/maze_v4.py:276-297, 299-379, 400-418
  * AntMazeEnv ctor/reset/step/_get_obs     envs/maze/ant_maze_v5.py:221-320 (inner AntEnv [ext]: frame_skip 5, RK4)
  * PointMazeEnv / PointEnv                 envs/maze/point_maze.py:316-434, envs/maze/point.py:22-77 (frame_skip 1, Euler)
  * compute_reward / compute_terminated     envs/maze/maze_v4.py:381-398
The per-step arithmetic (5 RK4 sub-steps, observation, reward, success) runs inside one CUDA kernel launch.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

from . import _lib
from .fetch import CudaBackend
from .models import build_maze_model, load_model
from .spaces import Box, Dict as DictSpace
from .vector import VectorEnv

R, G, C = "r", "g", "c"
MAPS = {
    "Open": [[1, 1, 1, 1, 1, 1, 1], [1, 0, 0, 0, 0, 0, 1], [1, 0, 0, 0, 0, 0, 1], [1, 0, 0, 0, 0, 0, 1], [1, 1, 1, 1, 1, 1, 1]],
    "Open_Diverse_G": [[1, 1, 1, 1, 1, 1, 1], [1, R, G, G, G, G, 1], [1, G, G, G, G, G, 1], [1, G, G, G, G, G, 1], [1, 1, 1, 1, 1, 1, 1]],
    "Open_Diverse_GR": [[1, 1, 1, 1, 1, 1, 1], [1, C, C, C, C, C, 1], [1, C, C, C, C, C, 1], [1, C, C, C, C, C, 1], [1, 1, 1, 1, 1, 1, 1]],
    "UMaze": [[1, 1, 1, 1, 1], [1, 0, 0, 0, 1], [1, 1, 1, 0, 1], [1, 0, 0, 0, 1], [1, 1, 1, 1, 1]],
    "Medium": [[1, 1, 1, 1, 1, 1, 1, 1], [1, 0, 0, 1, 1, 0, 0, 1], [1, 0, 0, 1, 0, 0, 0, 1], [1, 1, 0, 0, 0, 1, 1, 1],
               [1, 0, 0, 1, 0, 0, 0, 1], [1, 0, 1, 0, 0, 1, 0, 1], [1, 0, 0, 0, 1, 0, 0, 1], [1, 1, 1, 1, 1, 1, 1, 1]],
    "Medium_Diverse_G": [[1, 1, 1, 1, 1, 1, 1, 1], [1, R, 0, 1, 1, 0, 0, 1], [1, 0, 0, 1, 0, 0, G, 1], [1, 1, 0, 0, 0, 1, 1, 1],
                         [1, 0, 0, 1, 0, 0, 0, 1], [1, G, 1, 0, 0, 1, 0, 1], [1, 0, 0, 0, 1, G, 0, 1], [1, 1, 1, 1, 1, 1, 1, 1]],
    "Medium_Diverse_GR": [[1, 1, 1, 1, 1, 1, 1, 1], [1, C, 0, 1, 1, 0, 0, 1], [1, 0, 0, 1, 0, 0, C, 1], [1, 1, 0, 0, 0, 1, 1, 1],
                          [1, 0, 0, 1, 0, 0, 0, 1], [1, C, 1, 0, 0, 1, 0, 1], [1, 0, 0, 0, 1, C, 0, 1], [1, 1, 1, 1, 1, 1, 1, 1]],
    "Large": [[1] * 12, [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 1], [1, 0, 1, 1, 0, 1, 0, 1, 0, 1, 0, 1], [1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 1],
              [1, 0, 1, 1, 1, 1, 0, 1, 1, 1, 0, 1], [1, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0, 1], [1, 1, 0, 1, 0, 1, 0, 1, 0, 1, 1, 1],
              [1, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1], [1] * 12],
    "Large_Diverse_G": [[1] * 12, [1, R, 0, 0, 0, 1, G, 0, 0, 0, 0, 1], [1, 0, 1, 1, 0, 1, 0, 1, 0, 1, 0, 1], [1, 0, 0, 0, 0, G, 0, 1, 0, 0, G, 1],
                        [1, 0, 1, 1, 1, 1, 0, 1, 1, 1, 0, 1], [1, 0, G, 1, 0, 1, 0, 0, 0, 0, 0, 1], [1, 1, 0, 1, 0, 1, 0, 1, 0, 1, 1, 1],
                        [1, 0, 0, 1, G, 0, G, 1, 0, G, 0, 1], [1] * 12],
    "Large_Diverse_GR": [[1] * 12, [1, C, 0, 0, 0, 1, C, 0, 0, 0, 0, 1], [1, 0, 1, 1, 0, 1, 0, 1, 0, 1, 0, 1], [1, 0, 0, 0, 0, C, 0, 1, 0, 0, C, 1],
                         [1, 0, 1, 1, 1, 1, 0, 1, 1, 1, 0, 1], [1, 0, C, 1, 0, 1, 0, 0, 0, 0, 0, 1], [1, 1, 0, 1, 0, 1, 0, 1, 0, 1, 1, 1],
                         [1, 0, 0, 1, C, 0, C, 1, 0, C, 0, 1], [1] * 12],
}
# wall layout -> compiled physics model (the diverse variants only relabel free cells)
NOISE, SUCCESS_RADIUS = 0.25, 0.45
# per agent: maze_size_scaling, maze_height, frame_skip, first qpos entry in `observation`, velocity clip, episode lengths
AGENTS = {
    "ant": dict(scaling=4.0, height=0.5, frame_skip=5, obs_qpos_start=2, vel_clip=0.0, fps=50,
                steps={k: (700 if k.startswith(("Open", "UMaze")) else 1000) for k in MAPS}),     # __init__.py:839-958
    "point": dict(scaling=1.0, height=0.4, frame_skip=1, obs_qpos_start=0, vel_clip=5.0, fps=100,
                  steps={k: (300 if k.startswith(("Open", "UMaze")) else (600 if k.startswith("Medium") else 800)) for k in MAPS}),  # :960-1080
}
SCALING, HEIGHT, FRAME_SKIP = AGENTS["ant"]["scaling"], AGENTS["ant"]["height"], AGENTS["ant"]["frame_skip"]


def model_name(agent, maze):
    """wall layout -> compiled physics model (the diverse variants only relabel free cells)"""
    return f"{agent}maze_" + maze.split("_")[0].lower()


class MazeCells:
    """Cell bookkeeping of `Maze` (maze_v4.py:26-242) without the XML part.  fallbacks=False is the older `Maze` of AntMaze-v3
    (envs/maze/maze.py:86-157): a layout with no "r"/"c" cells gets no reset locations and one with no "g"/"c" cells no goal locations
    (maze_v4.py:223-230 would take the empty cells); an unlabelled layout still uses every free cell for both."""

    def __init__(self, maze_map, scaling=SCALING, fallbacks=True):
        self.maze_map, self.scaling = maze_map, scaling
        self.length, self.width = len(maze_map), len(maze_map[0])
        self.x_center, self.y_center = self.width / 2 * scaling, self.length / 2 * scaling
        goals, resets, combined, empty = [], [], [], []
        for i in range(self.length):
            for j in range(self.width):
                cell, xy = maze_map[i][j], self.cell_rowcol_to_xy((i, j))
                if cell == R:
                    resets.append(xy)
                elif cell == G:
                    goals.append(xy)
                elif cell == C:
                    combined.append(xy)
                elif cell == 0:
                    empty.append(xy)
        if not goals and not resets and not combined:
            combined = empty
        elif fallbacks and not resets and not combined:
            resets = empty
        elif fallbacks and not goals and not combined:
            goals = empty
        self.goal_locations = np.array(goals + combined)
        self.reset_locations = np.array(resets + combined)

    def cell_rowcol_to_xy(self, rowcol):
        return np.array([(rowcol[1] + 0.5) * self.scaling - self.x_center, self.y_center - (rowcol[0] + 0.5) * self.scaling])

    def cell_xy_to_rowcol(self, xy):
        return np.array([math.floor((self.y_center - xy[1]) / self.scaling), math.floor((xy[0] + self.x_center) / self.scaling)])


def check_maze_map(maze_map, scaling, fallbacks=True):
    """The cells of a user layout (`maze_map=`) as a list of rows, or ValueError with the reason.  fallbacks=False (AntMaze-v3,
    `MazeCells`) refuses a layout that labels cells but leaves no goal or no reset location.  Beyond the reference, a
    layout is refused when some goal location has no reset location in another cell: the reference's start draw
    (`generate_reset_pos`, maze_v4.py:276-297) would loop forever on it, and the device draw (csrc/reset_sample.cuh) would give up and start the env
    in its goal cell."""
    try:
        rows = [list(row) for row in maze_map]
    except TypeError:
        raise ValueError("maze_map must be a list of rows of cells") from None
    if not rows or not rows[0]:
        raise ValueError("maze_map is empty")
    if any(len(row) != len(rows[0]) for row in rows):
        raise ValueError(f"maze_map is not rectangular: row lengths {[len(row) for row in rows]}")
    for i, row in enumerate(rows):
        for j, cell in enumerate(row):
            if not (cell in (R, G, C) if isinstance(cell, str) else
                    (isinstance(cell, (int, np.integer)) and not isinstance(cell, bool) and cell in (0, 1))):
                raise ValueError(f"maze_map[{i}][{j}] = {cell!r}: a cell is 0, 1, {R!r}, {G!r} or {C!r}")
    cells = MazeCells(rows, scaling, fallbacks)
    if len(cells.goal_locations) == 0 or len(cells.reset_locations) == 0:
        raise ValueError(f"maze_map has no {'goal' if len(cells.goal_locations) == 0 else 'reset'} location")
    for g in cells.goal_locations:
        if not bool((np.linalg.norm(cells.reset_locations - g, axis=1) > 0.5 * scaling).any()):
            raise ValueError(f"maze_map: the goal cell {tuple(cells.cell_xy_to_rowcol(g).tolist())} has no reset location in another cell")
    return rows


def make_maze_task(model, reward_type, agent="ant", contact_forces=False, frame_skip=None, touch_mode=None):
    """contact_forces: append Ant-v5's clipped `cfrc_ext[1:]` (6 values per body) to the observation -- (105,) instead of (27,).
    touch_mode (the Ant's keywords, `AntKeywords.touch_mode`) overrides it: 2..4 select the ant kernel build, 4 appends all of
    `cfrc_ext`, world row included -- Ant-v4's (111,)."""
    cfg = AGENTS[agent]
    frame_skip = cfg["frame_skip"] if frame_skip is None else frame_skip
    mode = int(bool(contact_forces)) if touch_mode is None else touch_mode
    t = _lib.FetchTaskC()
    t.kind, t.nact, t.ngoal = 1, int(model.nu), 2
    t.n_substeps, t.reward_dense = frame_skip, int(reward_type == "dense")
    t.obs_qpos_start, t.vel_clip = cfg["obs_qpos_start"], cfg["vel_clip"]
    t.touch_mode = mode
    nmjb = len(model.mjbody_rt)
    t.nobs = int(model.nq - cfg["obs_qpos_start"] + model.nv) + {1: 6 * (nmjb - 1), 3: 6 * (nmjb - 1), 4: 6 * nmjb}.get(mode, 0)
    t.success_radius = SUCCESS_RADIUS
    t.dt = float(model.opt[0] * frame_skip)
    return t


# The info keys of the Ant (Ant.step [ext]), in the column order of the [N, 9] info rows the ant kernel build writes
# (b200sim_set_ant_info)
ANT_INFO_COLUMNS = ("x_position", "y_position", "distance_from_origin", "x_velocity", "y_velocity", "reward_forward", "reward_ctrl",
                    "reward_contact", "reward_survive")
# Gymnasium's Ant-v5 / Ant-v4 keywords [ext] that the maze forwards to its AntEnv (ant_maze_v5.py:249-255, ant_maze_v4.py:62-67) and
# their defaults.  AntMaze passes reset_noise_scale and exclude_current_positions_from_observation itself, so the reference refuses
# them with a TypeError; so are the keywords that the other version's AntEnv does not take.
ANT_KEYWORDS = {
    5: dict(frame_skip=5, forward_reward_weight=1.0, ctrl_cost_weight=0.5, contact_cost_weight=5e-4, healthy_reward=1.0, main_body=1,
            terminate_when_unhealthy=True, healthy_z_range=(0.2, 1.0), contact_force_range=(-1.0, 1.0), include_cfrc_ext_in_observation=True),
    4: dict(ctrl_cost_weight=0.5, use_contact_forces=False, contact_cost_weight=5e-4, healthy_reward=1.0, terminate_when_unhealthy=True,
            healthy_z_range=(0.2, 1.0), contact_force_range=(-1.0, 1.0)),
}


class AntKeywords:
    """The Ant keywords of one AntMaze env: parsed, refused as the reference refuses them, and turned into the kernel's settings."""

    def __init__(self, version, kwargs, include_cfrc):
        if version not in ANT_KEYWORDS:
            raise ValueError(f"ant_version must be 4 or 5, got {version!r}")
        for k in ("reset_noise_scale", "exclude_current_positions_from_observation"):
            if k in kwargs:
                raise TypeError(f"AntEnv got multiple values for keyword argument {k!r} (AntMaze passes it itself)")
        if "xml_file" in kwargs:
            if version == 4:
                raise TypeError("AntEnv got multiple values for keyword argument 'xml_file' (AntMaze-v4 passes it itself)")
            raise NotImplementedError("xml_file: the CUDA build steps the committed ant model only")
        other = ANT_KEYWORDS[9 - version]
        for k in list(kwargs):
            if k in other and k not in ANT_KEYWORDS[version]:
                raise TypeError(f"Ant-v{version} got an unexpected keyword argument {k!r}")
        if version == 4 and include_cfrc is not None:
            raise TypeError("Ant-v4 got an unexpected keyword argument 'include_cfrc_ext_in_observation'")
        kw = dict(ANT_KEYWORDS[version])
        self.frame_skip_given = "frame_skip" in kwargs
        kw.update({k: kwargs.pop(k) for k in list(kwargs) if k in kw})
        kw["include_cfrc_ext_in_observation"] = bool(include_cfrc) if version == 5 else False
        if version == 5 and kw["main_body"] not in (1, "torso"):
            raise NotImplementedError(f"main_body={kw['main_body']!r}: the CUDA build measures the torso (main_body 1) only")
        frame_skip = kw.get("frame_skip", 5)
        if isinstance(frame_skip, bool) or not isinstance(frame_skip, (int, np.integer)) or frame_skip < 1:
            raise ValueError(f"frame_skip must be a positive integer, got {frame_skip!r}")
        lo, hi = (float(v) for v in kw["contact_force_range"])
        if not lo <= hi:
            raise ValueError(f"contact_force_range must be (min, max), got {kw['contact_force_range']!r}")
        self.version, self.kw, self.frame_skip, self.cf_range = version, kw, int(frame_skip), (lo, hi)
        self.contact_obs = kw["include_cfrc_ext_in_observation"] or bool(kw.get("use_contact_forces", False))

    def needs_ant_build(self, ant_info):
        """The plain kernel build observes cfrc_ext[1:] clipped to (-1, 1) or nothing; anything else runs the ant build."""
        return ant_info or self.version == 4 and self.contact_obs or self.contact_obs and self.cf_range != (-1.0, 1.0)

    def touch_mode(self, ant_info):
        if not self.needs_ant_build(ant_info):
            return int(self.contact_obs)
        return 4 if self.version == 4 and self.contact_obs else (3 if self.contact_obs else 2)

    def params(self):
        kw, p = self.kw, _lib.AntParamsC()
        p.version = self.version
        p.forward_reward_weight = float(kw.get("forward_reward_weight", 1.0))
        p.ctrl_cost_weight, p.contact_cost_weight, p.healthy_reward = (float(kw[k]) for k in ("ctrl_cost_weight", "contact_cost_weight", "healthy_reward"))
        p.terminate_when_unhealthy, p.use_contact_forces = int(bool(kw["terminate_when_unhealthy"])), int(bool(kw.get("use_contact_forces", False)))
        p.healthy_z_range[0], p.healthy_z_range[1] = (float(v) for v in kw["healthy_z_range"])
        p.contact_force_range[0], p.contact_force_range[1] = self.cf_range
        return p

    def info_keys(self):
        """(step keys, reset keys) as (name, column) pairs: Ant-v5's, or Ant-v4's (no reward_contact, forward_reward = reward_forward)."""
        col = {k: i for i, k in enumerate(ANT_INFO_COLUMNS)}
        if self.version == 5:
            return tuple(col.items()), tuple((k, col[k]) for k in ANT_INFO_COLUMNS[:3])
        step = tuple((k, c) for k, c in col.items() if k != "reward_contact") + (("forward_reward", col["reward_forward"]),)
        return step, ()


def make_antmaze_task(model, reward_type):
    return make_maze_task(model, reward_type, "ant")


class MazeVectorEnv(VectorEnv):
    """`gym.make_vec("AntMaze_Large-v5" | "PointMaze_UMaze-v3", num_envs=N)` replacement (torch CUDA tensors, leading
    `num_envs` axis).  `maze` is a name from `MAPS` or (for the point agent's tests) an explicit cell list with its compiled
    `model`.  `maze_map=` is the reference's custom layout (point_maze.py:195-207, ant_maze_v5.py:221-229): a list of rows of
    0, 1, "r", "g", "c" cells (`check_maze_map`), built on the agent's committed model (`models.build_maze_model`) unless a
    `model` is given; the named `maze` still supplies the episode length.  The per-env numpy streams exist in every rng_mode:
    explicit `options` cells draw from them, and so does the goal update of `reset_target` except in rng_mode="device", where
    the step launch redraws the goals of the envs that succeeded (b200sim_set_goal_update).

    maze_version=3 (ant agent only) is AntMaze-v3's task logic, envs/maze/maze.py on Gymnasium's Ant-v4 (ant_maze_v3.py): the start
    is drawn farther than 0.5 (not half a cell) from the goal, a labelled layout gets no empty-cell fallbacks, `reset_target` does not
    exist, and in a continuing task with more than one goal location an env that reaches its goal gets one new goal inside the step
    (maze.py:283-302) whose reward is that of the new goal (ant_maze_v3.py:94-97).  The step's info is the Ant's (`ant_info` defaults
    to True) with no `success` key, and the reset info is empty."""

    metadata = {"render_modes": [], "render_fps": 50, "autoreset_mode": "next_step"}
    AGENT = "ant"
    AUTO_RECOVER = False
    SUCCESS_KEY = "success"

    def __init__(self, maze="Large", num_envs: int = 1, reward_type: str = "sparse", continuing_task: bool = True,
                 reset_target: Optional[bool] = None, max_episode_steps: Optional[int] = None, device="cuda:0", rng_mode: str = "auto",
                 autoreset_mode: str = "next_step", backend_factory=None, agent: Optional[str] = None, model=None,
                 include_cfrc_ext_in_observation: Optional[bool] = None, maze_map=None, ant_version: Optional[int] = None,
                 ant_info: Optional[bool] = None, maze_version: int = 4, **kwargs):
        self.agent = agent or self.AGENT
        cfg = AGENTS[self.agent]
        if maze_version not in (3, 4):
            raise ValueError(f"maze_version must be 3 or 4, got {maze_version!r}")
        v3 = self._v3 = maze_version == 3
        self.maze_version = maze_version
        if v3:
            if self.agent != "ant":
                raise ValueError("maze_version=3 (envs/maze/maze.py) is AntMaze-v3's; PointMaze-v3 runs the maze_v4 logic (maze_version=4)")
            if ant_version not in (None, 4):
                raise ValueError(f"AntMaze-v3 wraps Ant-v4, got ant_version={ant_version!r}")
            if reset_target is not None:   # v3's MazeEnv takes it into **kwargs and forwards it to Ant-v4, which refuses it
                raise TypeError("AntEnv.__init__() got an unexpected keyword argument 'reset_target'")
            ant_version = 4
        # the Ant's keywords (Gymnasium's Ant-v5 for the -v5 ids and by default, Ant-v4 for the -v4 and -v3 ids); they leave `kwargs`
        self.ant = AntKeywords(5 if ant_version is None else ant_version, kwargs, include_cfrc_ext_in_observation) if self.agent == "ant" else None
        if self.ant is None and (ant_info or ant_version is not None):
            raise ValueError("ant_version / ant_info are keywords of the ant agent")
        # AntMaze-v3's step info IS Ant-v4's (ant_maze_v3.py:91), so it is on by default there
        self.ant_info = v3 if ant_info is None else bool(ant_info)
        reset_target = bool(reset_target)
        if isinstance(maze, str) and maze not in MAPS:
            raise KeyError(f"unknown maze {maze!r}")
        if reward_type not in ("sparse", "dense"):
            raise ValueError("reward_type must be 'sparse' or 'dense'")
        self.maze_name, self.reward_type = maze, reward_type
        self.continuing_task, self.reset_target = continuing_task, reset_target
        self.scaling, self.frame_skip = cfg["scaling"], (self.ant.frame_skip if self.ant else cfg["frame_skip"])
        named = isinstance(maze, str)
        if maze_map is not None:
            if not named:
                raise ValueError("give the layout once: as `maze_map=` or as an explicit `maze` cell list, not both")
            layout = check_maze_map(maze_map, cfg["scaling"], fallbacks=not v3)
        else:
            layout = MAPS[maze] if named else maze
        self.cells = MazeCells(layout, cfg["scaling"], fallbacks=not v3)
        # generate_reset_pos draws the start again while it lies within this distance of the goal (maze_v4.py:290; maze.py:194)
        self.separation = 0.5 if v3 else 0.5 * cfg["scaling"]
        if model is None and not named:
            raise ValueError("an explicit maze map needs its compiled `model` (see models.compile_maze_model)")
        if model is not None:
            m = model
        else:
            m = build_maze_model(self.agent, layout) if maze_map is not None else load_model(model_name(self.agent, maze))
        # Ant-v5 keyword [ext]: AntMaze_*-v5 observes the clipped per-body contact forces (ant_maze_v5.py:99: (105,) = 27 + 13 x 6);
        # AntMaze_*-v4 (Ant-v4, use_contact_forces False) and the point agent do not.  The registry sets it per id.
        self.include_cfrc = bool(include_cfrc_ext_in_observation) and self.agent == "ant"
        t = make_maze_task(m, reward_type, self.agent, self.include_cfrc, self.frame_skip, self.ant.touch_mode(self.ant_info) if self.ant else None)
        box = lambda n: Box(-np.inf, np.inf, shape=(n,), dtype=np.float64)
        # "device": goal / reset cells and their noise are drawn inside the library (b200sim_reset_maze, csrc/reset_sample.cuh).
        # TimeLimit and compute_terminated (maze_v4.py:390-398: success ends the episode unless continuing_task) run inside the
        # step kernel
        super().__init__(model=m, task=t, fields=(("qpos", m.nq), ("qvel", m.nv), ("warm", m.nv), ("ctrl", m.nu), ("goal", 2)),
                         action_space=Box(-1.0, 1.0, shape=(m.nu,), dtype=np.float32),
                         observation_space=DictSpace(dict(observation=box(t.nobs), achieved_goal=box(2), desired_goal=box(2))),
                         backend_factory=backend_factory or CudaBackend, num_envs=num_envs, device=device,
                         max_episode_steps=(cfg["steps"][maze] if named else None) if max_episode_steps is None else max_episode_steps,
                         autoreset_mode=autoreset_mode, rng_mode=rng_mode, n_substeps=self.frame_skip, kwargs=kwargs,
                         terminate_on_success=not continuing_task)
        # the Ant's frame_skip: the inner AntEnv's render rate (MujocoEnv: round(1 / dt))
        self.metadata["render_fps"] = int(round(1.0 / self.dt)) if self.ant is not None and self.ant.frame_skip_given else cfg["fps"]
        # the ant kernel build (b200sim_set_ant_info): the Ant's keywords; with ant_info a fresh [N, 9] info row buffer per call
        # (_new_ant_rows) and the reset positions Ant-v5 measures distance_from_origin from
        self._ant_rows = self._ant_origin = None
        if self.ant is not None and t.touch_mode >= 2:
            if getattr(self.backend, "set_ant_info", None) is None:
                raise NotImplementedError(f"{type(self.backend).__name__} cannot run the Ant's keywords (no set_ant_info)")
            self._ant_params = self.ant.params()
            self._ant_origin = torch.zeros((self.num_envs, 2), dtype=torch.float32, device=self.device)
            self.backend.set_ant_info(self._ant_params, None, self._ant_origin)
        self._ant_keys = self.ant.info_keys() if self.ant_info else ((), ())
        if self._np_rngs is None:
            self._np_rngs = self._new_np_rngs([None] * self.num_envs)
        self.init_qpos = torch.as_tensor(np.array(m.qpos0), dtype=torch.float32, device=self.device)
        self._goal_loc = torch.as_tensor(self.cells.goal_locations, dtype=torch.float32, device=self.device)
        self._reset_loc = torch.as_tensor(self.cells.reset_locations, dtype=torch.float32, device=self.device)
        # update_goal (maze_v4.py:400-418) acts only in a continuing task with reset_target and more than one goal location; in
        # rng_mode="device" the step launch does it (b200sim_set_goal_update), keyed by each env's Philox key (vector.py)
        self._goal_update_on = continuing_task and reset_target and len(self.cells.goal_locations) > 1
        # AntMaze-v3's redraw (maze.py:283-302) acts in a continuing task with more than one goal location; in rng_mode="device" the
        # step launch does it (b200sim_set_goal_redraw), rewriting the reward too
        self._goal_redraw_on = v3 and continuing_task and len(self.cells.goal_locations) > 1
        self._goal_update_seed = None
        if self.rng_mode == "device" and self._goal_update_on and getattr(self.backend, "set_goal_update", None) is None:
            raise NotImplementedError(f"{type(self.backend).__name__} cannot update goals on the device (no set_goal_update)")
        if self.rng_mode == "device" and self._goal_redraw_on and getattr(self.backend, "set_goal_redraw", None) is None:
            raise NotImplementedError(f"{type(self.backend).__name__} cannot redraw goals on the device (no set_goal_redraw)")

    # ------------------------------------------------------------------ sampling (MazeEnv.reset, maze_v4.py:299-358)
    def _noise_np(self, rng, xy):
        nx = rng.uniform(low=-NOISE, high=NOISE) * self.scaling
        ny = rng.uniform(low=-NOISE, high=NOISE) * self.scaling
        return np.array([xy[0] + nx, xy[1] + ny])

    def _sample_np(self, i, options):
        rng, cells = self._np_rngs[i], self.cells
        options = options or {}
        if options.get("goal_cell") is not None:
            gc = options["goal_cell"]
            assert cells.length > gc[0] and cells.width > gc[1] and cells.maze_map[gc[0]][gc[1]] != 1, f"Goal can't be placed in a wall cell, {gc}"
            goal = cells.cell_rowcol_to_xy(gc)
        else:
            goal = cells.goal_locations[rng.integers(low=0, high=len(cells.goal_locations))].copy()
        goal = self._noise_np(rng, goal)
        if options.get("reset_cell") is not None:
            rc = options["reset_cell"]
            assert cells.length > rc[0] and cells.width > rc[1] and cells.maze_map[rc[0]][rc[1]] != 1, f"Reset can't be placed in a wall cell, {rc}"
            pos = cells.cell_rowcol_to_xy(rc)
        else:
            pos = goal.copy()
            while np.linalg.norm(pos - goal) <= self.separation:
                pos = cells.reset_locations[rng.integers(low=0, high=len(cells.reset_locations))].copy()
        return goal, self._noise_np(rng, pos)

    def _sample(self, idx, options=None):
        n = idx.numel()
        if self.rng_mode == "numpy" or options:  # explicit cells always go through the reference-ordered numpy path
            gs, ps = zip(*[self._sample_np(i, options) for i in idx.tolist()])
            return (torch.as_tensor(np.array(gs), dtype=torch.float32, device=self.device),
                    torch.as_tensor(np.array(ps), dtype=torch.float32, device=self.device))
        u = lambda *s: torch.rand(*s, generator=self._gen, device=self.device)
        ri = lambda hi, k: torch.randint(0, hi, (k,), generator=self._gen, device=self.device)
        goal = self._goal_loc[ri(len(self._goal_loc), n)] + (u(n, 2) * 2 - 1) * NOISE * self.scaling
        pos = self._reset_loc[ri(len(self._reset_loc), n)]
        bad = torch.linalg.norm(pos - goal, dim=1) <= self.separation
        while bool(bad.any()):
            pos[bad] = self._reset_loc[ri(len(self._reset_loc), int(bad.sum()))]
            bad = torch.linalg.norm(pos - goal, dim=1) <= self.separation
        return goal, pos + (u(n, 2) * 2 - 1) * NOISE * self.scaling

    def _rest_record(self):   # ant_env.init_qpos, zero velocities
        rest = torch.zeros(self.backend.state.shape[1], dtype=torch.float32, device=self.device)
        rest[self._sl["qpos"]] = self.init_qpos
        return rest

    def _device_tables(self):
        if self._dev_reset is None:
            from ._lib import MazeResetC

            p = MazeResetC()
            p.n_goal, p.n_reset, p.scaling, p.noise = len(self._goal_loc), len(self._reset_loc), float(self.scaling), float(NOISE)
            p.separation = self.separation if self._v3 else 0.0   # 0: the library's half cell, bit for bit the v4 draw
            self._dev_reset = (p, self._rest, self._goal_loc.contiguous(), self._reset_loc.contiguous())
        # first reset, or a new seed: the slot's seed keys the draws of a backend without per-env keys (vector.py)
        if (self._goal_update_on or self._goal_redraw_on) and self._goal_update_seed != self._dev_seed:
            setter = self.backend.set_goal_redraw if self._goal_redraw_on else self.backend.set_goal_update
            setter(self._dev_reset[2], self.scaling, NOISE, self._dev_seed, self.env_offset, self._episode)
            self._goal_update_seed = self._dev_seed
        return self._dev_reset

    def _device_reset(self, mask, out):
        p, rest, gl, rl = self._device_tables()
        self.backend.reset_maze(mask.to(torch.uint8), rest, p, gl, rl, self._dev_seed, self.env_offset, self._episode, out)
        self._elapsed.masked_fill_(mask, 0)
        self._set_origin(mask, out)

    def _reset_envs(self, mask, out, options=None):
        if self.rng_mode == "device":
            if not options:   # explicit cells keep the reference-ordered host path
                return self._device_reset(mask, out)
            # ... and start a new episode of the device streams too, so that the next goal updates draw fresh numbers
            self._device_tables()
            self._episode += mask.to(torch.int32)
        idx = self._mask_indices(mask)
        if idx.numel() == 0:
            return
        st, sl = self.backend.state, self._sl
        goal, pos = self._sample(idx, options)
        rec = self._rest.expand(idx.numel(), -1).clone()
        rec[:, sl["qpos"].start: sl["qpos"].start + 2] = pos    # ant_env.init_qpos with [:2] = reset_pos (ant_maze_v5.py:285)
        rec[:, sl["goal"]] = goal
        st[idx] = rec
        self._elapsed[idx] = 0
        self.backend.refresh(mask.to(torch.uint8), out)
        self._set_origin(mask, out)

    def _set_origin(self, mask, out):
        """Ant-v5's init_qpos[:2] <- the reset position of the envs just reset (ant_maze_v5.py:285); set_state leaves it alone."""
        if self._ant_origin is not None:
            torch.where(mask[:, None], out["achieved"], self._ant_origin, out=self._ant_origin)

    def _new_ant_rows(self):
        """Every call that returns info gets its own rows, so that the info of one step stays valid after the next."""
        if self.ant_info:
            self._ant_rows = torch.zeros((self.num_envs, len(ANT_INFO_COLUMNS)), dtype=torch.float32, device=self.device)
            self.backend.set_ant_info(self._ant_params, self._ant_rows, self._ant_origin)

    # ------------------------------------------------------------------ gymnasium API
    # ant_info=True adds the Ant's info (views of the call's [N, 9] rows, each key with its `_key` mask).  Gymnasium's vector
    # convention: an env reset instead of stepped (NEXT_STEP) reports the reset keys (the refresh of its reset wrote them) and 0 under the
    # other keys, which its mask marks absent; SAME_STEP puts the finished episodes' keys into final_info.
    def reset(self, *, seed=None, options=None):
        self._new_ant_rows()
        return super().reset(seed=seed, options=options)

    def _reset_info(self, out):
        info = {} if self._v3 else {"success": out["success"] > 0}   # v3: Ant-v4's reset info, {}
        for k, c in self._ant_keys[1]:
            info[k], info["_" + k] = self._ant_rows[:, c], self._const_true
        return info

    def _kernel_input(self, actions):
        self._new_ant_rows()
        return super()._kernel_input(actions)

    def _success(self, column):
        return column > 0

    def _step_results(self, out):
        reward, terminated, truncated, info = super()._step_results(out)
        if not self._v3:   # v3's step info is the Ant's alone (ant_maze_v3.py:91)
            info["success"] = self._success(out["success"])
        for k, c in self._ant_keys[0]:
            info[k], info["_" + k] = self._ant_rows[:, c], self._const_true
        return reward, terminated, truncated, info

    def _step_only_masks(self, info, absent):
        present = ~absent
        reset_keys = {k for k, _ in self._ant_keys[1]}
        for k, _ in self._ant_keys[0]:
            if k not in reset_keys:
                info["_" + k] = present

    def _mask_results(self, out, pre, reward, terminated, truncated, info):
        if "success" in info:
            info["success"] = info["success"] & ~pre
        if self.ant_info:
            self._step_only_masks(info, pre)
        return super()._mask_results(out, pre, reward, terminated, truncated, info)

    def _final_info(self, out, info, done):
        final = {} if self._v3 else super()._final_info(out, info, done)
        if self.ant_info:
            rows = self._ant_rows.clone()    # the refresh of the reset below rewrites the finished envs' rows with their reset info
            for k, c in self._ant_keys[0]:
                final[k], final["_" + k] = rows[:, c], done
            self._step_only_masks(info, done)
        return final

    def _after_autoreset(self, out, info):
        # rng_mode="device": the step launch has updated the goals already (the envs it reset got the reset draw after it)
        if self._goal_update_on and self.rng_mode != "device":
            self._update_goal(info["success"], out)  # maze_v4.py:400-418 (never for the envs that were just reset: `success` is masked)
        if self._goal_redraw_on and self.rng_mode != "device":
            self._redraw_goal(out)                   # maze.py:283-302 (the success column of the envs just reset is masked to 0)

    def _finish_info(self, out, info):
        pass   # `success` as of the step, before a SAME_STEP reset; no mask entry

    def _update_goal(self, success, out):
        """update_goal on the host, from each succeeding env's numpy stream in the reference's order: one read of their achieved
        goals and goals, one write of the new goals."""
        idx = torch.nonzero(success, as_tuple=False).flatten()
        if idx.numel() == 0:
            return
        st, sl = self.backend.state, self._sl
        cur = torch.cat([out["achieved"][idx], st[idx, sl["goal"]]], dim=1).double().cpu().numpy()
        new = cur[:, 2:].copy()
        for k, i in enumerate(idx.tolist()):
            ag, goal, rng = cur[k, :2], new[k], self._np_rngs[i]
            while np.linalg.norm(ag - goal) <= SUCCESS_RADIUS:
                goal = self._noise_np(rng, self.cells.goal_locations[rng.integers(low=0, high=len(self.cells.goal_locations))].copy())
            new[k] = goal
        st[idx, sl["goal"].start:sl["goal"].stop] = torch.as_tensor(new, dtype=torch.float32, device=self.device)

    def _redraw_goal(self, out):
        """AntMaze-v3's redraw on the host: each succeeding env gets one goal cell + noise, and its reward in the packed row becomes
        compute_reward against it (ant_maze_v3.py:94-97).  numpy mode: one draw from each succeeding env's stream in the reference's
        order (`integers`, then two `uniform`s).  torch mode: one candidate for every env from the device generator, applied where
        the success column is 1, with no host synchronisation."""
        st, sl, success = self.backend.state, self._sl["goal"], out["success"] > 0
        if self.rng_mode == "numpy":
            idx = torch.nonzero(success, as_tuple=False).flatten()
            if idx.numel() == 0:
                return
            cells = self.cells.goal_locations
            new = np.array([self._noise_np(self._np_rngs[i], cells[self._np_rngs[i].integers(low=0, high=len(cells))].copy())
                            for i in idx.tolist()])
            new = torch.as_tensor(new, dtype=torch.float32, device=self.device)
            st[idx, sl.start:sl.stop] = new
            out["reward"][idx] = self.backend.compute_reward(out["achieved"][idx], new)
            return
        n = self.num_envs
        gi = torch.randint(0, len(self._goal_loc), (n,), generator=self._gen, device=self.device)
        new = self._goal_loc[gi] + (torch.rand(n, 2, generator=self._gen, device=self.device) * 2 - 1) * NOISE * self.scaling
        st[:, sl] = torch.where(success[:, None], new, st[:, sl])
        out["reward"].copy_(torch.where(success, self.backend.compute_reward(out["achieved"], new), out["reward"]))

    def _reward_np_dtype(self):
        return np.float64

    def compute_terminated(self, achieved_goal, desired_goal, info=None):
        # pure in every version: AntMaze-v3's redraw of self.goal inside compute_terminated (maze.py:289-302) happens in step
        if not self.continuing_task:
            return bool(np.linalg.norm(np.asarray(achieved_goal) - np.asarray(desired_goal)) <= SUCCESS_RADIUS)
        return False


class AntMazeVectorEnv(MazeVectorEnv):
    AGENT = "ant"


class PointMazeVectorEnv(MazeVectorEnv):
    AGENT = "point"
