"""AntMaze-v3 restated on the fp64 oracle (test infrastructure): envs/maze/maze.py's task logic on Gymnasium's Ant-v4, as
ant_maze_v3.py wraps it.  The oracle module itself is unchanged; the Ant-v4 observation and info come from tests/ant_info_oracle.py.

  * the start draw: generate_reset_pos rejects starts within 0.5 of the goal (maze.py:189-200), not half a cell;
  * a labelled layout gets no empty-cell fallbacks (maze.py:140-150; the built-in maps are unaffected);
  * step (ant_maze_v3.py:90-102): compute_terminated redraws the goal once, with no rejection, when the ant is within 0.45 of it in a
    continuing task with more than one goal location (maze.py:283-302), and compute_reward runs after it, against the new goal; the
    observation's desired_goal was copied before, so it is the old goal;
  * the info is Ant-v4's: its step info, and {} at reset (no `success` key)."""
from __future__ import annotations

import numpy as np

from oracle.maze import MazeResetLogic, compute_reward
from tests.ant_info_oracle import OracleAntInfoEnv


class MazeResetLogicV3(MazeResetLogic):
    """MazeEnv.reset of envs/maze/maze.py:202-254: the same draw order as maze_v4 with the 0.5 start separation."""

    def generate_reset_pos(self, goal):
        reset_pos = goal.copy()
        while np.linalg.norm(reset_pos - goal) <= 0.5:   # maze.py:194
            idx = self.np_random.integers(low=0, high=len(self.maze.unique_reset_locations))
            reset_pos = self.maze.unique_reset_locations[idx].copy()
        return reset_pos


def redraw_v3(logic, achieved_goal, goal, continuing_task=True):
    """compute_terminated of maze.py:283-302 for a continuing task: (new goal, whether it was drawn)."""
    if continuing_task and bool(np.linalg.norm(achieved_goal - goal) <= 0.45) and len(logic.maze.unique_goal_locations) > 1:
        return logic.add_xy_position_noise(logic.generate_target_goal()), True
    return goal, False


class OracleAntMazeV3Env(OracleAntInfoEnv):
    def __init__(self, maze_map, model, reward_type="sparse", continuing_task=True, **ant_kw):
        super().__init__(maze_map, model, ant_version=4, **ant_kw)
        rng = self.logic.np_random
        self.logic = MazeResetLogicV3(maze_map, maze_size_scaling=4.0, position_noise_range=0.25)
        self.logic.np_random = rng
        self.reward_type, self.continuing_task = reward_type, continuing_task

    def reset(self, seed=None, options=None):
        obs, _ = super().reset(seed=seed, options=options)
        return obs, {}                                   # Ant-v4's reset info

    def step(self, action):
        obs, _, _, truncated, info = super().step(action)   # Ant-v4 physics, observation and info; its `success` is not v3's
        info.pop("success", None)
        ag = obs["achieved_goal"]
        terminated = (not self.continuing_task) and bool(np.linalg.norm(ag - self.goal) <= 0.45)
        self.goal, _ = redraw_v3(self.logic, ag, self.goal, self.continuing_task)
        reward = compute_reward(ag, self.goal, self.reward_type)      # after the redraw (ant_maze_v3.py:94-97)
        return obs, float(reward), terminated, truncated, info
