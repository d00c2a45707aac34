"""The Ant's keywords and per-step info restated on the fp64 oracle (test infrastructure): OracleAntMazeEnv with Ant-v5 / Ant-v4's
frame_skip, contact_force_range, observation and info [ext] (ant_v3.py:76-145 with the v4 / v5 changes), computed from the oracle's
own xpos and cfrc_ext.  The oracle module itself is unchanged."""
from __future__ import annotations

import numpy as np

from gymnasium_robotics_b200.maze import ANT_KEYWORDS
from oracle.ant_maze_env import OracleAntMazeEnv


class OracleAntInfoEnv(OracleAntMazeEnv):
    def __init__(self, maze_map, model, ant_version=5, include_cfrc_ext_in_observation=None, **kw):
        cfg = dict(ANT_KEYWORDS[ant_version])
        cfg.update(kw)
        self.version, self.cfg = ant_version, cfg
        self.include_v5 = ant_version == 5 and bool(include_cfrc_ext_in_observation)
        self.include_v4 = ant_version == 4 and bool(cfg.get("use_contact_forces", False))
        super().__init__(maze_map, model=model, include_cfrc_ext_in_observation=self.include_v5)
        self.FRAME_SKIP = int(cfg.get("frame_skip", 5))
        self.dt = float(model.opt[0]) * self.FRAME_SKIP
        self.torso = int(model.mjbody_rt[1])     # MJCF body 1 ("torso", main_body)
        self.xy = np.zeros(2)                    # the torso's xpos[:2] of the last forward pass

    def contact_forces(self):
        lo, hi = self.cfg["contact_force_range"]
        return np.clip(self._cfrc, lo, hi)

    def _ant_obs(self):
        o = [self.sim.qpos.copy(), self.sim.qvel.copy()]
        if self.include_v5:
            o.append(self.contact_forces()[1:].ravel())
        if self.include_v4:
            o.append(self.contact_forces().ravel())
        return np.concatenate(o)

    def set_state(self, qpos, qvel, goal):
        """MujocoEnv.set_state (mj_forward: xpos of the new state; cfrc_ext is left as it was -- zero here)."""
        self.sim.qpos[:] = qpos
        self.sim.qvel[:] = qvel
        self.goal = np.array(goal, dtype=np.float64)
        self.sim.forward()
        self._cfrc[:] = 0.0
        self.xy = self.sim.xpos[self.torso, :2].copy()

    def reset(self, seed=None, options=None):
        obs, info = super().reset(seed=seed, options=options)
        self.xy = self.sim.xpos[self.torso, :2].copy()
        if self.version == 5:   # Ant-v5 _get_reset_info
            q = self.sim.qpos
            info.update(x_position=q[0], y_position=q[1], distance_from_origin=float(np.linalg.norm(q[:2] - self.init_qpos[:2])))
        return obs, info

    def step(self, action):
        action = np.asarray(action, dtype=np.float64)
        before = self.xy.copy()
        obs, reward, terminated, truncated, info = super().step(action)
        after = self.sim.xpos[self.torso, :2].copy()
        self.xy = after
        vx, vy = (after - before) / self.dt
        cfg, q, v = self.cfg, self.sim.qpos, self.sim.qvel
        ctrl_cost = cfg["ctrl_cost_weight"] * float(np.sum(np.square(action)))
        contact_cost = cfg["contact_cost_weight"] * float(np.sum(np.square(self.contact_forces())))
        lo, hi = cfg["healthy_z_range"]
        healthy = bool(np.isfinite(np.concatenate([q, v])).all() and lo <= q[2] <= hi)
        if self.version == 5:
            info.update(x_position=q[0], y_position=q[1], distance_from_origin=float(np.linalg.norm(q[:2] - self.init_qpos[:2])),
                        x_velocity=vx, y_velocity=vy, reward_forward=cfg["forward_reward_weight"] * vx, reward_ctrl=-ctrl_cost,
                        reward_contact=-contact_cost, reward_survive=cfg["healthy_reward"] * float(healthy))
        else:
            info.update(x_position=after[0], y_position=after[1], distance_from_origin=float(np.linalg.norm(after)), x_velocity=vx,
                        y_velocity=vy, reward_forward=vx, forward_reward=vx,
                        reward_ctrl=-contact_cost if cfg["use_contact_forces"] else -ctrl_cost,
                        reward_survive=cfg["healthy_reward"] * float(healthy or cfg["terminate_when_unhealthy"]))
        return obs, reward, terminated, truncated, info
