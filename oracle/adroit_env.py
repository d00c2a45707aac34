"""Single-env numpy restatement of the reference's AdroitHandHammer environment on top of the CPU oracle.
TEST INFRASTRUCTURE ONLY (see oracle/oracle.c header; parity unpinned for the physics).

Restates envs/adroit_hand/adroit_hammer.py (AdroitHandHammerEnv) on top of what Gymnasium's un-vendored `MujocoEnv` does
(`do_simulation`: ctrl <- action, mj_step(nstep=frame_skip); `set_state`: qpos/qvel <- ..., mj_forward; `reset`:
mj_resetData then reset_model); every method cites the lines it follows (paths relative to /root/reference/gymnasium_robotics/).
The noslip post-solver the model asks for (adroit_assets.xml:3) is not restated (DESIGN.md).
"""
from __future__ import annotations

import numpy as np

from gymnasium_robotics_b200 import rotations
from .oracle_sim import OracleSim


class OracleAdroitHammerEnv:
    def __init__(self, model, reward_type="dense", frame_skip=5, noslip=True):
        self.model, self.frame_skip = model, frame_skip
        if reward_type.lower() not in ("dense", "sparse"):   # adroit_hammer.py:219-227
            raise ValueError(f"Unknown reward type, expected `dense` or `sparse` but got {reward_type}")
        self.sparse_reward = reward_type.lower() == "sparse"
        self.sim = OracleSim(model)
        # adroit_assets.xml:3 noslip_iterations="20": on, as in the reference; the CUDA path does not run the pass (DESIGN.md deviation
        # 12), so its parity tests build the oracle env with noslip=False and a separate test bounds the difference
        self.sim.set_noslip(noslip)
        m = model
        # adroit_hammer.py:264-270 (ids by name)
        self.target_obj_site_id = m.site_id("S_target")
        self.S_grasp_site_id = m.site_id("S_grasp")
        self.obj_body_id = int(m.names["body_map"]["Object"])
        self.tool_site_id = m.site_id("tool")
        self.goal_site_id = m.site_id("nail_goal")
        self.target_body_id = int(m.names["body_map"]["nail_board"])
        cr = np.asarray(m.act_ctrlrange, dtype=np.float64).reshape(-1, 2)
        self.act_mean = np.mean(cr, axis=1)                                  # :271
        self.act_rng = 0.5 * (cr[:, 1] - cr[:, 0])                           # :272-274
        self.np_random = np.random.Generator(np.random.PCG64(np.random.SeedSequence(None)))
        self.sim.forward()
        self.init_qpos, self.init_qvel = self.sim.qpos.copy(), self.sim.qvel.copy()   # MujocoEnv.__init__

    def step(self, a):  # adroit_hammer.py:291-335
        s = self.sim
        a = np.clip(a, -1.0, 1.0)
        a = self.act_mean + a * self.act_rng
        s.ctrl[:] = a                      # MujocoEnv.do_simulation
        s.step(self.frame_skip)
        obs = self._get_obs()
        reward, goal_achieved = self.reward()
        return obs, reward, False, False, dict(success=goal_achieved)

    def reward(self):
        """(reward, goal_achieved) of step() at the current, forwarded state."""
        s = self.sim
        hamm_pos = s.xpos[self.obj_body_id].ravel()
        palm_pos = s.site_xpos[self.S_grasp_site_id].ravel()
        head_pos = s.site_xpos[self.tool_site_id].ravel()
        nail_pos = s.site_xpos[self.target_obj_site_id].ravel()
        goal_pos = s.site_xpos[self.goal_site_id].ravel()
        goal_distance = np.linalg.norm(nail_pos - goal_pos)
        goal_achieved = goal_distance < 0.01
        reward = 10.0 if goal_achieved else -0.1
        if not self.sparse_reward:
            reward = -0.1 * np.linalg.norm(palm_pos - hamm_pos)
            reward -= np.linalg.norm(head_pos - nail_pos)
            reward -= 10 * np.linalg.norm(nail_pos - goal_pos)
            reward -= 1e-2 * np.linalg.norm(s.qvel.ravel())
            if hamm_pos[2] > 0.04 and head_pos[2] > 0.04:
                reward += 2
            if goal_distance < 0.020:
                reward += 25
            if goal_distance < 0.010:
                reward += 75
        return reward, goal_achieved

    def _get_obs(self):  # adroit_hammer.py:337-357
        s = self.sim
        qp = s.qpos.ravel()
        qv = np.clip(s.qvel.ravel(), -1.0, 1.0)
        obj_pos = s.xpos[self.obj_body_id].ravel()
        obj_rot = rotations.quat2euler(s.xquat[self.obj_body_id].ravel()).ravel()
        palm_pos = s.site_xpos[self.S_grasp_site_id].ravel()
        target_pos = s.site_xpos[self.target_obj_site_id].ravel()
        nail_impact = np.clip(s.sensordata[0], -1.0, 1.0)    # the compiled model keeps only "S_nail"
        return np.concatenate([qp[:-6], qv[-6:], palm_pos, obj_pos, obj_rot, target_pos, np.array([nail_impact])])

    def reset(self, *, seed=None, options=None):  # MujocoEnv.reset + adroit_hammer.py:359-370
        if seed is not None:
            self.np_random = np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))
        self.sim.reset_data()
        obs = self.reset_model()
        if options is not None and "initial_state_dict" in options:
            self.set_env_state(options["initial_state_dict"])
            obs = self._get_obs()
        return obs, {}

    def reset_model(self):  # adroit_hammer.py:372-378
        self.sim.body_pos[self.target_body_id, 2] = self.np_random.uniform(low=0.1, high=0.25)
        self.set_state(self.init_qpos, self.init_qvel)
        return self._get_obs()

    def set_state(self, qpos, qvel):  # MujocoEnv.set_state
        self.sim.qpos[:] = qpos
        self.sim.qvel[:] = qvel
        self.sim.forward()

    def get_env_state(self):  # adroit_hammer.py:380-388
        return dict(qpos=self.sim.qpos.ravel().copy(), qvel=self.sim.qvel.ravel().copy(),
                    board_pos=self.sim.body_pos[self.target_body_id].copy(),
                    target_pos=self.sim.site_xpos[self.target_obj_site_id].ravel().copy())

    def set_env_state(self, state_dict):  # adroit_hammer.py:390-402
        self.sim.body_pos[self.target_body_id] = state_dict["board_pos"]
        self.set_state(state_dict["qpos"], state_dict["qvel"])


class OracleAdroitRelocateEnv(OracleAdroitHammerEnv):
    """envs/adroit_hand/adroit_relocate.py (AdroitHandRelocateEnv).  The `target` site sits on the world body, so its
    site_xpos is its (per-episode) site_pos: kept as `self.target_pos`."""

    def __init__(self, model, reward_type="dense", frame_skip=5, noslip=True):
        self.model, self.frame_skip = model, frame_skip
        self.sparse_reward = reward_type.lower() == "sparse"
        self.sim = OracleSim(model)
        # adroit_assets.xml:3 noslip_iterations="20": on, as in the reference; the CUDA path does not run the pass (DESIGN.md deviation
        # 12), so its parity tests build the oracle env with noslip=False and a separate test bounds the difference
        self.sim.set_noslip(noslip)
        m = model
        self.S_grasp_site_id = m.site_id("S_grasp")                 # adroit_relocate.py:257-259
        self.obj_body_id = int(m.names["body_map"]["Object"])
        self.target_pos = np.asarray(m.site_pos).reshape(-1, 3)[m.site_id("target")].copy()
        cr = np.asarray(m.act_ctrlrange, dtype=np.float64).reshape(-1, 2)
        self.act_mean, self.act_rng = np.mean(cr, axis=1), 0.5 * (cr[:, 1] - cr[:, 0])
        self.np_random = np.random.Generator(np.random.PCG64(np.random.SeedSequence(None)))
        self.sim.forward()
        self.init_qpos, self.init_qvel = self.sim.qpos.copy(), self.sim.qvel.copy()

    def step(self, a):  # adroit_relocate.py:288-329
        s = self.sim
        a = np.clip(a, -1.0, 1.0)
        a = self.act_mean + a * self.act_rng
        s.ctrl[:] = a
        s.step(self.frame_skip)
        obs = self._get_obs()
        reward, goal_achieved = self.reward()
        return obs, reward, False, False, dict(success=goal_achieved)

    def reward(self):
        """(reward, goal_achieved) of step() at the current, forwarded state."""
        s = self.sim
        obj_pos = s.xpos[self.obj_body_id].ravel()
        palm_pos = s.site_xpos[self.S_grasp_site_id].ravel()
        target_pos = self.target_pos
        goal_distance = float(np.linalg.norm(obj_pos - target_pos))
        goal_achieved = goal_distance < 0.1
        reward = 10.0 if goal_achieved else -0.1
        if not self.sparse_reward:
            reward = -0.1 * np.linalg.norm(palm_pos - obj_pos)
            if obj_pos[2] > 0.04:
                reward += 1.0
                reward += -0.5 * np.linalg.norm(palm_pos - target_pos)
                reward += -0.5 * np.linalg.norm(obj_pos - target_pos)
            if goal_distance < 0.1:
                reward += 10.0
            if goal_distance < 0.05:
                reward += 20.0
        return reward, goal_achieved

    def _get_obs(self):  # adroit_relocate.py:331-339
        s = self.sim
        qpos = s.qpos.ravel()
        obj_pos = s.xpos[self.obj_body_id].ravel()
        palm_pos = s.site_xpos[self.S_grasp_site_id].ravel()
        return np.concatenate([qpos[:-6], palm_pos - obj_pos, palm_pos - self.target_pos, obj_pos - self.target_pos])

    def reset_model(self):  # adroit_relocate.py:354-373
        self.sim.body_pos[self.obj_body_id, 0] = self.np_random.uniform(low=-0.15, high=0.15)
        self.sim.body_pos[self.obj_body_id, 1] = self.np_random.uniform(low=-0.15, high=0.3)
        self.target_pos[0] = self.np_random.uniform(low=-0.2, high=0.2)
        self.target_pos[1] = self.np_random.uniform(low=-0.2, high=0.2)
        self.target_pos[2] = self.np_random.uniform(low=0.15, high=0.35)
        self.set_state(self.init_qpos, self.init_qvel)
        return self._get_obs()

    def get_env_state(self):  # adroit_relocate.py:375-388
        return dict(qpos=self.sim.qpos.ravel().copy(), qvel=self.sim.qvel.ravel().copy(),
                    hand_pos=self.sim.site_xpos[self.S_grasp_site_id].ravel().copy(),
                    obj_pos=self.sim.body_pos[self.obj_body_id].copy(), target_pos=self.target_pos.copy())

    def set_env_state(self, state_dict):  # adroit_relocate.py:390-402
        self.sim.body_pos[self.obj_body_id] = state_dict["obj_pos"]
        self.target_pos[:] = state_dict["target_pos"]
        self.set_state(state_dict["qpos"], state_dict["qvel"])


class OracleAdroitPenEnv(OracleAdroitHammerEnv):
    """envs/adroit_hand/adroit_pen.py (AdroitHandPenEnv)."""

    def __init__(self, model, reward_type="dense", frame_skip=5, noslip=True):
        self.model, self.frame_skip = model, frame_skip
        self.sparse_reward = reward_type.lower() == "sparse"
        self.sim = OracleSim(model)
        # adroit_assets.xml:3 noslip_iterations="20": on, as in the reference; the CUDA path does not run the pass (DESIGN.md deviation
        # 12), so its parity tests build the oracle env with noslip=False and a separate test bounds the difference
        self.sim.set_noslip(noslip)
        m = model
        self.target_obj_body_id = int(m.names["body_map"]["target"])       # adroit_pen.py:264-271
        self.obj_body_id = int(m.names["body_map"]["Object"])
        self.eps_ball_site_id = m.site_id("eps_ball")
        self.obj_t_site_id, self.obj_b_site_id = m.site_id("object_top"), m.site_id("object_bottom")
        self.tar_t_site_id, self.tar_b_site_id = m.site_id("target_top"), m.site_id("target_bottom")
        cr = np.asarray(m.act_ctrlrange, dtype=np.float64).reshape(-1, 2)
        self.act_mean, self.act_rng = np.mean(cr, axis=1), 0.5 * (cr[:, 1] - cr[:, 0])
        self.np_random = np.random.Generator(np.random.PCG64(np.random.SeedSequence(None)))
        self.sim.forward()
        self.init_qpos, self.init_qvel = self.sim.qpos.copy(), self.sim.qvel.copy()
        self.pen_length = self.tar_length = 1.0

    def _orien(self):
        s = self.sim
        return ((s.site_xpos[self.obj_t_site_id] - s.site_xpos[self.obj_b_site_id]) / self.pen_length,
                (s.site_xpos[self.tar_t_site_id] - s.site_xpos[self.tar_b_site_id]) / self.tar_length)

    def step(self, a):  # adroit_pen.py:288-337
        s = self.sim
        a = np.clip(a, -1.0, 1.0)
        a = self.act_mean + a * self.act_rng
        s.ctrl[:] = a
        s.step(self.frame_skip)
        obs = self._get_obs()
        reward, goal_achieved = self.reward()
        return obs, reward, False, False, dict(success=goal_achieved)

    def reward(self):
        """(reward, goal_achieved) of step() at the current, forwarded state."""
        s = self.sim
        obj_pos = s.xpos[self.obj_body_id].ravel()
        desired_loc = s.site_xpos[self.eps_ball_site_id].ravel()
        obj_orien, desired_orien = self._orien()
        goal_distance = np.linalg.norm(obj_pos - desired_loc)
        orien_similarity = np.dot(obj_orien, desired_orien)
        goal_achieved = goal_distance < 0.075 and orien_similarity > 0.95
        reward = 10.0 if goal_achieved else -0.1
        if not self.sparse_reward:
            reward = -goal_distance + orien_similarity
            if goal_distance < 0.075 and orien_similarity > 0.9:
                reward += 10
            if goal_distance < 0.075 and orien_similarity > 0.95:
                reward += 50
            if obj_pos[2] < 0.075:
                reward -= 5
        return reward, goal_achieved

    def _get_obs(self):  # adroit_pen.py:339-365
        s = self.sim
        qpos = s.qpos.ravel()
        obj_vel = s.qvel[-6:].ravel()
        obj_pos = s.xpos[self.obj_body_id].ravel()
        desired_pos = s.site_xpos[self.eps_ball_site_id].ravel()
        obj_orien, desired_orien = self._orien()
        return np.concatenate([qpos[:-6], obj_pos, obj_vel, obj_orien, desired_orien, obj_pos - desired_pos, obj_orien - desired_orien])

    def reset_model(self):  # adroit_pen.py:379-399
        desired_orien = np.zeros(3)
        desired_orien[0] = self.np_random.uniform(low=-1, high=1)
        desired_orien[1] = self.np_random.uniform(low=-1, high=1)
        self.sim.body_quat[self.target_obj_body_id] = rotations.euler2quat(desired_orien)
        self.set_state(self.init_qpos, self.init_qvel)
        s = self.sim
        self.pen_length = np.linalg.norm(s.site_xpos[self.obj_t_site_id] - s.site_xpos[self.obj_b_site_id])
        self.tar_length = np.linalg.norm(s.site_xpos[self.tar_t_site_id] - s.site_xpos[self.tar_b_site_id])
        return self._get_obs()

    def get_env_state(self):  # adroit_pen.py:401-409
        return dict(qpos=self.sim.qpos.ravel().copy(), qvel=self.sim.qvel.ravel().copy(),
                    desired_orien=self.sim.body_quat[self.target_obj_body_id].ravel().copy())

    def set_env_state(self, state_dict):  # adroit_pen.py:411-430
        self.sim.body_quat[self.target_obj_body_id] = state_dict["desired_orien"]
        self.set_state(state_dict["qpos"], state_dict["qvel"])


class OracleAdroitDoorEnv(OracleAdroitHammerEnv):
    """envs/adroit_hand/adroit_door.py (AdroitHandDoorEnv)."""

    def __init__(self, model, reward_type="dense", frame_skip=5, noslip=True):
        self.model, self.frame_skip = model, frame_skip
        self.sparse_reward = reward_type.lower() == "sparse"
        self.sim = OracleSim(model)
        # adroit_assets.xml:3 noslip_iterations="20": on, as in the reference; the CUDA path does not run the pass (DESIGN.md deviation
        # 12), so its parity tests build the oracle env with noslip=False and a separate test bounds the difference
        self.sim.set_noslip(noslip)
        m = model
        self.door_hinge_addrs = int(m.jnt_dofadr[m.joint_id("door_hinge")])      # adroit_door.py:258-263
        self.grasp_site_id, self.handle_site_id = m.site_id("S_grasp"), m.site_id("S_handle")
        self.door_body_id = int(m.names["body_map"]["frame"])
        cr = np.asarray(m.act_ctrlrange, dtype=np.float64).reshape(-1, 2)
        self.act_mean, self.act_rng = np.mean(cr, axis=1), 0.5 * (cr[:, 1] - cr[:, 0])
        self.np_random = np.random.Generator(np.random.PCG64(np.random.SeedSequence(None)))
        self.sim.forward()
        self.init_qpos, self.init_qvel = self.sim.qpos.copy(), self.sim.qvel.copy()

    def step(self, a):  # adroit_door.py:279-316
        s = self.sim
        a = np.clip(a, -1.0, 1.0)
        a = self.act_mean + a * self.act_rng
        s.ctrl[:] = a
        s.step(self.frame_skip)
        obs = self._get_obs()
        reward, goal_achieved = self.reward()
        return obs, reward, False, False, dict(success=goal_achieved)

    def reward(self):
        """(reward, goal_achieved) of step() at the current, forwarded state."""
        s = self.sim
        goal_distance = s.qpos[self.door_hinge_addrs]
        goal_achieved = goal_distance >= 1.35
        reward = 10.0 if goal_achieved else -0.1
        if not self.sparse_reward:
            handle_pos = s.site_xpos[self.handle_site_id].ravel()
            palm_pos = s.site_xpos[self.grasp_site_id].ravel()
            reward = -0.1 * np.linalg.norm(palm_pos - handle_pos)
            reward += -0.1 * (goal_distance - 1.57) * (goal_distance - 1.57)
            reward += -1e-5 * np.sum(s.qvel**2)
            if goal_distance > 0.2:
                reward += 2
            if goal_distance > 1.0:
                reward += 8
            if goal_distance > 1.35:
                reward += 10
        return reward, goal_achieved

    def _get_obs(self):  # adroit_door.py:318-344
        s = self.sim
        qpos = s.qpos.ravel()
        handle_pos = s.site_xpos[self.handle_site_id].ravel()
        palm_pos = s.site_xpos[self.grasp_site_id].ravel()
        door_pos = np.array([s.qpos[self.door_hinge_addrs]])
        door_open = 1.0 if door_pos > 1.0 else -1.0
        latch_pos = qpos[-1]
        return np.concatenate([qpos[1:-2], [latch_pos], door_pos, palm_pos, handle_pos, palm_pos - handle_pos, [door_open]])

    def reset_model(self):  # adroit_door.py:359-371
        self.sim.body_pos[self.door_body_id, 0] = self.np_random.uniform(low=-0.3, high=-0.2)
        self.sim.body_pos[self.door_body_id, 1] = self.np_random.uniform(low=0.25, high=0.35)
        self.sim.body_pos[self.door_body_id, 2] = self.np_random.uniform(low=0.252, high=0.35)
        self.set_state(self.init_qpos, self.init_qvel)
        return self._get_obs()

    def get_env_state(self):  # adroit_door.py:373-381
        return dict(qpos=self.sim.qpos.ravel().copy(), qvel=self.sim.qvel.ravel().copy(),
                    door_body_pos=self.sim.body_pos[self.door_body_id].ravel().copy())

    def set_env_state(self, state_dict):  # adroit_door.py:383-402
        self.sim.body_pos[self.door_body_id] = state_dict["door_body_pos"]
        self.set_state(state_dict["qpos"], state_dict["qvel"])
