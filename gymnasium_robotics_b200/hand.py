"""Batched Shadow-Hand block manipulation envs on the CUDA simulator: the vector-env replacement for
`gym.make_vec("HandManipulateBlockRotateXYZ-v1", num_envs=N)` and its Z / Parallel / Full siblings.

Mirrors (batched) the reference's Python around the hot path:
  * MujocoHandEnv._set_action                 envs/shadow_dexterous_hand/hand_env.py:42-61   (inside the step kernel)
  * MujocoManipulateEnv._get_obs / reward      envs/shadow_dexterous_hand/manipulate.py:88-138, 298-314 (inside the kernel)
  * MujocoManipulateEnv._reset_sim             manipulate.py:154-224 : randomised object pose, 10 x 20 settle sub-steps
                                               with zero action, retry while the block is not on the palm
  * MujocoManipulateEnv._sample_goal           manipulate.py:226-279
  * BaseRobotEnv.reset/step                    envs/robot_env.py:114-186 ; TimeLimit(100) of the registry (__init__.py:274-284)
The visual-only `target` free body of manipulate_block.xml is not simulated (it is contype 0, written only by
`_render_callback` and never observed), so nq = 24 + 7 and nv = 24 + 6.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import rotations
from ._lib import FetchTaskC
from .fetch import HAND_REF_POINT, CudaBackend, N_SUBSTEPS  # noqa: F401  (HAND_REF_POINT: re-exported)
from .models import load_model
from .spaces import Box, Dict as DictSpace
from .vector import VectorEnv

# target_position / target_rotation of the registered ids (__init__.py:105-395); TARGET_POSITION_RANGE manipulate_block.py:226
HAND_TASKS = {
    "HandManipulateBlockRotateZ": dict(target_position="ignore", target_rotation="z"),
    "HandManipulateBlockRotateParallel": dict(target_position="ignore", target_rotation="parallel"),
    "HandManipulateBlockRotateXYZ": dict(target_position="ignore", target_rotation="xyz"),
    "HandManipulateBlockFull": dict(target_position="random", target_rotation="xyz"),
    "HandManipulateBlock": dict(target_position="random", target_rotation="xyz"),
    # the egg (ellipsoid object, manipulate_egg.py:214-235: same defaults as the block; ids __init__.py:453-640)
    "HandManipulateEggRotate": dict(target_position="ignore", target_rotation="xyz", model="hand_egg", touch_model="hand_egg_touch"),
    "HandManipulateEggFull": dict(target_position="random", target_rotation="xyz", model="hand_egg", touch_model="hand_egg_touch"),
    "HandManipulateEgg": dict(target_position="random", target_rotation="xyz", model="hand_egg", touch_model="hand_egg_touch"),
    # the pen (manipulate_pen.py:216-235: no initial rotation randomisation, z rotation ignored, 5 cm position threshold;
    # ids __init__.py:651-780)
    "HandManipulatePenRotate": dict(target_position="ignore", target_rotation="xyz", model="hand_pen", touch_model="hand_pen_touch",
                                    randomize_initial_rotation=False, ignore_z_target_rotation=True, distance_threshold=0.05),
    "HandManipulatePenFull": dict(target_position="random", target_rotation="xyz", model="hand_pen", touch_model="hand_pen_touch",
                                  randomize_initial_rotation=False, ignore_z_target_rotation=True, distance_threshold=0.05),
    "HandManipulatePen": dict(target_position="random", target_rotation="xyz", model="hand_pen", touch_model="hand_pen_touch",
                              randomize_initial_rotation=False, ignore_z_target_rotation=True, distance_threshold=0.05),
}
TARGET_POSITION_RANGE = np.array([(-0.04, 0.04), (-0.06, 0.02), (0.0, 0.06)])
GOAL_USE_POS, GOAL_USE_ROT, GOAL_IGNORE_Z = 1, 2, 4


TOUCH_MODES = {"off": 0, "sensordata": 1, "boolean": 2, "log": 3}   # manipulate_touch_sensors.py:30-40 touch_get_obs


def make_hand_task(model, target_position, target_rotation, reward_type, distance_threshold, rotation_threshold, n_substeps,
                   touch_get_obs=None, ignore_z_target_rotation=False):
    """b200sim_fetch_task_t for kind 2 (ids resolved the way MujocoModelNames would, utils/mujoco_utils.py:327-469)."""
    m = model
    jobj = m.joint_id("object:joint")
    robot = [j for j, n in enumerate(m.names["joint"]) if n.startswith("robot")]
    assert robot == list(range(len(robot))) and jobj == len(robot), "robot joints must precede the object's free joint"
    t = FetchTaskC()
    t.kind, t.nact, t.ngoal = 2, int(m.nu), 7
    t.n_substeps, t.reward_dense = int(n_substeps), int(reward_type == "dense")
    t.obj_qadr, t.obj_dadr = int(m.jnt_qposadr[jobj]), int(m.jnt_dofadr[jobj])
    t.touch_mode = TOUCH_MODES.get(touch_get_obs, 0) if touch_get_obs is not None else 0
    t.nobs = t.obj_qadr + int(m.nv) + 7 + (int(m.nsensor) if t.touch_mode else 0)
    t.goal_flags = (GOAL_USE_POS if target_position != "ignore" else 0) | (GOAL_USE_ROT if target_rotation != "ignore" else 0) | \
        (GOAL_IGNORE_Z if ignore_z_target_rotation else 0)
    t.distance_threshold, t.rotation_threshold = float(distance_threshold), float(rotation_threshold)
    t.dt = float(m.opt[0] * n_substeps)
    return t


def _goal_space(ngoal, nobs):
    box = lambda n: Box(-np.inf, np.inf, shape=(n,), dtype=np.float64)
    return DictSpace(dict(desired_goal=box(ngoal), achieved_goal=box(ngoal), observation=box(nobs)))


class HandVectorEnv(VectorEnv):
    """Observations, rewards and flags are float32 / bool torch tensors on `device` with a leading `num_envs` axis."""

    def __init__(self, task: str = "HandManipulateBlockRotateXYZ", num_envs: int = 1, reward_type: str = "sparse",
                 max_episode_steps: Optional[int] = 100, device="cuda:0", rng_mode: str = "auto", autoreset_mode: str = "next_step",
                 n_substeps: int = N_SUBSTEPS, backend_factory=None, target_position=None, target_rotation=None,
                 randomize_initial_position=True, randomize_initial_rotation=None, distance_threshold=None,
                 rotation_threshold=0.1, relative_control=False, model=None, touch_get_obs=None,
                 touch_visualisation="on_touch", ignore_z_target_rotation=None, **kwargs):
        if task not in HAND_TASKS:
            raise KeyError(f"unknown Hand task {task!r}")
        if reward_type not in ("sparse", "dense"):
            raise ValueError("reward_type must be 'sparse' or 'dense'")
        if relative_control:
            # hand_env.py:47-57 calls data.get_joint_qpos, which the new mujoco bindings lack: dead code for the -v1 ids
            raise NotImplementedError("relative_control is not available in the reference's -v1 envs either")
        cfg = dict(HAND_TASKS[task])
        # per-object defaults of the reference's env classes (block: manipulate.py:24-40; pen: manipulate_pen.py:216-235)
        randomize_initial_rotation = cfg.get("randomize_initial_rotation", True) if randomize_initial_rotation is None else randomize_initial_rotation
        distance_threshold = cfg.get("distance_threshold", 0.01) if distance_threshold is None else distance_threshold
        ignore_z_target_rotation = cfg.get("ignore_z_target_rotation", False) if ignore_z_target_rotation is None else ignore_z_target_rotation
        self.ignore_z_target_rotation = ignore_z_target_rotation
        self.target_position = target_position or cfg["target_position"]
        self.target_rotation = target_rotation or cfg["target_rotation"]
        assert self.target_position in ("ignore", "fixed", "random")
        assert self.target_rotation in ("ignore", "fixed", "xyz", "z", "parallel")
        self.randomize_initial_position, self.randomize_initial_rotation = randomize_initial_position, randomize_initial_rotation
        self.distance_threshold, self.rotation_threshold = distance_threshold, rotation_threshold
        self.task_name, self.cfg, self.reward_type = task, cfg, reward_type
        # touch_get_obs is None for the plain ids; the *TouchSensors ids pass "boolean" / "sensordata" (or "log" / "off"):
        # they use the model with the 92 touch sites (manipulate_block_touch_sensors.py:72-92)
        self.touch_get_obs = touch_get_obs
        m = model if model is not None else load_model(
            cfg.get("model", "hand_block") if touch_get_obs is None else cfg.get("touch_model", "hand_block_touch"))
        t = make_hand_task(m, self.target_position, self.target_rotation, reward_type, distance_threshold,
                           rotation_threshold, n_substeps, touch_get_obs, ignore_z_target_rotation)
        # "device": start pose and goal are drawn inside the library (b200sim_reset_hand_pose / _goal, csrc/reset_sample.cuh)
        super().__init__(model=m, task=t, fields=(("qpos", m.nq), ("qvel", m.nv), ("warm", m.nv), ("ctrl", m.nu), ("goal", 7)),
                         action_space=Box(-1.0, 1.0, shape=(int(m.nu),), dtype=np.float32), observation_space=_goal_space(7, t.nobs),
                         backend_factory=backend_factory or CudaBackend, num_envs=num_envs, device=device,
                         max_episode_steps=max_episode_steps, autoreset_mode=autoreset_mode, rng_mode=rng_mode,
                         n_substeps=n_substeps, kwargs=kwargs)
        lay = self.backend.layout
        self._obj = slice(lay["qpos"] + t.obj_qadr, lay["qpos"] + t.obj_qadr + 7)
        # robot_env.py:301-303 after _env_setup with initial_qpos = {} (manipulate.py:148-151)
        self.initial_qpos = torch.as_tensor(np.array(m.qpos0), dtype=torch.float32, device=self.device)
        self.initial_qvel = torch.zeros(m.nv, dtype=torch.float32, device=self.device)
        cr = np.asarray(m.act_ctrlrange, dtype=np.float64).reshape(-1, 2)
        self._ctrl_center = torch.as_tensor((cr[:, 0] + cr[:, 1]) / 2.0, dtype=torch.float32, device=self.device)  # _set_action(zeros)
        self._parallel_np = rotations.parallel_quats()
        self._parallel = torch.as_tensor(np.array(self._parallel_np), dtype=torch.float32, device=self.device)
        self._range = torch.as_tensor(TARGET_POSITION_RANGE, dtype=torch.float32, device=self.device)
        self.reset_attempts = 0   # total settle passes run by resets (>= number of resets; diagnostics)

    def _rest_record(self):
        rest = torch.zeros(self.backend.state.shape[1], dtype=torch.float32, device=self.device)
        rest[self._sl["qpos"]] = self.initial_qpos
        rest[self._sl["qvel"]] = self.initial_qvel
        rest[self._sl["ctrl"]] = self._ctrl_center          # _set_action(np.zeros(20))
        return rest

    # ------------------------------------------------------------------ sampling
    @staticmethod
    def _quat_mul_t(a, b):
        aw, ax, ay, az = a.unbind(-1)
        bw, bx, by, bz = b.unbind(-1)
        return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                            aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], dim=-1)

    def _angle_axis_t(self, n, axis_mode):
        """Random (angle, axis) quaternion batch on the device RNG: angle ~ U(-pi, pi); axis = z or U(-1, 1)^3 normalised."""
        u = lambda *s: torch.rand(*s, generator=self._gen, device=self.device)
        angle = (u(n) * 2 - 1) * np.pi
        if axis_mode == "z":
            axis = torch.tensor([0.0, 0.0, 1.0], device=self.device).expand(n, 3)
        else:
            axis = u(n, 3) * 2 - 1
            axis = axis / torch.linalg.norm(axis, dim=1, keepdim=True)
        q = torch.cat([torch.cos(angle / 2).unsqueeze(1), torch.sin(angle / 2).unsqueeze(1) * axis], dim=1)
        return q / torch.linalg.norm(q, dim=1, keepdim=True)

    def _sample_initial_pose(self, idx):
        """manipulate.py:171-208: object start pose for the envs in `idx` -> float32 [n, 7]."""
        n = idx.numel()
        q0 = self.initial_qpos[self.task.obj_qadr:self.task.obj_qadr + 7]
        if self.rng_mode == "numpy":
            out = np.zeros((n, 7))
            q0n = q0.double().cpu().numpy()
            for k, i in enumerate(idx.tolist()):
                rng = self._np_rngs[i]
                pos, quat = q0n[:3].copy(), q0n[3:].copy()
                if self.randomize_initial_rotation:
                    if self.target_rotation == "z":
                        off = rotations.quat_from_angle_and_axis(rng.uniform(-np.pi, np.pi), np.array([0.0, 0.0, 1.0]))
                        quat = rotations.quat_mul(quat, off)
                    elif self.target_rotation == "parallel":
                        z = rotations.quat_from_angle_and_axis(rng.uniform(-np.pi, np.pi), np.array([0.0, 0.0, 1.0]))
                        par = self._parallel_np[rng.integers(24)]
                        quat = rotations.quat_mul(quat, rotations.quat_mul(z, par))
                    elif self.target_rotation in ("xyz", "ignore"):
                        angle = rng.uniform(-np.pi, np.pi)
                        quat = rotations.quat_mul(quat, rotations.quat_from_angle_and_axis(angle, rng.uniform(-1.0, 1.0, size=3)))
                if self.randomize_initial_position and self.target_position != "fixed":
                    pos = pos + rng.normal(size=3, scale=0.005)
                out[k, :3], out[k, 3:] = pos, quat / np.linalg.norm(quat)
            return torch.as_tensor(out, dtype=torch.float32, device=self.device)
        pos, quat = q0[:3].expand(n, 3).clone(), q0[3:].expand(n, 4).clone()
        if self.randomize_initial_rotation:
            if self.target_rotation == "z":
                quat = self._quat_mul_t(quat, self._angle_axis_t(n, "z"))
            elif self.target_rotation == "parallel":
                z = self._angle_axis_t(n, "z")
                par = self._parallel[torch.randint(0, 24, (n,), generator=self._gen, device=self.device)]
                quat = self._quat_mul_t(quat, self._quat_mul_t(z, par))
            elif self.target_rotation in ("xyz", "ignore"):
                quat = self._quat_mul_t(quat, self._angle_axis_t(n, "xyz"))
        if self.randomize_initial_position and self.target_position != "fixed":
            pos = pos + 0.005 * torch.randn(n, 3, generator=self._gen, device=self.device)
        return torch.cat([pos, quat / torch.linalg.norm(quat, dim=1, keepdim=True)], dim=1)

    def _sample_goals(self, idx, obj):
        """manipulate.py:226-279 given the settled object pose `obj` [n, 7]."""
        n = idx.numel()
        if self.rng_mode == "numpy":
            objn = obj.double().cpu().numpy()
            goals = np.zeros((n, 7))
            for k, i in enumerate(idx.tolist()):
                rng = self._np_rngs[i]
                pos = objn[k, :3].copy()
                if self.target_position == "random":
                    pos = pos + rng.uniform(TARGET_POSITION_RANGE[:, 0], TARGET_POSITION_RANGE[:, 1])
                if self.target_rotation == "z":
                    quat = rotations.quat_from_angle_and_axis(rng.uniform(-np.pi, np.pi), np.array([0.0, 0.0, 1.0]))
                elif self.target_rotation == "parallel":
                    quat = rotations.quat_from_angle_and_axis(rng.uniform(-np.pi, np.pi), np.array([0.0, 0.0, 1.0]))
                    quat = rotations.quat_mul(quat, self._parallel_np[rng.integers(24)])
                elif self.target_rotation == "xyz":
                    angle = rng.uniform(-np.pi, np.pi)
                    quat = rotations.quat_from_angle_and_axis(angle, rng.uniform(-1.0, 1.0, size=3))
                else:
                    quat = objn[k, 3:].copy()
                goals[k, :3], goals[k, 3:] = pos, quat / np.linalg.norm(quat)
            return torch.as_tensor(goals, dtype=torch.float32, device=self.device)
        pos = obj[:, :3].clone()
        if self.target_position == "random":
            u = torch.rand(n, 3, generator=self._gen, device=self.device)
            pos = pos + self._range[:, 0] + u * (self._range[:, 1] - self._range[:, 0])
        if self.target_rotation == "z":
            quat = self._angle_axis_t(n, "z")
        elif self.target_rotation == "parallel":
            quat = self._angle_axis_t(n, "z")
            quat = self._quat_mul_t(quat, self._parallel[torch.randint(0, 24, (n,), generator=self._gen, device=self.device)])
        elif self.target_rotation == "xyz":
            quat = self._angle_axis_t(n, "xyz")
        else:
            quat = obj[:, 3:].clone()
        return torch.cat([pos, quat / torch.linalg.norm(quat, dim=1, keepdim=True)], dim=1)

    def _device_reset(self, mask, out):
        """rng_mode="device": the same retry loop with the draws inside the library; the host only reads `pending.any()`."""
        if self._dev_reset is None:
            from ._lib import HandResetC

            modes = {"ignore": 0, "fixed": 0, "z": 1, "parallel": 2, "xyz": 3}
            p = HandResetC()
            p.obj_qadr = int(self.task.obj_qadr)
            p.rot_mode = 3 if self.target_rotation == "ignore" else modes[self.target_rotation]     # manipulate.py:188-194
            p.randomize_rotation = int(bool(self.randomize_initial_rotation))
            p.randomize_position = int(bool(self.randomize_initial_position) and self.target_position != "fixed")
            p.goal_rot_mode, p.goal_random_position = modes[self.target_rotation], int(self.target_position == "random")
            for k in range(3):
                p.pos_lo[k], p.pos_hi[k] = float(TARGET_POSITION_RANGE[k, 0]), float(TARGET_POSITION_RANGE[k, 1])
            self._dev_reset = (p, self._rest, self._parallel.contiguous())
        p, rest, par = self._dev_reset
        st = self.backend.state
        pending = mask.clone()
        for attempt in range(100):
            if not bool(pending.any()):
                break
            m8 = pending.to(torch.uint8)
            self.backend.reset_hand_pose(m8, rest, p, par, self._dev_seed, self.env_offset, self._episode, attempt)
            self.backend.raw_step(10 * self.n_substeps, out, mask=m8)
            self.reset_attempts += 1
            pending = pending & ~(st[:, self._obj.start + 2] > 0.04)
        else:
            raise RuntimeError("hand reset did not settle on the palm within 100 attempts")
        self.backend.reset_hand_goal(mask.to(torch.uint8), p, par, self._dev_seed, self.env_offset, self._episode, out)
        self._elapsed.masked_fill_(mask, 0)

    def _reset_envs(self, mask, out, options=None):
        """BaseRobotEnv.reset (robot_env.py:154-186): retry `_reset_sim` until the block rests on the palm, then sample
        the goal.  Every attempt settles the pending envs together with one masked raw-step launch (10 x 20 sub-steps)."""
        if self.rng_mode == "device":
            return self._device_reset(mask, out)
        idx_all = torch.nonzero(mask, as_tuple=False).flatten()
        if idx_all.numel() == 0:
            return
        st, sl = self.backend.state, self._sl
        pending = mask.clone()
        for attempt in range(100):
            idx = torch.nonzero(pending, as_tuple=False).flatten()
            if idx.numel() == 0:
                break
            rec = self._rest.expand(idx.numel(), -1).clone()  # time, qpos, qvel reset; _set_action(np.zeros(20))
            rec[:, self._obj] = self._sample_initial_pose(idx)
            rec[:, sl["goal"]] = st[idx][:, sl["goal"]]
            st[idx] = rec
            self.backend.raw_step(10 * self.n_substeps, out, mask=pending.to(torch.uint8))
            self.reset_attempts += 1
            on_palm = st[:, self._obj.start + 2] > 0.04     # site "object:center" sits at the body origin
            pending = pending & ~on_palm
        else:
            raise RuntimeError("hand reset did not settle on the palm within 100 attempts")
        st[idx_all, sl["goal"]] = self._sample_goals(idx_all, st[idx_all][:, self._obj])
        self._elapsed[idx_all] = 0
        self.backend.refresh(mask.to(torch.uint8), out)  # mj_forward + _get_obs for the reset envs


# ---------------------------------------------------------------------------------------------------------------- HandReach
FINGERTIP_SITE_NAMES = ["robot0:S_fftip", "robot0:S_mftip", "robot0:S_rftip", "robot0:S_lftip", "robot0:S_thtip"]  # reach.py:8-14
# reach.py:15-40 DEFAULT_INITIAL_QPOS (joint order of the model)
REACH_INITIAL_QPOS = {
    "robot0:WRJ1": -0.16514339750464327, "robot0:WRJ0": -0.31973286565062153, "robot0:FFJ3": 0.14340512546557435,
    "robot0:FFJ2": 0.32028208333591573, "robot0:FFJ1": 0.7126053607727917, "robot0:FFJ0": 0.6705281001412586,
    "robot0:MFJ3": 0.000246444303701037, "robot0:MFJ2": 0.3152655251085491, "robot0:MFJ1": 0.7659800313729842,
    "robot0:MFJ0": 0.7323156897425923, "robot0:RFJ3": 0.00038520700007378114, "robot0:RFJ2": 0.36743546201985233,
    "robot0:RFJ1": 0.7119514095008576, "robot0:RFJ0": 0.6699446327514138, "robot0:LFJ4": 0.0525442258033891,
    "robot0:LFJ3": -0.13615534724474673, "robot0:LFJ2": 0.39872030433433003, "robot0:LFJ1": 0.7415570009679252,
    "robot0:LFJ0": 0.704096378652974, "robot0:THJ4": 0.003673823825070126, "robot0:THJ3": 0.5506291436028695,
    "robot0:THJ2": -0.014515151997119306, "robot0:THJ1": -0.0015229223564485414, "robot0:THJ0": -0.7894883021600622,
}


def body_xpos(model, qpos, body_name):
    """World position of a body frame for hinge/slide chains (host-side forward kinematics over the compiled tables;
    the reference reads `data.xpos[body]` after `mj_forward`, reach.py:292-296)."""
    m = model
    b = m.names["body_map"][body_name]
    chain = []
    while b > 0:
        chain.append(b)
        b = int(m.body_parent[b])
    pos, quat = np.zeros(3), np.array([1.0, 0.0, 0.0, 0.0])
    bpos, bquat = np.asarray(m.body_pos).reshape(-1, 3), np.asarray(m.body_quat).reshape(-1, 4)
    jpos, jaxis = np.asarray(m.jnt_pos).reshape(-1, 3), np.asarray(m.jnt_axis).reshape(-1, 3)
    rot = lambda q, v: rotations.quat2mat(q) @ v
    for b in reversed(chain):
        pos = pos + rot(quat, bpos[b])
        quat = rotations.quat_mul(quat, bquat[b])
        for j in range(int(m.body_jntadr[b]), int(m.body_jntadr[b]) + int(m.body_jntnum[b])):
            dq = qpos[int(m.jnt_qposadr[j])] - m.qpos0[int(m.jnt_qposadr[j])]
            if int(m.jnt_type[j]) == 2:   # slide
                pos = pos + rot(quat, jaxis[j]) * dq
            else:                         # hinge about the joint anchor
                anchor = pos + rot(quat, jpos[j])
                quat = rotations.quat_mul(quat, rotations.quat_from_angle_and_axis(dq, jaxis[j].copy()))
                pos = anchor - rot(quat, jpos[j])
    return pos


class HandReachVectorEnv(VectorEnv):
    """`gym.make_vec("HandReach-v3", num_envs=N)` replacement (envs/shadow_dexterous_hand/reach.py, MujocoHandReachEnv)."""

    def __init__(self, num_envs: int = 1, reward_type: str = "sparse", max_episode_steps: Optional[int] = 50, device="cuda:0",
                 rng_mode: str = "auto", autoreset_mode: str = "next_step", n_substeps: int = N_SUBSTEPS, backend_factory=None,
                 distance_threshold=0.01, relative_control=False, initial_qpos=None, model=None, **kwargs):
        if reward_type not in ("sparse", "dense"):
            raise ValueError("reward_type must be 'sparse' or 'dense'")
        if relative_control:
            raise NotImplementedError("relative_control is not available in the reference's new-binding envs either")
        self.task_name, self.reward_type, self.distance_threshold = "HandReach", reward_type, distance_threshold
        m = model if model is not None else load_model("hand_reach")
        t = FetchTaskC()
        t.kind, t.nact, t.ngoal = 3, int(m.nu), 15
        t.n_substeps, t.reward_dense = int(n_substeps), int(reward_type == "dense")
        t.nobs = int(m.nq) + int(m.nv) + 15
        t.distance_threshold, t.dt = float(distance_threshold), float(m.opt[0] * n_substeps)
        for k, name in enumerate(FINGERTIP_SITE_NAMES):
            t.tip_site[k] = m.site_id(name)
        super().__init__(model=m, task=t, fields=(("qpos", m.nq), ("qvel", m.nv), ("warm", m.nv), ("ctrl", m.nu), ("goal", 15)),
                         action_space=Box(-1.0, 1.0, shape=(int(m.nu),), dtype=np.float32), observation_space=_goal_space(15, t.nobs),
                         backend_factory=backend_factory or CudaBackend, num_envs=num_envs, device=device,
                         max_episode_steps=max_episode_steps, autoreset_mode=autoreset_mode, rng_mode=rng_mode,
                         n_substeps=n_substeps, kwargs=kwargs)
        # _env_setup (reach.py:286-296): initial joint angles, mj_forward, initial fingertip positions and palm position
        q0 = np.array(m.qpos0, dtype=np.float64)
        for name, value in (initial_qpos or REACH_INITIAL_QPOS).items():
            q0[int(m.jnt_qposadr[m.joint_id(name)])] = value
        self.initial_qpos = torch.as_tensor(q0, dtype=torch.float32, device=self.device)
        self.initial_qvel = torch.zeros(m.nv, dtype=torch.float32, device=self.device)
        st = self.backend.state
        st.zero_()
        st[:, self._sl["qpos"]] = self.initial_qpos
        out = self.backend.new_outputs()
        self.backend.refresh(None, out)
        self.initial_goal = out["achieved"][0].clone()
        self.palm_xpos = body_xpos(m, q0, "robot0:palm")
        self._last = out

    def _rest_record(self):   # mj_resetData (robot_env.py:305-316)
        rest = torch.zeros(self.backend.state.shape[1], dtype=torch.float32, device=self.device)
        rest[self._sl["qpos"]] = self.initial_qpos
        rest[self._sl["qvel"]] = self.initial_qvel
        return rest

    def _sample_goals(self, idx):
        """reach.py:95-121."""
        n = idx.numel()
        init = self.initial_goal.double().cpu().numpy().reshape(5, 3)
        if self.rng_mode == "numpy":
            goals = np.zeros((n, 15))
            finger_names = [name for name in FINGERTIP_SITE_NAMES if name != "robot0:S_thtip"]
            for k, i in enumerate(idx.tolist()):
                rng = self._np_rngs[i]
                finger_idx = FINGERTIP_SITE_NAMES.index(rng.choice(finger_names))
                meeting = self.palm_xpos + np.array([0.0, -0.09, 0.05])
                meeting = meeting + rng.normal(scale=0.005, size=3)
                goal = init.copy()
                for j in (4, finger_idx):
                    d = meeting - goal[j]
                    goal[j] = meeting - 0.005 * d / np.linalg.norm(d)
                if rng.uniform() < 0.1:
                    goal = init.copy()
                goals[k] = goal.flatten()
            return torch.as_tensor(goals, dtype=torch.float32, device=self.device)
        dev = self.device
        init_t = self.initial_goal.reshape(5, 3)
        finger = torch.randint(0, 4, (n,), generator=self._gen, device=dev)
        meeting = torch.as_tensor(self.palm_xpos + np.array([0.0, -0.09, 0.05]), dtype=torch.float32, device=dev) \
            + 0.005 * torch.randn(n, 3, generator=self._gen, device=dev)
        goal = init_t.expand(n, 5, 3).clone()
        ar = torch.arange(n, device=dev)
        for sel in (torch.full((n,), 4, device=dev, dtype=torch.long), finger):
            d = meeting - goal[ar, sel]
            goal[ar, sel] = meeting - 0.005 * d / torch.linalg.norm(d, dim=1, keepdim=True)
        keep = torch.rand(n, generator=self._gen, device=dev) < 0.1
        goal[keep] = init_t
        return goal.reshape(n, 15)

    def _device_reset(self, mask, out):
        if self._dev_reset is None:
            from ._lib import ReachResetC

            p = ReachResetC()
            meeting = self.palm_xpos + np.array([0.0, -0.09, 0.05])
            init = self.initial_goal.double().cpu().numpy()
            for k in range(3):
                p.meeting[k] = float(meeting[k])
            for k in range(15):
                p.initial_goal[k] = float(init[k])
            self._dev_reset = (p, self._rest)
        p, rest = self._dev_reset
        self.backend.reset_reach(mask.to(torch.uint8), rest, p, self._dev_seed, self.env_offset, self._episode, out)
        self._elapsed.masked_fill_(mask, 0)

    def _reset_envs(self, mask, out, options=None):
        if self.rng_mode == "device":
            return self._device_reset(mask, out)
        idx = torch.nonzero(mask, as_tuple=False).flatten()
        if idx.numel() == 0:
            return
        rec = self._rest.expand(idx.numel(), -1).clone()
        rec[:, self._sl["goal"]] = self._sample_goals(idx)
        self.backend.state[idx] = rec
        self._elapsed[idx] = 0
        self.backend.refresh(mask.to(torch.uint8), out)  # mj_forward + _get_obs


def make_hand_vec(task, **kwargs):
    if task == "HandReach":
        return HandReachVectorEnv(**kwargs)
    return HandVectorEnv(task=task, **kwargs)
