"""Batched FrankaKitchen-v1 on the CUDA simulator (kernel build csrc/b200sim_kitchen*.cu: joint equalities, condim 6).

Mirrors (batched) the reference's Python around the hot path:
  * FrankaRobot.step / _ctrl_velocity_limits / _ctrl_position_limits / _get_obs   envs/franka_kitchen/franka_env.py:92-170
      action -> clip -> x2 -> velocity bounds -> position target from the LAST NOISY robot observation -> position bounds,
      `do_simulation(ctrl, 40)` (the kernel launch, task kind 8), observation noise on robot qpos / qvel
  * KitchenEnv.step / _get_obs / compute_reward / reset                         envs/franka_kitchen/kitchen_env.py:356-437
      object observation noise (amplitude offsets 8 / 9 as in the reference), per-task goal distances on qpos slices,
      completion / removal / termination bookkeeping -- here as [N, n_tasks] boolean tensors
  * registry: FrankaKitchen-v1, max_episode_steps = 280 (__init__.py:1117-1121)
The target computation, the noise and the bookkeeping are a few elementwise tensor operations per step (they are Python in
the reference as well); the 40 sub-steps of physics are one kernel launch.  With rng_mode="device" the kernel adds the noise itself.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

from ._lib import FetchTaskC
from .fetch import KITCHEN_REF_POINT, CudaBackend  # noqa: F401  (KITCHEN_REF_POINT: re-exported)
from .models import load_franka_config, load_model
from .spaces import Box
from .vector import VectorEnv, _int64

FRAME_SKIP = 40
# kitchen_env.py:27-45
OBS_ELEMENT_INDICES = {
    "bottom burner": [11, 12], "top burner": [15, 16], "light switch": [17, 18], "slide cabinet": [19],
    "hinge cabinet": [20, 21], "microwave": [22], "kettle": [23, 24, 25, 26, 27, 28, 29],
}
OBS_ELEMENT_GOALS = {
    "bottom burner": [-0.88, -0.01], "top burner": [-0.92, -0.01], "light switch": [-0.69, -0.05], "slide cabinet": [0.37],
    "hinge cabinet": [0.0, 1.45], "microwave": [-0.75], "kettle": [-0.23, 0.75, 1.62, 0.99, 0.0, 0.0, -0.06],
}
BONUS_THRESH = 0.3
# kitchen_env.py:246-279
INIT_QPOS = [1.48388023e-01, -1.76848573e00, 1.84390296e00, -2.47685760e00, 2.60252026e-01, 7.12533105e-01, 1.59515394e00,
             4.79267505e-02, 3.71350919e-02, -2.66279850e-04, -5.18043486e-05, 3.12877220e-05, -4.51199853e-05, -3.90842156e-06,
             -4.22629655e-05, 6.28065475e-05, 4.04984708e-05, 4.62730939e-04, -2.26906415e-04, -4.65501369e-04, -6.44129196e-03,
             -1.77048263e-03, 1.08009684e-03, -2.69397440e-01, 3.50383255e-01, 1.61944683e00, 1.00618764e00, 4.06395120e-03,
             -6.62095997e-03, -2.68278933e-04]


def make_kitchen_task(model, frame_skip=FRAME_SKIP):
    t = FetchTaskC()
    t.kind, t.nact, t.ngoal = 8, int(model.nu), int(model.nq)
    t.n_substeps, t.reward_dense = int(frame_skip), 0
    t.nobs = int(model.nq) + int(model.nv)
    t.dt = float(model.opt[0] * frame_skip)
    t.penv_body = -1
    return t


class KitchenVectorEnv(VectorEnv):
    """`gym.make_vec("FrankaKitchen-v1", num_envs=N)`.  Observation dict: `observation` [N, 59], `achieved_goal` /
    `desired_goal` dicts task -> [N, k]; reward = number of tasks completed in the step; `terminated` when every task of the
    episode is completed; info carries the bookkeeping as boolean [N, n_tasks] tensors (column order `self.tasks`).
    The observation is noisy, and the next step's control targets start from it.  rng_mode="numpy" / "torch" draw the noise on
    the host and have no `set_state`.  rng_mode="device" draws it in the step kernel (b200sim_set_obs_noise) as a function of
    (seed, global env index, episode, step), so a run does not depend on batch shape or sharding, and `get_state` / `set_state`
    checkpoint the env: the record's goal slot, which the kitchen task does not use, carries what the state record lacks --
    word 0 the episode counter, words 1-2 the env's Philox key (int32 bits, low word first), then `tasks_to_complete` and `episode_task_completions` (0 / 1)."""

    metadata = {"render_modes": [], "render_fps": 12, "autoreset_mode": "next_step"}
    AUTO_RECOVER = False

    def __init__(self, num_envs: int = 1, tasks_to_complete=None, terminate_on_tasks_completed: bool = True,
                 remove_task_when_completed: bool = True, object_noise_ratio: float = 0.0005, robot_noise_ratio: float = 0.01,
                 max_episode_steps: Optional[int] = 280, device="cuda:0", rng_mode: str = "auto", autoreset_mode: str = "next_step",
                 frame_skip: int = FRAME_SKIP, backend_factory=None, model=None, **kwargs):
        tasks = list(OBS_ELEMENT_GOALS.keys()) if tasks_to_complete is None else list(tasks_to_complete)
        for task in tasks:                                                      # kitchen_env.py:291-297
            if task not in OBS_ELEMENT_GOALS:
                raise ValueError(f"The task {task} cannot be found the the list of possible goals: {OBS_ELEMENT_GOALS.keys()}")
        self.tasks = tasks
        self.terminate_on_tasks_completed, self.remove_task_when_completed = terminate_on_tasks_completed, remove_task_when_completed
        self.object_noise_ratio, self.robot_noise_ratio = object_noise_ratio, robot_noise_ratio
        self.frame_skip = int(frame_skip)
        # mesh_collision="hull": the nine Franka collision meshes collide through support maps on their reduced convex hulls (32 vertices
        # each; blob franka_kitchen_hull, kernels of csrc/b200sim_kitchen_hull.cu) instead of box proxies (DESIGN.md deviation 1)
        mesh_collision = kwargs.get("mesh_collision", "box")
        if mesh_collision not in ("box", "hull"):
            raise ValueError("mesh_collision must be 'box' or 'hull'")
        self.mesh_collision = mesh_collision
        m = model if model is not None else load_model("franka_kitchen_hull" if mesh_collision == "hull" else "franka_kitchen")
        # broadphase="groups" (default): the kernel build with the two-level broad phase (csrc/b200sim_kitchen_groups.cu) -- it
        # matches the flat-scan build bit for bit (tests/test_zz_kitchen_gpu.py) and tests far fewer pairs per sub-step; "flat": one
        # scan over all 3 708 pairs.  The library reads the choice from the
        # environment when the handle is created.
        broadphase = kwargs.get("broadphase", "flat" if os.environ.get("B200SIM_KITCHEN_GROUPS", "1") in ("0",) else "groups")
        if broadphase not in ("flat", "groups"):
            raise ValueError("broadphase must be 'flat' or 'groups'")
        if mesh_collision == "hull" and broadphase != "groups":
            raise ValueError("mesh_collision='hull' exists for the two-level broad phase only")
        self.broadphase = broadphase
        factory = backend_factory or CudaBackend

        def make_backend(*args):
            prev = os.environ.get("B200SIM_KITCHEN_GROUPS")
            os.environ["B200SIM_KITCHEN_GROUPS"] = "1" if broadphase == "groups" else "0"
            try:
                return factory(*args)
            finally:
                if prev is None:
                    del os.environ["B200SIM_KITCHEN_GROUPS"]
                else:
                    os.environ["B200SIM_KITCHEN_GROUPS"] = prev

        t = make_kitchen_task(m, frame_skip)
        # `terminated` is the task bookkeeping below, not a kernel flag
        super().__init__(model=m, task=t, fields=(("qpos", m.nq), ("qvel", m.nv), ("warm", m.nv), ("ctrl", m.nu)),
                         action_space=Box(-1.0, 1.0, shape=(9,), dtype=np.float64),  # franka_env.py:90
                         observation_space=Box(-np.inf, np.inf, shape=(int(t.nobs),), dtype=np.float64),
                         backend_factory=make_backend, num_envs=num_envs, device=device, max_episode_steps=max_episode_steps,
                         autoreset_mode=autoreset_mode, rng_mode=rng_mode, n_substeps=frame_skip, kwargs=kwargs)
        self._can_terminate = bool(terminate_on_tasks_completed)
        if self.rng_mode == "device" and getattr(self.backend, "set_obs_noise", None) is None:
            self.backend.close()
            raise NotImplementedError("rng_mode='device' needs a backend that draws the observation noise in the step "
                                      f"(set_obs_noise, b200sim_set_obs_noise); {type(self.backend).__name__} has none")
        dev = self.device
        assert int(np.round(1.0 / self.dt)) == self.metadata["render_fps"]      # kitchen_env.py:311-313
        cfg = load_franka_config()                                              # franka_env.py:172-202
        nv = int(m.nv)
        f32 = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float64), dtype=torch.float32, device=dev)
        pb, vb = np.array(cfg["pos_bound"][:nv]), np.array(cfg["vel_bound"][:nv])
        self._pos_lo, self._pos_hi, self._vel_lo, self._vel_hi = f32(pb[:9, 0]), f32(pb[:9, 1]), f32(vb[:9, 0]), f32(vb[:9, 1])
        pa, va = np.array(cfg["pos_noise_amp"][:nv]), np.array(cfg["vel_noise_amp"][:nv])
        # observation = robot qpos (9) | robot qvel (9) | object qpos (21) | object qvel (20), one noise scale per entry
        self._noise_scale = f32(np.concatenate([robot_noise_ratio * pa[:9], robot_noise_ratio * va[:9],
                                                object_noise_ratio * pa[8:], object_noise_ratio * va[9:]]))
        self.init_qpos, self.init_qvel = f32(INIT_QPOS), torch.zeros(nv, dtype=torch.float32, device=dev)
        self._idx = {t: torch.as_tensor(OBS_ELEMENT_INDICES[t], device=dev) for t in tasks}
        self._goal = {t: f32(OBS_ELEMENT_GOALS[t]) for t in tasks}
        # every task's qpos entries are one contiguous run (kitchen_env.py:20-38): `achieved_goal[t]` is a view, not a gather
        self._run = {}
        for t in tasks:
            ii = [int(i) for i in OBS_ELEMENT_INDICES[t]]
            self._run[t] = slice(ii[0], ii[-1] + 1) if ii == list(range(ii[0], ii[-1] + 1)) else None
        # all tasks' distance tests in one pass: entries padded to the longest task, padding masked out of the squared distance
        kmax = max(len(OBS_ELEMENT_INDICES[t]) for t in tasks)
        idx_pad = np.zeros((len(tasks), kmax), dtype=np.int64)
        goal_pad, live = np.zeros((len(tasks), kmax)), np.zeros((len(tasks), kmax))
        for j, t in enumerate(tasks):
            k = len(OBS_ELEMENT_INDICES[t])
            idx_pad[j, :k], goal_pad[j, :k], live[j, :k] = OBS_ELEMENT_INDICES[t], OBS_ELEMENT_GOALS[t], 1.0
        self._idx_pad = torch.as_tensor(idx_pad.reshape(-1), device=dev)
        self._goal_pad, self._live_pad = f32(goal_pad), f32(live)
        n, k = self.num_envs, len(tasks)
        self._todo = torch.ones((n, k), dtype=torch.bool, device=dev)            # tasks_to_complete
        self._episode_done = torch.zeros((n, k), dtype=torch.bool, device=dev)  # episode_task_completions
        self._last_robot_qpos = self.init_qpos[:9].expand(n, 9).clone()
        self._obs = torch.zeros((n, int(self.task.nobs)), dtype=torch.float32, device=dev)   # the noisy observation of the last call

    # ------------------------------------------------------------------ noise / observation
    def _noise(self, idx):
        """59 uniform draws in [-1, 1) per env in the reference's order (robot qpos 9, robot qvel 9, object qpos 21, object
        qvel 20: franka_env.py:114-124 then kitchen_env.py:374-385), scaled per entry."""
        n = idx.numel()
        if self.rng_mode == "numpy":
            u = np.stack([self._np_rngs[i].uniform(low=-1.0, high=1.0, size=self._noise_scale.numel()) for i in idx.tolist()])
            u = torch.as_tensor(u, dtype=torch.float32, device=self.device)
        else:
            u = torch.rand((n, self._noise_scale.numel()), generator=self._gen, device=self.device) * 2 - 1
        return u * self._noise_scale

    def _obs_dict(self, out):
        q = out["achieved"]
        return self._cast_obs({"observation": out["obs"] if self.rng_mode == "device" else self._obs,
                               "achieved_goal": {t: (q[:, self._run[t]] if self._run[t] is not None else q[:, self._idx[t]]) for t in self.tasks},
                               "desired_goal": {t: self._goal[t].expand(self.num_envs, -1) for t in self.tasks}})

    # ------------------------------------------------------------------ reset
    def _rest_record(self):
        rest = torch.zeros(self.backend.state.shape[1], dtype=torch.float32, device=self.device)
        rest[self._sl["qpos"]] = self.init_qpos
        rest[self._sl["qvel"]] = self.init_qvel
        return rest

    def _device_noise(self):
        """rng_mode="device": the episode counters, the reset without draws and the noise stream of the handle (seed as it stands)."""
        if self._dev_reset is None:
            from ._lib import UniformResetC

            p = UniformResetC()
            p.n, p.quat_slot = 0, -1   # reset_model draws nothing but the observation noise
            self._dev_reset = p
        self.backend.set_obs_noise(self._noise_scale, self._dev_seed, self.env_offset, self._episode)
        return self._dev_reset

    def _reset_envs(self, mask, out, options=None):
        """MujocoEnv.reset -> mj_resetData -> reset_model (franka_env.py:130-137), then KitchenEnv.reset (kitchen_env.py:425-437)."""
        if self.rng_mode == "device":
            # record <- rest record, elapsed <- 0, episode += 1, then the refresh draws the noise of (episode, step 0)
            p = self._device_noise()
            every = self._reset_all
            self.backend.reset_uniform(None if every else mask.to(torch.uint8), self._rest, p, self._dev_seed, self.env_offset, self._episode, out)
            self._todo = self._todo | mask[:, None]
            self._episode_done = self._episode_done & ~mask[:, None]
            self._last_robot_qpos = out["obs"][:, :9].clone()
            return
        idx = self._mask_indices(mask)
        if idx.numel() == 0:
            return
        self.backend.state[idx] = self._rest.expand(idx.numel(), -1).clone()
        self._elapsed[idx] = 0
        self._todo[idx] = True
        self._episode_done[idx] = False
        self.backend.refresh(mask.to(torch.uint8), out)   # set_state -> mj_forward, noise-free observation
        noisy = out["obs"][idx] + self._noise(idx)
        self._last_robot_qpos[idx] = noisy[:, :9]
        self._obs = self._obs.clone()
        self._obs[idx] = noisy

    def _reset_info(self, out):
        return {"tasks_to_complete": self._todo.clone(), "episode_task_completions": self._episode_done.clone(),
                "step_task_completions": torch.zeros_like(self._todo)}

    # ------------------------------------------------------------------ step
    def control_targets(self, a):
        """franka_env.py:92-100, 139-170: clip, act_mid + a * act_rng (0, 2), velocity bounds, position target from the last noisy
        robot observation, position bounds -- the `ctrl` the step kernel receives."""
        vel = torch.clamp(torch.clamp(a, -1.0, 1.0) * 2.0, self._vel_lo, self._vel_hi)
        return torch.clamp(self._last_robot_qpos + vel * self.dt, self._pos_lo, self._pos_hi).contiguous()

    def _kernel_input(self, actions):
        return self.control_targets(actions)

    def _step_results(self, out):
        if self.rng_mode == "device":   # the kernel returned the noisy observation
            self._last_robot_qpos = out["obs"][:, :9].clone()
        else:
            # the observation noise of every env is drawn before a NEXT_STEP reset draws its reset noise
            self._obs = out["obs"] + self._noise(self._all_idx)
            self._last_robot_qpos = self._obs[:, :9].clone()
        q = out["achieved"]
        # kitchen_env.py:356-369, 399-423
        # (|| q[task] - goal || < BONUS_THRESH for every task at once; the norm itself, as the reference compares it)
        diff = (q[:, self._idx_pad].view(self.num_envs, len(self.tasks), -1) - self._goal_pad) * self._live_pad
        close = torch.linalg.norm(diff, dim=2) < BONUS_THRESH
        step_done = close & self._todo
        reward = step_done.sum(dim=1).to(torch.float32)
        if self.remove_task_when_completed:
            self._todo = self._todo & ~step_done
        self._episode_done = self._episode_done | step_done
        terminated = self._episode_done.all(dim=1) if self.terminate_on_tasks_completed else torch.zeros_like(self._needs_reset)
        info = {"tasks_to_complete": self._todo.clone(), "step_task_completions": step_done,
                "episode_task_completions": self._episode_done.clone()}
        return reward, terminated, out["truncated"], info

    def _mask_results(self, out, pre, reward, terminated, truncated, info):
        info = {"tasks_to_complete": self._todo.clone(), "step_task_completions": info["step_task_completions"] & ~pre[:, None],
                "episode_task_completions": self._episode_done.clone()}
        return torch.where(pre, torch.zeros_like(reward), reward), terminated & ~pre, truncated & ~pre, info

    def _final_info(self, out, info, done):
        return None   # the bookkeeping tensors of the step already describe the finished episodes

    def _finish_info(self, out, info):
        pass

    # GoalEnv-style reward on (achieved, desired) dicts of tensors: the number of listed tasks within BONUS_THRESH
    def compute_reward(self, achieved_goal, desired_goal, info=None):
        return sum((torch.linalg.norm(torch.as_tensor(achieved_goal[t]) - torch.as_tensor(desired_goal[t]), dim=-1) < BONUS_THRESH)
                   .to(torch.float32) for t in achieved_goal)

    # ------------------------------------------------------------------ state access (rng_mode="device")
    def get_state(self):
        state, elapsed = super().get_state()
        if self.rng_mode == "device":
            self._device_noise()
            g, k = self.backend.layout["goal"], len(self.tasks)
            state[:, g].view(torch.int32).copy_(self._episode)
            keys = self._keys if self._keys is not None else torch.full((self.num_envs,), _int64(self._dev_seed), dtype=torch.int64, device=self.device)
            state[:, g + 1:g + 3].view(torch.int32).copy_(keys.view(torch.int32).view(self.num_envs, 2))   # each env's key, low word first
            state[:, g + 3:g + 3 + k] = self._todo.to(torch.float32)
            state[:, g + 3 + k:g + 3 + 2 * k] = self._episode_done.to(torch.float32)
        return state, elapsed

    def set_state(self, state, elapsed=None):
        """rng_mode="device" only: a record of `get_state` (with its bookkeeping) and the step counters; the refresh redraws the
        noise of (seed, env, episode, step), so the observation and the next control targets are those of the saved env."""
        if self.rng_mode != "device":
            raise NotImplementedError("FrankaKitchen has set_state in rng_mode='device' only: with host-drawn noise the noisy observation "
                                      "and the last robot pose are not part of the record")
        state = torch.as_tensor(state).to(self.device, torch.float32)
        g, k = self.backend.layout["goal"], len(self.tasks)
        words = state[:, g:g + 3].contiguous().view(torch.int32)
        keys = words[:, 1:3].contiguous().view(torch.int64).view(self.num_envs)
        self._dev_seed = int(keys[0]) & 0xFFFFFFFFFFFFFFFF   # the noise seed of a backend without per-env keys
        if self._keys is not None:
            self._keys.copy_(keys)
        self._device_noise()
        self._episode.copy_(words[:, 0])
        self._todo = state[:, g + 3:g + 3 + k] != 0
        self._episode_done = state[:, g + 3 + k:g + 3 + 2 * k] != 0
        obs = super().set_state(state, elapsed)
        self._last_robot_qpos = self._last["obs"][:, :9].clone()
        return obs
