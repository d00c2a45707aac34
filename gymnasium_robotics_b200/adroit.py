"""Batched Adroit hand environments on the CUDA simulator: `gym.make_vec("AdroitHandHammer-v2", num_envs=N)` and
`gym.make_vec("AdroitHandRelocate-v2", num_envs=N)`, `"AdroitHandPen-v2"`, `"AdroitHandDoor-v2"` (+ the `Sparse` ids).

Mirrors (batched) the reference's Python around the hot path:
  * AdroitHandHammerEnv.step / _get_obs        envs/adroit_hand/adroit_hammer.py:291-357   (inside the step kernel,
                                               csrc/fetch_task.cuh `adroit_hammer_observe`, task kind 4)
  * MujocoEnv.do_simulation(a, frame_skip=5)   ctrl = act_mean + clip(a) * act_rng, 5 x mj_step (un-vendored Gymnasium base)
  * reset_model                                adroit_hammer.py:372-378: model.body_pos[nail_board].z ~ U(0.1, 0.25) per
                                               episode (a per-env body position in the state record), init_qpos / init_qvel
  * get_env_state / set_env_state              adroit_hammer.py:380-402
  * registry                                   __init__.py:1082-1101: ids AdroitHandHammer-v2 (dense) / AdroitHandHammerSparse-v2,
                                               max_episode_steps = 200
The ctor's actuator gain / bias overwrite (adroit_hammer.py:235-262) writes the values the MJCF already holds
(adroit_assets.xml actuator block), so the compiled model needs no edit.  The model has 33 dofs: it runs on the wide
kernel build (64-bit dof masks, bordered register Cholesky, csrc/b200sim_wide.cu).
Not restated: the noslip post-solver (`noslip_iterations=20`, adroit_assets.xml:3) -- listed in DESIGN.md.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import rotations
from ._lib import FetchTaskC
from .fetch import ADROIT_REF_POINT, CudaBackend  # noqa: F401  (ADROIT_REF_POINT: re-exported)
from .models import load_model
from .spaces import Box
from .vector import VectorEnv

FRAME_SKIP = 5
BOARD_Z_RANGE = (0.1, 0.25)           # adroit_hammer.py:374-376


def make_hammer_task(model, reward_type, frame_skip=FRAME_SKIP):
    """b200sim_fetch_task_t for kind 4 (ids resolved as MujocoModelNames would, adroit_hammer.py:264-270)."""
    m = model
    t = FetchTaskC()
    t.kind, t.nact, t.ngoal = 4, int(m.nu), 3
    t.n_substeps, t.reward_dense = int(frame_skip), int(reward_type == "dense")
    t.grip_site = m.site_id("S_grasp")
    t.obj_site = m.frame_site("Object")
    t.frame_site = m.site_id("S_target")
    t.tip_site[0], t.tip_site[1] = m.site_id("tool"), m.site_id("nail_goal")
    t.penv_body = int(m.names["body_map"]["nail_board"])
    t.nobs = int(m.nq) - 6 + 6 + 13
    t.dt = float(m.opt[0] * frame_skip)
    return t


def make_relocate_task(model, reward_type, frame_skip=FRAME_SKIP):
    """b200sim_fetch_task_t for kind 5 (adroit_relocate.py:257-259)."""
    m = model
    t = FetchTaskC()
    t.kind, t.nact, t.ngoal = 5, int(m.nu), 3
    t.n_substeps, t.reward_dense = int(frame_skip), int(reward_type == "dense")
    t.grip_site = m.site_id("S_grasp")
    t.obj_site = m.frame_site("Object")
    t.penv_body = int(m.names["body_map"]["Object"])
    t.nobs = int(m.nq) - 6 + 9
    t.dt = float(m.opt[0] * frame_skip)
    return t


def make_pen_task(model, reward_type, frame_skip=FRAME_SKIP):
    """b200sim_fetch_task_t for kind 6 (adroit_pen.py:264-271; the two lengths of :392-399 are model constants)."""
    m = model
    t = FetchTaskC()
    t.kind, t.nact, t.ngoal = 6, int(m.nu), 3
    t.n_substeps, t.reward_dense = int(frame_skip), int(reward_type == "dense")
    t.obj_site = m.frame_site("Object")
    t.frame_site = m.site_id("eps_ball")
    names = ("object_top", "object_bottom", "target_top", "target_bottom")
    for k, n in enumerate(names):
        t.tip_site[k] = m.site_id(n)
    sp = np.asarray(m.site_pos).reshape(-1, 3)
    t.distance_threshold = float(np.linalg.norm(sp[t.tip_site[0]] - sp[t.tip_site[1]]))   # pen_length
    t.rotation_threshold = float(np.linalg.norm(sp[t.tip_site[2]] - sp[t.tip_site[3]]))   # tar_length
    t.penv_body = int(m.names["body_map"]["target"])
    t.nobs = int(m.nq) - 6 + 21
    t.dt = float(m.opt[0] * frame_skip)
    return t


def make_door_task(model, reward_type, frame_skip=FRAME_SKIP):
    """b200sim_fetch_task_t for kind 7 (adroit_door.py:258-263)."""
    m = model
    t = FetchTaskC()
    t.kind, t.nact, t.ngoal = 7, int(m.nu), 3
    t.n_substeps, t.reward_dense = int(frame_skip), int(reward_type == "dense")
    t.grip_site, t.frame_site = m.site_id("S_grasp"), m.site_id("S_handle")
    t.obj_qadr = int(m.jnt_qposadr[m.joint_id("door_hinge")])
    assert m.names["joint"][-1] == "latch" and t.obj_qadr == int(m.nq) - 2
    t.penv_body = int(m.names["body_map"]["frame"])
    t.nobs = int(m.nq) - 3 + 12
    t.dt = float(m.opt[0] * frame_skip)
    return t


class _AdroitVectorEnv(VectorEnv):
    """Observations, rewards and flags are float32 / bool torch tensors on `device` with a leading `num_envs` axis;
    `info["success"]` mirrors the reference's `dict(success=goal_achieved)`.  A task class names its model and task struct and
    gives two tables:
      * RESET_DRAWS: reset_model's uniform draws, in the reference's order: (record field, offset inside it, low, high); the
        field "euler" is Euler angle `offset` of the orientation written to penv[3:7] (the Pen's target);
      * STATE_KEYS: the get_env_state / set_env_state entries besides qpos and qvel: (key, record field, offset inside it, width)."""

    metadata = {"render_modes": [], "render_fps": 100, "autoreset_mode": "next_step"}
    RECOVERY_KEEP = ("goal", "penv")   # a recovered env keeps its per-episode model pose and target
    SUCCESS_KEY = "success"

    def __init__(self, num_envs: int = 1, reward_type: str = "dense", max_episode_steps: Optional[int] = 200, device="cuda:0",
                 rng_mode: str = "auto", autoreset_mode: str = "next_step", frame_skip: int = FRAME_SKIP, backend_factory=None,
                 model=None, **kwargs):
        if reward_type.lower() not in ("sparse", "dense"):
            raise ValueError(f"Unknown reward type, expected `dense` or `sparse` but got {reward_type}")   # adroit_hammer.py:224-227
        self.task_name, self.reward_type = self.TASK_NAME, reward_type.lower()
        self.sparse_reward = self.reward_type == "sparse"
        self.frame_skip = int(frame_skip)
        m = model if model is not None else load_model(self.MODEL_NAME)
        t = self.make_task(m, self.reward_type, frame_skip)
        super().__init__(model=m, task=t, fields=(("qpos", m.nq), ("qvel", m.nv), ("warm", m.nv), ("ctrl", m.nu), ("goal", 3), ("penv", 7)),
                         action_space=Box(-1.0, 1.0, shape=(int(m.nu),), dtype=np.float32),                  # adroit_hammer.py:229-232
                         observation_space=Box(-np.inf, np.inf, shape=(int(t.nobs),), dtype=np.float64),
                         backend_factory=backend_factory or CudaBackend, num_envs=num_envs, device=device,
                         max_episode_steps=max_episode_steps, autoreset_mode=autoreset_mode, rng_mode=rng_mode,
                         n_substeps=frame_skip, kwargs=kwargs)
        self.init_qpos = torch.as_tensor(np.array(m.qpos0), dtype=torch.float32, device=self.device)   # MujocoEnv: data.qpos at load
        self.init_qvel = torch.zeros(m.nv, dtype=torch.float32, device=self.device)
        # model pose (position 3 + quaternion 4) of the body whose pose is per-env state
        self._board_pos0 = torch.as_tensor(np.concatenate([np.asarray(m.body_pos).reshape(-1, 3)[t.penv_body],
                                                           np.asarray(m.body_quat).reshape(-1, 4)[t.penv_body]]),
                                           dtype=torch.float32, device=self.device)
        cr = np.asarray(m.act_ctrlrange, dtype=np.float64).reshape(-1, 2)
        self.act_mean, self.act_rng = cr.mean(axis=1), 0.5 * (cr[:, 1] - cr[:, 0])                      # adroit_hammer.py:271-274
        self._draw_bounds = tuple(torch.tensor([d[i] for d in self.RESET_DRAWS], dtype=torch.float32, device=self.device) for i in (2, 3))

    # ------------------------------------------------------------------ reset
    def _rest_record(self):
        rest = torch.zeros(self.backend.state.shape[1], dtype=torch.float32, device=self.device)   # ctrl, warm start, time <- 0
        rest[self._sl["qpos"]] = self.init_qpos
        rest[self._sl["qvel"]] = self.init_qvel
        rest[self._sl["penv"]] = self._board_pos0
        return rest

    def _device_reset(self, mask, out):
        """rng_mode="device": the uniform draws of reset_model happen inside the library (csrc/reset_sample.cuh)."""
        if self._dev_reset is None:
            from ._lib import UniformResetC

            p, sl = UniformResetC(), self._sl
            p.n = len(self.RESET_DRAWS)
            p.quat_slot = -1
            for k, (field, off, lo, hi) in enumerate(self.RESET_DRAWS):
                if field == "euler":
                    p.slot[k], p.quat_slot = -1 - off, sl["penv"].start + 3
                else:
                    p.slot[k] = sl[field].start + off
                p.lo[k], p.hi[k] = lo, hi
            self._dev_reset = (p, self._rest)
        every = self._reset_all
        p, rest = self._dev_reset
        self.backend.reset_uniform(None if every else mask.to(torch.uint8), rest, p, self._dev_seed, self.env_offset, self._episode, out)
        if every:
            self._elapsed.zero_()
        else:
            self._elapsed.masked_fill_(mask, 0)

    def _reset_envs(self, mask, out, options=None):
        """MujocoEnv.reset -> mj_resetData -> reset_model (the RESET_DRAWS, in the reference's order) for the envs in `mask`."""
        if self.rng_mode == "device":
            return self._device_reset(mask, out)
        idx = self._mask_indices(mask)
        n = idx.numel()
        if n == 0:
            return
        if self.rng_mode == "numpy":
            u = np.array([[self._np_rngs[i].uniform(low=d[2], high=d[3]) for d in self.RESET_DRAWS] for i in idx.tolist()])
        else:
            lo, hi = self._draw_bounds
            u = lo + (hi - lo) * torch.rand((n, lo.numel()), generator=self._gen, device=self.device)
        u32 = torch.as_tensor(u, dtype=torch.float32, device=self.device)
        rec = self._rest.expand(n, -1).clone()
        for k, (field, off, _, _) in enumerate(self.RESET_DRAWS):
            if field != "euler":
                rec[:, self._sl[field].start + off] = u32[:, k]
        angles = [(k, off) for k, (field, off, _, _) in enumerate(self.RESET_DRAWS) if field == "euler"]
        if angles:            # body_quat = euler2quat([u, u, 0]), from the float64 draws of rng_mode="numpy"
            drawn = u if self.rng_mode == "numpy" else u32.double().cpu().numpy()
            euler = np.zeros((n, 3))
            for k, off in angles:
                euler[:, off] = drawn[:, k]
            pq = self._sl["penv"].start + 3
            rec[:, pq:pq + 4] = torch.as_tensor(rotations.euler2quat(euler), dtype=torch.float32, device=self.device)
        self.backend.state[idx] = rec
        self._elapsed[idx] = 0
        self.backend.refresh(mask.to(torch.uint8), out)   # set_state -> mj_forward, then _get_obs

    # ------------------------------------------------------------------ gymnasium API (flat observation, `success` info)
    def _obs_dict(self, out):
        return self._cast_obs(out["obs"])

    def _success(self, column):
        return column > 0.5

    def reset(self, *, seed=None, options=None):
        """adroit_hammer.py:359-370 (and the siblings): `options={"initial_state_dict": {...}}` sets the state after the
        ordinary reset through `set_env_state` (entries [width] for every env or [num_envs, width])."""
        if options is not None and "initial_state_dict" in options and "reset_mask" in options:
            raise ValueError("initial_state_dict sets the state of every env: it does not combine with reset_mask")
        obs, info = super().reset(seed=seed, options=options)
        if options is not None and "initial_state_dict" in options:
            obs = self._cast_obs(self.set_env_state(options["initial_state_dict"]))
        return obs, info

    def compute_reward(self, *a, **k):
        raise NotImplementedError("Adroit environments are not GoalEnvs (no compute_reward in the reference)")

    # adroit_*.py get_env_state / set_env_state, batched: dicts of [N, .] tensors
    def _state_keys(self):
        return (("qpos", "qpos", 0, self.model.nq), ("qvel", "qvel", 0, self.model.nv)) + self.STATE_KEYS

    def get_env_state(self):
        st, sl = self.backend.state, self._sl
        return {key: st[:, sl[f].start + off:sl[f].start + off + w].clone() for key, f, off, w in self._state_keys()}

    def set_env_state(self, state_dict):
        st, sl = self.backend.state, self._sl
        for key, f, off, width in self._state_keys():
            v = torch.as_tensor(np.asarray(state_dict[key]) if not torch.is_tensor(state_dict[key]) else state_dict[key])
            assert v.shape[-1] == width, f"The state dictionary entry {key} must have {width} columns"
            start = sl[f].start + off
            st[:, start:start + width] = v.to(self.device, torch.float32).reshape(-1, width).expand(self.num_envs, width)
        st[:, sl["warm"]] = 0
        out = self.backend.new_outputs()
        self.backend.refresh(None, out)   # set_state -> mj_forward
        self._last = out
        return out["obs"]
class AdroitHammerVectorEnv(_AdroitVectorEnv):
    """`gym.make_vec("AdroitHandHammer-v2", num_envs=N)`: obs 46; the nail board height (model.body_pos[nail_board].z) is per-env
    state."""

    TASK_NAME, MODEL_NAME = "AdroitHandHammer", "adroit_hammer"
    make_task = staticmethod(make_hammer_task)
    RESET_DRAWS = (("penv", 2, BOARD_Z_RANGE[0], BOARD_Z_RANGE[1]),)                                        # adroit_hammer.py:372-378
    STATE_KEYS = (("board_pos", "penv", 0, 3),)                                                              # adroit_hammer.py:380-402

    def get_env_state(self):
        s = super().get_env_state()
        s["target_pos"] = self._last["achieved"].clone() if self._last is not None else None
        return s


class AdroitRelocateVectorEnv(_AdroitVectorEnv):
    """`gym.make_vec("AdroitHandRelocate-v2", num_envs=N)`: 36 dofs (6-dof arm + 24 hand joints + 6-dof ball) on the wide
    build; obs 39; per-episode ball start (model.body_pos[Object] x, y) and target (model.site_pos[target]) as per-env state
    (envs/adroit_hand/adroit_relocate.py:288-402)."""

    TASK_NAME, MODEL_NAME = "AdroitHandRelocate", "adroit_relocate"
    make_task = staticmethod(make_relocate_task)
    # body_pos of "Object" (z stays the model's), then site_pos of "target" (a world site)
    RESET_DRAWS = (("penv", 0, -0.15, 0.15), ("penv", 1, -0.15, 0.3), ("goal", 0, -0.2, 0.2), ("goal", 1, -0.2, 0.2),
                   ("goal", 2, 0.15, 0.35))                                                                    # adroit_relocate.py:354-373
    STATE_KEYS = (("obj_pos", "penv", 0, 3), ("target_pos", "goal", 0, 3))                                     # adroit_relocate.py:375-402

    def get_env_state(self):
        s = super().get_env_state()
        hand = self._last["obs"][:, -9:-6] if self._last is not None else None   # palm - ball; palm = that + ball
        s["hand_pos"] = (hand + self._last["achieved"]).clone() if hand is not None else None
        return s


class AdroitPenVectorEnv(_AdroitVectorEnv):
    """`gym.make_vec("AdroitHandPen-v2", num_envs=N)`: 30 dofs (24 hand joints + 6-dof pen; the arm is fixed), obs 45; the
    target orientation (model.body_quat[target], two Euler angles ~ U(-1, 1)) is per-env state
    (envs/adroit_hand/adroit_pen.py:288-430)."""

    TASK_NAME, MODEL_NAME = "AdroitHandPen", "adroit_pen"
    make_task = staticmethod(make_pen_task)
    RESET_DRAWS = (("euler", 0, -1.0, 1.0), ("euler", 1, -1.0, 1.0))    # adroit_pen.py:379-384: body_quat[target] = euler2quat([u, u, 0])
    STATE_KEYS = (("desired_orien", "penv", 3, 4),)                      # adroit_pen.py:401-430


class AdroitDoorVectorEnv(_AdroitVectorEnv):
    """`gym.make_vec("AdroitHandDoor-v2", num_envs=N)`: 30 dofs (4-dof arm + 24 hand joints + door hinge + latch), obs 39; the
    door frame position (model.body_pos[frame]) is per-env state (envs/adroit_hand/adroit_door.py:279-402)."""

    TASK_NAME, MODEL_NAME = "AdroitHandDoor", "adroit_door"
    make_task = staticmethod(make_door_task)
    RESET_DRAWS = (("penv", 0, -0.3, -0.2), ("penv", 1, 0.25, 0.35), ("penv", 2, 0.252, 0.35))               # adroit_door.py:359-371
    STATE_KEYS = (("door_body_pos", "penv", 0, 3),)                                                           # adroit_door.py:373-402


ADROIT_TASKS = {"AdroitHandHammer": AdroitHammerVectorEnv, "AdroitHandRelocate": AdroitRelocateVectorEnv,
                "AdroitHandPen": AdroitPenVectorEnv, "AdroitHandDoor": AdroitDoorVectorEnv}


def make_adroit_vec(task, num_envs=1, **kwargs):
    if task not in ADROIT_TASKS:
        raise KeyError(f"unknown Adroit task {task!r}")
    return ADROIT_TASKS[task](num_envs=num_envs, **kwargs)
