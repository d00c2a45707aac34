"""Batched Fetch environments (`gym.vector.VectorEnv`-style) on the b200sim CUDA path.

Host-side mirror of the reference's Fetch stack, batched over `num_envs`:
  * task tables              envs/fetch/{reach,push,slide,pick_and_place}.py ctor kwargs (e.g. pick_and_place.py:139-162)
  * construction/_env_setup  envs/fetch/fetch_env.py:404-428, envs/robot_env.py:292-303
  * reset/_reset_sim/_sample_goal   envs/robot_env.py:154-186, envs/fetch/fetch_env.py:375-402, 153-166
  * step                     envs/robot_env.py:114-152  (runs entirely inside one CUDA kernel, csrc/fetch_task.cuh)
  * compute_reward/_is_success      envs/fetch/fetch_env.py:74-80, 168-170
  * TimeLimit (max_episode_steps=50) and vector autoreset as gymnasium's wrappers/vector envs do.
All per-step arithmetic happens on the GPU; this file only owns reset-time sampling and bookkeeping.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import numpy as np
import torch

from . import _lib
from .mjcf import EQ_WELD, JNT_FREE
from .models import load_model
from .spaces import Box, Dict as DictSpace
from .vector import VectorEnv

FETCH_TASKS = {
    "FetchReach": dict(model="fetch_reach", has_object=False, block_gripper=True, gripper_extra_height=0.2,
                       target_in_the_air=True, target_offset=0.0, obj_range=0.15, target_range=0.15, distance_threshold=0.05,
                       initial_qpos={"robot0:slide0": 0.4049, "robot0:slide1": 0.48, "robot0:slide2": 0.0}),
    "FetchPush": dict(model="fetch_push", has_object=True, block_gripper=True, gripper_extra_height=0.0,
                      target_in_the_air=False, target_offset=0.0, obj_range=0.15, target_range=0.15, distance_threshold=0.05,
                      initial_qpos={"robot0:slide0": 0.405, "robot0:slide1": 0.48, "robot0:slide2": 0.0,
                                    "object0:joint": [1.25, 0.53, 0.4, 1.0, 0.0, 0.0, 0.0]}),
    "FetchPickAndPlace": dict(model="fetch_pick_and_place", has_object=True, block_gripper=False, gripper_extra_height=0.2,
                              target_in_the_air=True, target_offset=0.0, obj_range=0.15, target_range=0.15,
                              distance_threshold=0.05,
                              initial_qpos={"robot0:slide0": 0.405, "robot0:slide1": 0.48, "robot0:slide2": 0.0,
                                            "object0:joint": [1.25, 0.53, 0.4, 1.0, 0.0, 0.0, 0.0]}),
    # envs/fetch/slide.py:160-190 (cylinder puck; target_offset = [0.4, 0, 0])
    "FetchSlide": dict(model="fetch_slide", has_object=True, block_gripper=True, gripper_extra_height=-0.02,
                       target_in_the_air=False, target_offset=(0.4, 0.0, 0.0), obj_range=0.1, target_range=0.3, distance_threshold=0.05,
                       initial_qpos={"robot0:slide0": 0.05, "robot0:slide1": 0.48, "robot0:slide2": 0.0,
                                     "object0:joint": [1.7, 1.1, 0.41, 1.0, 0.0, 0.0, 0.0]}),
}
N_SUBSTEPS = 20
REF_POINT = (1.0, 0.75, 0.4)  # fixed world point the device spatial algebra is expressed about
# the same point of the other families, inside each robot's workspace
HAND_REF_POINT = (1.0, 0.9, 0.2)
ADROIT_REF_POINT = (0.0, -0.2, 0.2)
KITCHEN_REF_POINT = (-0.2, 0.3, 1.8)


def reference_point(task):
    """The fixed world point of a task's spatial algebra, by task kind: Fetch (0) and maze (1) REF_POINT, Hand (2, 3) HAND_REF_POINT,
    Adroit (4-7) ADROIT_REF_POINT, Kitchen (8) KITCHEN_REF_POINT."""
    k = int(task.kind)
    return HAND_REF_POINT if k in (2, 3) else ADROIT_REF_POINT if 4 <= k <= 7 else KITCHEN_REF_POINT if k == 8 else REF_POINT


def make_task_struct(model, cfg, reward_type, n_substeps=N_SUBSTEPS):
    t = _lib.FetchTaskC()
    t.has_object, t.block_gripper = int(cfg["has_object"]), int(cfg["block_gripper"])
    t.n_substeps, t.reward_dense = n_substeps, int(reward_type == "dense")
    t.grip_site = model.site_id("robot0:grip")
    t.obj_site = model.site_id("object0") if cfg["has_object"] else -1
    t.frame_site = model.frame_site("robot0:gripper_link")
    robot = [j for j, n in enumerate(model.names["joint"]) if n.startswith("robot")]
    t.nrobot = len(robot)
    for i, j in enumerate(robot):
        t.robot_qadr[i], t.robot_dadr[i] = int(model.jnt_qposadr[j]), int(model.jnt_dofadr[j])
    t.finger_qadr[0] = int(model.jnt_qposadr[model.joint_id("robot0:l_gripper_finger_joint")])
    t.finger_qadr[1] = int(model.jnt_qposadr[model.joint_id("robot0:r_gripper_finger_joint")])
    t.nobs = 25 if cfg["has_object"] else 10
    t.distance_threshold = float(cfg["distance_threshold"])
    t.dt = float(model.opt[0] * n_substeps)
    return t


def welded_eq_data(model):
    """utils/mujoco_utils.py:74-80 reset_mocap_welds, applied to the model constants before upload."""
    eq = np.array(model.eq_data, dtype=np.float64).reshape(-1, 11).copy()
    for i in range(model.neq):
        if model.eq_type[i] == EQ_WELD:
            eq[i, :7] = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]
    return eq


class _DevArray:
    def __init__(self, ptr, shape, typestr="<f4"):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (int(ptr), False), "version": 3, "strides": None}


class CudaBackend:
    """Thin owner of a `b200sim_t` handle; all arguments are torch CUDA tensors passed as raw device pointers.

    Outputs are PACKED (b200sim_set_packed): one [N, W] fp32 row per env, obs | achieved | desired | reward | success | terminated |
    truncated; `new_outputs()` hands out that buffer under "packed" next to column views of it under the classic names, so one
    device->host copy (or one all-gather) moves everything a step produced."""

    def __init__(self, model, eq_data, task, num_envs, device):
        if not torch.cuda.is_available():
            raise RuntimeError("b200sim needs a CUDA device: there is no CPU fallback on the product path")
        self.device = torch.device(device)
        self.L = _lib.lib()
        blob = model.to_blob()
        h = ctypes.c_void_p()
        self.ref = reference_point(task)
        ref = np.asarray(self.ref, dtype=np.float32)
        # eq_data: NULL (keep the blob's equality data) or exactly neq x 11 doubles (include/b200sim.h); the C side cannot see the
        # length, so an empty override must become NULL here -- a pointer to a zero-length array would be read out of bounds
        eq = np.ascontiguousarray(eq_data, dtype=np.float64)
        if eq.size not in (0, 11 * int(model.neq)):
            raise ValueError(f"eq_data must be empty or [neq = {int(model.neq)}, 11], got shape {eq.shape}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        rc = self.L.b200sim_create(blob, len(blob), eq.ctypes.data if eq.size else None, ref.ctypes.data, ctypes.byref(task), num_envs,
                                   self.device.index, ctypes.byref(h))
        if rc != 0:
            raise RuntimeError(f"b200sim_create failed ({rc}): {self.L.b200sim_last_error(None).decode()}")
        self.h = h
        self.num_envs, self.nobs = num_envs, task.nobs
        self.ngoal, self.nact = (3, 4) if task.kind == 0 else (task.ngoal, task.nact)
        lay = (ctypes.c_int * 9)()
        self.L.b200sim_layout(h, lay)
        self.layout = dict(zip(("qpos", "qvel", "warm", "ctrl", "mocap", "pose", "goal", "stride", "penv"), list(lay)))
        self.state = torch.as_tensor(_DevArray(self.L.b200sim_state(h), (num_envs, self.layout["stride"])), device=self.device)
        # per-env step counters of the in-kernel TimeLimit (b200sim_set_time_limit), capacity-overflow counter, info words
        self.elapsed = torch.as_tensor(_DevArray(self.L.b200sim_elapsed(h), (num_envs,), "<i4"), device=self.device)
        self.overflow_counter = torch.as_tensor(_DevArray(self.L.b200sim_overflow_counter(h), (1,), "<i8"), device=self.device)
        self.info = torch.zeros(num_envs, dtype=torch.int32, device=self.device)
        self.packed_w = int(self.L.b200sim_set_packed(h, 1))

    def set_time_limit(self, max_episode_steps, terminate_on_success=False):
        self._check(self.L.b200sim_set_time_limit(self.h, int(max_episode_steps or 0), int(bool(terminate_on_success))))

    def close(self):
        if getattr(self, "h", None):
            self.state = None
            self.L.b200sim_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(f"b200sim call failed ({rc}): {self.L.b200sim_last_error(self.h).decode()}")

    def new_outputs(self):
        n, d, no, ng = self.num_envs, self.device, self.nobs, self.ngoal
        p = torch.zeros((n, self.packed_w), dtype=torch.float32, device=d)   # zeros: refresh / raw launches do not write the flags
        flags = torch.zeros((2, n), dtype=torch.uint8, device=d)
        k = no + 2 * ng
        return dict(packed=p, obs=p[:, :no], achieved=p[:, no:no + ng], desired=p[:, no + ng:k], reward=p[:, k], success=p[:, k + 1],
                    terminated=flags[0].view(torch.bool), truncated=flags[1].view(torch.bool), flags=flags)

    def _ptrs(self, out):
        return [out["packed"].data_ptr(), None, None, None, None]

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def step(self, actions, out, info=None):
        """One env-step of every env; the flags of the step land in out["terminated"] / out["truncated"], the solver's info word
        (Newton iterations | capacity-overflow bits << 16) in `info` (default: the backend's persistent `self.info`)."""
        assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous() and actions.shape == (self.num_envs, self.nact)
        info = self.info if info is None else info
        f = out["flags"]
        self._check(self.L.b200sim_step(self.h, actions.data_ptr(), *self._ptrs(out), f[0].data_ptr(), f[1].data_ptr(), info.data_ptr(),
                                        self._stream()))

    def refresh(self, mask, out):
        self._check(self.L.b200sim_refresh(self.h, mask.data_ptr() if mask is not None else None, *self._ptrs(out), self._stream()))

    def raw_step(self, nstep, out, mask=None):
        if mask is None:
            self._check(self.L.b200sim_raw_step(self.h, int(nstep), *self._ptrs(out), self._stream()))
        else:
            self._check(self.L.b200sim_raw_step_masked(self.h, mask.data_ptr(), int(nstep), *self._ptrs(out), self._stream()))

    def reset_draw(self, mask, rest_record, params, seed, env_offset, episode, out):
        """b200sim_reset: in-kernel draw of object start + goal for the masked envs (None = all), then mj_forward + _get_obs."""
        assert rest_record.is_cuda and rest_record.dtype == torch.float32 and rest_record.numel() == self.layout["stride"]
        assert episode.is_cuda and episode.dtype == torch.int32 and episode.numel() == self.num_envs
        self._check(self.L.b200sim_reset(self.h, mask.data_ptr() if mask is not None else None, rest_record.data_ptr(), ctypes.byref(params),
                                         int(seed) & 0xFFFFFFFFFFFFFFFF, int(env_offset), episode.data_ptr(), *self._ptrs(out), self._stream()))

    def reset_uniform(self, mask, rest_record, params, seed, env_offset, episode, out):
        """b200sim_reset_uniform: record <- rest record + a fixed list of uniform draws, then mj_forward + _get_obs."""
        assert rest_record.is_cuda and rest_record.dtype == torch.float32 and rest_record.numel() == self.layout["stride"]
        assert episode.is_cuda and episode.dtype == torch.int32 and episode.numel() == self.num_envs
        self._check(self.L.b200sim_reset_uniform(self.h, mask.data_ptr() if mask is not None else None, rest_record.data_ptr(), ctypes.byref(params),
                                                 int(seed) & 0xFFFFFFFFFFFFFFFF, int(env_offset), episode.data_ptr(), *self._ptrs(out), self._stream()))

    def set_obs_noise(self, scale, seed, env_offset, episode):
        """b200sim_set_obs_noise (kitchen builds): later launches add u * scale to the observation, u drawn per (seed, env, episode,
        step); scale None turns the noise off.  The handle keeps both pointers: the tensors must outlive its launches."""
        if scale is not None:
            assert scale.is_cuda and scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == self.nobs
            assert episode.is_cuda and episode.dtype == torch.int32 and episode.is_contiguous() and episode.numel() == self.num_envs
        self._check(self.L.b200sim_set_obs_noise(self.h, scale.data_ptr() if scale is not None else None, int(seed) & 0xFFFFFFFFFFFFFFFF,
                                                 int(env_offset), episode.data_ptr() if scale is not None else None))

    def set_env_keys(self, keys):
        """b200sim_set_env_keys: every later draw of env i (resets, goal update / redraw, observation noise) is keyed by keys[i]
        (int64 [N] on the device, read as unsigned) in place of the seed; None turns the table off.  The handle keeps the pointer:
        the tensor must outlive its launches."""
        if keys is not None:
            assert keys.is_cuda and keys.dtype == torch.int64 and keys.is_contiguous() and keys.numel() == self.num_envs
        self._check(self.L.b200sim_set_env_keys(self.h, keys.data_ptr() if keys is not None else None))

    def set_goal_update(self, goal_xy, scaling, noise, seed, env_offset, episode, fn="b200sim_set_goal_update"):
        """b200sim_set_goal_update (maze tasks): every later step redraws the goal of the envs that succeeded, per (seed, env,
        episode, step); goal_xy None turns the update off.  The handle keeps both pointers: the tensors must outlive its steps."""
        if goal_xy is not None:
            assert goal_xy.is_cuda and goal_xy.dtype == torch.float32 and goal_xy.is_contiguous() and goal_xy.dim() == 2 and goal_xy.shape[1] == 2
            assert episode.is_cuda and episode.dtype == torch.int32 and episode.is_contiguous() and episode.numel() == self.num_envs
        on = goal_xy is not None
        self._check(getattr(self.L, fn)(self.h, goal_xy.data_ptr() if on else None, len(goal_xy) if on else 0, float(scaling),
                                        float(noise), int(seed) & 0xFFFFFFFFFFFFFFFF, int(env_offset), episode.data_ptr() if on else None))

    def set_goal_redraw(self, goal_xy, scaling, noise, seed, env_offset, episode):
        """b200sim_set_goal_redraw (AntMaze-v3): every later step draws ONE new goal for the envs that succeeded and writes their
        reward again against it; it shares the handle's slot with set_goal_update (setting one replaces the other)."""
        self.set_goal_update(goal_xy, scaling, noise, seed, env_offset, episode, fn="b200sim_set_goal_redraw")

    def set_ant_info(self, params, rows, origin):
        """b200sim_set_ant_info (ant-build handles): the Ant's keywords, and the [N, 9] info rows later launches write (None: no rows)
        with the [N, 2] Ant-v5 reset positions.  The handle keeps both pointers: the tensors must outlive its launches."""
        for t, w in ((rows, 9), (origin, 2)):
            if t is not None:
                assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == (self.num_envs, w)
        self._check(self.L.b200sim_set_ant_info(self.h, ctypes.byref(params), rows.data_ptr() if rows is not None else None,
                                                origin.data_ptr() if origin is not None else None))

    def reset_maze(self, mask, rest_record, params, goal_xy, reset_xy, seed, env_offset, episode, out):
        """b200sim_reset_maze: goal cell + noise, reset cell away from the goal + noise, then mj_forward + _get_obs."""
        assert rest_record.is_cuda and rest_record.dtype == torch.float32 and rest_record.numel() == self.layout["stride"]
        assert episode.is_cuda and episode.dtype == torch.int32 and episode.numel() == self.num_envs
        for t, n in ((goal_xy, params.n_goal), (reset_xy, params.n_reset)):
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == (n, 2)
        self._check(self.L.b200sim_reset_maze(self.h, mask.data_ptr() if mask is not None else None, rest_record.data_ptr(), ctypes.byref(params),
                                              goal_xy.data_ptr(), reset_xy.data_ptr(), int(seed) & 0xFFFFFFFFFFFFFFFF, int(env_offset),
                                              episode.data_ptr(), *self._ptrs(out), self._stream()))

    def reset_hand_pose(self, mask, rest_record, params, parallel, seed, env_offset, episode, attempt):
        """b200sim_reset_hand_pose: records of the masked envs <- rest record + drawn object start pose (goal kept); no refresh."""
        assert rest_record.is_cuda and rest_record.numel() == self.layout["stride"] and parallel.is_cuda and tuple(parallel.shape) == (24, 4)
        self._check(self.L.b200sim_reset_hand_pose(self.h, mask.data_ptr() if mask is not None else None, rest_record.data_ptr(), ctypes.byref(params),
                                                   parallel.data_ptr(), int(seed) & 0xFFFFFFFFFFFFFFFF, int(env_offset), episode.data_ptr(),
                                                   int(attempt), self._stream()))

    def reset_hand_goal(self, mask, params, parallel, seed, env_offset, episode, out):
        """b200sim_reset_hand_goal: goal drawn from the settled object pose, episode counters incremented, then the refresh."""
        self._check(self.L.b200sim_reset_hand_goal(self.h, mask.data_ptr() if mask is not None else None, ctypes.byref(params), parallel.data_ptr(),
                                                   int(seed) & 0xFFFFFFFFFFFFFFFF, int(env_offset), episode.data_ptr(), *self._ptrs(out),
                                                   self._stream()))

    def reset_reach(self, mask, rest_record, params, seed, env_offset, episode, out):
        """b200sim_reset_reach: HandReach goal drawn on the device, then mj_forward + _get_obs."""
        assert rest_record.is_cuda and rest_record.numel() == self.layout["stride"] and episode.is_cuda and episode.dtype == torch.int32
        self._check(self.L.b200sim_reset_reach(self.h, mask.data_ptr() if mask is not None else None, rest_record.data_ptr(), ctypes.byref(params),
                                               int(seed) & 0xFFFFFFFFFFFFFFFF, int(env_offset), episode.data_ptr(), *self._ptrs(out), self._stream()))

    def check_state(self, bad, rest_record, keep):
        """b200sim_check_state: bad[i] = record i holds NaN / |x| > 1e10; such records are put back to `rest_record` (if given)."""
        assert bad.is_cuda and bad.dtype == torch.uint8 and bad.numel() == self.num_envs
        self._check(self.L.b200sim_check_state(self.h, bad.data_ptr(), rest_record.data_ptr() if rest_record is not None else None,
                                               ctypes.byref(keep) if keep is not None else None, self._stream()))

    def compute_reward(self, ag, dg):
        ag = ag.to(self.device, torch.float32).contiguous().reshape(-1, self.ngoal)
        dg = dg.to(self.device, torch.float32).contiguous().reshape(-1, self.ngoal)
        out = torch.empty(ag.shape[0], dtype=torch.float32, device=self.device)
        self._check(self.L.b200sim_compute_reward(self.h, ag.data_ptr(), dg.data_ptr(), ag.shape[0], out.data_ptr(), self._stream()))
        return out

    @property
    def launches(self):
        return int(self.L.b200sim_launch_count(self.h))


class FetchVectorEnv(VectorEnv):
    """`gym.make_vec("FetchPickAndPlace-v4", num_envs=N)` replacement.  Observations, rewards and flags are torch
    tensors on `device` (float32 / bool) with a leading `num_envs` axis."""

    def __init__(self, task: str = "FetchPickAndPlace", num_envs: int = 1, reward_type: str = "sparse",
                 max_episode_steps: Optional[int] = 50, device="cuda:0", rng_mode: str = "auto",
                 autoreset_mode: str = "next_step", n_substeps: int = N_SUBSTEPS, backend_factory=None, **kwargs):
        if task not in FETCH_TASKS:
            raise KeyError(f"unknown Fetch task {task!r}")
        if reward_type not in ("sparse", "dense"):
            raise ValueError("reward_type must be 'sparse' or 'dense'")
        cfg = dict(FETCH_TASKS[task])
        self.task_name, self.cfg, self.reward_type = task, cfg, reward_type
        m = load_model(cfg["model"])
        t = make_task_struct(m, cfg, reward_type, n_substeps)
        box = lambda n: Box(-np.inf, np.inf, shape=(n,), dtype=np.float64)
        # robot_env.py:106-112: compute_terminated is constant False, so the kernel's TimeLimit is the only episode end
        super().__init__(model=m, task=t, fields=(("qpos", m.nq), ("qvel", m.nv), ("warm", m.nv), ("ctrl", m.nu), ("mocap", 7),
                                                  ("pose", 7), ("goal", 3)),
                         action_space=Box(-1.0, 1.0, shape=(4,), dtype=np.float32),
                         observation_space=DictSpace(dict(desired_goal=box(3), achieved_goal=box(3), observation=box(t.nobs))),
                         backend_factory=backend_factory or CudaBackend, eq_data=welded_eq_data(m), num_envs=num_envs, device=device,
                         max_episode_steps=max_episode_steps, autoreset_mode=autoreset_mode, rng_mode=rng_mode,
                         n_substeps=n_substeps, kwargs=kwargs)
        self._env_setup()

    # ------------------------------------------------------------------ construction
    def _env_setup(self):
        """envs/fetch/fetch_env.py:404-428 run once for every env in lock-step (all envs are identical here)."""
        m, st, sl = self.model, self.backend.state, self._sl
        qpos = np.array(m.qpos0, dtype=np.float64)
        for name, value in self.cfg["initial_qpos"].items():
            j = m.joint_id(name)
            a = int(m.jnt_qposadr[j])
            n = 7 if m.jnt_type[j] == JNT_FREE else 1
            qpos[a:a + n] = value
        st.zero_()
        st[:, sl["qpos"]] = torch.as_tensor(qpos, dtype=torch.float32, device=self.device)
        st[:, sl["mocap"]] = torch.tensor([0, 0, 0, 1, 0, 0, 0], dtype=torch.float32, device=self.device)
        out = self.backend.new_outputs()
        self.backend.refresh(None, out)  # mj_forward
        grip = out["obs"][:, 0:3]
        target = grip + torch.tensor([-0.498, 0.005, -0.431 + self.cfg["gripper_extra_height"]], dtype=torch.float32, device=self.device)
        st[:, sl["mocap"]] = torch.cat([target, torch.tensor([1.0, 0.0, 1.0, 0.0], device=self.device).expand(self.num_envs, 4)], dim=1)
        self.backend.raw_step(10 * self.n_substeps, out)  # 10 x mj_step(nstep=n_substeps)
        # site positions as of the last forward pass (the reference reads data.site_xpos without a new mj_forward)
        self.initial_gripper_xpos = out["obs"][0, 0:3].clone()
        self.height_offset = float(out["obs"][0, 5]) if self.cfg["has_object"] else None
        self.initial_qpos = st[0, sl["qpos"]].clone()
        self.initial_qvel = st[0, sl["qvel"]].clone()
        self._mocap_rest = torch.tensor([0, 0, 0, 1, 0, 0, 0], dtype=torch.float32, device=self.device)
        self._obj_qadr = int(m.jnt_qposadr[m.joint_id("object0:joint")]) if self.cfg["has_object"] else -1
        self._last = out

    def _rest_record(self):
        rest = torch.zeros(self.backend.state.shape[1], dtype=torch.float32, device=self.device)
        rest[self._sl["qpos"]] = self.initial_qpos
        rest[self._sl["qvel"]] = self.initial_qvel
        rest[self._sl["mocap"]] = self._mocap_rest
        return rest

    # ------------------------------------------------------------------ sampling
    def _sample_reset(self, idx):
        """Object start position (fetch_env.py:386-399) and goal (fetch_env.py:153-166) for the envs in `idx`."""
        cfg, n = self.cfg, idx.numel()
        g0 = self.initial_gripper_xpos
        off = cfg["target_offset"]
        if self.rng_mode == "numpy":
            g0n = g0.double().cpu().numpy()
            obj = np.zeros((n, 2))
            goals = np.zeros((n, 3))
            for k, i in enumerate(idx.tolist()):
                rng = self._np_rngs[i]
                if cfg["has_object"]:
                    xy = g0n[:2]
                    while np.linalg.norm(xy - g0n[:2]) < 0.1:
                        xy = g0n[:2] + rng.uniform(-cfg["obj_range"], cfg["obj_range"], size=2)
                    obj[k] = xy
                    goal = g0n[:3] + rng.uniform(-cfg["target_range"], cfg["target_range"], size=3)
                    goal += off
                    goal[2] = self.height_offset
                    if cfg["target_in_the_air"] and rng.uniform() < 0.5:
                        goal[2] += rng.uniform(0, 0.45)
                else:
                    goal = g0n[:3] + rng.uniform(-cfg["target_range"], cfg["target_range"], size=3)
                goals[k] = goal
            return (torch.as_tensor(obj, dtype=torch.float32, device=self.device) if cfg["has_object"] else None,
                    torch.as_tensor(goals, dtype=torch.float32, device=self.device))
        # device RNG (Philox): same distributions, different stream
        u = lambda *s: torch.rand(*s, generator=self._gen, device=self.device)
        obj = None
        if cfg["has_object"]:
            # rejection sampling (fetch_env.py:386-392) without a host round trip: masked redraws until a rejected sample is
            # left with probability p^(k+1) < 1e-11 per env, p = pi 0.1^2 / (2 obj_range)^2 -- 24 redraws for obj_range 0.15
            # (p = 0.35), 105 for FetchSlide's 0.1 (p = 0.79; 24 would leave 0.2 % of its resets inside the excluded disc)
            p_rej = min(np.pi * 0.01 / (2 * cfg["obj_range"]) ** 2, 0.999)
            redraws = 24 if p_rej < 0.36 else int(np.ceil(np.log(1e-11) / np.log(p_rej)))
            obj = g0[:2] + (u(n, 2) * 2 - 1) * cfg["obj_range"]
            for _ in range(redraws):
                bad = torch.linalg.norm(obj - g0[:2], dim=1) < 0.1
                obj = torch.where(bad[:, None], g0[:2] + (u(n, 2) * 2 - 1) * cfg["obj_range"], obj)
        goals = g0[:3] + (u(n, 3) * 2 - 1) * cfg["target_range"]
        if cfg["has_object"]:
            goals = goals + torch.as_tensor(off, dtype=torch.float32, device=self.device)
            goals[:, 2] = self.height_offset
            if cfg["target_in_the_air"]:
                air = u(n) < 0.5
                goals[:, 2] += torch.where(air, u(n) * 0.45, torch.zeros(n, device=self.device))
        return obj, goals

    def _device_reset_params(self):
        from ._lib import FetchResetC

        cfg, p = self.cfg, FetchResetC()
        p.has_object, p.target_in_the_air, p.obj_qadr = int(cfg["has_object"]), int(cfg["target_in_the_air"]), max(self._obj_qadr, 0)
        p.obj_range, p.target_range = float(cfg.get("obj_range", 0.0)), float(cfg["target_range"])
        g0 = self.initial_gripper_xpos.cpu().tolist()
        for k in range(3):
            p.target_offset[k] = float(np.broadcast_to(np.asarray(cfg["target_offset"], dtype=np.float64), (3,))[k])
            p.gripper_xpos[k] = float(g0[k])
        p.height_offset = float(self.height_offset or 0.0)
        return p, self._rest

    def _reset_envs(self, mask, out, options=None):
        if self.rng_mode == "device":
            if self._dev_reset is None:
                self._dev_reset = self._device_reset_params()
            p, rest = self._dev_reset
            every = self._reset_all
            self.backend.reset_draw(None if every else mask.to(torch.uint8), rest, p, self._dev_seed, self.env_offset, self._episode, out)
            if every:
                self._elapsed.zero_()
            else:
                self._elapsed.masked_fill_(mask, 0)
            return
        idx = self._mask_indices(mask)
        if idx.numel() == 0:
            return
        st, sl = self.backend.state, self._sl
        obj, goals = self._sample_reset(idx)
        rec = self._rest.expand(idx.numel(), -1).clone()  # mj_resetData
        if obj is not None:
            rec[:, sl["qpos"].start + self._obj_qadr: sl["qpos"].start + self._obj_qadr + 2] = obj
        rec[:, sl["goal"]] = goals
        st[idx] = rec
        self._elapsed[idx] = 0
        self.backend.refresh(mask.to(torch.uint8), out)  # mj_forward + _get_obs for the reset envs
