"""The base class of the batched vector envs: construction plumbing, seeding, the gymnasium autoreset state machine and the
state access every family shares.

A family passes its model, task struct, state-record fields, spaces and backend to `VectorEnv.__init__`, and supplies
  * `_rest_record()`: the state record `mj_resetData` leaves (host reset template, device reset, `auto_recover`);
  * `_reset_envs(mask, out, options=None)`: reset the envs in `mask` (every env while `_reset_all` is set) and refresh `out`;
  * `_obs_dict(out)`: the observation of the step's outputs;
and, where the family's step results are not the packed row's columns, the step hooks below (`_kernel_input`, `_step_results`,
`_mask_results`, `_after_autoreset`).
"""
from __future__ import annotations

import functools

import numpy as np
import torch

from .rollout import CtorPickle
from .spaces import batch_space

AUTORESET_MODES = ("next_step", "same_step", "disabled")
RNG_MODES = ("auto", "numpy", "torch", "device")


def _clone(x):
    return {k: _clone(v) for k, v in x.items()} if isinstance(x, dict) else x.clone()


def _int64(seed):
    """A seed as the signed 64-bit word the library reads back as unsigned."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s - (1 << 64) if s >= 1 << 63 else s


class VectorEnv(CtorPickle):
    """Observations, rewards and flags are torch tensors on `device` with a leading `num_envs` axis."""

    metadata = {"render_modes": [], "render_fps": 25, "autoreset_mode": "next_step"}
    AUTO_RECOVER = True            # the family can put envs with NaN / huge state values back to their rest record
    DEVICE_RESET = True            # the family has rng_mode="device" (reset draws inside the library)
    RECOVERY_KEEP = ("goal",)      # record fields a recovered env keeps
    SUCCESS_KEY = "is_success"     # info key of the packed row's success column

    def __init__(self, *, model, task, fields, action_space, observation_space, backend_factory, num_envs, device,
                 max_episode_steps, autoreset_mode, rng_mode, n_substeps, kwargs, eq_data=None, terminate_on_success=False):
        if autoreset_mode not in AUTORESET_MODES:
            raise ValueError("autoreset_mode must be next_step, same_step or disabled")
        if rng_mode not in RNG_MODES:
            raise ValueError("rng_mode must be auto, numpy, torch or device")
        if rng_mode == "device" and not self.DEVICE_RESET:
            raise NotImplementedError(f"rng_mode='device' (in-kernel reset draws) does not exist for {type(self).__name__}")
        if kwargs.get("render_mode") is not None:
            raise NotImplementedError("rendering is out of scope for the batched CUDA path")
        # opt-in failure detection: after every step the state records are scanned for NaN / huge values and such envs are put
        # back to their rest record with the goal kept ([ext] mj_checkPos / mj_checkVel / mj_checkAcc + mj_resetData in mj_step)
        self.auto_recover = bool(kwargs.get("auto_recover", False))
        if self.auto_recover and not self.AUTO_RECOVER:
            raise NotImplementedError(f"auto_recover is not available for {type(self).__name__}")
        self.model, self.task = model, task
        self.num_envs, self.max_episode_steps, self.autoreset_mode = int(num_envs), max_episode_steps, autoreset_mode
        self.metadata = dict(self.metadata, autoreset_mode=autoreset_mode)
        self.n_substeps = int(n_substeps)
        self.dt = float(model.opt[0] * n_substeps)
        self.backend = backend_factory(model, np.zeros((0, 11)) if eq_data is None else eq_data, task, self.num_envs, device)
        self.device = self.backend.device
        lay = self.backend.layout
        self._sl = {k: slice(lay[k], lay[k] + n) for k, n in fields}
        self.single_action_space, self.single_observation_space = action_space, observation_space
        self.action_space = batch_space(action_space, self.num_envs)
        self.observation_space = batch_space(observation_space, self.num_envs)
        # "numpy": per-env PCG64 streams in the reference's draw order (value-equal resets); "torch": torch's device generator;
        # "device": the draws happen inside the library (csrc/reset_sample.cuh) -- no host work per reset
        self.rng_mode = rng_mode if rng_mode != "auto" else ("numpy" if self.num_envs <= 64 else "torch")
        self.env_offset = int(kwargs.get("env_offset", 0))   # global index of env 0 (sharded runs, sharding.py)
        self._np_rngs = self._new_np_rngs([None] * self.num_envs) if self.rng_mode == "numpy" else None
        self._gen = torch.Generator(device=self.device)
        self._gen.seed()
        self._dev_seed = int(self._gen.initial_seed())
        # TimeLimit and the terminated / truncated flags are computed by the step kernel (b200sim_set_time_limit); the per-env
        # step counters live in the library and are visible here as a tensor
        self._elapsed = self.backend.elapsed
        self.backend.set_time_limit(max_episode_steps, terminate_on_success)
        self._can_terminate = bool(terminate_on_success)
        n, dev = self.num_envs, self.device
        self._needs_reset = torch.zeros(n, dtype=torch.bool, device=dev)
        self._all_idx = torch.arange(n, device=dev)
        self._const_true = torch.ones(n, dtype=torch.bool, device=dev)
        # autoreset state: `_elapsed_ub` is a host-side upper bound of max(_elapsed); `_in_phase`: every env was reset together and
        # none can terminate, so the bound IS every env's step count and the TimeLimit is known without reading the device
        self._elapsed_ub, self._pending_reset, self._in_phase, self._reset_all = 0, False, False, False
        self._episode = self._keys = self._dev_reset = self._recovery = None   # built below / by the first device reset / recovery
        if self.rng_mode == "device":
            # per-env episode counters and Philox keys of the library's draws (b200sim_set_env_keys): a full reset with a seed gives every
            # env that key, a partial one gives it to the envs it resets and leaves the others' streams alone.  A backend without
            # the hook draws every env with the batch seed and refuses only a partial reset with a seed
            self._episode = torch.zeros(n, dtype=torch.int32, device=dev)
            if getattr(self.backend, "set_env_keys", None) is not None:
                self._keys = torch.full((n,), _int64(self._dev_seed), dtype=torch.int64, device=dev)
                self.backend.set_env_keys(self._keys)
        self._last = None
        self.closed = False

    @staticmethod
    def _new_np_rngs(seeds):
        return [np.random.Generator(np.random.PCG64(np.random.SeedSequence(s))) for s in seeds]

    @functools.cached_property
    def _rest(self):
        return self._rest_record()

    def _rest_record(self):
        """The state record mj_resetData leaves (ctrl, warm start and time zero)."""
        raise NotImplementedError

    def _mask_indices(self, mask):
        """Indices of the envs in `mask`; no device round trip when every env is due (`_reset_all`)."""
        return self._all_idx if self._reset_all else torch.nonzero(mask, as_tuple=False).flatten()

    def _reset(self, mask, out, every, options=None):
        self._reset_all = every
        try:
            self._reset_envs(mask, out, options)
        finally:
            self._reset_all = False

    # ------------------------------------------------------------------ gymnasium API
    def _obs_dict(self, out):
        return self._cast_obs({"observation": out["obs"], "achieved_goal": out["achieved"], "desired_goal": out["desired"]})

    def _reset_info(self, out):
        return {}

    def _seeds(self, seed):
        return [seed + i for i in range(self.num_envs)] if isinstance(seed, (int, np.integer)) else list(seed)

    def reset(self, *, seed=None, options=None):
        """Gymnasium's vector reset.  `options={"reset_mask": mask}` resets only the envs in `mask` (a numpy bool array of shape
        (num_envs,), Gymnasium's form, with at least one True; or a torch.bool tensor, the GPU-native form, which is not read, so an
        all-False one is a no-op); the other options go to the family's reset.  The whole batch comes back: the masked rows hold
        their new episode's first observation, the others their current one.  A reset of mask M with `seed=x` leaves each env of M
        as a full `reset(seed=x)` would (record, observation, step counter and RNG stream) and every other env as it was: in
        rng_mode="numpy" env i of M gets the generator of seed x + i (or x[i]); in "device" it gets the key x (or x[0]) and its
        episode counter restarts, so it replays its episode of a full reset bit for bit, later goal updates and observation noise
        included; in "torch" x reseeds the one device generator and the masked envs draw from it, which promises equal
        distributions only.  With seed=None the masked envs continue their own streams."""
        if options and "reset_mask" in options:
            options = dict(options)
            mask, every = self._reset_mask(options.pop("reset_mask"))
            return self._partial_reset(mask, every, seed, options or None)
        if seed is not None:
            seeds = self._seeds(seed)
            if self._np_rngs is not None:
                self._np_rngs = self._new_np_rngs(seeds)
            self._gen.manual_seed(int(seeds[0]))
            self._dev_seed = int(seeds[0])   # rng_mode="device": one key for the batch; env index and episode counter select the stream
            if self._episode is not None:
                self._episode.zero_()
            if self._keys is not None:
                self._keys.fill_(_int64(self._dev_seed))
        out = self.backend.new_outputs()
        self._reset(torch.ones(self.num_envs, dtype=torch.bool, device=self.device), out, True, options)
        self._needs_reset.zero_()
        self._elapsed_ub, self._pending_reset, self._in_phase = 0, False, not self._can_terminate
        self._last = out
        return self._obs_dict(out), self._reset_info(out)

    def _reset_mask(self, mask):
        """The mask on the device, and whether it holds every env (None for a torch mask: finding out would read the device)."""
        shape = (self.num_envs,)
        if isinstance(mask, np.ndarray):
            if mask.dtype != np.bool_ or mask.shape != shape:
                raise ValueError(f"reset_mask must be a bool array of shape {shape}, got {mask.dtype} {mask.shape}")
            if not mask.any():
                raise ValueError("reset_mask has no True entry: no env would be reset")
            return torch.from_numpy(mask).to(self.device), bool(mask.all())
        if torch.is_tensor(mask):
            if mask.dtype != torch.bool or tuple(mask.shape) != shape:
                raise ValueError(f"reset_mask must be a torch.bool tensor of shape {shape}, got {mask.dtype} {tuple(mask.shape)}")
            return mask.to(self.device), None
        raise ValueError(f"reset_mask must be a numpy bool array or a torch.bool tensor, got {type(mask).__name__}")

    def _partial_reset(self, mask, every, seed, options):
        if seed is not None and self.rng_mode == "device" and self._keys is None:
            raise NotImplementedError(f"a partial reset with a seed in rng_mode='device' needs per-env keys (set_env_keys, "
                                      f"b200sim_set_env_keys); {type(self.backend).__name__} has none")
        if seed is not None:
            seeds = self._seeds(seed)
            if self._np_rngs is not None:   # the host streams need the mask on the host
                for i in torch.nonzero(mask.cpu(), as_tuple=False).flatten().tolist():
                    self._np_rngs[i] = self._new_np_rngs([seeds[i]])[0]
            self._gen.manual_seed(int(seeds[0]))
            if self._keys is not None:
                self._keys.masked_fill_(mask, _int64(seeds[0]))
                self._episode.masked_fill_(mask, 0)
        out = self.backend.new_outputs()
        if self._last is not None:   # the rows outside the mask keep their current observation
            out["packed"].copy_(self._last["packed"])
            out["packed"].masked_fill_(mask[:, None], 0.0)
            out["flags"].copy_(self._last["flags"])
            out["flags"].masked_fill_(mask[None, :], 0)
        self._reset(mask, out, False, options)
        self._needs_reset = self._needs_reset & ~mask   # a pending NEXT_STEP autoreset of a masked env is cancelled
        # the step bound stays valid (reset envs count from 0); the envs are in phase again only when every one was reset
        if every:
            self._elapsed_ub, self._pending_reset, self._in_phase = 0, False, not self._can_terminate
        else:
            self._in_phase = False
        self._last = out
        info = self._reset_info(out)
        for k in info:
            if k.startswith("_"):
                info[k] = mask
        return self._obs_dict(out), info

    # step hooks: the defaults serve the families whose step results are the packed row's columns
    def _kernel_input(self, actions):
        return actions.contiguous()

    def _step_results(self, out):
        """(reward, terminated, truncated, info) of the step the kernel just took.  solver_info: Newton iterations (low 16 bits) |
        capacity-overflow flags << 16 of this step, per env (the backend's persistent tensor: valid until the next step)."""
        return out["reward"], out["terminated"], out["truncated"], {"solver_info": self.backend.info}

    def _mask_results(self, out, pre, reward, terminated, truncated, info):
        """NEXT_STEP autoreset: the envs in `pre` were reset instead of stepped -- reward 0, no success, no flags (in place, so the
        packed row stays the single source of the step's results)."""
        k = self.backend.nobs + 2 * self.backend.ngoal
        out["packed"][:, k:k + 4].masked_fill_(pre[:, None], 0.0)
        out["flags"].masked_fill_(pre[None, :], 0)
        return reward, terminated, truncated, info

    def _after_autoreset(self, out, info):
        pass

    def _success(self, column):
        """The info value of the packed row's success column."""
        return column

    def _final_info(self, out, info, done):
        """gymnasium's SAME_STEP convention: the info of the finished episodes next to their last observation."""
        return {self.SUCCESS_KEY: self._success(out["success"].clone()), "_" + self.SUCCESS_KEY: done.clone()}

    def _finish_info(self, out, info):
        # the success column as it stands after this call's resets, and a mask saying every env reports it
        info[self.SUCCESS_KEY] = self._success(out["success"])
        info["_" + self.SUCCESS_KEY] = self._const_true

    def step(self, actions):
        if not torch.is_tensor(actions):
            actions = torch.as_tensor(np.asarray(actions, dtype=np.float32))
        if tuple(actions.shape) != (self.num_envs, self.single_action_space.shape[0]):
            raise ValueError("Action dimension mismatch")
        a = self._kernel_input(actions.to(self.device, torch.float32, non_blocking=True))
        out = self.backend.new_outputs()
        # physics + observation + reward + success + TimeLimit / terminated / truncated flags: one kernel
        self.backend.step(a, out)
        self._elapsed_ub += 1
        reward, terminated, truncated, info = self._step_results(out)
        if self.auto_recover:
            self._check_and_recover(out, info)
        # while no env can terminate, the host knows from its step bound when a TimeLimit may be due and reads the device only then
        lazy, in_phase = not self._can_terminate, self._in_phase
        if self.autoreset_mode == "next_step" and (not lazy or self._pending_reset):
            self._pending_reset = False
            if in_phase or bool(self._needs_reset.any()):
                # envs that finished on the previous call are reset now; their action is ignored (gymnasium NEXT_STEP)
                pre = self._needs_reset.clone()
                self._reset(pre, out, in_phase)
                reward, terminated, truncated, info = self._mask_results(out, pre, reward, terminated, truncated, info)
                self._needs_reset.zero_()
                if lazy:
                    self._elapsed_ub = 0 if in_phase else int(self._elapsed.max())
        self._after_autoreset(out, info)
        if not lazy or (self.max_episode_steps is not None and self._elapsed_ub >= self.max_episode_steps):
            done = truncated | terminated
            if self.autoreset_mode == "next_step":
                self._needs_reset = done
                self._pending_reset = True
            elif self.autoreset_mode == "same_step":
                if in_phase or bool(done.any()):
                    info["final_obs"] = _clone(self._obs_dict(out))
                    info["_final_obs"] = done.clone()
                    final_info = self._final_info(out, info, done)
                    if final_info is not None:
                        info["final_info"], info["_final_info"] = final_info, done.clone()
                    self._reset(done, out, in_phase)
                if lazy:
                    self._elapsed_ub = 0 if in_phase else int(self._elapsed.max())
        self._finish_info(out, info)
        self._last = out
        return self._obs_dict(out), reward, terminated, truncated, info

    # ------------------------------------------------------------------ failure recovery (auto_recover=True)
    def _check_and_recover(self, out, info):
        if self._recovery is None:
            from ._lib import KeepC

            keep = KeepC()
            keep.n = len(self.RECOVERY_KEEP)
            for k, f in enumerate(self.RECOVERY_KEEP):
                keep.start[k], keep.len[k] = self._sl[f].start, self._sl[f].stop - self._sl[f].start
            self._recovery = (self._rest, keep)
            self._bad = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
            self.bad_state_count = torch.zeros((), dtype=torch.int64, device=self.device)
        rest, keep = self._recovery
        self.backend.check_state(self._bad, rest, keep)
        self.backend.refresh(self._bad, out)          # mj_forward + _get_obs of the recovered envs (none, almost always)
        bad = self._bad.bool()
        self.bad_state_count += bad.sum()
        info["bad_state"] = bad

    @property
    def solver_overflow_count(self):
        """Env-steps so far in which a capacity limit (broad-phase candidates, contacts, contact groups, limit rows) dropped
        something (DESIGN.md deviation 5); reads the device counter (synchronises)."""
        return int(self.backend.overflow_counter[0])

    # GoalEnv API (core.py:45-114), batched; accepts numpy or torch, any leading shape
    def _reward_np_dtype(self):
        return np.float32 if self.reward_type == "sparse" else np.float64

    def compute_reward(self, achieved_goal, desired_goal, info=None):
        is_np = not torch.is_tensor(achieved_goal)
        ag = torch.as_tensor(np.asarray(achieved_goal)) if is_np else achieved_goal
        dg = torch.as_tensor(np.asarray(desired_goal)) if not torch.is_tensor(desired_goal) else desired_goal
        r = self.backend.compute_reward(ag, dg).reshape(ag.shape[:-1])
        return r.cpu().numpy().astype(self._reward_np_dtype()) if is_np else r

    def compute_terminated(self, achieved_goal, desired_goal, info=None):
        return False

    def compute_truncated(self, achieved_goal, desired_goal, info=None):
        return False

    # state access (checkpoint / parity injection), SURVEY.md section 5
    def get_state(self):
        return self.backend.state.clone(), self._elapsed.clone()

    def set_state(self, state, elapsed=None):
        self.backend.state.copy_(state)
        if elapsed is not None:
            self._elapsed.copy_(elapsed)
            self._in_phase = False
        self._elapsed_ub = int(self._elapsed.max())
        out = self.backend.new_outputs()
        self.backend.refresh(None, out)
        self._last = out
        return self._obs_dict(out)

    def close(self):
        if not self.closed:
            self.backend.close()
            self.closed = True
