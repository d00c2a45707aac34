"""CPU test backend for the vector envs: drives the host emulation of the kernel source, one env at a time, with the handle surface of
CudaBackend (gymnasium_robotics_b200/fetch.py) and the refusals, launch counts and episode bookkeeping of csrc/b200sim.cu.  Lets the
`-m "not gpu"` suite cover the host logic (reset sampling, autoreset, TimeLimit, spaces) and the kernel arithmetic without a GPU.
Test infrastructure only."""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from tests.hostsim import FLAGS, AntInfoArgsC, FetchTaskC as HostTaskC, HostSim, ObsNoiseKey, goal_redraw, goal_update, host_flavor

_U64 = 0xFFFFFFFFFFFFFFFF


class HostSimBackend:
    """The emulation of the kernel build b200sim_create would pick (tests.hostsim.host_flavor), or of `flavor` when it is given (as a
    keyword, functools.partial(HostSimBackend, flavor=...), or as the class attribute FLAVOR); the reference point is the task's."""
    FLAVOR = None
    NGRP_CAP = 0   # the contact-group capacity of the device model (0: the model's own)

    def __init__(self, model, eq_data, task, num_envs, device, flavor=None):
        from gymnasium_robotics_b200.fetch import reference_point

        self.device = torch.device("cpu")
        self.num_envs, self.nobs = num_envs, task.nobs
        flavor = self.FLAVOR if flavor is None else flavor
        self.flavor = host_flavor(model, task) if flavor is None else flavor
        penv = int(task.penv_body) if task.kind in (4, 5, 6, 7) else -1
        self.sim = HostSim(model, eq_data=eq_data if len(eq_data) else None, ref=reference_point(task), penv_body=penv, ngrp_cap=self.NGRP_CAP,
                           flavor=self.flavor)
        self.L = self.sim._L
        t = HostTaskC()
        for name, _ in task._fields_:
            setattr(t, name, getattr(task, name))
        o = 0
        lay = {}
        fetch = task.kind == 0
        if fetch:
            t.nact, t.ngoal = 4, 3
        self.ngoal, self.nact = int(t.ngoal), int(t.nact)
        for k, n in (("qpos", model.nq), ("qvel", model.nv), ("warm", model.nv), ("ctrl", model.nu), ("mocap", 7 * model.nmocap),
                     ("pose", 7 if fetch else 0), ("goal", self.ngoal), ("penv", 7 if penv > 0 else 0)):
            lay[k] = o
            o += n
        lay["stride"] = (o + 3) & ~3
        for k in ("qpos", "qvel", "warm", "ctrl", "mocap", "pose", "goal", "stride", "penv"):
            setattr(t, "st_" + k, lay[k])
        self.task, self.layout = t, lay
        self.state = torch.zeros((num_envs, lay["stride"]), dtype=torch.float32)
        self.launches = 0
        # the same episode bookkeeping as the step kernel (csrc/step_kernel.cuh): per-env step counters, flags, info words
        self.elapsed = torch.zeros(num_envs, dtype=torch.int32)
        self.info = torch.zeros(num_envs, dtype=torch.int32)
        self.overflow_counter = torch.zeros(1, dtype=torch.int64)
        self.overflow_bits = 0   # the capacity flags of every info word so far
        self.max_steps, self.term_on_success = 0, False
        self.packed_w = (self.nobs + 2 * self.ngoal + 4 + 3) & ~3
        # the handle's settings: observation noise (kitchen builds), the goal slot (maze tasks), the Ant's keywords (ant build) -- the
        # library's defaults: Ant-v5's keywords, no info rows
        self.kitchen_build, self.ant_build = "-DB200_KITCHEN" in FLAGS[self.flavor][1], self.flavor == "ant"
        self.noise = self.goal_args = None
        self.redraw = False
        self.ant = AntInfoArgsC(-1.0, 1.0, 1.0, 0.5, 5e-4, 1.0, 0.2, 1.0, 0, 0, 0, None, None)
        self.ant_rows = self.ant_origin = None
        if self.ant_build:
            assert lay["stride"] - (lay["goal"] + 2) >= 2   # the torso position is kept in the two record words after the goal

    def set_time_limit(self, max_episode_steps, terminate_on_success=False):
        self.max_steps, self.term_on_success = int(max_episode_steps or 0), bool(terminate_on_success)

    def close(self):
        pass

    def new_outputs(self):
        n, no, ng = self.num_envs, self.nobs, self.ngoal
        p = torch.zeros((n, self.packed_w))
        flags = torch.zeros((2, n), dtype=torch.uint8)
        k = no + 2 * ng
        return dict(packed=p, obs=p[:, :no], achieved=p[:, no:no + ng], desired=p[:, no + ng:k], reward=p[:, k], success=p[:, k + 1],
                    terminated=flags[0].view(torch.bool), truncated=flags[1].view(torch.bool), flags=flags)

    @staticmethod
    def _fail(code, msg):
        raise RuntimeError(f"b200sim call failed ({code}): {msg}")

    def set_obs_noise(self, scale, seed, env_offset, episode):
        """b200sim_set_obs_noise: later launches add u * scale to the observation, u drawn per (seed, env, episode, step)."""
        if not self.kitchen_build:
            self._fail(-6, "b200sim_set_obs_noise: observation noise exists in the kitchen kernel builds only")
        if scale is not None and episode is None:
            self._fail(-1, "b200sim_set_obs_noise: episode is NULL")
        if int(env_offset) < 0:
            self._fail(-1, "b200sim_set_obs_noise: negative env_offset")
        self.noise = None if scale is None else (scale.numpy(), int(seed) & _U64, int(env_offset), episode)

    def _set_goal_slot(self, fn, redraw, goal_xy, scaling, noise, seed, env_offset, episode):
        if self.task.kind != 1:
            self._fail(-6, f"{fn}: not a maze task")
        if goal_xy is not None and episode is None:
            self._fail(-1, f"{fn}: episode is NULL")
        if goal_xy is not None and len(goal_xy) < 2:
            self._fail(-1, f"{fn}: fewer than two goal cells")
        if int(env_offset) < 0:
            self._fail(-1, f"{fn}: negative env_offset")
        self.goal_args = None if goal_xy is None else (goal_xy.numpy(), float(scaling), float(noise), int(seed), int(env_offset), episode)
        self.redraw = goal_xy is not None and redraw

    def set_goal_update(self, goal_xy, scaling, noise, seed, env_offset, episode):
        """b200sim_set_goal_update: after each step, every env's record goes through rs_maze_goal_update with the key the update kernel
        builds (global index, episode counter, step counter after the step); one more launch per step while it is set."""
        self._set_goal_slot("b200sim_set_goal_update", False, goal_xy, scaling, noise, seed, env_offset, episode)

    def set_goal_redraw(self, goal_xy, scaling, noise, seed, env_offset, episode):
        """b200sim_set_goal_redraw: rs_maze_goal_redraw in place of the update, which also rewrites the changed envs' reward; it shares
        the goal slot with set_goal_update, as on the handle."""
        self._set_goal_slot("b200sim_set_goal_redraw", True, goal_xy, scaling, noise, seed, env_offset, episode)

    def set_ant_info(self, params, rows, origin):
        """b200sim_set_ant_info: the Ant's keywords, and the [N, 9] info rows later launches write with the [N, 2] reset positions."""
        if not self.ant_build:
            self._fail(-6, "b200sim_set_ant_info: not an ant-build handle (maze task with touch_mode 2..4)")
        p = params
        if p.version not in (4, 5):
            self._fail(-1, "b200sim_set_ant_info: params NULL or version not 4 / 5")
        if not p.contact_force_range[0] <= p.contact_force_range[1]:
            self._fail(-1, "b200sim_set_ant_info: contact_force_range is not (min, max)")
        if rows is not None and p.version == 5 and origin is None:
            self._fail(-1, "b200sim_set_ant_info: Ant-v5 info needs origin")
        v4 = p.version == 4
        self.ant = AntInfoArgsC(p.contact_force_range[0], p.contact_force_range[1], 1.0 if v4 else p.forward_reward_weight, p.ctrl_cost_weight,
                                p.contact_cost_weight, p.healthy_reward, p.healthy_z_range[0], p.healthy_z_range[1], int(v4),
                                int(v4 and bool(p.terminate_when_unhealthy)), int(v4 and bool(p.use_contact_forces)), None, None)
        self.ant_rows, self.ant_origin = rows, origin

    def _extra(self, i, mode, rows, origin):
        """Env i's build-specific argument of hostsim_env_step: its noise key as the step kernel builds it (global index, episode counter,
        step counter after the launch), or its Ant arguments (info row, reset position); () on the other builds."""
        if self.kitchen_build:
            if self.noise is None:
                return (None,)
            scale, seed, offset, episode = self.noise
            step = int(self.elapsed[i]) + (1 if mode == 0 else 0)
            return (ctypes.byref(ObsNoiseKey(scale.ctypes.data, seed, offset + i, int(episode[i]), step)),)
        if self.ant_build:
            a = AntInfoArgsC.from_buffer_copy(self.ant)
            a.rows = rows[i].ctypes.data if rows is not None else None
            a.origin = origin[i].ctypes.data if origin is not None else None
            return (ctypes.byref(a),)
        return ()

    def _run(self, mode, nraw, actions, mask, out, info=None):
        st = self.state.numpy()
        k = self.nobs + 2 * self.ngoal
        rows = self.ant_rows.numpy() if self.ant_rows is not None else None
        origin = self.ant_origin.numpy() if self.ant_origin is not None else None
        for i in range(self.num_envs):
            if mask is not None and not bool(mask[i]):
                continue
            a = actions[i].numpy() if actions is not None else np.zeros(self.nact, dtype=np.float32)
            obs, ag, dg, rew, suc, it = self.sim.env_step(self.task, mode, nraw, st[i], a, self.nobs, self.ngoal, *self._extra(i, mode, rows, origin))
            self.overflow_bits |= it >> 16
            out["obs"][i] = torch.from_numpy(obs); out["achieved"][i] = torch.from_numpy(ag); out["desired"][i] = torch.from_numpy(dg)
            out["reward"][i] = rew; out["success"][i] = suc
            if mode == 0:   # flags are written by step launches only (refresh / raw leave them alone)
                self.elapsed[i] += 1
                trunc = self.max_steps > 0 and int(self.elapsed[i]) >= self.max_steps
                term = self.term_on_success and suc != 0
                out["flags"][0, i], out["flags"][1, i] = int(term), int(trunc)
                out["packed"][i, k + 2], out["packed"][i, k + 3] = float(term), float(trunc)
            if info is not None:
                info[i] = it
            if it >> 16:
                self.overflow_counter += 1
        self.launches += 1

    def step(self, actions, out, info=None):
        self._run(0, 0, actions, None, out, self.info if info is None else info)
        if self.goal_args is None:
            return
        # the goal update or redraw launch after the step (csrc/b200sim.cu b200sim_step)
        goal_xy, scaling, noise, seed, offset, episode = self.goal_args
        st, q, g, radius = self.state.numpy(), self.layout["qpos"], self.layout["goal"], self.task.success_radius
        for i in range(self.num_envs):
            key = (seed, offset + i, int(episode[i]), int(self.elapsed[i]), st[i, q:q + 2], st[i, g:g + 2])
            if self.redraw:
                new, r = goal_redraw(goal_xy, scaling, noise, radius, self.task.reward_dense, *key)
                if r is not None:
                    st[i, g:g + 2] = new
                    out["reward"][i] = float(r)
            else:
                new, n = goal_update(goal_xy, scaling, noise, radius, *key)
                if n:
                    st[i, g:g + 2] = new
        self.launches += 1

    def refresh(self, mask, out):
        self._run(1, 0, None, mask, out)

    def raw_step(self, nstep, out, mask=None):
        self._run(2, nstep, None, mask, out)

    def _per_env(self, mask, fn, episode=None, out=None):
        """One reset-style launch: fn(i, record of env i) for the envs in `mask` (None: all); with `episode` their episode counters move
        on and their step counters restart; with `out` the refresh launch follows."""
        st = self.state.numpy()
        for i in range(self.num_envs):
            if mask is None or bool(mask[i]):
                fn(i, st[i])
                if episode is not None:
                    episode[i] += 1
                    self.elapsed[i] = 0
        self.launches += 1
        if out is not None:
            self.refresh(mask, out)

    def reset_draw(self, mask, rest_record, params, seed, env_offset, episode, out):
        """b200sim_reset on the emulation: the same csrc/reset_sample.cuh code, env by env, then the refresh."""
        rest, lay, p = rest_record.numpy(), self.layout, ctypes.byref(params)
        self._per_env(mask, lambda i, rec: self.L.hostsim_fetch_reset_record(p, int(seed) & _U64, i + int(env_offset), int(episode[i]), rest.ctypes.data,
                                                                             lay["stride"], lay["qpos"], lay["goal"], rec.ctypes.data), episode, out)

    def reset_uniform(self, mask, rest_record, params, seed, env_offset, episode, out):
        rest, p = rest_record.numpy(), ctypes.byref(params)
        self._per_env(mask, lambda i, rec: self.L.hostsim_uniform_reset_record(p, int(seed) & _U64, i + int(env_offset), int(episode[i]),
                                                                               rest.ctypes.data, self.layout["stride"], rec.ctypes.data), episode, out)

    def reset_maze(self, mask, rest_record, params, goal_xy, reset_xy, seed, env_offset, episode, out):
        rest, g, r, lay, p = rest_record.numpy(), goal_xy.numpy(), reset_xy.numpy(), self.layout, ctypes.byref(params)
        self._per_env(mask, lambda i, rec: self.L.hostsim_maze_reset_record(p, g.ctypes.data, r.ctypes.data, int(seed) & _U64, i + int(env_offset),
                                                                            int(episode[i]), rest.ctypes.data, lay["stride"], lay["qpos"], lay["goal"],
                                                                            rec.ctypes.data), episode, out)

    def reset_hand_pose(self, mask, rest_record, params, parallel, seed, env_offset, episode, attempt):
        rest, par, lay, p = rest_record.numpy(), parallel.numpy(), self.layout, ctypes.byref(params)
        self._per_env(mask, lambda i, rec: self.L.hostsim_hand_pose_record(p, par.ctypes.data, int(seed) & _U64, i + int(env_offset), int(episode[i]),
                                                                           int(attempt), rest.ctypes.data, lay["stride"], lay["qpos"], lay["goal"],
                                                                           self.ngoal, rec.ctypes.data))

    def reset_hand_goal(self, mask, params, parallel, seed, env_offset, episode, out):
        par, lay, p = parallel.numpy(), self.layout, ctypes.byref(params)
        self._per_env(mask, lambda i, rec: self.L.hostsim_hand_goal(p, par.ctypes.data, int(seed) & _U64, i + int(env_offset), int(episode[i]),
                                                                    lay["qpos"], lay["goal"], rec.ctypes.data), episode, out)

    def reset_reach(self, mask, rest_record, params, seed, env_offset, episode, out):
        rest, p = rest_record.numpy(), ctypes.byref(params)
        self._per_env(mask, lambda i, rec: self.L.hostsim_reach_reset_record(p, int(seed) & _U64, i + int(env_offset), int(episode[i]), rest.ctypes.data,
                                                                             self.layout["stride"], self.layout["goal"], rec.ctypes.data), episode, out)

    def check_state(self, bad, rest_record, keep):
        rest = rest_record.numpy().ctypes.data if rest_record is not None else None
        k = ctypes.byref(keep) if keep is not None else None

        def one(i, rec):
            bad[i] = self.L.hostsim_check_record(rec.ctypes.data, self.layout["stride"], rest, k)

        self._per_env(None, one)

    def compute_reward(self, ag, dg):
        ag = ag.to(torch.float32).reshape(-1, self.ngoal); dg = dg.to(torch.float32).reshape(-1, self.ngoal)
        if self.task.kind == 2:  # same arithmetic as the kernel's hand_goal_distance / hand_reward (fetch_task.cuh)
            t = self.task
            dp = torch.sqrt(((ag[:, :3] - dg[:, :3]) ** 2).sum(-1)) if t.goal_flags & 1 else torch.zeros(ag.shape[0])
            qa = ag[:, 3:]
            if t.goal_flags & 4:   # ignore_z_target_rotation (the pen)
                from gymnasium_robotics_b200 import rotations as R
                ea, eb = R.quat2euler(qa.double().numpy()), R.quat2euler(dg[:, 3:].double().numpy())
                ea[:, 2] = eb[:, 2]
                qa = torch.as_tensor(R.euler2quat(ea), dtype=torch.float32)
            dr = 2 * torch.acos(torch.clamp((qa * dg[:, 3:]).sum(-1), -1, 1)) if t.goal_flags & 2 else torch.zeros(ag.shape[0])
            suc = (dp < t.distance_threshold).to(torch.float32) * (dr < t.rotation_threshold).to(torch.float32)
            return -(10 * dp + dr) if t.reward_dense else suc - 1
        d = torch.sqrt(((ag - dg) ** 2).sum(-1))
        if self.task.kind == 1:
            return torch.exp(-d) if self.task.reward_dense else (d <= self.task.success_radius).to(torch.float32)
        return -d if self.task.reward_dense else -(d > self.task.distance_threshold).to(torch.float32)
