"""The handle's per-env key table (b200sim_set_env_keys) on the host emulation: HostSimBackend with `set_env_keys`.  While a table is
set, env i draws with keys[i] in place of the seed: a reset draws each group of envs that share a key with that key as the seed (the
emulation runs one env at a time, so this is the device's per-env draw), the goal update / redraw after a step and the kitchen's
observation noise take env i's key.  Test infrastructure only."""
from __future__ import annotations

import ctypes

import torch

from tests.hostsim import ObsNoiseKey, goal_redraw, goal_update
from tests.hostsim_backend import HostSimBackend

_U64 = 0xFFFFFFFFFFFFFFFF


class KeyedHostSimBackend(HostSimBackend):
    keys = None

    def set_env_keys(self, keys):
        """b200sim_set_env_keys: int64 [N] (read as unsigned), or None to turn the table off."""
        self.keys = keys

    def _groups(self, mask, seed):
        """(mask, key) per key of the masked envs; (mask, seed) without a table."""
        if self.keys is None:
            return [(mask, seed)]
        sel = torch.ones(self.num_envs, dtype=torch.bool) if mask is None else torch.as_tensor(mask).bool()
        return [((sel & (self.keys == k)).to(torch.uint8), int(k)) for k in torch.unique(self.keys[sel]).tolist()]

    def reset_draw(self, mask, rest_record, params, seed, env_offset, episode, out):
        for m, k in self._groups(mask, seed):
            super().reset_draw(m, rest_record, params, k, env_offset, episode, out)

    def reset_uniform(self, mask, rest_record, params, seed, env_offset, episode, out):
        for m, k in self._groups(mask, seed):
            super().reset_uniform(m, rest_record, params, k, env_offset, episode, out)

    def reset_maze(self, mask, rest_record, params, goal_xy, reset_xy, seed, env_offset, episode, out):
        for m, k in self._groups(mask, seed):
            super().reset_maze(m, rest_record, params, goal_xy, reset_xy, k, env_offset, episode, out)

    def reset_hand_pose(self, mask, rest_record, params, parallel, seed, env_offset, episode, attempt):
        for m, k in self._groups(mask, seed):
            super().reset_hand_pose(m, rest_record, params, parallel, k, env_offset, episode, attempt)

    def reset_hand_goal(self, mask, params, parallel, seed, env_offset, episode, out):
        for m, k in self._groups(mask, seed):
            super().reset_hand_goal(m, params, parallel, k, env_offset, episode, out)

    def reset_reach(self, mask, rest_record, params, seed, env_offset, episode, out):
        for m, k in self._groups(mask, seed):
            super().reset_reach(m, rest_record, params, k, env_offset, episode, out)

    def _extra(self, i, mode, rows, origin):
        if self.keys is None or not self.kitchen_build or self.noise is None:
            return super()._extra(i, mode, rows, origin)
        scale, _, offset, episode = self.noise
        step = int(self.elapsed[i]) + (1 if mode == 0 else 0)
        return (ctypes.byref(ObsNoiseKey(scale.ctypes.data, int(self.keys[i]) & _U64, offset + i, int(episode[i]), step)),)

    def step(self, actions, out, info=None):
        if self.keys is None or self.goal_args is None:
            return super().step(actions, out, info)
        args, self.goal_args = self.goal_args, None
        try:
            super().step(actions, out, info)   # the step launch alone
        finally:
            self.goal_args = args
        # the goal update or redraw launch, env i keyed by keys[i]
        goal_xy, scaling, noise, _, offset, episode = args
        st, q, g, radius = self.state.numpy(), self.layout["qpos"], self.layout["goal"], self.task.success_radius
        for i in range(self.num_envs):
            key = (int(self.keys[i]) & _U64, offset + i, int(episode[i]), int(self.elapsed[i]), st[i, q:q + 2], st[i, g:g + 2])
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
