"""Test-only ctypes wrapper of maze_redraw.cpp (AntMaze-v3's goal redraw, hostsim_maze_goal_redraw) and GoalRedrawHostBackend: the host
emulation backend with b200sim_set_goal_redraw, which runs the redraw after every step as the redraw kernel does."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from tests.hostsim.maze_goal import GoalUpdateHostBackend

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_OUT = os.path.join(_HERE, "libhostsim_maze_redraw.so")
_LIB = None


def build(force=False):
    """Compile libhostsim_maze_redraw.so when it is older than a source (under a file lock, renamed into place)."""
    srcs = [os.path.join(_HERE, "maze_redraw.cpp"), os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc", "reset_sample.cuh"),
            os.path.join(_ROOT, "include", "b200sim.h")]

    def stale():
        return force or not os.path.exists(_OUT) or os.path.getmtime(_OUT) < max(os.path.getmtime(s) for s in srcs)

    if stale():
        import fcntl

        with open(_OUT + ".lock", "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                tmp = f"{_OUT}.{os.getpid()}.tmp"
                subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-function", "-o", tmp, srcs[0]])
                os.replace(tmp, _OUT)
    return _OUT


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        vp, ci, cu, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_float
        L.hostsim_maze_goal_redraw.argtypes = [vp, ci, cf, cf, cf, ci, ctypes.c_ulonglong, cu, cu, cu, vp, vp, vp]
        L.hostsim_maze_goal_redraw.restype = ci
        _LIB = L
    return _LIB


def goal_redraw(goal_xy, scaling, noise, radius, dense, seed, env, episode, step, ach, goal):
    """rs_maze_goal_redraw on the host: (new goal as float32 [2], reward against it as float32 or None when the goal stays)."""
    g = np.ascontiguousarray(goal_xy, dtype=np.float32)
    a, out, r = np.asarray(ach, dtype=np.float32).copy(), np.asarray(goal, dtype=np.float32).copy(), np.zeros(1, dtype=np.float32)
    changed = lib().hostsim_maze_goal_redraw(g.ctypes.data, len(g), float(scaling), float(noise), float(radius), int(bool(dense)),
                                             int(seed) & 0xFFFFFFFFFFFFFFFF, int(env), int(episode), int(step), a.ctypes.data, out.ctypes.data,
                                             r.ctypes.data)
    return out, (r[0] if changed else None)


class GoalRedrawHostBackend(GoalUpdateHostBackend):
    """GoalUpdateHostBackend with b200sim_set_goal_redraw: the two share one slot, as on the handle.  With the redraw set, every step
    runs rs_maze_goal_redraw on each env's record with the redraw kernel's key and writes the changed envs' goal and packed reward."""
    redraw = False

    def set_goal_update(self, goal_xy, scaling, noise, seed, env_offset, episode):
        super().set_goal_update(goal_xy, scaling, noise, seed, env_offset, episode)
        self.redraw = False

    def set_goal_redraw(self, goal_xy, scaling, noise, seed, env_offset, episode):
        super().set_goal_update(goal_xy, scaling, noise, seed, env_offset, episode)
        self.redraw = goal_xy is not None

    def step(self, actions, out, info=None):
        if not self.redraw:
            return super().step(actions, out, info)
        args, self.goal_args = self.goal_args, None      # the plain step, then the redraw below in place of the update
        try:
            super().step(actions, out, info)
        finally:
            self.goal_args = args
        goal_xy, scaling, noise, seed, offset, episode = args
        st, q, g = self.state.numpy(), self.layout["qpos"], self.layout["goal"]
        for i in range(self.num_envs):
            new, r = goal_redraw(goal_xy, scaling, noise, self.task.success_radius, self.task.reward_dense, seed, offset + i, int(episode[i]),
                                 int(self.elapsed[i]), st[i, q:q + 2], st[i, g:g + 2])
            if r is not None:
                st[i, g:g + 2] = new
                out["reward"][i] = float(r)
        self.launches += 1
