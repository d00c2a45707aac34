"""Test-only ctypes wrapper of maze_goal.cpp (the maze goal update, hostsim_maze_goal_update) and GoalUpdateHostBackend: the host
emulation backend with b200sim_set_goal_update, which runs the update after every step as the update kernel does."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from tests.hostsim_backend import HostSimBackend

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_OUT = os.path.join(_HERE, "libhostsim_maze_goal.so")
_LIB = None


def build(force=False):
    """Compile libhostsim_maze_goal.so when it is older than a source (under a file lock, renamed into place)."""
    srcs = [os.path.join(_HERE, "maze_goal.cpp"), os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc", "reset_sample.cuh"),
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
        L.hostsim_maze_goal_update.argtypes = [vp, ci, cf, cf, cf, ctypes.c_ulonglong, cu, cu, cu, vp, vp]
        L.hostsim_maze_goal_update.restype = ci
        _LIB = L
    return _LIB


def goal_update(goal_xy, scaling, noise, radius, seed, env, episode, step, ach, goal):
    """rs_maze_goal_update on the host: (new goal as float32 [2], candidates drawn)."""
    g = np.ascontiguousarray(goal_xy, dtype=np.float32)
    a, out = np.asarray(ach, dtype=np.float32).copy(), np.asarray(goal, dtype=np.float32).copy()
    n = lib().hostsim_maze_goal_update(g.ctypes.data, len(g), float(scaling), float(noise), float(radius), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                       int(env), int(episode), int(step), a.ctypes.data, out.ctypes.data)
    return out, n


class GoalUpdateHostBackend(HostSimBackend):
    """HostSimBackend with b200sim_set_goal_update: after each step, every env's record goes through rs_maze_goal_update with the
    key the update kernel builds (global index, episode counter, step counter after the step); one more launch when it runs."""
    goal_args = None

    def set_goal_update(self, goal_xy, scaling, noise, seed, env_offset, episode):
        if goal_xy is not None:
            assert len(goal_xy) >= 2 and episode is not None and int(env_offset) >= 0
        self.goal_args = None if goal_xy is None else (goal_xy.numpy(), float(scaling), float(noise), int(seed), int(env_offset), episode)

    def step(self, actions, out, info=None):
        super().step(actions, out, info)
        if self.goal_args is None:
            return
        goal_xy, scaling, noise, seed, offset, episode = self.goal_args
        st, q, g = self.state.numpy(), self.layout["qpos"], self.layout["goal"]
        for i in range(self.num_envs):
            new, n = goal_update(goal_xy, scaling, noise, self.task.success_radius, seed, offset + i, int(episode[i]), int(self.elapsed[i]),
                                 st[i, q:q + 2], st[i, g:g + 2])
            if n:
                st[i, g:g + 2] = new
        self.launches += 1
