"""Test-only ctypes wrapper of ant_info.cpp (the host emulation as the ant kernel build, -DB200_ANT) and AntInfoHostBackend: the host
emulation backend with b200sim_set_ant_info, which runs each env as fetch_kernel_ant does (the Ant's keywords, the info row, the
torso position kept in the state record)."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np
import torch

from tests.hostsim import HostSim
from tests.hostsim_backend import HostSimBackend

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_OUT = os.path.join(_HERE, "libhostsim_ant.so")
_LIB = None


class AntInfoArgsC(ctypes.Structure):
    """AntInfoArgs (csrc/fetch_task.cuh)"""
    _fields_ = [(n, ctypes.c_float) for n in ("cf_lo", "cf_hi", "forward_w", "ctrl_w", "contact_w", "healthy_reward", "z_lo", "z_hi")] + \
               [(n, ctypes.c_int) for n in ("v4", "survive_always", "contact_in_ctrl")] + [("rows", ctypes.c_void_p), ("origin", ctypes.c_void_p)]


def build(force=False):
    """Compile libhostsim_ant.so when it is older than a source (under a file lock, renamed into place)."""
    csrc = os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc")
    srcs = [os.path.join(_HERE, "ant_info.cpp"), os.path.join(_HERE, "hostsim.cpp"), os.path.join(_HERE, "hostwarp.h")] + \
           [os.path.join(csrc, f) for f in ("sim_core.cuh", "dmodel.h", "fetch_task.cuh", "reset_sample.cuh")] + \
           [os.path.join(_ROOT, "include", f) for f in ("b200sim_model.h", "b200sim.h")]

    def stale():
        return force or not os.path.exists(_OUT) or os.path.getmtime(_OUT) < max(os.path.getmtime(s) for s in srcs)

    if stale():
        import fcntl

        with open(_OUT + ".lock", "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                tmp = f"{_OUT}.{os.getpid()}.tmp"
                subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-function", "-DB200_ANT", "-o", tmp, srcs[0]])
                os.replace(tmp, _OUT)
    return _OUT


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        vp = ctypes.c_void_p
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, vp, vp, ctypes.c_int, ctypes.c_int]
        L.hostsim_scr_words.argtypes = [vp]
        L.hostsim_scratch.restype = ctypes.POINTER(ctypes.c_float)
        L.hostsim_scratch.argtypes = [vp]
        L.hostsim_offset.argtypes = [vp, ctypes.c_char_p]
        L.hostsim_ant_env_step.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, vp] + [vp] * 7
        L.hostsim_ant_env_step.restype = ctypes.c_int
        _LIB = L
    return _LIB


class AntHostSim(HostSim):
    """HostSim on the ant-build emulation."""

    def __init__(self, model, ref):
        self.model, self._L = model, lib()
        blob = model.to_blob()
        r = np.asarray(ref, dtype=np.float32)
        self._h = self._L.hostsim_create(blob, len(blob), None, r.ctypes.data, -1, 0)
        if not self._h:
            raise RuntimeError("hostsim_create failed")
        n = self._L.hostsim_scr_words(self._h)
        self.scratch = np.ctypeslib.as_array(self._L.hostsim_scratch(self._h), shape=(n,))
        self.ref = r.astype(np.float64)


class AntInfoHostBackend(HostSimBackend):
    """HostSimBackend with b200sim_set_ant_info, for maze tasks with touch_mode 2..4 (the handles b200sim_create gives the ant build);
    refuses it for any other task, as the library does."""

    def __init__(self, model, eq_data, task, num_envs, device):
        super().__init__(model, eq_data, task, num_envs, device)
        self.ant_build = task.kind == 1 and task.touch_mode >= 2
        if self.ant_build:
            from gymnasium_robotics_b200.fetch import REF_POINT

            self.sim = AntHostSim(model, getattr(self, "REF", REF_POINT))
            assert self.layout["stride"] - (self.layout["goal"] + 2) >= 2
        # b200sim's defaults: Ant-v5's keywords, no info rows
        self.ant = AntInfoArgsC(-1.0, 1.0, 1.0, 0.5, 5e-4, 1.0, 0.2, 1.0, 0, 0, 0, None, None)
        self.ant_rows = self.ant_origin = None

    def set_ant_info(self, params, rows, origin):
        if not self.ant_build:
            raise RuntimeError("b200sim call failed (-6): b200sim_set_ant_info: not an ant-build handle (maze task with touch_mode 2..4)")
        p = params
        assert p.version in (4, 5) and p.contact_force_range[0] <= p.contact_force_range[1]
        assert rows is None or p.version == 4 or origin is not None
        v4 = p.version == 4
        self.ant = AntInfoArgsC(p.contact_force_range[0], p.contact_force_range[1], 1.0 if v4 else p.forward_reward_weight, p.ctrl_cost_weight,
                                p.contact_cost_weight, p.healthy_reward, p.healthy_z_range[0], p.healthy_z_range[1], int(v4),
                                int(v4 and bool(p.terminate_when_unhealthy)), int(v4 and bool(p.use_contact_forces)), None, None)
        self.ant_rows, self.ant_origin = rows, origin

    def _run(self, mode, nraw, actions, mask, out, info=None):
        if not self.ant_build:
            return super()._run(mode, nraw, actions, mask, out, info)
        st = self.state.numpy()
        rows = self.ant_rows.numpy() if self.ant_rows is not None else None
        origin = self.ant_origin.numpy() if self.ant_origin is not None else None
        k = self.nobs + 2 * self.ngoal
        L = self.sim._L
        for i in range(self.num_envs):
            if mask is not None and not bool(mask[i]):
                continue
            a = np.zeros(max(32, self.nact), dtype=np.float32)
            if actions is not None:
                a[:self.nact] = actions[i].numpy()
            args = AntInfoArgsC.from_buffer_copy(self.ant)
            args.rows = rows[i].ctypes.data if rows is not None else None
            args.origin = origin[i].ctypes.data if origin is not None else None
            obs, ag, dg = np.zeros(self.nobs, np.float32), np.zeros(self.ngoal, np.float32), np.zeros(self.ngoal, np.float32)
            rew, suc = np.zeros(1, np.float32), np.zeros(1, np.float32)
            it = L.hostsim_ant_env_step(self.sim._h, ctypes.byref(self.task), mode, nraw, ctypes.byref(args), st[i].ctypes.data, a.ctypes.data,
                                        obs.ctypes.data, ag.ctypes.data, dg.ctypes.data, rew.ctypes.data, suc.ctypes.data)
            out["obs"][i] = torch.from_numpy(obs); out["achieved"][i] = torch.from_numpy(ag); out["desired"][i] = torch.from_numpy(dg)
            out["reward"][i] = float(rew[0]); out["success"][i] = float(suc[0])
            if mode == 0:
                self.elapsed[i] += 1
                trunc = self.max_steps > 0 and int(self.elapsed[i]) >= self.max_steps
                term = self.term_on_success and suc[0] != 0
                out["flags"][0, i], out["flags"][1, i] = int(term), int(trunc)
                out["packed"][i, k + 2], out["packed"][i, k + 3] = float(term), float(trunc)
            if info is not None:
                info[i] = it
        self.launches += 1
