"""Test-only ctypes wrapper of kitchen_noise.cpp: the kitchen flavors of the host emulation (hostsim.cpp) with the observation-noise
entry points of FrankaKitchen rng_mode="device" (hostsim_kitchen_noise, hostsim_kitchen_env_step, and every hostsim_* function)."""
from __future__ import annotations

import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
FLAGS = {"kitchen": ["-DB200_KITCHEN"], "kitchen_groups": ["-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS"],
         "kitchen_hull": ["-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS", "-DB200_HULL"]}
_LIB = {}


def build(flavor, force=False):
    """Compile libhostsim_noise_<flavor>.so when it is older than a source (under a file lock, renamed into place)."""
    out = os.path.join(_HERE, f"libhostsim_noise_{flavor}.so")
    csrc = os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc")
    srcs = [os.path.join(_HERE, "kitchen_noise.cpp"), os.path.join(_HERE, "hostsim.cpp"), os.path.join(_HERE, "hostwarp.h")] + \
           [os.path.join(csrc, f) for f in ("sim_core.cuh", "dmodel.h", "fetch_task.cuh", "reset_sample.cuh")] + \
           [os.path.join(_ROOT, "include", f) for f in ("b200sim_model.h", "b200sim.h")]

    def stale():
        return force or not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs)

    if stale():
        import fcntl

        with open(out + ".lock", "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                tmp = f"{out}.{os.getpid()}.tmp"
                subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-function"] + FLAGS[flavor] +
                                      ["-o", tmp, srcs[0]])
                os.replace(tmp, out)
    return out


def lib(flavor):
    if flavor not in _LIB:
        L = ctypes.CDLL(build(flavor))
        vp, ci, cu = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, vp, vp, ci, ci]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_destroy.restype = None
        L.hostsim_kitchen_noise.argtypes = [ctypes.c_ulonglong, cu, cu, cu, vp]
        L.hostsim_kitchen_noise.restype = None
        L.hostsim_kitchen_env_step.argtypes = [vp, vp, ci, ci, vp, ctypes.c_ulonglong, cu, cu, cu] + [vp] * 7
        L.hostsim_kitchen_env_step.restype = ci
        _LIB[flavor] = L
    return _LIB[flavor]
