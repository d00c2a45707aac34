"""Test-only ctypes wrapper for the host emulation (WARP_W == 1) of the CUDA physics core.  See hostsim.cpp."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from gymnasium_robotics_b200 import _lib
from gymnasium_robotics_b200.mjcf import EQ_JOINT, GEOM_MESH

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = {}


class FetchTaskC(ctypes.Structure):
    """FetchTask (csrc/fetch_task.cuh): b200sim_fetch_task_t and the state-record offsets b200sim_create adds to it."""
    _fields_ = _lib.FetchTaskC._fields_ + [(n, ctypes.c_int) for n in ("st_qpos", "st_qvel", "st_warm", "st_ctrl", "st_mocap", "st_pose",
                                                                       "st_goal", "st_stride", "st_penv")]


class ObsNoiseKey(ctypes.Structure):
    """ObsNoiseKey (csrc/fetch_task.cuh): one env's observation-noise stream in one launch."""
    _fields_ = [("scale", ctypes.c_void_p), ("seed", ctypes.c_ulonglong), ("env", ctypes.c_uint), ("episode", ctypes.c_uint), ("t", ctypes.c_uint)]


class AntInfoArgsC(ctypes.Structure):
    """AntInfoArgs (csrc/fetch_task.cuh)"""
    _fields_ = [(n, ctypes.c_float) for n in ("cf_lo", "cf_hi", "forward_w", "ctrl_w", "contact_w", "healthy_reward", "z_lo", "z_hi")] + \
               [(n, ctypes.c_int) for n in ("v4", "survive_always", "contact_in_ctrl")] + [("rows", ctypes.c_void_p), ("origin", ctypes.c_void_p)]


_WARP = ["-DB200_HOST_WARP", "-Wno-unknown-pragmas"]   # WARP_W == 32 on lock-step fibers (hostwarp.h): the lane-parallel code paths
_KITCHEN, _GROUPS = ["-DB200_KITCHEN"], ["-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS"]
# one row per emulated kernel build: flavor -> (library, g++ defines)
#   False: the plain build; True: the 64-bit dof-mask build (models with more than 32 dofs, csrc/b200sim_wide.cu);
#   "kitchen": the Franka-Kitchen kernel features with the flat-scan broad phase (csrc/b200sim_kitchen.cu); "kitchen_groups": the
#   two-level broad phase (regrouped pair list, group table, csrc/b200sim_kitchen_groups.cu); "kitchen_flat": the groups build's data
#   layout scanned in one level, the bit-exact A/B reference of the two-level scan; "kitchen_hull": the groups build plus the
#   support-map narrow phase for mesh geoms (csrc/b200sim_kitchen_hull.cu); "ant": the Ant's keywords and info (csrc/b200sim_ant.cu);
#   "warp*": those builds on the 32-lane emulated warp; "warp_timing" with the stage timer's collective counts
FLAGS = {False: ("libhostsim.so", []), True: ("libhostsim_wide.so", ["-DB200_WIDE"]),
         "kitchen": ("libhostsim_kitchen.so", _KITCHEN), "kitchen_groups": ("libhostsim_kitchen_groups.so", _GROUPS),
         "kitchen_flat": ("libhostsim_kitchen_flat.so", _GROUPS + ["-DB200_KITCHEN_FLATSCAN"]),
         "kitchen_hull": ("libhostsim_kitchen_hull.so", _GROUPS + ["-DB200_HULL"]), "ant": ("libhostsim_ant.so", ["-DB200_ANT"]),
         "warp": ("libhostsim_warp.so", _WARP), "warp_wide": ("libhostsim_warp_wide.so", _WARP + ["-DB200_WIDE"]),
         "warp_kitchen": ("libhostsim_warp_kitchen.so", _WARP + _KITCHEN), "warp_kitchen_groups": ("libhostsim_warp_kitchen_groups.so", _WARP + _GROUPS),
         "warp_kitchen_hull": ("libhostsim_warp_kitchen_hull.so", _WARP + _GROUPS + ["-DB200_HULL"]),
         "warp_timing": ("libhostsim_warp_timing.so", _WARP + ["-DB200_STAGE_TIMING"])}
FLAVORS = tuple(f for f in FLAGS if f != "warp_timing")   # what the package build compiles; tests/count_stage_collectives.py builds the last
_SRCS = [os.path.join(_HERE, "hostsim.cpp"), os.path.join(_HERE, "hostwarp.h")] + \
        [os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc", f) for f in ("sim_core.cuh", "dmodel.h", "fetch_task.cuh", "reset_sample.cuh")] + \
        [os.path.join(_ROOT, "include", f) for f in ("b200sim_model.h", "b200sim.h")]


def host_flavor(model, task):
    """The flavor that emulates the kernel build b200sim_create picks for (model, task) (csrc/b200sim.cu): a mesh geom -> the hull build;
    a joint equality or a condim-6 pair -> a kitchen build (flat scan when B200SIM_KITCHEN_GROUPS=0, else the two-level broad phase);
    more than 32 dofs -> the wide build; a maze task with touch_mode 2..4 -> the ant build; else the plain build."""
    if (np.asarray(model.geom_type) == GEOM_MESH).any():
        return "kitchen_hull"
    if (np.asarray(model.eq_type)[:model.neq] == EQ_JOINT).any() or (np.asarray(model.pair_condim) == 6).any():
        return "kitchen" if os.environ.get("B200SIM_KITCHEN_GROUPS") == "0" else "kitchen_groups"
    if model.nv > 32:
        return True
    return "ant" if task.kind == 1 and task.touch_mode >= 2 else False


def build(force=False, wide=False):
    """Compile the library of flavor `wide` (a key of FLAGS) when it is older than a source.  Several processes may get here at once
    (the 2-rank gloo tests, pytest-xdist): one compiles under a file lock into a temporary name and renames it into place, the others
    wait and then find the library fresh."""
    name, defines = FLAGS[wide]
    out = os.path.join(_HERE, name)

    def stale():
        return force or not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in _SRCS)

    if stale():
        import fcntl

        with open(out + ".lock", "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                tmp = f"{out}.{os.getpid()}.tmp"
                subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-function"] + defines + ["-o", tmp, _SRCS[0]])
                os.replace(tmp, out)
                force = False
    return out


def lib(wide=False):
    """The library of flavor `wide`, every hostsim_* function it exports with its argument and result types."""
    if _LIB.get(wide) is None:
        L = ctypes.CDLL(build(wide=wide))
        vp, ci, cu, cf, cu64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_float, ctypes.c_ulonglong
        defines = FLAGS[wide][1]
        step_extra = [vp] if "-DB200_KITCHEN" in defines or "-DB200_ANT" in defines else []   # the noise key / the Ant's arguments
        sigs = {"hostsim_create": (vp, [ctypes.c_char_p, ctypes.c_size_t, vp, vp, ci, ci]),
                "hostsim_destroy": (None, [vp]), "hostsim_scratch": (ctypes.POINTER(ctypes.c_float), [vp]),
                "hostsim_scr_words": (ci, [vp]), "hostsim_npair": (ci, [vp]), "hostsim_nbgrp": (ci, [vp]),
                "hostsim_offset": (ci, [vp, ctypes.c_char_p]), "hostsim_model_offset": (ci, [vp, ctypes.c_char_p]),
                "hostsim_forward": (None, [vp]), "hostsim_kinematics": (None, [vp]), "hostsim_step": (None, [vp, ci]),
                "hostsim_collide": (None, [vp, ci]), "hostsim_problem": (None, [vp, ci]), "hostsim_jv": (None, [vp, ci]),
                "hostsim_build_h": (None, [vp, ci]), "hostsim_touch": (None, [vp, vp]),
                "hostsim_ray_hits": (None, [ci, vp, ci, vp, vp, vp]),
                "hostsim_model": (ctypes.POINTER(ctypes.c_uint32), [vp]), "hostsim_model_words": (ci, [vp]), "hostsim_hot_words": (ci, [vp]),
                "hostsim_layout": (None, [vp]), "hostsim_task_size": (ci, []),
                "hostsim_env_step": (ci, [vp, vp, ci, ci] + [vp] * 7 + step_extra),
                "hostsim_spd": (ci, [ci, ci, vp, vp, cf, vp, vp]),
                "hostsim_philox4x32_10": (None, [vp] * 3),
                "hostsim_fetch_reset_record": (None, [vp, cu64, cu, cu, vp, ci, ci, ci, vp]),
                "hostsim_uniform_reset_record": (None, [vp, cu64, cu, cu, vp, ci, vp]),
                "hostsim_maze_reset_record": (None, [vp, vp, vp, cu64, cu, cu, vp, ci, ci, ci, vp]),
                "hostsim_hand_pose_record": (None, [vp, vp, cu64, cu, cu, cu, vp, ci, ci, ci, ci, vp]),
                "hostsim_hand_goal": (None, [vp, vp, cu64, cu, cu, ci, ci, vp]),
                "hostsim_reach_reset_record": (None, [vp, cu64, cu, cu, vp, ci, ci, vp]),
                "hostsim_check_record": (ci, [vp, ci, vp, vp]),
                "hostsim_maze_goal_update": (ci, [vp, ci, cf, cf, cf, cu64, cu, cu, cu, vp, vp]),
                "hostsim_maze_goal_redraw": (ci, [vp, ci, cf, cf, cf, ci, cu64, cu, cu, cu, vp, vp, vp]),
                "hostsim_kitchen_noise": (None, [cu64, cu, cu, cu, vp]),       # kitchen flavors
                "hostsim_collectives": (ctypes.c_long, []),                    # warp flavors
                "hostsim_stage_rounds": (ci, [ctypes.POINTER(ctypes.c_longlong), ci])}   # warp_timing
        for name, (res, args) in sigs.items():
            f = getattr(L, name, None)      # (a function of some flavors only is absent from the others)
            if f is not None:
                f.restype, f.argtypes = res, args
        assert L.hostsim_task_size() == ctypes.sizeof(FetchTaskC)
        _LIB[wide] = L
    return _LIB[wide]


def goal_update(goal_xy, scaling, noise, radius, seed, env, episode, step, ach, goal):
    """rs_maze_goal_update on the host: (new goal as float32 [2], candidates drawn)."""
    g = np.ascontiguousarray(goal_xy, dtype=np.float32)
    a, out = np.asarray(ach, dtype=np.float32).copy(), np.asarray(goal, dtype=np.float32).copy()
    n = lib().hostsim_maze_goal_update(g.ctypes.data, len(g), float(scaling), float(noise), float(radius), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                       int(env), int(episode), int(step), a.ctypes.data, out.ctypes.data)
    return out, n


def goal_redraw(goal_xy, scaling, noise, radius, dense, seed, env, episode, step, ach, goal):
    """rs_maze_goal_redraw on the host: (new goal as float32 [2], reward against it as float32 or None when the goal stays)."""
    g = np.ascontiguousarray(goal_xy, dtype=np.float32)
    a, out, r = np.asarray(ach, dtype=np.float32).copy(), np.asarray(goal, dtype=np.float32).copy(), np.zeros(1, dtype=np.float32)
    changed = lib().hostsim_maze_goal_redraw(g.ctypes.data, len(g), float(scaling), float(noise), float(radius), int(bool(dense)),
                                             int(seed) & 0xFFFFFFFFFFFFFFFF, int(env), int(episode), int(step), a.ctypes.data, out.ctypes.data,
                                             r.ctypes.data)
    return out, (r[0] if changed else None)


def kitchen_noise(seed, env, episode, t):
    """The 59 uniforms in [-1, 1) of the kitchen observation-noise stream (seed; env, episode, step t), float32 [59]."""
    out = np.zeros(59, dtype=np.float32)
    lib("kitchen").hostsim_kitchen_noise(int(seed) & 0xFFFFFFFFFFFFFFFF, int(env), int(episode), int(t), out.ctypes.data)
    return out


def ray_hits(flavor, tp, size, p, d):
    """ray_hits_site(tp, size, p[i], d[i]) of the kernel source for rays in the site frame: bool [n]."""
    p, d = np.ascontiguousarray(p, np.float32), np.ascontiguousarray(d, np.float32)
    sz, hit = np.ascontiguousarray(size, np.float32), np.zeros(len(p), np.int32)
    lib(wide=flavor).hostsim_ray_hits(int(tp), sz.ctypes.data, len(p), p.ctypes.data, d.ctypes.data, hit.ctypes.data)
    return hit.astype(bool)


def spd(flavor, nvp, nv, A, x, dadd, hh, H, use_dadd, inplace):
    """spd_solve<nvp> of the given flavor (on the 32-lane flavors the register Cholesky, bordered for nvp > 32) for a batch of cases,
    one call each; the same buffers as tests.devsim.spd.  A, x and H are overwritten with their contents after the solve."""
    L = lib(wide=flavor)
    for e in range(len(nv)):
        pa, px, ph = A[e].ctypes.data, x[e].ctypes.data, H[e].ctypes.data
        rc = L.hostsim_spd(int(nvp), int(nv[e]), pa, dadd[e].ctypes.data if use_dadd else None, float(hh), px, pa if inplace else ph)
        if rc != 0:
            raise RuntimeError(f"hostsim_spd: flavor {flavor!r} does not instantiate NVP {nvp}")


class HostSim:
    """fp32 single-env emulation of the kernel; arrays are views into the emulated shared-memory scratch."""

    def __init__(self, model, eq_data=None, ref=(1.0, 0.75, 0.4), penv_body=-1, ngrp_cap=0, flavor=None):
        self.model = model
        blob = model.to_blob()
        L = lib(wide=flavor if flavor is not None else model.nv > 32)
        self._L = L
        eq = np.ascontiguousarray(eq_data, dtype=np.float64) if eq_data is not None else None
        r = np.asarray(ref, dtype=np.float32)
        self._h = L.hostsim_create(blob, len(blob), eq.ctypes.data if eq is not None else None, r.ctypes.data, int(penv_body), int(ngrp_cap))
        if not self._h:
            raise RuntimeError("hostsim_create failed")
        n = L.hostsim_scr_words(self._h)
        self.scratch = np.ctypeslib.as_array(L.hostsim_scratch(self._h), shape=(n,))
        self.ref = r.astype(np.float64)

    def arr(self, name, count, dtype=np.float32):
        o = self._L.hostsim_offset(self._h, name.encode())
        assert o >= 0, name
        v = self.scratch[o:o + count]
        return v if dtype == np.float32 else v.view(dtype)

    def __getattr__(self, k):
        m = self.__dict__["model"]
        sizes = {"qpos": m.nq, "qvel": m.nv, "qacc": m.nv, "ctrl": m.nu, "mocap_pos": 3 * m.nmocap,
                 "mocap_quat": 4 * m.nmocap, "xpos": 3 * m.nbody, "xquat": 4 * m.nbody,
                 "fsmooth": m.nv, "fcon": m.nv, "M": m.nv * (m.nv + 1) // 2, "cdof": 6 * m.nv, "cinert": 10 * m.nbody}
        if k in sizes:
            return self.arr(k, sizes[k])
        raise AttributeError(k)

    def counters(self):
        return self.arr("counters", 8, np.int32)

    def dense_M(self):
        nv = self.model.nv
        P = self.M
        M = np.zeros((nv, nv))
        for i in range(nv):
            for j in range(i + 1):
                M[i, j] = M[j, i] = P[i * (i + 1) // 2 + j]
        return M

    def kinematics(self):
        self._L.hostsim_kinematics(self._h)

    def collide(self, nvp):
        """The collision stage alone, compiled as forward<nvp> compiles it (HF, CX)."""
        self._L.hostsim_collide(self._h, int(nvp))

    def problem(self, nvp):
        """Every stage forward<nvp> runs up to the first direction solve (tests/devsim STAGE_PROBLEM)."""
        self._L.hostsim_problem(self._h, int(nvp))

    def jv(self, nvp):
        """The rows' JV slots <- J search, rows_from_vec<HF> (tests/devsim STAGE_JV)."""
        self._L.hostsim_jv(self._h, int(nvp))

    def build_h(self, nvp):
        """build_H<HF> alone (tests/devsim STAGE_BUILD_H)."""
        self._L.hostsim_build_h(self._h, int(nvp))

    def touch(self):
        """touch_observe with touch_mode 1 on the current scratch (tests/devsim STAGE_TOUCH): float32 [nsensor]."""
        out = np.zeros(self.model.nsensor, np.float32)
        self._L.hostsim_touch(self._h, out.ctypes.data)
        return out

    def offset(self, name):
        o = self._L.hostsim_offset(self._h, name.encode())
        assert o >= 0, name
        return o

    def model_offset(self, name):
        o = self._L.hostsim_model_offset(self._h, name.encode())
        assert o >= 0, name
        return o

    @property
    def layout(self):
        """This flavor's contact-record and group layout (dmodel.h enums)."""
        names = ("C_MU", "C_U", "C_DIMGRP", "CON_WORDS", "GRP_WORDS", "G_RANGE", "C_W", "C_D", "CX_POS", "CX_PAIR", "CX_WORDS")
        lay = np.zeros(len(names), np.int32)
        self._L.hostsim_layout(lay.ctypes.data)
        return dict(zip(names, lay.tolist()))

    @property
    def words(self):
        """The device model buffer (header and arrays, 4-byte words)."""
        return np.ctypeslib.as_array(self._L.hostsim_model(self._h), shape=(self._L.hostsim_model_words(self._h),))

    def forward(self):
        self._L.hostsim_forward(self._h)

    def step(self, n=1):
        self._L.hostsim_step(self._h, int(n))

    def env_step(self, task, mode, nraw, st, action, nobs, ngoal=3, *extra):
        """One env's launch; `extra`: the kitchen flavors' noise key or the ant flavor's arguments (hostsim_env_step)."""
        obs = np.zeros(nobs, dtype=np.float32)
        ag, dg = np.zeros(ngoal, dtype=np.float32), np.zeros(ngoal, dtype=np.float32)
        rew, suc = np.zeros(1, dtype=np.float32), np.zeros(1, dtype=np.float32)
        a = np.zeros(max(32, len(action)), dtype=np.float32)
        a[:len(action)] = action
        it = self._L.hostsim_env_step(self._h, ctypes.byref(task), mode, nraw, st.ctypes.data, a.ctypes.data, obs.ctypes.data,
                                      ag.ctypes.data, dg.ctypes.data, rew.ctypes.data, suc.ctypes.data, *extra)
        return obs, ag, dg, float(rew[0]), float(suc[0]), it
