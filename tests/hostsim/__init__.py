"""Test-only ctypes wrapper for the host emulation (WARP_W == 1) of the CUDA physics core.  See hostsim.cpp."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = {}


class FetchTaskC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("has_object", "block_gripper", "n_substeps", "reward_dense", "grip_site",
                                             "obj_site", "frame_site", "nrobot")] + \
               [("robot_qadr", ctypes.c_int * 16), ("robot_dadr", ctypes.c_int * 16), ("finger_qadr", ctypes.c_int * 2),
                ("nobs", ctypes.c_int), ("distance_threshold", ctypes.c_float), ("dt", ctypes.c_float),
                ("kind", ctypes.c_int), ("nact", ctypes.c_int), ("ngoal", ctypes.c_int), ("success_radius", ctypes.c_float),
                ("obs_qpos_start", ctypes.c_int), ("vel_clip", ctypes.c_float),
                ("obj_qadr", ctypes.c_int), ("obj_dadr", ctypes.c_int), ("goal_flags", ctypes.c_int),
                ("rotation_threshold", ctypes.c_float), ("touch_mode", ctypes.c_int), ("tip_site", ctypes.c_int * 5),
                ("penv_body", ctypes.c_int)] + \
               [(n, ctypes.c_int) for n in ("st_qpos", "st_qvel", "st_warm", "st_ctrl", "st_mocap", "st_pose", "st_goal",
                                             "st_stride", "st_penv")]


def build(force=False, wide=False):
    """wide = True: the 64-bit dof-mask build (models with more than 32 dofs, -DB200_WIDE as in csrc/b200sim_wide.cu);
    wide = "kitchen": the bring-up build of the Franka-Kitchen kernel features (-DB200_KITCHEN, DESIGN.md section 7);
    wide = "kitchen_groups": that build with the two-level broad phase (-DB200_KITCHEN_GROUPS: regrouped pair list, group table);
    wide = "kitchen_flat": the groups build's data layout scanned in one level, the bit-exact A/B reference of the two-level scan
    (-DB200_KITCHEN_FLATSCAN)"""
    out = os.path.join(_HERE, {True: "libhostsim_wide.so", "kitchen": "libhostsim_kitchen.so", "kitchen_groups": "libhostsim_kitchen_groups.so",
                               "kitchen_flat": "libhostsim_kitchen_flat.so", "warp": "libhostsim_warp.so", "warp_wide": "libhostsim_warp_wide.so",
                               "warp_kitchen_groups": "libhostsim_warp_kitchen_groups.so", "warp_kitchen": "libhostsim_warp_kitchen.so", "warp_timing": "libhostsim_warp_timing.so",
                               "kitchen_hull": "libhostsim_kitchen_hull.so", "warp_kitchen_hull": "libhostsim_warp_kitchen_hull.so"}.get(wide, "libhostsim.so"))
    srcs = [os.path.join(_HERE, "hostsim.cpp")] + [os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc", f)
                                                   for f in ("sim_core.cuh", "dmodel.h", "fetch_task.cuh")] + \
           [os.path.join(_ROOT, "include", "b200sim_model.h"), os.path.join(_ROOT, "include", "b200sim.h"), os.path.join(_HERE, "hostwarp.h"),
            os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc", "reset_sample.cuh")]
    def stale():
        return force or not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs)

    if stale():
        # several processes may get here at once (the 2-rank gloo tests, pytest-xdist): one compiles under a file lock into a
        # temporary name and renames it into place, the others wait and then find the library fresh
        import fcntl

        with open(out + ".lock", "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                tmp = f"{out}.{os.getpid()}.tmp"
                subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unused-function"] +
                                      ({"kitchen": ["-DB200_KITCHEN"], "kitchen_groups": ["-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS"],
                                        "kitchen_flat": ["-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS", "-DB200_KITCHEN_FLATSCAN"],
                                        # WARP_W == 32 on lock-step fibers (hostwarp.h): the lane-parallel code paths themselves
                                        "warp": ["-DB200_HOST_WARP", "-Wno-unknown-pragmas"],
                                        "warp_wide": ["-DB200_HOST_WARP", "-DB200_WIDE", "-Wno-unknown-pragmas"],
                                        "warp_timing": ["-DB200_HOST_WARP", "-DB200_STAGE_TIMING", "-Wno-unknown-pragmas"],
                                        "warp_kitchen": ["-DB200_HOST_WARP", "-DB200_KITCHEN", "-Wno-unknown-pragmas"],
                                        "warp_kitchen_groups": ["-DB200_HOST_WARP", "-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS",
                                                                "-Wno-unknown-pragmas"],
                                        # the kitchen groups build + the support-map narrow phase for mesh geoms (csrc/b200sim_kitchen_hull.cu)
                                        "kitchen_hull": ["-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS", "-DB200_HULL"],
                                        "warp_kitchen_hull": ["-DB200_HOST_WARP", "-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS",
                                                              "-DB200_HULL", "-Wno-unknown-pragmas"]}.get(wide) or
                                       (["-DB200_WIDE"] if wide else [])) + ["-o", tmp, srcs[0]])
                os.replace(tmp, out)
                force = False
    return out


def lib(wide=False):
    if _LIB.get(wide) is None:
        L = ctypes.CDLL(build(wide=wide))
        L.hostsim_create.restype = ctypes.c_void_p
        L.hostsim_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.hostsim_scratch.restype = ctypes.POINTER(ctypes.c_float)
        L.hostsim_scratch.argtypes = [ctypes.c_void_p]
        for f in ("hostsim_destroy", "hostsim_forward", "hostsim_kinematics"):
            getattr(L, f).argtypes = [ctypes.c_void_p]
            getattr(L, f).restype = None
        L.hostsim_step.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.hostsim_step.restype = None
        L.hostsim_offset.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.hostsim_scr_words.argtypes = [ctypes.c_void_p]
        L.hostsim_env_step.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 7
        L.hostsim_spd.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]
        L.hostsim_spd.restype = ctypes.c_int
        for f in ("hostsim_collide", "hostsim_problem", "hostsim_jv", "hostsim_build_h"):
            getattr(L, f).argtypes = [ctypes.c_void_p, ctypes.c_int]
            getattr(L, f).restype = None
        L.hostsim_model_offset.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.hostsim_model.restype = ctypes.POINTER(ctypes.c_uint32)
        L.hostsim_model.argtypes = [ctypes.c_void_p]
        L.hostsim_model_words.argtypes = [ctypes.c_void_p]
        L.hostsim_layout.argtypes = [ctypes.c_void_p]
        L.hostsim_layout.restype = None
        assert L.hostsim_task_size() == ctypes.sizeof(FetchTaskC)
        _LIB[wide] = L
    return _LIB[wide]


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
        lay = np.zeros(6, np.int32)
        self._L.hostsim_layout(lay.ctypes.data)
        return dict(zip(("C_MU", "C_U", "C_DIMGRP", "CON_WORDS", "GRP_WORDS", "G_RANGE"), lay.tolist()))

    @property
    def words(self):
        """The device model buffer (header and arrays, 4-byte words)."""
        return np.ctypeslib.as_array(self._L.hostsim_model(self._h), shape=(self._L.hostsim_model_words(self._h),))

    def forward(self):
        self._L.hostsim_forward(self._h)

    def step(self, n=1):
        self._L.hostsim_step(self._h, int(n))

    def env_step(self, task, mode, nraw, st, action, nobs, ngoal=3):
        obs = np.zeros(nobs, dtype=np.float32)
        ag, dg = np.zeros(ngoal, dtype=np.float32), np.zeros(ngoal, dtype=np.float32)
        rew, suc = np.zeros(1, dtype=np.float32), np.zeros(1, dtype=np.float32)
        a = np.zeros(max(32, len(action)), dtype=np.float32)
        a[:len(action)] = action
        it = self._L.hostsim_env_step(self._h, ctypes.byref(task), mode, nraw, st.ctypes.data, a.ctypes.data, obs.ctypes.data,
                                      ag.ctypes.data, dg.ctypes.data, rew.ctypes.data, suc.ctypes.data)
        return obs, ag, dg, float(rew[0]), float(suc[0]), it
