"""Test-only ctypes wrapper for the device harness (devsim.cu): single stages of the kernel source on the GPU.

One shared library per product translation unit, built with the product's nvcc flags and that unit's defines, so that each
stage runs in exactly the instantiation and arithmetic the product kernels use (nvcc's FMA contraction, -prec-div=false,
-prec-sqrt=false, the hardware rsqrtf).  nvcc cross-compiles them without a GPU; running them needs one.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = {}

# flavor -> (the product translation unit it mirrors, its extra defines, the NVPs that unit instantiates)
FLAVORS = {
    "plain": ("b200sim.cu", [], (14, 15, 21, 22, 30)),
    "wide": ("b200sim_wide.cu", ["-DB200_WIDE"], (36,)),
    "kitchen": ("b200sim_kitchen.cu", ["-DB200_KITCHEN"], (31,)),
    "kitchen_groups": ("b200sim_kitchen_groups.cu", ["-DB200_KITCHEN", "-DB200_KITCHEN_GROUPS"], (31,)),
}
# the library that runs the register Cholesky of an NVP (the kitchen units share one spd_solve<31>)
NVP_FLAVOR = {v: f for f, (_, _, vs) in FLAVORS.items() for v in vs if f != "kitchen_groups"}


def build(flavor="plain", force=False):
    """Compile libdevsim_<flavor>.so (lazily, under a file lock, into a temporary name renamed into place)."""
    from gymnasium_robotics_b200 import _lib

    out = os.path.join(_HERE, f"libdevsim_{flavor}.so")
    csrc = os.path.join(_ROOT, "gymnasium_robotics_b200", "csrc")
    srcs = [os.path.join(_HERE, "devsim.cu")] + [os.path.join(csrc, f) for f in ("sim_core.cuh", "dmodel.h", "fetch_task.cuh")] + \
           [os.path.join(_ROOT, "include", f) for f in ("b200sim_model.h", "b200sim.h")]

    def stale():
        return force or not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs)

    if stale():
        import fcntl

        with open(out + ".lock", "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                tmp = f"{out}.{os.getpid()}.tmp"
                subprocess.check_call(["nvcc"] + list(_lib.NVCC_FLAGS) + FLAVORS[flavor][1] + ["-o", tmp, srcs[0]])
                os.replace(tmp, out)
                force = False
    return out


def lib(flavor="plain"):
    if _LIB.get(flavor) is None:
        L = ctypes.CDLL(build(flavor))
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.devsim_spd.argtypes = [ci, ci, vp, vp, vp, ctypes.c_float, ci, vp, vp, ci, ci, ci, ci]
        L.devsim_spd.restype = ci
        L.devsim_last_error.restype = ctypes.c_char_p
        L.devsim_model_create.restype = vp
        L.devsim_model_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, vp, vp, ci, ci]
        L.devsim_model_destroy.argtypes = [vp]
        L.devsim_model_words.restype = ctypes.POINTER(ctypes.c_uint32)
        L.devsim_model_words.argtypes = [vp]
        L.devsim_scr_words.argtypes = [vp]
        L.devsim_model_nwords.argtypes = [vp]
        L.devsim_layout.argtypes = [vp]
        L.devsim_layout.restype = None
        L.devsim_offset.argtypes = [vp, ctypes.c_char_p, ci]
        L.devsim_stage.argtypes = [vp, ci, ci, ci, vp, vp]
        L.devsim_stage.restype = ci
        L.devsim_ray_hits.argtypes = [ci, vp, ci, vp, vp, vp]
        L.devsim_ray_hits.restype = ci
        _LIB[flavor] = L
    return _LIB[flavor]


def spd(nvp, nv, A, x, dadd, hh, H, use_dadd, inplace):
    """spd_solve<nvp> on the GPU for a batch of cases, one block each.  nv: [n] int; A: [n, la], x and dadd: [n, lx], H: [n, lh]
    float32 buffers (la, lx, lh multiples of 4).  A, x and H are overwritten with their contents after the solve."""
    L = lib(NVP_FLAVOR[nvp])
    nv = np.ascontiguousarray(nv, dtype=np.int32)
    for a in (A, x, dadd, H):
        assert a.dtype == np.float32 and a.flags.c_contiguous and a.shape[0] == len(nv) and a.shape[1] % 4 == 0
    rc = L.devsim_spd(int(nvp), len(nv), nv.ctypes.data, A.ctypes.data, dadd.ctypes.data, float(hh), int(bool(use_dadd)), x.ctypes.data,
                      H.ctypes.data, A.shape[1], x.shape[1], H.shape[1], int(bool(inplace)))
    if rc != 0:
        raise RuntimeError(f"devsim_spd(nvp={nvp}): {L.devsim_last_error().decode()}")


def ray_hits(flavor, tp, size, p, d):
    """ray_hits_site(tp, size, p[i], d[i]) of the `flavor` unit on the GPU for rays in the site frame: bool [n]."""
    L = lib(flavor)
    p, d = np.ascontiguousarray(p, np.float32), np.ascontiguousarray(d, np.float32)
    sz, hit = np.ascontiguousarray(size, np.float32), np.zeros(len(p), np.int32)
    if L.devsim_ray_hits(int(tp), sz.ctypes.data, len(p), p.ctypes.data, d.ctypes.data, hit.ctypes.data) != 0:
        raise RuntimeError(f"devsim_ray_hits({flavor}): {L.devsim_last_error().decode()}")
    return hit.astype(bool)


STAGE_COLLIDE, STAGE_KIN, STAGE_PROBLEM, STAGE_JV, STAGE_BUILD_H, STAGE_TOUCH = 0, 1, 2, 3, 4, 5
LAYOUT = ("C_MU", "C_U", "C_DIMGRP", "CON_WORDS", "GRP_WORDS", "G_RANGE", "C_W", "C_D", "CX_POS", "CX_PAIR", "CX_WORDS")


class DevModel:
    """The device model of `model` as the `flavor` unit builds it, and single stages of that unit on batches of scratch images."""

    def __init__(self, flavor, model, eq_data=None, ref=(1.0, 0.75, 0.4), penv_body=-1, ngrp_cap=0):
        self.flavor, self.model, self.ref = flavor, model, np.asarray(ref, np.float32).astype(np.float64)
        L = self._L = lib(flavor)
        blob = model.to_blob()
        eq = np.ascontiguousarray(eq_data, dtype=np.float64) if eq_data is not None else None
        r = np.asarray(ref, dtype=np.float32)
        self._h = L.devsim_model_create(blob, len(blob), eq.ctypes.data if eq is not None else None, r.ctypes.data, int(penv_body),
                                        int(ngrp_cap))
        if not self._h:
            raise RuntimeError(f"devsim_model_create({flavor}): {L.devsim_last_error().decode()}")
        self.scr_words = L.devsim_scr_words(self._h)
        self.words = np.ctypeslib.as_array(L.devsim_model_words(self._h), shape=(L.devsim_model_nwords(self._h),)).copy()
        lay = np.zeros(len(LAYOUT), np.int32)
        L.devsim_layout(lay.ctypes.data)
        self.layout = dict(zip(LAYOUT, lay.tolist()))

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.devsim_model_destroy(self._h)
            self._h = None

    def model_words(self):
        """A view of the device model words this handle uploads for every run (`words` is a copy): an edit reaches the next run."""
        return np.ctypeslib.as_array(self._L.devsim_model_words(self._h), shape=(len(self.words),))

    def offset(self, name):
        o = self._L.devsim_offset(self._h, name.encode(), 0)
        assert o >= 0, name
        return o

    def model_offset(self, name):
        o = self._L.devsim_offset(self._h, name.encode(), 1)
        assert o >= 0, name
        return o

    def run(self, nvp, stage, scratch):
        """stage (STAGE_COLLIDE / STAGE_KIN / STAGE_PROBLEM / STAGE_JV / STAGE_BUILD_H / STAGE_TOUCH) of the NVP = nvp instantiation on
        scratch images [n, scr_words] float32, in place.  STAGE_TOUCH returns the sensor values, float32 [n, nsensor]."""
        assert scratch.dtype == np.float32 and scratch.flags.c_contiguous and scratch.shape[1] == self.scr_words
        out = np.zeros((scratch.shape[0], self.model.nsensor), np.float32) if stage == STAGE_TOUCH else None
        rc = self._L.devsim_stage(self._h, int(nvp), int(stage), scratch.shape[0], scratch.ctypes.data,
                                  out.ctypes.data if out is not None else None)
        if rc != 0:
            raise RuntimeError(f"devsim_stage({self.flavor}, nvp={nvp}): {self._L.devsim_last_error().decode()}")
        return out
