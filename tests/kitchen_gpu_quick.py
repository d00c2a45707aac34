"""Torch-free check of the CUDA kitchen build (csrc/b200sim_kitchen.cu) through the C-ABI: numpy + ctypes + libcudart only, so
that it starts in a second on a fresh GPU box.  Replays tests/golden/kitchen_quick.npz (made by tests/golden/
make_kitchen_quick.py from the host emulation of the same kernel source) and prints the result as one JSON line.
Usage: python tests/kitchen_gpu_quick.py"""
import ctypes
import json
import os
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
t0 = time.time()
g = np.load(os.path.join(ROOT, "tests", "golden", "kitchen_quick.npz"))
rt = ctypes.CDLL("libcudart.so.12") if not os.path.exists("/usr/local/cuda/lib64/libcudart.so") else ctypes.CDLL("/usr/local/cuda/lib64/libcudart.so")
L = ctypes.CDLL(os.path.join(ROOT, "gymnasium_robotics_b200", "libb200sim.so"))
vp, ci = ctypes.c_void_p, ctypes.c_int
L.b200sim_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, vp, vp, vp, ci, ci, ctypes.POINTER(vp)]
L.b200sim_last_error.argtypes, L.b200sim_last_error.restype = [vp], ctypes.c_char_p
L.b200sim_state.argtypes, L.b200sim_state.restype = [vp], vp
L.b200sim_layout.argtypes = [vp, ctypes.POINTER(ci)]
L.b200sim_step.argtypes = [vp] * 9
L.b200sim_refresh.argtypes = [vp] * 8
rt.cudaMalloc.argtypes = [ctypes.POINTER(vp), ctypes.c_size_t]
rt.cudaMemcpy.argtypes = [vp, vp, ctypes.c_size_t, ci]
res = {"ok": False}


def finish():
    res["seconds"] = time.time() - t0
    print(json.dumps(res))


def dev(nbytes):
    p = vp()
    assert rt.cudaMalloc(ctypes.byref(p), nbytes) == 0
    return p


try:
    blob, task, ref = g["blob"].tobytes(), g["task"].tobytes(), np.ascontiguousarray(g["ref"], dtype=np.float32)
    state0, ctrls, exp = g["state0"], g["ctrls"], g["obs"]
    N, stride, nq, nv = state0.shape[0], int(g["stride"]), int(g["nq"]), int(g["nv"])
    h = vp()
    tbuf = ctypes.create_string_buffer(task, len(task))
    rc = L.b200sim_create(blob, len(blob), None, ref.ctypes.data, ctypes.cast(tbuf, vp), N, 0, ctypes.byref(h))
    if rc != 0:
        res["error"] = "create: " + L.b200sim_last_error(None).decode()
        raise SystemExit
    lay = (ci * 9)()
    L.b200sim_layout(h, lay)
    assert lay[7] == stride, (lay[7], stride)
    st = L.b200sim_state(h)
    assert rt.cudaMemcpy(st, state0.ctypes.data, state0.nbytes, 1) == 0
    nobs = nq + nv
    d_obs, d_ag, d_dg, d_r, d_s, d_a = dev(4 * N * nobs), dev(4 * N * nq), dev(4 * N * nq), dev(4 * N), dev(4 * N), dev(4 * N * 9)
    d_info = dev(4 * N)
    obs = np.zeros((N, nobs), dtype=np.float32)
    info = np.zeros(N, dtype=np.int32)
    errs = []
    rc = L.b200sim_refresh(h, None, d_obs, d_ag, d_dg, d_r, d_s, None)
    assert rc == 0, L.b200sim_last_error(h).decode()
    assert rt.cudaDeviceSynchronize() == 0
    rt.cudaMemcpy(obs.ctypes.data, d_obs, obs.nbytes, 2)
    errs.append(float(np.abs(obs - exp[0]).max()))
    t1 = time.time()
    for k in range(ctrls.shape[0]):
        a = np.ascontiguousarray(ctrls[k], dtype=np.float32)
        rt.cudaMemcpy(d_a, a.ctypes.data, a.nbytes, 1)
        rc = L.b200sim_step(h, d_a, d_obs, d_ag, d_dg, d_r, d_s, d_info, None)
        assert rc == 0, L.b200sim_last_error(h).decode()
        e = rt.cudaDeviceSynchronize()
        if e != 0:
            res["error"] = f"cuda error {e} after step {k}"
            raise SystemExit
        rt.cudaMemcpy(obs.ctypes.data, d_obs, obs.nbytes, 2)
        rt.cudaMemcpy(info.ctypes.data, d_info, info.nbytes, 2)
        errs.append(float(np.abs(obs - exp[k + 1]).max()))
        res.setdefault("overflow", []).append(int((info >> 16).max()))
        res.setdefault("iters", []).append(int((info & 0xffff).max()))
    res["step_seconds"] = time.time() - t1
    res["max_abs_err_vs_emulation"] = errs
    res["finite"] = bool(np.isfinite(obs).all())
    # fp32 on both sides, different summation orders (32 lanes vs 1): positions to 1e-4, velocities to 1e-2
    pos_cols = list(range(9)) + list(range(18, 18 + nq - 9))
    res["pos_err"] = float(np.abs(obs - exp[-1])[:, pos_cols].max())
    res["ok"] = res["finite"] and res["pos_err"] < 5e-4 and max(errs) < 5e-2
except SystemExit:
    pass
except Exception as ex:   # noqa: BLE001
    res["error"] = repr(ex)
finish()
