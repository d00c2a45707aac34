"""Which kernel build and block size b200sim_create picks for each committed model family (run with -m gpu on an H100, 132 SMs).

The choice depends on the model (its nv and features pick the NVP and the translation unit), on num_envs (the waves rule, the
kitchen's 7 / 10 / 11 warps) and on the shared memory one block can hold.  The tables below were recorded on an NVIDIA H100 80GB
HBM3 and pin, per family:
  * for num_envs in NUM_ENVS, what b200sim_launch_config reports: dynamic shared memory in bytes, envs per block, blocks;
  * for B200SIM_WPB = 1..32 (one env), whether b200sim_create accepts the forced block size, and the return code and message
    of a refusal.
A change to the instantiation lists or to the selection code that moves any of these fails here rather than as a slower or
refused launch.
"""
import ctypes

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.fetch import welded_eq_data

pytestmark = pytest.mark.gpu

NUM_ENVS = (1, 61, 1024, 2048, 4096)
FAMILIES = {
    "fetch_pick": ("FetchPickAndPlace-v4", {}),
    "fetch_slide": ("FetchSlide-v4", {}),
    "hand": ("HandManipulateBlock-v1", {}),
    "hand_touch": ("HandManipulateBlock_ContinuousTouchSensors-v1", {}),
    "hand_reach": ("HandReach-v3", {}),
    "adroit_door": ("AdroitHandDoor-v2", {}),
    "adroit_hammer": ("AdroitHandHammer-v2", {}),
    "adroit_pen": ("AdroitHandPen-v2", {}),
    "adroit_relocate": ("AdroitHandRelocate-v2", {}),
    "antmaze": ("AntMaze_Large-v5", {}),
    "pointmaze": ("PointMaze_Large-v3", {}),
    "kitchen_flat": ("FrankaKitchen-v1", {"broadphase": "flat"}),
    "kitchen_groups": ("FrankaKitchen-v1", {}),
    "kitchen_hull": ("FrankaKitchen-v1", {"mesh_collision": "hull"}),
}

# family -> {num_envs: (smem bytes, envs per block, blocks)}
LAUNCH = {
    "fetch_pick": {1: (56384, 7, 1), 61: (56384, 7, 9), 1024: (63376, 8, 128), 2048: (119312, 16, 128), 4096: (231184, 32, 128)},
    "fetch_slide": {1: (56288, 7, 1), 61: (56288, 7, 9), 1024: (63280, 8, 128), 2048: (119216, 16, 128), 4096: (231088, 32, 128)},
    "hand": {1: (95312, 7, 1), 61: (95312, 7, 9), 1024: (178080, 14, 74), 2048: (178080, 14, 147), 4096: (178080, 14, 293)},
    "hand_touch": {1: (100496, 7, 1), 61: (100496, 7, 9), 1024: (185504, 14, 74), 2048: (185504, 14, 147), 4096: (185504, 14, 293)},
    "hand_reach": {1: (84176, 7, 1), 61: (84176, 7, 9), 1024: (156304, 14, 74), 2048: (156304, 14, 147), 4096: (156304, 14, 293)},
    "adroit_door": {1: (102544, 7, 1), 61: (102544, 7, 9), 1024: (188336, 14, 74), 2048: (188336, 14, 147), 4096: (188336, 14, 293)},
    "adroit_hammer": {1: (110784, 7, 1), 61: (110784, 7, 9), 1024: (151104, 10, 103), 2048: (151104, 10, 205), 4096: (191424, 13, 316)},
    "adroit_pen": {1: (97472, 7, 1), 61: (97472, 7, 9), 1024: (180688, 14, 74), 2048: (180688, 14, 147), 4096: (180688, 14, 293)},
    "adroit_relocate": {1: (114352, 7, 1), 61: (114352, 7, 9), 1024: (156880, 10, 103), 2048: (156880, 10, 205), 4096: (199408, 13, 316)},
    "antmaze": {1: (49952, 7, 1), 61: (49952, 7, 9), 1024: (56416, 8, 128), 2048: (108128, 16, 128), 4096: (211552, 32, 128)},
    "pointmaze": {1: (30016, 7, 1), 61: (30016, 7, 9), 1024: (34096, 8, 128), 2048: (66736, 16, 128), 4096: (132016, 32, 128)},
    "kitchen_flat": {1: (160112, 7, 1), 61: (160112, 7, 9), 1024: (203120, 10, 103), 2048: (203120, 10, 205), 4096: (203120, 10, 410)},
    "kitchen_groups": {1: (150656, 7, 1), 61: (150656, 7, 9), 1024: (209536, 11, 94), 2048: (209536, 11, 187), 4096: (209536, 11, 373)},
    "kitchen_hull": {1: (148032, 7, 1), 61: (148032, 7, 9), 1024: (206912, 11, 94), 2048: (206912, 11, 187), 4096: (206912, 11, 373)},
}

# family -> (accepted B200SIM_WPB values, (return code, message) of every refused value)
FORCED = {
    "fetch_pick": ((7, 8, 14, 16, 28, 32), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "fetch_slide": ((7, 8, 14, 16, 28, 32), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "hand": ((7, 14), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "hand_touch": ((7, 14), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "hand_reach": ((7, 14), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "adroit_door": ((7, 14), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "adroit_hammer": ((7, 10, 13, 14), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "adroit_pen": ((7, 14), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "adroit_relocate": ((7, 10, 13, 14), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "antmaze": ((7, 8, 14, 16, 28, 32), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "pointmaze": ((7, 8, 14, 16, 28, 32), [(-8, "b200sim_create: B200SIM_WPB names no kernel variant that fits")]),
    "kitchen_flat": ((7, 10), [(-8, "b200sim_create: B200SIM_WPB names no kitchen kernel variant that fits")]),
    "kitchen_groups": ((7, 10, 11), [(-8, "b200sim_create: B200SIM_WPB names no kitchen kernel variant that fits")]),
    "kitchen_hull": ((7, 10, 11), [(-8, "b200sim_create: B200SIM_WPB names no kitchen kernel variant that fits")]),
}


def _create(env, eq, n, wpb, mp):
    """b200sim_create for n envs of the env's model and task: (0, launch config) or (return code, message)."""
    if wpb is None:
        mp.delenv("B200SIM_WPB", raising=False)
    else:
        mp.setenv("B200SIM_WPB", str(wpb))
    if hasattr(env, "broadphase"):
        mp.setenv("B200SIM_KITCHEN_GROUPS", "1" if env.broadphase == "groups" else "0")
    L, blob = env.backend.L, env.model.to_blob()
    ref = np.asarray(env.backend.ref, dtype=np.float32)
    eq = np.ascontiguousarray(eq, dtype=np.float64)
    h = ctypes.c_void_p()
    rc = L.b200sim_create(blob, len(blob), eq.ctypes.data if eq.size else None, ref.ctypes.data, ctypes.byref(env.task), n,
                          env.device.index or 0, ctypes.byref(h))
    if rc != 0:
        return rc, L.b200sim_last_error(None).decode()
    smem, w, b = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert L.b200sim_launch_config(h, ctypes.byref(smem), ctypes.byref(w), ctypes.byref(b)) == 0
    L.b200sim_destroy(h)
    return 0, (smem.value, w.value, b.value)


def observe(family, mp):
    """The launch configurations and the forced-block-size answers of one family (the form of LAUNCH and FORCED)."""
    env_id, kw = FAMILIES[family]
    env = pkg.make_vec(env_id, num_envs=1, device="cuda:0", **kw)
    if not hasattr(env.backend, "L"):
        pytest.skip("needs the C-ABI (block-size override, launch config)")
    eq = welded_eq_data(env.model) if type(env).__name__ == "FetchVectorEnv" else np.zeros((0, 11))
    launch = {}
    for n in NUM_ENVS:
        rc, cfg = _create(env, eq, n, None, mp)
        assert rc == 0, f"{family}, {n} envs: b200sim_create failed ({rc}): {cfg}"
        launch[n] = cfg
    accepted, refused = [], set()
    for w in range(1, 33):
        rc, what = _create(env, eq, 1, w, mp)
        if rc == 0:
            assert what[1] == w
            accepted.append(w)
        else:
            refused.add((rc, what))
    env.close()
    return launch, (tuple(accepted), sorted(refused))


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_launch_config_and_forced_block_sizes(family, monkeypatch):
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the tables were recorded on a 132-SM H100")
    launch, forced = observe(family, monkeypatch)
    assert launch == LAUNCH[family]
    assert forced == FORCED[family]
