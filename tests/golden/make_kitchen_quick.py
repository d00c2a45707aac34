"""Generates tests/golden/kitchen_quick.npz: inputs and expected outputs (kitchen-flavor host emulation of the kernel source,
fp32) for tests/kitchen_gpu_quick.py, a torch-free ctypes check of the CUDA kitchen build through the C-ABI."""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from gymnasium_robotics_b200.kitchen import INIT_QPOS, KITCHEN_REF_POINT, make_kitchen_task   # noqa: E402
from gymnasium_robotics_b200.models import load_franka_config, load_model                     # noqa: E402
from tests.hostsim_backend import HostSimBackend                                               # noqa: E402
import torch                                                                                   # noqa: E402


class KB(HostSimBackend):
    FLAVOR = "kitchen"   # the flat-scan build's layout


m = load_model("franka_kitchen")
task = make_kitchen_task(m)
N, STEPS = 8, 3
be = KB(m, np.zeros((0, 11)), task, N, "cpu")
lay = be.layout
be.state[:, lay["qpos"]:lay["qpos"] + m.nq] = torch.as_tensor(INIT_QPOS, dtype=torch.float32)
state0 = be.state.numpy().copy()
out = be.new_outputs()
be.refresh(None, out)
obs = [out["obs"].numpy().copy()]
cfg = load_franka_config()
pb, vb = np.array(cfg["pos_bound"][:9]), np.array(cfg["vel_bound"][:9])
rng = np.random.default_rng(5)
ctrls = []
for k in range(STEPS):
    a = rng.uniform(-1, 1, size=(N, 9))
    ctrl = np.clip(obs[-1][:, :9] + np.clip(2 * a, vb[:, 0], vb[:, 1]) * float(task.dt), pb[:, 0], pb[:, 1]).astype(np.float32)
    ctrls.append(ctrl)
    out = be.new_outputs()
    be.step(torch.as_tensor(ctrl), out)
    obs.append(out["obs"].numpy().copy())
assert getattr(be, "overflow_bits", 0) == 0
from gymnasium_robotics_b200._lib import FetchTaskC   # noqa: E402
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "kitchen_quick.npz"), blob=np.frombuffer(m.to_blob(), dtype=np.uint8),
                    task=np.frombuffer(bytes(task), dtype=np.uint8), ref=np.asarray(KITCHEN_REF_POINT, dtype=np.float32),
                    state0=state0, ctrls=np.stack(ctrls), obs=np.stack(obs), stride=lay["stride"], nq=m.nq, nv=m.nv)
print("ok", np.stack(obs).shape, ctypes.sizeof(FetchTaskC), os.path.getsize(os.path.join(ROOT, "tests", "golden", "kitchen_quick.npz")))
