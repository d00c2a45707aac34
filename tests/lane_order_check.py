"""Race sensitivity check on the 32-lane fiber emulation (tests/hostsim/hostwarp.h): the lanes of every interval between two warp
collectives run in ascending, descending and shuffled order in three separate processes; an output that depends on the order is a
shared-memory race between lanes (the CPU stand-in for compute-sanitizer racecheck).  Prints one digest per family and order:
    PYTHONPATH=. python tests/lane_order_check.py            # runs the three orders and compares
"""
import functools
import hashlib
import os
import subprocess
import sys

import numpy as np


def digests():
    import torch

    import gymnasium_robotics_b200 as pkg
    from gymnasium_robotics_b200.fetch import welded_eq_data
    from tests.hostsim_backend import HostSimBackend
    from tests.test_warp_emulation import CASES

    out = {}
    for env_id, ref, flavor1, flavor32, warm, tol in CASES:
        W1, W32 = (functools.partial(HostSimBackend, flavor=f) for f in (flavor1, flavor32))

        kw = dict(experimental=True) if env_id.startswith("Franka") else {}
        env = pkg.make_vec(env_id, num_envs=1, backend_factory=W1, rng_mode="numpy", **kw)
        env.reset(seed=3)
        rng = np.random.default_rng(5)
        for _ in range(warm):
            env.step(rng.uniform(-1, 1, size=(1, env.single_action_space.shape[0])).astype(np.float32))
        eq = welded_eq_data(env.model) if env.model.nmocap > 0 else np.zeros((0, 11))
        b = W32(env.model, eq, env.task, 1, "cpu")
        b.state.copy_(env.backend.state)
        o = b.new_outputs()
        for _ in range(2):
            b.step(torch.as_tensor(rng.uniform(-1, 1, size=(1, b.nact)).astype(np.float32)), o)
        out[env_id] = hashlib.sha1(b.state.numpy().tobytes() + o["obs"].numpy().tobytes()).hexdigest()[:16]
    return out


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        for k, v in digests().items():
            print(k, v)
        sys.exit(0)
    res = {}
    for order in ("ascending", "reverse", "shuffle"):
        env = dict(os.environ, HOSTWARP_ORDER=order)
        txt = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True).stdout
        res[order] = dict(l.split() for l in txt.strip().splitlines() if len(l.split()) == 2)
    bad = 0
    for fam in res["ascending"]:
        same = res["reverse"].get(fam) == res["ascending"][fam] == res["shuffle"].get(fam)
        bad += not same
        print(f"{fam:58s} {'order-independent' if same else 'ORDER-DEPENDENT: ' + str([res[o].get(fam) for o in res])}")
    sys.exit(1 if bad else 0)
