"""Dynamic proxy without a GPU: warp collectives (shuffles, ballots, __syncwarp) executed per kitchen sub-step by the flat-scan build and by
the two-level broad-phase build, counted by the 32-lane fiber emulation (tests/hostsim/hostwarp.h scheduler rounds).
    PYTHONPATH=. python tests/count_collectives.py"""
import functools
import numpy as np, torch
from gymnasium_robotics_b200.kitchen import KitchenVectorEnv
from gymnasium_robotics_b200.models import load_model
from tests.hostsim_backend import HostSimBackend
from tests import hostsim
m = load_model("franka_kitchen")
res={}
for fl in ("warp_kitchen", "warp_kitchen_groups"):
    env = KitchenVectorEnv(num_envs=1, backend_factory=functools.partial(HostSimBackend, flavor=fl), device="cpu", rng_mode="numpy", model=m)
    env.reset(seed=4)
    L = hostsim.lib(fl)
    rng = np.random.default_rng(0)
    c0 = L.hostsim_collectives()
    for k in range(3):
        env.step(rng.uniform(-1,1,size=(1,9)))
    res[fl] = (L.hostsim_collectives()-c0)/3/40
    print(fl, "warp collectives (scheduler rounds) per sub-step: %.0f" % res[fl])
print("saved per sub-step: %.0f (%.1f %%)" % (res["warp_kitchen"]-res["warp_kitchen_groups"], 100*(1-res["warp_kitchen_groups"]/res["warp_kitchen"])))
