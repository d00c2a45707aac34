"""Random-action soak of the kernel source on the CPU emulation: several env families, aggressive actions (every fourth
step saturated), TimeLimit + same-step autoreset.  Observations must stay finite and capacity overflow may only show up as
flags in the info word (the counted-but-unwritten contact record was found by exactly this kind of run at scale)."""
import functools

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.adroit import ADROIT_REF_POINT
from gymnasium_robotics_b200.fetch import REF_POINT
from gymnasium_robotics_b200.hand import HAND_REF_POINT
from tests.hostsim_backend import HostSimBackend

CASES = [("FetchPickAndPlace-v4", REF_POINT), ("FetchSlide-v4", REF_POINT), ("HandManipulateEggFull-v1", HAND_REF_POINT),
         ("AdroitHandDoor-v2", ADROIT_REF_POINT), ("AdroitHandHammer-v2", ADROIT_REF_POINT), ("AdroitHandRelocate-v2", ADROIT_REF_POINT),
         ("AntMaze_UMaze-v5", REF_POINT)]


@pytest.mark.parametrize("env_id,ref", CASES)
def test_random_action_soak_stays_finite(env_id, ref):
    n, steps = 6, 36
    env = pkg.make_vec(env_id, num_envs=n, backend_factory=HostSimBackend, rng_mode="torch", autoreset_mode="same_step", max_episode_steps=15)
    assert tuple(env.backend.sim.ref) == pytest.approx(ref)
    env.reset(seed=0)
    g = torch.Generator().manual_seed(7)
    for k in range(steps):
        a = torch.rand((n, env.single_action_space.shape[0]), generator=g) * 2 - 1
        if k % 4 == 0:
            a = torch.sign(a)
        o, r, te, tr, info = env.step(a)
        x = o["observation"] if isinstance(o, dict) else o
        assert torch.isfinite(x).all() and torch.isfinite(r).all(), f"{env_id}: non-finite output at step {k}"
    assert float(x.abs().max()) < 1e3
    assert getattr(env.backend, "overflow_bits", 0) & ~0xF == 0   # only the four documented capacity flags can ever be set


@pytest.mark.parametrize("flavor", ["kitchen", "kitchen_groups"])
def test_kitchen_soak_with_the_two_level_broad_phase(flavor):
    """FrankaKitchen-v1 on the kitchen-flavor emulation (29 dofs, 3 708 pairs in 1 010 groups): saturated actions sweep the arm
    through the scene; no capacity flag at all (a longer run of 5 600 env-steps saw none either, up to 57 candidates)."""
    from gymnasium_robotics_b200.kitchen import KitchenVectorEnv

    env = KitchenVectorEnv(num_envs=4, backend_factory=functools.partial(HostSimBackend, flavor=flavor), device="cpu", rng_mode="torch", autoreset_mode="same_step",
                           max_episode_steps=25)
    env.reset(seed=0)
    g = torch.Generator().manual_seed(3)
    for k in range(60):
        a = torch.rand((4, 9), generator=g) * 2 - 1
        if k % 3 == 0:
            a = torch.sign(a)
        o, r, te, tr, info = env.step(a)
        assert torch.isfinite(o["observation"]).all() and float(o["observation"].abs().max()) < 1e3, k
    assert getattr(env.backend, "overflow_bits", 0) == 0
