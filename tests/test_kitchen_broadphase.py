"""Two-level broad phase of the kitchen build (-DB200_KITCHEN_GROUPS: csrc/sim_core.cuh `collision`, csrc/dmodel.h group table), on CPU:
(1) the emulation of the two-level scan is bit-identical to the one-level scan over the same regrouped pair list
(-DB200_KITCHEN_FLATSCAN), so the candidate set and order are the flat scan's; (2) a 32-lane model of the level-1 compaction
(exclusive scans, running pair counts, the slot-overflow branch) and of the level-2 bisection against a sequential one."""
import numpy as np
import pytest
import torch

from gymnasium_robotics_b200.kitchen import KITCHEN_REF_POINT, KitchenVectorEnv
from gymnasium_robotics_b200.models import load_model
from tests.hostsim import HostSim
from tests.hostsim_backend import HostSimBackend


class TwoLevel(HostSimBackend):
    FLAVOR = "kitchen_groups"


class FlatScan(HostSimBackend):
    FLAVOR = "kitchen_flat"


def test_group_table_covers_every_pair_once():
    m = load_model("franka_kitchen")
    s = HostSim(m, ref=KITCHEN_REF_POINT, flavor="kitchen_groups")
    assert s._L.hostsim_npair(s._h) == len(m.pair_geom1) == 3708
    assert 0 < s._L.hostsim_nbgrp(s._h) <= 1100          # 1 010 groups: 32 warp iterations instead of 116
    # shared-memory footprint of the staged constants: the 44 KB pair list is gone, the group table is in
    assert s._L.hostsim_hot_words(s._h) * 4 < 48 * 1024


def test_two_level_scan_is_bit_identical_to_the_flat_scan():
    m = load_model("franka_kitchen")
    ea, eb = (KitchenVectorEnv(num_envs=2, backend_factory=F, device="cpu", rng_mode="numpy", model=m) for F in (TwoLevel, FlatScan))
    oa, _ = ea.reset(seed=4)
    ob, _ = eb.reset(seed=4)
    assert torch.equal(oa["observation"], ob["observation"])
    rng = np.random.default_rng(0)
    ncand_max = 0
    for k in range(24):
        a = rng.uniform(-1, 1, size=(2, 9))
        if k >= 8:
            a[:, :7] = np.sign(a[:, :7])      # saturated joint velocities: the arm sweeps through the scene
        ra, rb = ea.step(a), eb.step(a)
        assert torch.equal(ra[0]["observation"], rb[0]["observation"]), k
        ca, cb = ea.backend.sim.counters(), eb.backend.sim.counters()
        assert np.array_equal(ca, cb)
        ncand_max = max(ncand_max, int(ca[3]))
    assert ncand_max >= 8 and getattr(ea.backend, "overflow_bits", 0) == 0


# ---------------------------------------------------------------------------------------------------------------
W = 32


def _exscan(v):
    out = np.concatenate([[0], np.cumsum(v)[:-1]])
    return out, int(np.sum(v))


def lanes_level1(hit, count, start, nsurv_max):
    """Transcription of the level-1 loop for a 32-lane warp; returns (surv entries incl. end marker, overflowed)."""
    surv, nsurv, npexp, over = {}, 0, 0, False
    n = len(hit)
    for base in range(0, n, W):
        idx = np.arange(base, base + W)
        h = np.array([bool(hit[i]) if i < n else False for i in idx])
        npg = np.array([count[i] if i < n and hit[i] else 0 for i in idx])
        slot, total = _exscan(h.astype(int))
        poff, ptotal = _exscan(npg)
        for l in range(W):
            if h[l] and nsurv + slot[l] < nsurv_max:
                surv[nsurv + slot[l]] = (start[idx[l]], npexp + poff[l])
        if nsurv + total > nsurv_max:
            keep = nsurv_max - nsurv
            kept_lanes = [l for l in range(W) if h[l] and slot[l] < keep]
            kept_pairs = (poff[kept_lanes[-1]] + npg[kept_lanes[-1]]) if (kept_lanes and keep > 0) else 0
            over = True
            nsurv, npexp = nsurv_max, npexp + kept_pairs
        else:
            nsurv, npexp = nsurv + total, npexp + ptotal
    surv[nsurv] = (0, npexp)
    return [surv[i] for i in range(nsurv + 1)], over


def lanes_level2(surv):
    nsurv, npexp = len(surv) - 1, surv[-1][1]
    pairs = []
    for ei in range(npexp):
        lo, hi = 0, nsurv
        while hi - lo > 1:
            mid = (lo + hi) >> 1
            if surv[mid][1] <= ei:
                lo = mid
            else:
                hi = mid
        pairs.append(surv[lo][0] + ei - surv[lo][1])
    return pairs


@pytest.mark.parametrize("nsurv_max", [96, 5])
def test_lane_model_of_the_compaction(nsurv_max):
    rng = np.random.default_rng(1)
    for trial in range(50):
        n = int(rng.integers(1, 200))
        count = rng.integers(1, 14, size=n)
        start = np.concatenate([[0], np.cumsum(count)[:-1]])
        hit = rng.random(n) < rng.choice([0.02, 0.2, 0.6])
        surv, over = lanes_level1(hit, count, start, nsurv_max)
        kept = [g for g in range(n) if hit[g]][:nsurv_max]
        assert over == (int(hit.sum()) > nsurv_max)
        want = [p for g in kept for p in range(start[g], start[g] + count[g])]
        assert lanes_level2(surv) == want        # ascending pair order: the flat scan's candidate order


def test_groups_build_tracks_the_validated_flat_build():
    """The two kernel builds scan different pair orders (original list vs regrouped list), so contacts are numbered differently and
    results agree to solver precision rather than bit for bit."""
    from tests.test_kitchen_host import KitchenHostBackend

    m = load_model("franka_kitchen")
    ea, eb = (KitchenVectorEnv(num_envs=2, backend_factory=F, device="cpu", rng_mode="numpy", model=m) for F in (TwoLevel, KitchenHostBackend))
    oa, _ = ea.reset(seed=4)
    ob, _ = eb.reset(seed=4)
    assert torch.equal(oa["observation"], ob["observation"])
    rng = np.random.default_rng(0)
    for k in range(6):
        a = rng.uniform(-1, 1, size=(2, 9))
        oa, ob = ea.step(a)[0], eb.step(a)[0]
        e = (oa["observation"] - ob["observation"]).abs()
        assert float(e[:, :9].max()) < 1e-4 and float(e[:, 18:39].max()) < 1e-4, k
