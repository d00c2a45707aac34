"""AntMaze's `ant_info=True` and Ant keywords on the ant kernel build (run with -m gpu on an H100): CUDA vs the fp64 oracle per info
key, the rest of the step bit-identical with the info on and off, the info rows invariant to block size, batch shape and neighbours,
and no extra synchronising call per step."""
import json
import os
import subprocess
import sys
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

import gymnasium_robotics_b200 as pkg  # noqa: E402
from gymnasium_robotics_b200.maze import ANT_INFO_COLUMNS, MAPS  # noqa: E402
from tests.ant_info_oracle import OracleAntInfoEnv  # noqa: E402
from tests.test_ant_info import V4_KEYS, V5_KEYS  # noqa: E402

pytestmark = pytest.mark.gpu


def gpu(env_id, n, **kw):
    return pkg.make_vec(env_id, num_envs=n, device="cuda:0", **kw)


def inject(env, oracles):
    lay = env.backend.layout
    rec = np.zeros((len(oracles), lay["stride"]))
    for i, o in enumerate(oracles):
        rec[i, lay["qpos"]:lay["qpos"] + 15] = o.sim.qpos
        rec[i, lay["qvel"]:lay["qvel"] + 14] = o.sim.qvel
        rec[i, lay["warm"]:lay["warm"] + 14] = o.sim.qacc_warmstart
        rec[i, lay["goal"]:lay["goal"] + 2] = o.goal
    env.set_state(torch.as_tensor(rec, dtype=torch.float32, device="cuda:0"))
    for o in oracles:
        o.set_state(o.sim.qpos.copy(), o.sim.qvel.copy(), o.goal)


# CUDA (fp32) vs the fp64 oracle, one step from one injected state of a landed ant.  Largest errors over the 32 compared env-steps of
# each id, measured on an H100 80GB HBM3 (700 W): positions and distance 4.6e-6, velocities and reward_forward 6.1e-5, the ctrl cost
# 1.8e-7, the contact cost 5.6e-7 (Ant-v4's reward_ctrl under use_contact_forces too), reward_survive exact.  The envelopes are 5x to 10x
# that; the costs are relative to max(1, |value|).
TOL = dict(x_position=3e-5, y_position=3e-5, distance_from_origin=3e-5, x_velocity=5e-4, y_velocity=5e-4, reward_forward=5e-4,
           forward_reward=5e-4, reward_ctrl=2e-6, reward_contact=5e-6, reward_survive=0.0)


@pytest.mark.parametrize("env_id,kw", [("AntMaze_Large-v5", {}), ("AntMaze_Large-v4", dict(use_contact_forces=True))])
def test_cuda_matches_the_oracle_per_key(env_id, kw):
    n = 8
    env = gpu(env_id, n, ant_info=True, rng_mode="numpy", **kw)
    env.reset(seed=11)
    oracles = [OracleAntInfoEnv(MAPS["Large"], env.model, ant_version=env.ant.version, include_cfrc_ext_in_observation=env.include_cfrc, **kw)
               for _ in range(n)]
    for i, o in enumerate(oracles):
        o.reset(seed=11 + i)
        for _ in range(10):
            o.step(np.zeros(8))
    keys = V5_KEYS if env.ant.version == 5 else V4_KEYS
    tols = dict(TOL, reward_ctrl=TOL["reward_contact"]) if kw.get("use_contact_forces") else TOL
    worst = {k: 0.0 for k in keys}
    rng = np.random.default_rng(2)
    for trial in range(4):
        inject(env, oracles)
        a = rng.uniform(-1, 1, (n, 8)).astype(np.float32)
        _, _, _, _, info = env.step(torch.as_tensor(a, device="cuda:0"))
        got = {k: info[k].double().cpu().numpy() for k in keys}
        for i, orc in enumerate(oracles):
            _, _, _, _, oi = orc.step(a[i])
            for k in keys:
                want = float(oi[k])
                err = abs(got[k][i] - want)
                worst[k] = max(worst[k], err)
                assert err <= tols[k] * (max(1.0, abs(want)) if k in ("reward_contact", "reward_ctrl") else 1.0), (k, i, got[k][i], want)
    print(env_id, {k: f"{v:.2e}" for k, v in sorted(worst.items())})
    env.close()


@pytest.mark.parametrize("env_id,kw", [("AntMaze_Large-v5", {}), ("AntMaze_Medium-v4", {})])
def test_info_on_leaves_the_step_bit_identical(env_id, kw):
    """A seeded 50-step rollout (autoresets included) with ant_info on and off: packed rows, flags, the used words of the state records
    and the solver's info words are bit-identical (the ant build keeps the torso position in two of the record's spare words)."""
    n, steps = 256, 50
    envs = [gpu(env_id, n, ant_info=on, rng_mode="device", max_episode_steps=20, **kw) for on in (False, True)]
    assert envs[0].task.touch_mode in (0, 1) and envs[1].task.touch_mode >= 2
    used = envs[0].backend.layout["goal"] + 2
    for e in envs:
        e.reset(seed=5)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    for s in range(steps):
        a = torch.rand((n, 8), generator=g, device="cuda:0") * 2 - 1
        outs = [e.step(a) for e in envs]
        p0, p1 = (e._last for e in envs)
        assert torch.equal(p0["packed"], p1["packed"]) and torch.equal(p0["flags"], p1["flags"]), s
        assert torch.equal(envs[0].backend.state[:, :used], envs[1].backend.state[:, :used]), s
        assert torch.equal(outs[0][4]["solver_info"], outs[1][4]["solver_info"]), s
    for e in envs:
        e.close()


def test_info_rows_invariant_to_block_size_batch_shape_and_neighbours(monkeypatch):
    n, sub = 96, 13
    monkeypatch.delenv("B200SIM_WPB", raising=False)
    ref = gpu("AntMaze_Large-v5", n, ant_info=True, rng_mode="device")
    monkeypatch.setenv("B200SIM_WPB", "7")
    small_blocks = gpu("AntMaze_Large-v5", n, ant_info=True, rng_mode="device")
    monkeypatch.delenv("B200SIM_WPB")
    part = gpu("AntMaze_Large-v5", sub, ant_info=True, rng_mode="device")
    ref.reset(seed=3)
    for _ in range(15):     # let the ants land: contacts, costs
        ref.step(torch.zeros((n, 8), device="cuda:0"))
    state, elapsed = ref.get_state()
    perm = torch.randperm(n, device="cuda:0")
    for e, st, el in ((small_blocks, state, elapsed), (part, state[perm[:sub]], elapsed[perm[:sub]])):
        e.reset(seed=3)
        e.set_state(st.clone(), el.clone())
        e._ant_origin.copy_(ref._ant_origin if e is small_blocks else ref._ant_origin[perm[:sub]])
    g = torch.Generator(device="cuda:0").manual_seed(1)
    for s in range(10):
        a = torch.rand((n, 8), generator=g, device="cuda:0") * 2 - 1
        info_r = ref.step(a)[4]
        info_b = small_blocks.step(a)[4]
        info_p = part.step(a[perm[:sub]])[4]
        if s == 0:   # ref kept its stale torso positions; the others' set_state refreshed them to qpos: compare from the second step on
            continue
        rows_r = torch.stack([info_r[k] for k in ANT_INFO_COLUMNS], 1)
        rows_b = torch.stack([info_b[k] for k in ANT_INFO_COLUMNS], 1)
        rows_p = torch.stack([info_p[k] for k in ANT_INFO_COLUMNS], 1)
        assert torch.equal(rows_r, rows_b), s
        assert torch.equal(rows_r[perm[:sub]], rows_p), s
    for e in (ref, small_blocks, part):
        e.close()


def _syncs(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(x.message) for x in w)


def _sync_counts(mode):
    counts = []
    for on in (False, True):
        env = gpu("AntMaze_UMaze-v5", 64, ant_info=on, rng_mode="device", max_episode_steps=4, autoreset_mode=mode)
        a = torch.zeros((64, 8), device="cuda:0")
        env.reset(seed=3)
        env.step(a)
        counts.append([_syncs(lambda: env.step(a)) for _ in range(10)])
        env.close()
    return counts


@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_no_extra_synchronising_call(mode):
    """Steps with the info make no more synchronising calls than without (the rows are allocated, not read; the reset positions are a
    masked copy on the device).  Counted in a process of its own: PyTorch reports some synchronising calls once per process, so
    counting here would change what later tests of the session count."""
    out = subprocess.run([sys.executable, __file__, "syncs", mode], capture_output=True, text=True, check=True,
                         cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    counts = json.loads(out.stdout.strip().splitlines()[-1])
    assert all(on <= off for on, off in zip(counts[1], counts[0])), counts


if __name__ == "__main__" and sys.argv[1:2] == ["syncs"]:
    print(json.dumps(_sync_counts(sys.argv[2])))
