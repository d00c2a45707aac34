"""The AntMaze_*-v3 ids on the GPU: the v3 start draw of b200sim_reset_maze (separation 0.5) and the goal redraw kernel that
b200sim_step launches after the step kernel (b200sim_set_goal_redraw) against the restatements in tests/test_antmaze_v3.py, their
invariance to batch shape, block size and sharding, seeded parity against the v3 oracle env, and steps that make no synchronising
call in the device and torch modes.  Models come from the committed blobs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.maze import MAPS, NOISE
from tests.antmaze_v3_oracle import OracleAntMazeV3Env
from tests.parity_util import check_envelope, inject_records
from tests.test_antmaze_v3 import py_maze_draw_sep, py_redraw
from tests.test_gpu_parity import ENVELOPE
from tests.test_maze_goal_update_gpu import _goals, _place_on_goals, _shift, _sync_messages, _zeros

pytestmark = pytest.mark.gpu
f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _make(env_id="AntMaze_Large-v3", n=1024, **kw):
    kw = {"rng_mode": "device", "device": "cuda:0", **kw}
    return pkg.make_vec(env_id, num_envs=n, **kw)


@pytest.mark.parametrize("env_id", ["AntMaze_Large-v3", "AntMaze_LargeDense-v3"])
def test_device_starts_and_redraws_equal_the_restatement(env_id):
    seed, offset = 31, 7
    env = _make(env_id, env_offset=offset)
    obs, info = env.reset(seed=seed)
    assert info == {}
    st, _ = env.get_state()
    gl, rl = env._goal_loc.cpu().numpy(), env._reset_loc.cpu().numpy()
    g, q = obs["desired_goal"].cpu().numpy(), st[:, :2].cpu().numpy()
    for i in range(env.num_envs):
        wg, wp = py_maze_draw_sep(gl, rl, env.scaling, NOISE, 0.5, seed, offset + i, 0)
        assert np.array_equal(g[i], wg) and np.array_equal(q[i], wp), i
    for step in range(1, 3):
        _place_on_goals(env, _shift(env.num_envs))
        old = _goals(env).cpu().numpy()
        o, r, te, tr, info = env.step(_zeros(env))
        assert "success" not in info
        new, ach = _goals(env).cpu().numpy(), o["achieved_goal"].cpu().numpy()
        assert np.array_equal(o["desired_goal"].cpu().numpy(), old)         # the observation carries the old goal
        changed = (new != old).any(axis=1)
        near = np.linalg.norm(ach.astype(np.float64) - old, axis=1)
        assert not changed[near > 0.45 + 1e-5].any() and changed[near < 0.45 - 1e-5].all()   # fires for the success column
        assert changed.sum() > env.num_envs // 2 and (~changed).sum() > env.num_envs // 6
        for i in range(env.num_envs):
            if changed[i]:
                assert np.array_equal(new[i], py_redraw(gl, env.scaling, seed, offset + i, 1, step)), (step, i)
        # the reward is compute_reward against the goal the env holds now, bit for bit
        assert torch.equal(r, env.compute_reward(o["achieved_goal"], _goals(env)))
        assert not te.any()
    env.close()


def test_device_draws_are_invariant_to_batch_block_size_and_sharding(monkeypatch):
    seed, steps, n = 5, 3, 1024

    def run(n, offset=0, wpb=None):
        if wpb is None:
            monkeypatch.delenv("B200SIM_WPB", raising=False)
        else:
            monkeypatch.setenv("B200SIM_WPB", str(wpb))
        env = _make(n=n, env_offset=offset)
        monkeypatch.delenv("B200SIM_WPB", raising=False)
        env.reset(seed=seed)
        out = [_goals(env).cpu()]
        for _ in range(steps):
            _place_on_goals(env)
            o, r, *_ = env.step(_zeros(env))
            out += [_goals(env).cpu(), r.cpu()]
        env.close()
        return out

    full = run(n)
    for wpb in (7, 16):
        assert all(torch.equal(a, b) for a, b in zip(full, run(n, wpb=wpb)))
    assert all(torch.equal(a[:n // 4], b) for a, b in zip(full, run(n // 4)))
    for k in range(2):
        o = n // 2 + k * (n // 4)
        assert all(torch.equal(a[o:o + n // 4], b) for a, b in zip(full, run(n // 4, offset=o)))


def test_goal_redraw_and_goal_update_share_the_slot():
    """set_goal_update after set_goal_redraw runs the rejection update (the reward untouched); set_goal_redraw(None) turns both off."""
    env = _make(n=256)
    env.reset(seed=3)
    be = env.backend
    args = (env._goal_loc, env.scaling, NOISE, 3, 0, env._episode)
    res = []
    for setter in (be.set_goal_redraw, be.set_goal_update):
        setter(*args)
        saved = env.get_state()
        _place_on_goals(env)
        out = be.new_outputs()
        be.step(_zeros(env), out)
        res.append((out["reward"].clone(), _goals(env), out["achieved"].clone()))
        env.set_state(*saved)
    (r_red, g_red, ach), (r_upd, g_upd, _) = res
    assert torch.equal(r_red, env.compute_reward(ach, g_red)) and (r_upd == 1).all()
    d = torch.linalg.norm(ach.double() - g_upd.double(), dim=1)
    assert (d > 0.45 - 1e-6).all()
    be.set_goal_redraw(None, 0, 0, 0, 0, None)
    g0 = _goals(env)
    _place_on_goals(env)
    be.step(_zeros(env), be.new_outputs())
    assert torch.equal(_goals(env), g0)
    env.close()


def test_antmaze_v3_oracle_parity():
    """AntMaze_Large-v3 in the numpy mode against the v3 oracle env, from the oracle's state at every step; half the ants sit on their
    goals so that goals are redrawn.  Inside the stated antmaze/* envelopes."""
    n, seed = 8, 12
    env = pkg.make_vec("AntMaze_Large-v3", num_envs=n, device="cuda:0", rng_mode="numpy")
    obs, _ = env.reset(seed=seed)
    oracles = [OracleAntMazeV3Env(MAPS["Large"], env.model) for _ in range(n)]
    for i, o in enumerate(oracles):
        oo, _ = o.reset(seed=seed + i)
        np.testing.assert_allclose(obs["desired_goal"][i].double().cpu().numpy(), oo["desired_goal"], rtol=1e-6, atol=2e-6)
    rng = np.random.default_rng(2)
    epos, evel, redraws = [], [], 0
    for step in range(6):
        for i, o in enumerate(oracles):
            if (i + step) % 2 == 0:
                o.sim.qpos[:2] = o.goal
                o.sim.forward()
        env.set_state(inject_records(env, oracles, lambda i, o, rec, lay: rec.__setitem__(slice(lay["goal"], lay["goal"] + 2), o.goal)))
        for o in oracles:
            o.set_state(o.sim.qpos.copy(), o.sim.qvel.copy(), o.goal)
        a = rng.uniform(-1, 1, (n, 8)).astype(np.float32)
        o_, r, te, tr, info = env.step(torch.as_tensor(a))
        goals = _goals(env).cpu().numpy()
        for i, orc in enumerate(oracles):
            before = orc.goal.copy()
            oo, orr, ote, otr, oi = orc.step(a[i].astype(np.float64))
            d = np.abs(o_["observation"][i].double().cpu().numpy() - oo["observation"])
            epos.append(d[:13].max()); evel.append(d[13:27].max())
            assert set(oi) <= set(info) and "success" not in info
            assert float(r[i]) == float(orr) and bool(te[i]) == ote
            np.testing.assert_array_equal(goals[i], orc.goal.astype(f32))
            redraws += int(not np.array_equal(before, orc.goal))
    assert redraws >= 10
    check_envelope("antmaze/pos", epos, *ENVELOPE["antmaze/pos"])
    check_envelope("antmaze/vel", evel, *ENVELOPE["antmaze/vel"])
    env.close()


def _redraw_step_syncs(rng_mode):
    """The synchronising calls of 8 steps of AntMaze_UMaze-v3 x 128 with every ant on its goal before the first, and whether goals
    were redrawn on the way."""
    n = 128
    env = _make("AntMaze_UMaze-v3", n=n, rng_mode=rng_mode)
    env.reset(seed=3)
    gen = torch.Generator(device="cuda:0").manual_seed(3)
    actions = [torch.rand((n, 8), generator=gen, device="cuda:0") * 2 - 1 for _ in range(9)]
    env.step(actions[0])                 # first calls of this env: not counted
    _place_on_goals(env)                 # (set_state reads the step counters: not counted)
    g0 = _goals(env)
    torch.cuda.synchronize()
    syncs = [_sync_messages(lambda a=a: env.step(a)) for a in actions[1:]]
    torch.cuda.synchronize()
    redrawn = not torch.equal(_goals(env), g0)
    env.close()
    return syncs, redrawn


@pytest.mark.parametrize("rng_mode", ["device", "torch"])
def test_steps_with_redraws_make_no_synchronising_call(rng_mode):
    # In a process of its own: torch prints its notice about the sync debug mode once per process, the first time the mode is
    # switched on, and tests/test_env_host_syncs_gpu.py counts that notice in the first reset it observes.
    code = f"import json; from tests.test_antmaze_v3_gpu import _redraw_step_syncs; print(json.dumps(_redraw_step_syncs({rng_mode!r})))"
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    syncs, redrawn = json.loads(res.stdout.strip().splitlines()[-1])
    assert syncs == [[]] * 8
    assert redrawn                       # goals were redrawn on the way
