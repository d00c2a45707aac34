"""HandVectorEnv (host logic + the kernel source emulated with WARP_W == 1) against the oracle restatement of the
reference's MujocoHandBlockEnv.  CPU only; the GPU parity proper is in tests/test_gpu_parity.py."""
import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.hand import HandVectorEnv
from gymnasium_robotics_b200.models import load_model
from oracle.hand_env import OracleHandBlockEnv
from tests.hostsim_backend import HostSimBackend




def make(task="HandManipulateBlockRotateXYZ", n=1, **kw):
    return HandVectorEnv(task, num_envs=n, backend_factory=HostSimBackend, rng_mode="numpy", **kw)


def test_spaces_and_ids():
    env = pkg.make_vec("HandManipulateBlockRotateXYZ-v1", num_envs=2, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.single_action_space.shape == (20,)
    assert env.single_observation_space["observation"].shape == (61,)
    assert env.single_observation_space["achieved_goal"].shape == (7,)
    assert env.max_episode_steps == 100
    obs, info = env.reset(seed=3)
    assert obs["observation"].shape == (2, 61) and obs["desired_goal"].shape == (2, 7)
    with pytest.raises(ValueError):
        env.step(np.zeros((2, 4), dtype=np.float32))
    assert "HandManipulateBlockDense-v1" in pkg.ENV_IDS and "HandManipulateBlockRotateParallel-v1" in pkg.ENV_IDS


@pytest.mark.parametrize("task,kw", [("HandManipulateBlockRotateXYZ", dict(target_position="ignore", target_rotation="xyz")),
                                     ("HandManipulateBlockFull", dict(target_position="random", target_rotation="xyz")),
                                     ("HandManipulateBlockRotateParallel", dict(target_position="ignore", target_rotation="parallel"))])
def test_reset_matches_oracle_sampling(task, kw):
    """Same seed -> same RNG draws (numpy PCG64 parity mode): identical goal; settled state within fp32 tolerance."""
    model = load_model("hand_block")
    env = make(task)
    orc = OracleHandBlockEnv(model=model, **kw)
    obs, _ = env.reset(seed=11)
    oobs, _ = orc.reset(seed=11)
    g, og = obs["desired_goal"][0].double().numpy(), oobs["desired_goal"]
    np.testing.assert_allclose(g[3:], og[3:], atol=2e-6)          # rotation goal: pure RNG + quaternion algebra
    np.testing.assert_allclose(g[:3], og[:3], atol=2e-3)          # position goal rides on the settled block position
    a, oa = obs["achieved_goal"][0].double().numpy(), oobs["achieved_goal"]
    np.testing.assert_allclose(a[:3], oa[:3], atol=2e-3)
    assert a[2] > 0.04 and oa[2] > 0.04
    # robot joints after the 200 settle sub-steps
    np.testing.assert_allclose(obs["observation"][0, :24].double().numpy(), oobs["observation"][:24], atol=5e-3)


def test_step_tracks_oracle_from_injected_state():
    """Free-running env steps from identical state: fp32 kernel arithmetic vs the fp64 oracle."""
    model = load_model("hand_block")
    env = make()
    orc = OracleHandBlockEnv(model=model)
    env.reset(seed=5)
    orc.reset(seed=5)
    lay, m = env.backend.layout, model
    rec = np.zeros(lay["stride"])
    s = orc.sim
    rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
    rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
    rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
    rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
    rec[lay["goal"]:lay["goal"] + 7] = orc.goal
    env.set_state(torch.as_tensor(rec[None], dtype=torch.float32))
    rng = np.random.default_rng(0)
    for k in range(3):
        a = rng.uniform(-1, 1, size=20)
        obs, rew, term, trunc, info = env.step(a[None].astype(np.float32))
        oobs, orew, _, _, oinfo = orc.step(a)
        o, oo = obs["observation"][0].double().numpy(), oobs["observation"]
        # joint angles and block pose; velocities are looser (contact forces on a 70 g block, see DESIGN.md)
        np.testing.assert_allclose(o[:24], oo[:24], atol=2e-3)
        np.testing.assert_allclose(o[54:57], oo[54:57], atol=2e-3)
        assert float(rew[0]) == float(orew)
        assert float(info["is_success"][0]) == float(oinfo["is_success"])
    assert not bool(term.any()) and not bool(trunc.any())


def test_compute_reward_matches_oracle():
    model = load_model("hand_block")
    rng = np.random.default_rng(1)
    ag, dg = rng.normal(size=(64, 7)), rng.normal(size=(64, 7))
    ag[:, 3:] /= np.linalg.norm(ag[:, 3:], axis=1, keepdims=True)
    dg[:, 3:] /= np.linalg.norm(dg[:, 3:], axis=1, keepdims=True)
    dg[:8] = ag[:8]                       # exact successes
    dg[8:16, :3] = ag[8:16, :3] + 0.004   # near the 0.01 m threshold
    for task, kw in (("HandManipulateBlockRotateXYZ", dict(target_position="ignore", target_rotation="xyz")),
                     ("HandManipulateBlockFull", dict(target_position="random", target_rotation="xyz"))):
        for rt in ("sparse", "dense"):
            env = make(task, reward_type=rt)
            orc = OracleHandBlockEnv(model=model, reward_type=rt, **kw)
            r = env.compute_reward(ag, dg, {})
            ro = orc.compute_reward(ag, dg, {})
            np.testing.assert_allclose(r, ro, atol=2e-3 if rt == "dense" else 0)


def test_touch_sensor_observation_tracks_oracle():
    """HandManipulateBlockRotateXYZ_ContinuousTouchSensors-v1 / _BooleanTouchSensors-v1: 92 extra observation entries."""
    model = load_model("hand_block_touch")
    assert model.nsensor == 92
    env = pkg.make_vec("HandManipulateBlockRotateXYZ_ContinuousTouchSensors-v1", num_envs=1, backend_factory=HostSimBackend,
                       rng_mode="numpy")
    envb = pkg.make_vec("HandManipulateBlockRotateXYZ_BooleanTouchSensors-v1", num_envs=1, backend_factory=HostSimBackend,
                        rng_mode="numpy")
    assert env.single_observation_space["observation"].shape == (153,)
    orc = OracleHandBlockEnv(model=model, touch_get_obs="sensordata")
    obs, _ = env.reset(seed=2)
    obsb, _ = envb.reset(seed=2)
    oobs, _ = orc.reset(seed=2)
    t, tb, ot = obs["observation"][0, 61:].double().numpy(), obsb["observation"][0, 61:].double().numpy(), oobs["observation"][61:]
    assert ot.shape == (92,) and ot.sum() > 0.3   # the 70 g block rests on the hand: about m g = 0.69 N of normal force
    # the same sensors fire; forces agree to a few percent (fp32 contact geometry, see DESIGN.md)
    assert set(np.nonzero(t > 1e-3)[0]) == set(np.nonzero(ot > 1e-3)[0])
    np.testing.assert_allclose(t, ot, atol=0.03 * max(1.0, ot.max()))
    assert np.array_equal(tb, (t > 0).astype(np.float64))
    # one step with identical state: touch values follow
    lay, m, s = env.backend.layout, model, orc.sim
    rec = np.zeros(lay["stride"])
    rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
    rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
    rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
    rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
    rec[lay["goal"]:lay["goal"] + 7] = orc.goal
    env.set_state(torch.as_tensor(rec[None], dtype=torch.float32))
    a = np.random.default_rng(3).uniform(-1, 1, 20)
    obs, *_ = env.step(a[None].astype(np.float32))
    oobs, *_ = orc.step(a)
    t, ot = obs["observation"][0, 61:].double().numpy(), oobs["observation"][61:]
    np.testing.assert_allclose(t, ot, atol=0.05 * max(1.0, ot.max()))


def test_hand_reach_matches_oracle():
    """HandReach-v3: construction (initial fingertip goal, palm position by host FK), goal sampling with the reference's
    draw order, and env-steps from identical state."""
    from gymnasium_robotics_b200.hand import HandReachVectorEnv
    from oracle.hand_env import OracleHandReachEnv

    model = load_model("hand_reach")
    env = pkg.make_vec("HandReach-v3", num_envs=2, backend_factory=HostSimBackend, rng_mode="numpy")
    assert isinstance(env, HandReachVectorEnv) and env.max_episode_steps == 50
    assert env.single_observation_space["observation"].shape == (63,) and env.single_action_space.shape == (20,)
    orc = OracleHandReachEnv(model=model)
    np.testing.assert_allclose(env.palm_xpos, orc.palm_xpos, atol=1e-12)
    np.testing.assert_allclose(env.initial_goal.double().numpy(), orc.initial_goal, atol=2e-6)
    for seed in (0, 1, 2, 3):   # covers both branches of the 10 % "keep the initial pose" draw over the seeds
        obs, _ = env.reset(seed=seed)
        oobs, _ = orc.reset(seed=seed)
        np.testing.assert_allclose(obs["desired_goal"][0].double().numpy(), oobs["desired_goal"], atol=2e-6)
        np.testing.assert_allclose(obs["observation"][0].double().numpy(), oobs["observation"], atol=2e-6)
    rng = np.random.default_rng(0)
    for k in range(4):
        a = rng.uniform(-1, 1, size=(2, 20)).astype(np.float32)
        a[1] = a[0]
        obs, rew, term, trunc, info = env.step(a)
        oobs, orew, _, _, oinfo = orc.step(a[0].astype(np.float64))
        np.testing.assert_allclose(obs["observation"][0].double().numpy(), oobs["observation"], atol=2e-3)
        np.testing.assert_allclose(obs["achieved_goal"][0].double().numpy(), oobs["achieved_goal"], atol=2e-4)
        assert float(rew[0]) == float(orew) and float(info["is_success"][0]) == float(oinfo["is_success"])
    r = env.compute_reward(obs["achieved_goal"], obs["desired_goal"], {})
    assert torch.equal(r, rew)


def test_pen_env_matches_oracle():
    """HandManipulatePen*-v1: capsule object, no initial rotation randomisation, z rotation ignored in the goal distance,
    5 cm position threshold (manipulate_pen.py:216-235)."""
    model = load_model("hand_pen")
    env = pkg.make_vec("HandManipulatePenRotate-v1", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.ignore_z_target_rotation and env.distance_threshold == 0.05 and not env.randomize_initial_rotation
    orc = OracleHandBlockEnv(model=model, target_position="ignore", target_rotation="xyz", randomize_initial_rotation=False,
                             ignore_z_target_rotation=True, distance_threshold=0.05)
    obs, _ = env.reset(seed=21)
    oobs, _ = orc.reset(seed=21)
    np.testing.assert_allclose(obs["desired_goal"][0, 3:].double().numpy(), oobs["desired_goal"][3:], atol=2e-6)
    a, oa = obs["achieved_goal"][0].double().numpy(), oobs["achieved_goal"]
    assert a[2] > 0.04 and oa[2] > 0.04
    np.testing.assert_allclose(a[:3], oa[:3], atol=5e-3)
    # env-steps from identical state
    lay, m, s = env.backend.layout, model, orc.sim
    rng = np.random.default_rng(5)
    for k in range(3):
        rec = np.zeros(lay["stride"])
        rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
        rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
        rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
        rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
        rec[lay["goal"]:lay["goal"] + 7] = orc.goal
        env.set_state(torch.as_tensor(rec[None], dtype=torch.float32))
        act = rng.uniform(-1, 1, 20)
        obs, rew, *_ , info = env.step(act[None].astype(np.float32))
        oobs, orew, _, _, oinfo = orc.step(act)
        np.testing.assert_allclose(obs["observation"][0, :24].double().numpy(), oobs["observation"][:24], atol=2e-3)
        np.testing.assert_allclose(obs["observation"][0, 54:57].double().numpy(), oobs["observation"][54:57], atol=2e-3)
        assert float(rew[0]) == float(orew)
    # ignore-z goal distance: dense reward on random pose pairs against the oracle's numpy restatement
    envd = pkg.make_vec("HandManipulatePenRotateDense-v1", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    orcd = OracleHandBlockEnv(model=model, target_position="ignore", target_rotation="xyz", reward_type="dense",
                              randomize_initial_rotation=False, ignore_z_target_rotation=True, distance_threshold=0.05)
    ag, dg = rng.normal(size=(32, 7)), rng.normal(size=(32, 7))
    ag[:, 3:] /= np.linalg.norm(ag[:, 3:], axis=1, keepdims=True)
    dg[:, 3:] /= np.linalg.norm(dg[:, 3:], axis=1, keepdims=True)
    np.testing.assert_allclose(envd.compute_reward(ag, dg, {}), orcd.compute_reward(ag, dg, {}), atol=2e-3)
    # the in-kernel (emulated) ignore-z distance: dense step reward against the oracle
    envd.reset(seed=21)
    orcd.reset(seed=21)
    s = orcd.sim
    rec = np.zeros(lay["stride"])
    rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
    rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
    rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
    rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
    rec[lay["goal"]:lay["goal"] + 7] = orcd.goal
    envd.set_state(torch.as_tensor(rec[None], dtype=torch.float32))
    act = rng.uniform(-1, 1, 20)
    _, rew, *_ = envd.step(act[None].astype(np.float32))
    _, orew, *_ = orcd.step(act)
    assert abs(float(rew[0]) - float(orew)) < 5e-3 and float(orew) < -0.05


def test_egg_env_matches_oracle():
    """HandManipulateEgg*-v1 (manipulate_egg.py:214-235): ellipsoid object through the general convex collider, otherwise
    the block env's defaults."""
    model = load_model("hand_egg")
    env = pkg.make_vec("HandManipulateEggRotate-v1", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    assert not env.ignore_z_target_rotation and env.distance_threshold == 0.01 and env.randomize_initial_rotation
    orc = OracleHandBlockEnv(model=model, target_position="ignore", target_rotation="xyz")
    obs, _ = env.reset(seed=21)
    oobs, _ = orc.reset(seed=21)
    np.testing.assert_allclose(obs["desired_goal"][0, 3:].double().numpy(), oobs["desired_goal"][3:], atol=2e-6)
    a, oa = obs["achieved_goal"][0].double().numpy(), oobs["achieved_goal"]
    assert a[2] > 0.04 and oa[2] > 0.04
    np.testing.assert_allclose(a[:3], oa[:3], atol=5e-3)
    lay, m, s = env.backend.layout, model, orc.sim
    rng = np.random.default_rng(5)
    seen_contact = False
    for k in range(4):
        rec = np.zeros(lay["stride"])
        rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
        rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
        rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
        rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
        rec[lay["goal"]:lay["goal"] + 7] = orc.goal
        env.set_state(torch.as_tensor(rec[None], dtype=torch.float32))
        act = rng.uniform(-1, 1, 20)
        obs, rew, *_ , info = env.step(act[None].astype(np.float32))
        oobs, orew, _, _, oinfo = orc.step(act)
        seen_contact = seen_contact or s.ncon > 0
        np.testing.assert_allclose(obs["observation"][0, :24].double().numpy(), oobs["observation"][:24], atol=2e-4)
        np.testing.assert_allclose(obs["observation"][0, 54:61].double().numpy(), oobs["observation"][54:61], atol=2e-4)
        assert float(rew[0]) == float(orew)
    assert seen_contact
    assert {"HandManipulateEgg-v1", "HandManipulateEggFull-v1", "HandManipulateEggRotate_BooleanTouchSensors-v1",
            "HandManipulateEgg_ContinuousTouchSensorsDense-v1"} <= set(pkg.ENV_IDS)


# ------------------------------------------------------------------------------------------------ Adroit hammer (config 5a)
def test_adroit_hammer_env_matches_oracle():
    """AdroitHandHammer-v2 on the wide build (33 dofs: 64-bit dof masks, bordered Cholesky; emulated here with -DB200_WIDE):
    reset (board height from the same PCG64 draw), env-steps from injected oracle states, dense and sparse reward,
    get/set_env_state round trip (adroit_hammer.py:291-402)."""
    from oracle.adroit_env import OracleAdroitHammerEnv

    m = load_model("adroit_hammer")
    assert m.nv == 33 and m.nu == 26
    env = pkg.make_vec("AdroitHandHammer-v2", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.single_observation_space.shape == (46,) and env.single_action_space.shape == (26,) and env.max_episode_steps == 200
    orc = OracleAdroitHammerEnv(m, noslip=False)
    obs, info = env.reset(seed=4)
    oobs, _ = orc.reset(seed=4)
    assert obs.shape == (1, 46) and info == {}
    np.testing.assert_allclose(obs[0].double().numpy(), oobs, atol=1e-6)
    board_z = float(env.get_env_state()["board_pos"][0, 2])
    assert 0.1 <= board_z <= 0.25 and board_z == pytest.approx(orc.sim.body_pos[orc.target_body_id, 2], abs=1e-7)
    lay, s = env.backend.layout, orc.sim
    rng = np.random.default_rng(1)
    errs = []
    for k in range(8):
        rec = np.zeros(lay["stride"])
        rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
        rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
        rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
        rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
        rec[lay["penv"]:lay["penv"] + 3] = s.body_pos[orc.target_body_id]
        rec[lay["penv"] + 3:lay["penv"] + 7] = np.asarray(m.body_quat).reshape(-1, 4)[orc.target_body_id]
        env.backend.state[0] = torch.as_tensor(rec, dtype=torch.float32)
        a = rng.uniform(-1, 1, 26)
        if k >= 4:
            a[:2] = [-1, -0.5]     # lower the arm onto the hammer
        o, r, te, tr, info = env.step(a[None].astype(np.float32))
        oo, orr, _, _, oi = orc.step(a)
        d = np.abs(o[0].double().numpy() - oo)
        errs.append(d.max())
        assert d.max() < 2e-5                            # all 46 entries (measured: < 1e-6)
        assert abs(float(r[0]) - orr) < 2e-5 and bool(info["success"][0]) == bool(oi["success"])
        assert not bool(te.any()) and not bool(tr.any())
    assert np.median(errs) < 5e-6
    # sparse reward ids and the state round trip
    envs = pkg.make_vec("AdroitHandHammerSparse-v2", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    envs.reset(seed=4)
    _, r, *_ = envs.step(np.zeros((1, 26), dtype=np.float32))
    assert float(r[0]) == pytest.approx(-0.1)
    st = env.get_env_state()
    o1 = env.set_env_state(st)
    st2 = env.get_env_state()
    assert torch.equal(st["qpos"], st2["qpos"]) and torch.equal(st["board_pos"], st2["board_pos"]) and o1.shape == (1, 46)
    with pytest.raises(ValueError):
        pkg.make_vec("AdroitHandHammer-v2", num_envs=1, backend_factory=HostSimBackend, reward_type="shaped")


def test_adroit_relocate_env_matches_oracle():
    """AdroitHandRelocate-v2 (36 dofs, wide build): five reset draws in the reference's order (ball x, y; target x, y, z),
    env-steps from injected oracle states, reward / success, state round trip (adroit_relocate.py:288-402)."""
    from oracle.adroit_env import OracleAdroitRelocateEnv

    m = load_model("adroit_relocate")
    assert m.nv == 36 and m.nu == 30
    env = pkg.make_vec("AdroitHandRelocate-v2", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.single_observation_space.shape == (39,) and env.single_action_space.shape == (30,)
    orc = OracleAdroitRelocateEnv(m, noslip=False)
    obs, _ = env.reset(seed=4)
    oobs, _ = orc.reset(seed=4)
    np.testing.assert_allclose(obs[0].double().numpy(), oobs, atol=1e-6)
    st = env.get_env_state()
    np.testing.assert_allclose(st["target_pos"][0].double().numpy(), orc.target_pos, atol=1e-7)
    np.testing.assert_allclose(st["obj_pos"][0].double().numpy(), orc.sim.body_pos[orc.obj_body_id], atol=1e-7)
    np.testing.assert_allclose(st["hand_pos"][0].double().numpy(), orc.get_env_state()["hand_pos"], atol=1e-6)
    lay, s = env.backend.layout, orc.sim
    rng = np.random.default_rng(1)
    for k in range(6):
        rec = np.zeros(lay["stride"])
        rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
        rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
        rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
        rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
        rec[lay["penv"]:lay["penv"] + 3] = s.body_pos[orc.obj_body_id]
        rec[lay["penv"] + 3:lay["penv"] + 7] = np.asarray(m.body_quat).reshape(-1, 4)[orc.obj_body_id]
        rec[lay["goal"]:lay["goal"] + 3] = orc.target_pos
        env.backend.state[0] = torch.as_tensor(rec, dtype=torch.float32)
        a = rng.uniform(-1, 1, 30)
        if k >= 3:
            a[:3] = [0, 0.5, -1]     # arm forward and down onto the table
        o, r, te, tr, info = env.step(a[None].astype(np.float32))
        oo, orr, _, _, oi = orc.step(a)
        assert np.abs(o[0].double().numpy() - oo).max() < 2e-5
        assert abs(float(r[0]) - orr) < 2e-5 and bool(info["success"][0]) == bool(oi["success"])
    o1 = env.set_env_state(env.get_env_state())
    assert o1.shape == (1, 39) and {"AdroitHandRelocate-v2", "AdroitHandRelocateSparse-v2"} <= set(pkg.ENV_IDS)


def test_adroit_pen_env_matches_oracle():
    """AdroitHandPen-v2 (30 dofs): the pen is a cylinder (portal-refinement collider) and the static target pen's
    quaternion is per-env state (two Euler draws per reset); obs 45, dense / sparse reward (adroit_pen.py:288-430)."""
    from oracle.adroit_env import OracleAdroitPenEnv

    m = load_model("adroit_pen")
    env = pkg.make_vec("AdroitHandPen-v2", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.single_observation_space.shape == (45,) and env.single_action_space.shape == (24,)
    orc = OracleAdroitPenEnv(m, noslip=False)
    obs, _ = env.reset(seed=4)
    oobs, _ = orc.reset(seed=4)
    np.testing.assert_allclose(obs[0].double().numpy(), oobs, atol=2e-6)
    assert orc.pen_length == pytest.approx(0.13, abs=1e-12) and env.task.distance_threshold == pytest.approx(0.13, abs=1e-7)
    np.testing.assert_allclose(env.get_env_state()["desired_orien"][0].double().numpy(), orc.get_env_state()["desired_orien"], atol=1e-7)
    lay, s = env.backend.layout, orc.sim
    rng = np.random.default_rng(1)
    errs = []
    for k in range(8):
        rec = np.zeros(lay["stride"])
        rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
        rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
        rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
        rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
        rec[lay["penv"]:lay["penv"] + 3] = s.body_pos[orc.target_obj_body_id]
        rec[lay["penv"] + 3:lay["penv"] + 7] = s.body_quat[orc.target_obj_body_id]
        env.backend.state[0] = torch.as_tensor(rec, dtype=torch.float32)
        a = rng.uniform(-1, 1, 24)
        o, r, te, tr, info = env.step(a[None].astype(np.float32))
        oo, orr, _, _, oi = orc.step(a)
        d = np.abs(o[0].double().numpy() - oo)
        errs.append(d.max())
        assert np.delete(d, [30, 31, 32]).max() < 2e-4      # everything but the pen's angular velocity
        assert d.max() < 2e-2                               # fp32 vs fp64 portal normals (1e-4) torque the light pen
        assert abs(float(r[0]) - orr) < 2e-4 and bool(info["success"][0]) == bool(oi["success"])
    assert np.median(errs) < 2e-3
    envs = pkg.make_vec("AdroitHandPenSparse-v2", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    envs.reset(seed=4)
    _, r, *_ = envs.step(np.zeros((1, 24), dtype=np.float32))
    assert float(r[0]) == pytest.approx(-0.1)
    assert env.set_env_state(env.get_env_state()).shape == (1, 45)


def test_adroit_door_env_matches_oracle():
    """AdroitHandDoor-v2 (30 dofs, 278 candidate geom pairs -> two-byte broad-phase candidates; cylinder door posts and
    latch through the portal-refinement collider; per-env door frame position) (adroit_door.py:279-402)."""
    from oracle.adroit_env import OracleAdroitDoorEnv

    m = load_model("adroit_door")
    assert len(m.pair_geom1) > 255
    env = pkg.make_vec("AdroitHandDoor-v2", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    assert env.single_observation_space.shape == (39,) and env.single_action_space.shape == (28,)
    orc = OracleAdroitDoorEnv(m, noslip=False)
    obs, _ = env.reset(seed=4)
    oobs, _ = orc.reset(seed=4)
    np.testing.assert_allclose(obs[0].double().numpy(), oobs, atol=2e-6)
    np.testing.assert_allclose(env.get_env_state()["door_body_pos"][0].double().numpy(), orc.get_env_state()["door_body_pos"], atol=1e-7)
    lay, s = env.backend.layout, orc.sim
    rng = np.random.default_rng(1)
    for k in range(8):
        rec = np.zeros(lay["stride"])
        rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
        rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
        rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
        rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
        rec[lay["penv"]:lay["penv"] + 3] = s.body_pos[orc.door_body_id]
        rec[lay["penv"] + 3:lay["penv"] + 7] = s.body_quat[orc.door_body_id]
        env.backend.state[0] = torch.as_tensor(rec, dtype=torch.float32)
        a = rng.uniform(-1, 1, 28)
        if k >= 4:
            a[0] = 1.0     # push the arm towards the door
        o, r, te, tr, info = env.step(a[None].astype(np.float32))
        oo, orr, _, _, oi = orc.step(a)
        assert np.abs(o[0].double().numpy() - oo).max() < 2e-4
        assert abs(float(r[0]) - orr) < 2e-4 and bool(info["success"][0]) == bool(oi["success"])
    assert env.set_env_state(env.get_env_state()).shape == (1, 39)
    assert {"AdroitHandDoor-v2", "AdroitHandDoorSparse-v2", "AdroitHandPenSparse-v2"} <= set(pkg.ENV_IDS)


def test_adroit_reset_honours_initial_state_dict():
    """adroit_hammer.py:359-370: reset(options={"initial_state_dict": ...}) = ordinary reset, then set_env_state."""

    env = pkg.make_vec("AdroitHandHammer-v2", num_envs=2, backend_factory=HostSimBackend, rng_mode="numpy")
    obs0, _ = env.reset(seed=3)
    sd = env.get_env_state()
    q = sd["qpos"][0].clone()
    q[2] += 0.1                                   # bend one arm joint
    want = dict(qpos=q.numpy(), qvel=np.zeros(env.model.nv), board_pos=np.array([0.05, 0.0, 0.2]))
    obs, _ = env.reset(seed=3, options={"initial_state_dict": want})
    sd2 = env.get_env_state()
    assert torch.allclose(sd2["qpos"], torch.as_tensor(want["qpos"], dtype=torch.float32).expand(2, -1))
    assert torch.allclose(sd2["board_pos"], torch.as_tensor(want["board_pos"], dtype=torch.float32).expand(2, -1))
    assert float((obs - obs0).abs().max()) > 1e-3 and abs(float(obs[0, 2]) - float(q[2])) < 1e-6
    env.close()
