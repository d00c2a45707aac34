"""Host logic of FetchVectorEnv on CPU: the kernel source runs through the WARP_W == 1 emulation backend
(tests/hostsim_backend.py), so reset sampling, seeding, TimeLimit, autoreset and the GoalEnv contract are covered
without a GPU -- and the emulated kernel arithmetic is compared with the fp64 oracle env along the way."""
import numpy as np
import pytest
import torch

from gymnasium_robotics_b200.fetch import FetchVectorEnv
from tests.hostsim_backend import HostSimBackend
from tests.parity_util import inject_oracle_state, oracle_env_from_model


def mk(task="FetchPickAndPlace", n=2, **kw):
    return FetchVectorEnv(task, num_envs=n, backend_factory=HostSimBackend, **kw)


@pytest.fixture(scope="module")
def pnp():
    return mk("FetchPickAndPlace", 3, rng_mode="numpy")


def test_spaces_and_shapes(pnp):
    obs, info = pnp.reset(seed=1)
    assert info == {}
    assert obs["observation"].shape == (3, 25) and obs["achieved_goal"].shape == (3, 3) and obs["desired_goal"].shape == (3, 3)
    assert pnp.single_action_space.shape == (4,) and pnp.single_action_space.dtype == np.float32
    assert pnp.single_observation_space["observation"].shape == (25,)
    assert pnp.action_space.shape == (3, 4)
    o, r, te, tr, inf = pnp.step(np.zeros((3, 4), dtype=np.float32))
    assert r.shape == (3,) and te.dtype == torch.bool and tr.dtype == torch.bool and "is_success" in inf
    with pytest.raises(ValueError, match="Action dimension mismatch"):  # robot_env.py:129-130
        pnp.step(np.zeros((3, 5), dtype=np.float32))


def test_initial_state_matches_oracle_and_published_value(pnp):
    orc = oracle_env_from_model("FetchPickAndPlace", pnp.model)
    assert np.allclose(pnp.initial_gripper_xpos.double().numpy(), orc.initial_gripper_xpos, atol=2e-5)
    # gripper rest position quoted by the reference's own docs/tests era (remembered public value, see DESIGN.md)
    assert np.allclose(orc.initial_gripper_xpos, [1.3419, 0.7491, 0.5347], atol=5e-4)
    assert pnp.height_offset == pytest.approx(orc.height_offset, abs=2e-6)


def test_reset_sampling_follows_the_reference_rng_stream(pnp):
    """numpy mode: env i is seeded seed+i with Generator(PCG64(SeedSequence)) and draws in the reference's order
    (fetch_env.py:386-399 then :153-166), so goals/object starts equal the oracle env's for the same seed."""
    obs, _ = pnp.reset(seed=40)
    for i in range(3):
        orc = oracle_env_from_model("FetchPickAndPlace", pnp.model)
        oo, _ = orc.reset(seed=40 + i)
        assert np.allclose(obs["desired_goal"][i].double().numpy(), oo["desired_goal"], atol=1e-6)
        assert np.allclose(obs["achieved_goal"][i].double().numpy(), oo["achieved_goal"], atol=2e-5)
        assert np.allclose(obs["observation"][i].double().numpy(), oo["observation"], atol=5e-5)
    # reset-state invariant of the reference (tests/test_envs.py:175-231): qpos == initial_qpos except object xy
    st, _ = pnp.get_state()
    q = st[:, :22]
    assert torch.equal(q[:, :15], pnp.initial_qpos[:15].expand(3, 15)) and torch.equal(q[:, 17:], pnp.initial_qpos[17:].expand(3, 5))
    assert torch.count_nonzero(st[:, 22:22 + 21] - pnp.initial_qvel) == 0


def test_same_seed_determinism():
    outs = []
    for _ in range(2):
        env = mk("FetchPush", 2, rng_mode="numpy")
        env.reset(seed=5)
        rng = np.random.default_rng(0)
        acc = []
        for _ in range(6):
            o, r, *_ = env.step(rng.uniform(-1, 1, (2, 4)).astype(np.float32))
            acc.append(torch.cat([o["observation"], o["desired_goal"], r[:, None]], 1))
        outs.append(torch.stack(acc))
    assert torch.equal(outs[0], outs[1])


def test_step_tracks_oracle_and_reward_contract(pnp):
    pnp.reset(seed=9)
    oracles = [oracle_env_from_model("FetchPickAndPlace", pnp.model) for _ in range(3)]
    for i, o in enumerate(oracles):
        o.reset(seed=9 + i)
    rng = np.random.default_rng(3)
    for _ in range(4):
        inject_oracle_state(pnp, oracles)
        a = rng.uniform(-1, 1, (3, 4)).astype(np.float32)
        o, r, te, tr, info = pnp.step(a)
        for i, orc in enumerate(oracles):
            oo, orr, _, _, oi = orc.step(a[i].astype(np.float64))
            assert np.abs(o["observation"][i].double().numpy() - oo["observation"]).max() < 2e-4
            assert float(r[i]) == float(orr)
        # GoalEnv invariant (core.py:61-62)
        assert torch.equal(pnp.compute_reward(o["achieved_goal"], o["desired_goal"], {}), r)
        rn = pnp.compute_reward(o["achieved_goal"].numpy(), o["desired_goal"].numpy(), {})
        assert rn.dtype == np.float32 and np.array_equal(rn, r.numpy())


def test_fetch_slide_tracks_oracle():
    """FetchSlide-v4 (envs/fetch/slide.py:160-190): the cylinder puck goes through the general convex collider.  A flat
    cylinder keeps rocking on its single portal contact, so its Euler angles (obs 11:14) and angular velocity (obs
    17:20) are chaotic between an fp32 and an fp64 run; everything else is compared."""
    env = mk("FetchSlide", 2, rng_mode="numpy")
    orc0 = oracle_env_from_model("FetchSlide", env.model)
    assert np.allclose(env.initial_gripper_xpos.double().numpy(), orc0.initial_gripper_xpos, atol=5e-5)
    assert env.height_offset == pytest.approx(orc0.height_offset, abs=5e-4)
    assert env.height_offset == pytest.approx(0.414, abs=2e-3)       # puck resting on the table top
    obs, _ = env.reset(seed=3)
    oracles = [oracle_env_from_model("FetchSlide", env.model) for _ in range(2)]
    keep = np.array([i for i in range(25) if not 11 <= i < 14 and not 17 <= i < 20])
    for i, o in enumerate(oracles):
        oo, _ = o.reset(seed=3 + i)
        assert np.abs(obs["desired_goal"][i].double().numpy() - oo["desired_goal"]).max() < 5e-4
        assert np.abs(obs["observation"][i].double().numpy() - oo["observation"])[keep].max() < 2e-3
        # slide.py: target_offset 0.4 in x, goal on the table
        assert oo["desired_goal"][2] == pytest.approx(o.height_offset)
    rng = np.random.default_rng(0)
    for _ in range(3):
        inject_oracle_state(env, oracles)
        a = rng.uniform(-1, 1, (2, 4)).astype(np.float32)
        o, r, *_ = env.step(a)
        for i, orc in enumerate(oracles):
            oo, orr, *_ = orc.step(a[i].astype(np.float64))
            assert np.abs(o["observation"][i].double().numpy() - oo["observation"])[keep].max() < 5e-4
            assert float(r[i]) == float(orr)


def test_free_motion_parity_outlier_is_one_ulp_away():
    """Step 0, env 7 of the free-motion phase of test_gpu_parity.py's FetchPickAndPlace step parity (fingers in contact): one ulp on
    the injected wrist-flex angle moves the emulated finger velocity (obs 23) by 2.2e-5, the error the sm_90a build shows there."""
    n = 8
    env = mk("FetchPickAndPlace", n, rng_mode="numpy")
    env.reset(seed=100)
    oracles = [oracle_env_from_model("FetchPickAndPlace", env.model) for _ in range(n)]
    for i, o in enumerate(oracles):
        o.reset(seed=100 + i)
    a = np.random.default_rng(7).uniform(-1, 1, (n, 4)).astype(np.float32)   # the parity test's first actions
    inject_oracle_state(env, oracles)
    base = env.backend.state.clone()
    want = oracles[7].step(a[7].astype(np.float64))[0]["observation"]
    o, *_ = env.step(a)
    assert np.abs(o["observation"][7].double().numpy() - want).max() < 2e-7
    slot = env.backend.layout["qpos"] + int(env.model.jnt_qposadr[env.model.joint_id("robot0:wrist_flex_joint")])
    st = base.clone()
    st[7, slot] = float(np.nextafter(np.float32(st[7, slot].item()), np.float32(-np.inf)))
    env.backend.state.copy_(st)
    o, *_ = env.step(a)
    d = np.abs(o["observation"][7].double().numpy() - want)
    assert int(d.argmax()) == 23 and 1e-5 < d.max() < 8e-5


def test_timelimit_and_next_step_autoreset():
    env = mk("FetchReach", 2, rng_mode="numpy", max_episode_steps=3)
    env.reset(seed=0)
    a = np.full((2, 4), 0.5, dtype=np.float32)
    for t in range(3):
        o, r, te, tr, info = env.step(a)
        assert not bool(te.any()) and bool(tr.all()) == (t == 2)
    moved = o["observation"].clone()
    o2, r2, te2, tr2, info2 = env.step(a)  # NEXT_STEP: this call resets, action ignored, reward 0
    assert not bool(tr2.any()) and torch.count_nonzero(r2) == 0
    assert torch.allclose(o2["observation"][:, :3], env.initial_gripper_xpos.expand(2, 3), atol=1e-4)
    assert not torch.allclose(o2["observation"], moved)
    o3, *_ = env.step(a)
    assert int(env._elapsed.max()) == 1


def test_same_step_autoreset_reports_final_obs():
    env = mk("FetchReach", 2, rng_mode="torch", autoreset_mode="same_step", max_episode_steps=2)
    env.reset(seed=0)
    a = np.full((2, 4), 1.0, dtype=np.float32)
    env.step(a)
    o, r, te, tr, info = env.step(a)
    assert bool(tr.all()) and "final_obs" in info and bool(info["_final_obs"].all())
    assert bool(info["_final_info"].all()) and info["final_info"]["is_success"].shape == (2,)
    assert not torch.allclose(info["final_obs"]["observation"], o["observation"])
    assert torch.allclose(o["observation"][:, :3], env.initial_gripper_xpos.expand(2, 3), atol=1e-4)


def test_dense_reward_and_registry():
    import gymnasium_robotics_b200 as pkg

    assert set(pkg.ENV_IDS) >= {"FetchReach-v4", "FetchPickAndPlace-v4", "FetchPickAndPlaceDense-v4", "FetchPush-v4", "FetchSlide-v4", "FetchSlideDense-v4"}
    assert pkg.ENV_IDS["FetchPickAndPlace-v4"]["max_episode_steps"] == 50  # reference __init__.py:47-52
    env = pkg.make_vec("FetchReachDense-v4", num_envs=1, backend_factory=HostSimBackend, rng_mode="numpy")
    obs, _ = env.reset(seed=2)
    o, r, *_ = env.step(np.zeros((1, 4), dtype=np.float32))
    d = torch.linalg.norm(o["achieved_goal"] - o["desired_goal"], dim=1)
    assert torch.allclose(r, -d)
    with pytest.raises(KeyError):
        pkg.make_vec("AdroitHandHammer-v1", num_envs=1)   # not on the CUDA path (and not a registered id of the reference)


def test_contact_group_overflow_is_flagged_and_harmless():
    """Regression: a geom pair beyond the per-env contact-group capacity must be dropped together with its contacts before
    they are numbered.  (Counted-but-unwritten contact records used to be finalised from stale words: garbage pair index,
    illegal address on the GPU with 2 048 Adroit envs pressing the hand onto the table.)  The capacity is shrunk to 3 groups
    (weld + 2 geom pairs) so that the gripper pressed onto the table and the object overflows it at once."""
    class TinyGroups(HostSimBackend):
        NGRP_CAP = 4

    env = FetchVectorEnv("FetchPickAndPlace", num_envs=1, backend_factory=TinyGroups, rng_mode="numpy")
    env.reset(seed=0)
    a = np.array([[0.0, 0.0, -1.0, -1.0]], dtype=np.float32)
    for _ in range(12):
        o, r, *_ = env.step(a)
        assert torch.isfinite(o["observation"]).all()
    assert env.backend.overflow_bits & 4, "the scenario was meant to overflow the group capacity"
    # the same scenario with the production capacity never flags
    env2 = mk("FetchPickAndPlace", 1, rng_mode="numpy")
    env2.reset(seed=0)
    for _ in range(12):
        env2.step(a)
    assert getattr(env2.backend, "overflow_bits", 0) == 0


def test_auto_recover_detects_and_resets_bad_states():
    """SURVEY.md section 5 failure detection ([ext] mj_checkPos / mj_checkVel: NaN or |x| > 1e10 => mj_resetData): opt-in scan of the
    state records after each step (C-ABI b200sim_check_state); a bad env goes back to its rest state and keeps its goal."""
    env = mk("FetchPickAndPlace", 4, rng_mode="numpy", auto_recover=True)
    obs, _ = env.reset(seed=3)
    goals = obs["desired_goal"].clone()
    o, r, te, tr, info = env.step(np.zeros((4, 4), dtype=np.float32))
    assert not info["bad_state"].any() and int(env.bad_state_count) == 0
    st = env.backend.state
    st[1, env._sl["qvel"].start + 3] = float("nan")
    st[2, env._sl["qpos"].start + 1] = 3e10
    o, r, te, tr, info = env.step(np.full((4, 4), 0.5, dtype=np.float32))
    assert info["bad_state"].tolist() == [False, True, True, False] and int(env.bad_state_count) == 2
    assert torch.isfinite(o["observation"]).all() and torch.isfinite(r).all()
    assert torch.equal(o["desired_goal"], goals)                               # the goal survives the recovery
    rest, _ = env._recovery
    q = env._sl["qpos"]
    assert torch.equal(st[1, q], rest[q]) and torch.equal(st[2, q], rest[q])   # back at initial_qpos / initial_qvel
    assert not torch.equal(st[0, q], rest[q])                                  # the healthy envs moved on
    o, r, te, tr, info = env.step(np.zeros((4, 4), dtype=np.float32))
    assert not info["bad_state"].any() and torch.isfinite(o["observation"]).all()


def test_auto_recover_on_other_families():
    """The scan keeps what an episode drew: the Adroit door's frame position (per-env model pose) survives a recovery."""
    import gymnasium_robotics_b200 as pkg
    from gymnasium_robotics_b200.adroit import ADROIT_REF_POINT

    class AdroitHostBackend(HostSimBackend):
        REF = ADROIT_REF_POINT

    env = pkg.make_vec("AdroitHandDoor-v2", num_envs=2, backend_factory=AdroitHostBackend, rng_mode="numpy", auto_recover=True)
    env.reset(seed=1)
    frame = env.get_env_state()["door_body_pos"].clone()
    st = env.backend.state
    st[1, env._sl["qvel"].start + 5] = float("inf")
    o, r, te, tr, info = env.step(np.zeros((2, 28), dtype=np.float32))
    assert info["bad_state"].tolist() == [False, True] and torch.isfinite(o).all()
    s = env.get_env_state()
    assert torch.equal(s["door_body_pos"], frame) and torch.equal(s["qpos"][1], env.init_qpos)


def test_torch_mode_rejection_sampling_on_fetch_slide():
    """FetchSlide's obj_range 0.1 rejects 79 % of the candidate start positions (fetch_env.py:386-392): the masked-redraw loop of the
    torch RNG mode must run long enough that no env keeps a rejected one."""
    env = mk("FetchSlide", 256, rng_mode="torch")
    env._gen.manual_seed(0)
    obj, goals = env._sample_reset(torch.arange(256))
    g0 = env.initial_gripper_xpos
    d = torch.linalg.norm(obj - g0[:2], dim=1)
    assert float(d.min()) >= 0.1 and float((obj - g0[:2]).abs().max()) <= 0.1 + 1e-6


def test_packed_row_flags_and_solver_info():
    """The step's results live in ONE packed row per env (obs | achieved | desired | reward | success | terminated | truncated,
    include/b200sim.h b200sim_set_packed) that the classic outputs are views of; TimeLimit / terminated / truncated come from
    the step itself (b200sim_set_time_limit) in every autoreset mode; info carries the solver's per-env info word."""
    env = mk("FetchPickAndPlace", 2, rng_mode="numpy", autoreset_mode="same_step", max_episode_steps=3)
    env.reset(seed=5)
    for k in range(3):
        o, r, te, tr, info = env.step(np.full((2, 4), 0.1, dtype=np.float32))
        out = env._last
        p, no = out["packed"], 25
        assert p.shape[1] % 4 == 0 and p.shape[1] >= no + 6 + 4
        # final_obs holds the pre-reset observation on the truncation step; the packed row holds what step() returned
        assert torch.equal(p[:, :no], o["observation"]) and torch.equal(p[:, no:no + 3], o["achieved_goal"]) and torch.equal(p[:, no + 3:no + 6], o["desired_goal"])
        assert torch.equal(p[:, no + 6], r) and torch.equal(p[:, no + 8] > 0, te) and torch.equal(p[:, no + 9] > 0, tr)
        assert bool(tr.all()) == (k == 2) and not bool(te.any())
        assert info["solver_info"].shape == (2,) and int((info["solver_info"] & 0xffff).min()) >= 0
    assert "final_obs" in info and int(env._elapsed.max()) == 0   # same-step autoreset zeroed the library's step counters
    assert env.solver_overflow_count == 0
    env.close()
    # NEXT_STEP: the call after a truncation resets instead of stepping and reports neutral results for those envs
    env = mk("FetchReach", 2, rng_mode="numpy", autoreset_mode="next_step", max_episode_steps=2)
    env.reset(seed=5)
    env.step(np.zeros((2, 4), dtype=np.float32))
    _, _, _, tr, _ = env.step(np.zeros((2, 4), dtype=np.float32))
    assert bool(tr.all())
    o, r, te, tr, info = env.step(np.ones((2, 4), dtype=np.float32))
    assert not bool(tr.any()) and float(r.abs().max()) == 0.0 and float(info["is_success"].max()) == 0.0 and int(env._elapsed.max()) == 0
    assert float(env._last["packed"][:, 10 + 6:10 + 10].abs().max()) == 0.0
    env.close()


def test_register_envs_against_a_gymnasium_stub(monkeypatch):
    """`register_envs()` (gymnasium is absent from this image): executed against a stub of `gymnasium.envs.registration` -- every
    id of the reference's registry that the CUDA path provides is registered once with a `vector_entry_point` that resolves to a
    constructor of this package and kwargs that constructor accepts (checked by building two of them on the host emulation)."""
    import importlib
    import sys
    import types

    import gymnasium_robotics_b200 as pkg

    calls, registry = [], {}
    gym = types.ModuleType("gymnasium")
    envs = types.ModuleType("gymnasium.envs")
    reg = types.ModuleType("gymnasium.envs.registration")

    def register(id, vector_entry_point=None, kwargs=None, **kw):
        calls.append((id, vector_entry_point, dict(kwargs or {})))
        registry[id] = vector_entry_point

    reg.register, reg.registry = register, registry
    gym.envs, envs.registration = envs, reg
    for name, mod in (("gymnasium", gym), ("gymnasium.envs", envs), ("gymnasium.envs.registration", reg)):
        monkeypatch.setitem(sys.modules, name, mod)
    assert pkg.register_envs() is True
    ids = [c[0] for c in calls]
    assert len(ids) == len(set(ids)) == len(pkg.ENV_IDS)
    assert {"FetchPickAndPlace-v4", "AntMaze_Large-v5", "HandManipulateBlockRotateXYZ_ContinuousTouchSensors-v1", "AdroitHandHammer-v2",
            "FrankaKitchen-v1", "PointMaze_UMaze-v3"} <= set(ids)
    n0 = len(calls)
    assert pkg.register_envs() is True and len(calls) == n0           # idempotent: ids already in the registry are skipped
    by_id = {c[0]: c for c in calls}
    for env_id in ids:                                                # every entry point resolves
        mod, attr = by_id[env_id][1].split(":")
        assert callable(getattr(importlib.import_module(mod), attr)), env_id
    # gymnasium.make_vec(id, num_envs=N, vectorization_mode="vector_entry_point") calls entry_point(num_envs=N, **kwargs)
    for env_id in ("FetchReach-v4", "AntMaze_UMaze-v4"):
        mod, attr = by_id[env_id][1].split(":")
        env = getattr(importlib.import_module(mod), attr)(num_envs=2, backend_factory=HostSimBackend, rng_mode="numpy", **by_id[env_id][2])
        obs, _ = env.reset(seed=0)
        assert obs["observation"].shape[0] == 2 and env.max_episode_steps == pkg.ENV_IDS[env_id]["max_episode_steps"]
        env.close()
