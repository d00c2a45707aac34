"""In-kernel reset draws (csrc/reset_sample.cuh, C-ABI b200sim_reset; SURVEY.md 8f row 1) on CPU: the Philox4x32-10 rounds against
the published known answers, the draw logic against a pure-Python restatement of fetch_env.py:386-399 / :153-166 on the same
random numbers, the distributions, and the vector env in rng_mode="device" on the host emulation backend."""
import ctypes

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200._lib import FetchResetC
from tests import hostsim
from tests.hostsim_backend import HostSimBackend

M32 = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Salmon et al. 2011, written independently of the C code (python ints)."""
    c, k = list(ctr), list(key)
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & M32, p1 & M32, ((p0 >> 32) ^ c[3] ^ k[1]) & M32, p0 & M32]
        k = [(k[0] + 0x9E3779B9) & M32, (k[1] + 0xBB67AE85) & M32]
    return c


def c_philox(ctr, key):
    L = hostsim.lib()
    a, b, o = (ctypes.c_uint32 * 4)(*ctr), (ctypes.c_uint32 * 2)(*key), (ctypes.c_uint32 * 4)()
    L.hostsim_philox4x32_10(a, b, o)
    return list(o)


def test_philox_known_answers():
    """Random123 kat_vectors, philox4x32 10 rounds."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((M32, M32, M32, M32), (M32, M32), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert tuple(philox4x32_10(ctr, key)) == want
        assert tuple(c_philox(ctr, key)) == want
    rng = np.random.default_rng(0)
    for _ in range(200):
        ctr, key = [int(x) for x in rng.integers(0, 2 ** 32, 4)], [int(x) for x in rng.integers(0, 2 ** 32, 2)]
        assert c_philox(ctr, key) == philox4x32_10(ctr, key)


def u01(x):
    return np.float32(x >> 8) * np.float32(1.0 / 16777216.0)


def py_fetch_draw(p, seed, env, episode):
    """fetch_env.py:386-392 and :153-166 on the generator's numbers, float32 like the kernel."""
    f = np.float32
    key = (seed & M32, (seed >> 32) & M32)
    g0 = np.array(list(p.gripper_xpos), dtype=f)
    xy = np.zeros(2, dtype=f)
    if p.has_object:
        done = False
        for b in range(64):
            r = philox4x32_10((env, episode, b, 0x5EED), key)
            for h in range(2):
                d = np.array([(f(2) * u01(r[2 * h]) - f(1)) * f(p.obj_range), (f(2) * u01(r[2 * h + 1]) - f(1)) * f(p.obj_range)], dtype=f)
                xy = g0[:2] + d
                if np.sqrt(d[0] * d[0] + d[1] * d[1]) >= f(0.1):
                    done = True
                    break
            if done:
                break
    r = philox4x32_10((env, episode, 64, 0x5EED), key)
    goal = np.array([g0[k] + (f(2) * u01(r[k]) - f(1)) * f(p.target_range) for k in range(3)], dtype=f)
    if p.has_object:
        goal = goal + np.array(list(p.target_offset), dtype=f)
        goal[2] = f(p.height_offset)
        if p.target_in_the_air and u01(r[3]) < f(0.5):
            r2 = philox4x32_10((env, episode, 65, 0x5EED), key)
            goal[2] += u01(r2[0]) * f(0.45)
    return xy, goal


def c_fetch_record(p, seed, env, episode, rest, st_qpos, st_goal):
    L = hostsim.lib()
    rec = np.zeros_like(rest)
    L.hostsim_fetch_reset_record(ctypes.byref(p), seed, env, episode, rest.ctypes.data, len(rest), st_qpos, st_goal, rec.ctypes.data)
    return rec


def params(has_object=True, air=True, obj_range=0.15, target_range=0.15, offset=(0.0, 0.0, 0.0)):
    p = FetchResetC()
    p.has_object, p.target_in_the_air, p.obj_qadr = int(has_object), int(air), 15
    p.obj_range, p.target_range, p.height_offset = obj_range, target_range, 0.42
    for k in range(3):
        p.target_offset[k] = offset[k]
        p.gripper_xpos[k] = (1.34, 0.75, 0.53)[k]
    return p


@pytest.mark.parametrize("cfg", [dict(), dict(air=False, obj_range=0.1, target_range=0.3, offset=(0.4, 0.0, 0.0)), dict(has_object=False)])
def test_draw_matches_the_python_restatement_and_the_reference_distributions(cfg):
    p = params(**cfg)
    rest = np.arange(60, dtype=np.float32)
    g0 = np.array(list(p.gripper_xpos))
    xs, gs = [], []
    for env in range(400):
        rec = c_fetch_record(p, 0x1234567890ABCDEF, env, env % 3, rest, 0, 56)
        xy, goal = py_fetch_draw(p, 0x1234567890ABCDEF, env, env % 3)
        assert np.array_equal(rec[56:59], goal)
        untouched = np.ones(60, dtype=bool)
        untouched[56:59] = False
        if p.has_object:
            assert np.array_equal(rec[15:17], xy)
            untouched[15:17] = False
        assert np.array_equal(rec[untouched], rest[untouched])      # everything else is the rest record
        xs.append(rec[15:17].astype(np.float64)); gs.append(rec[56:59].astype(np.float64))
    xs, gs = np.array(xs), np.array(gs)
    off = np.array(list(p.target_offset))
    if p.has_object:
        d = np.linalg.norm(xs - g0[:2], axis=1)
        assert d.min() >= 0.1 - 1e-6 and np.abs(xs - g0[:2]).max() <= p.obj_range + 1e-6      # fetch_env.py:386-392
        assert np.abs(gs[:, :2] - g0[:2] - off[:2]).max() <= p.target_range + 1e-6
        lifted = gs[:, 2] > p.height_offset + 1e-9
        if p.target_in_the_air:
            assert 0.4 < lifted.mean() < 0.6 and gs[:, 2].max() <= p.height_offset + 0.45       # :160-161
        else:
            assert not lifted.any()
        assert abs(np.mean(gs[:, 0] - g0[0] - off[0])) < 4 * p.target_range / np.sqrt(3 * 400)
    else:
        assert np.abs(gs - g0).max() <= p.target_range + 1e-6 and gs[:, 2].std() > 0.02


def mk(task, n, **kw):
    kw.setdefault("rng_mode", "device")
    return pkg.make_vec(task, num_envs=n, backend_factory=HostSimBackend, **kw)


def test_vector_env_with_in_kernel_resets():
    env = mk("FetchPickAndPlace-v4", 4, max_episode_steps=3)
    o1, _ = env.reset(seed=7)
    g0 = env.initial_gripper_xpos.numpy()
    st, _ = env.get_state()
    q = st[:, :22]
    # reset-state invariant (reference tests/test_envs.py:175-231): qpos == initial_qpos except the object's xy
    assert torch.equal(q[:, :15], env.initial_qpos[:15].expand(4, 15)) and torch.equal(q[:, 17:], env.initial_qpos[17:].expand(4, 5))
    assert (np.linalg.norm(q[:, 15:17].numpy() - g0[:2], axis=1) >= 0.1 - 1e-6).all()
    assert len({tuple(r) for r in o1["desired_goal"].numpy().round(6).tolist()}) == 4          # every env its own stream
    env2 = mk("FetchPickAndPlace-v4", 4, max_episode_steps=3)
    o2, _ = env2.reset(seed=7)
    assert torch.equal(o1["desired_goal"], o2["desired_goal"]) and torch.equal(o1["observation"], o2["observation"])
    o3, _ = env2.reset(seed=8)
    assert not torch.equal(o1["desired_goal"], o3["desired_goal"])
    # next-step autoreset: new goals for the next episode, drawn from the episode counter
    goals = [o1["desired_goal"].clone()]
    for k in range(8):
        o, r, te, tr, info = env.step(np.zeros((4, 4), dtype=np.float32))
        if k in (3, 7):      # the call after a truncation is the reset call
            goals.append(o["desired_goal"].clone())
    assert not torch.equal(goals[0], goals[1]) and not torch.equal(goals[1], goals[2])
    assert int(env._episode.min()) == 3 and int(env._episode.max()) == 3
    # a shard that starts at global env 2 draws what envs 2, 3 of the big batch drew
    shard = mk("FetchPickAndPlace-v4", 2, env_offset=2)
    os_, _ = shard.reset(seed=7)
    assert torch.equal(os_["desired_goal"], o1["desired_goal"][2:])
    with pytest.raises(ValueError):
        mk("FetchReach-v4", 1, rng_mode="philox")


def test_reach_has_no_object_draw():
    env = mk("FetchReach-v4", 3)
    o, _ = env.reset(seed=1)
    g0 = env.initial_gripper_xpos.numpy()
    assert np.abs(o["desired_goal"].numpy() - g0).max() <= 0.15 + 1e-6
    st, _ = env.get_state()
    assert torch.equal(st[:, :15], env.initial_qpos.expand(3, 15))


def test_uniform_slot_reset_against_python():
    """b200sim_reset_uniform's record: slot k <- lo + (hi - lo) * u, u = word k % 4 of Philox block k / 4."""
    from gymnasium_robotics_b200._lib import UniformResetC

    L = hostsim.lib()
    p = UniformResetC()
    slots, lo, hi = [3, 40, 41, 7, 12, 13], [-0.15, -0.15, -0.2, 0.1, 0.0, 5.0], [0.15, 0.3, 0.2, 0.25, 1.0, 5.0]
    p.n, p.quat_slot = 6, -1
    for k in range(6):
        p.slot[k], p.lo[k], p.hi[k] = slots[k], lo[k], hi[k]
    rest = np.arange(48, dtype=np.float32)
    seed = 99
    vals = []
    for env in range(300):
        rec = np.zeros_like(rest)
        L.hostsim_uniform_reset_record(ctypes.byref(p), seed, env, 2, rest.ctypes.data, 48, rec.ctypes.data)
        f = np.float32
        for k in range(6):
            r = philox4x32_10((env, 2, k // 4, 0x0A11), (seed, 0))
            want = f(lo[k]) + (f(hi[k]) - f(lo[k])) * u01(r[k % 4])
            assert rec[slots[k]] == want
        keep = np.ones(48, dtype=bool)
        keep[slots] = False
        assert np.array_equal(rec[keep], rest[keep])
        vals.append(rec[slots])
    vals = np.array(vals)
    assert (vals >= np.array(lo, dtype=np.float32) - 1e-7).all() and (vals <= np.array(hi, dtype=np.float32) + 1e-7).all()
    assert abs(vals[:, 0].mean()) < 0.03 and (vals[:, 5] == 5.0).all()


def test_adroit_door_env_with_in_kernel_resets():
    """adroit_door.py:359-371: the frame position is three uniform draws per episode; everything else is the model's rest state."""
    env = pkg.make_vec("AdroitHandDoor-v2", num_envs=3, backend_factory=HostSimBackend, rng_mode="device", max_episode_steps=2)
    o, _ = env.reset(seed=5)
    s = env.get_env_state()
    pos = s["door_body_pos"].numpy()
    assert ((pos >= [-0.3, 0.25, 0.252]) & (pos <= [-0.2, 0.35, 0.35])).all() and len({tuple(r) for r in pos.round(6).tolist()}) == 3
    assert torch.equal(s["qpos"], env.init_qpos.expand(3, -1)) and torch.count_nonzero(s["qvel"]) == 0
    env2 = pkg.make_vec("AdroitHandDoor-v2", num_envs=3, backend_factory=HostSimBackend, rng_mode="device")
    o2, _ = env2.reset(seed=5)
    assert torch.equal(o, o2)
    for _ in range(3):     # TimeLimit 2: the third call is the next-step reset with new draws
        o, *_ = env.step(np.zeros((3, 28), dtype=np.float32))
    assert not np.array_equal(env.get_env_state()["door_body_pos"].numpy(), pos)
    # the Pen's target orientation: euler2quat of two draws (adroit_pen.py:379-384), against utils/rotations.py's restatement
    from gymnasium_robotics_b200 import rotations

    pen = pkg.make_vec("AdroitHandPen-v2", num_envs=4, backend_factory=HostSimBackend, rng_mode="device")
    pen.reset(seed=9)
    quat = pen.get_env_state()["desired_orien"].numpy()
    for i in range(4):
        r = philox4x32_10((i, 0, 0, 0x0A11), (9, 0))
        e = [float(np.float32(-1) + np.float32(2) * u01(r[0])), float(np.float32(-1) + np.float32(2) * u01(r[1])), 0.0]
        assert np.abs(quat[i] - rotations.euler2quat(np.array(e))).max() < 1e-6
    assert abs(np.linalg.norm(quat, axis=1) - 1).max() < 1e-6


def py_maze_draw(goal_xy, reset_xy, scaling, noise, seed, env, episode):
    """maze_v4.py:256-297 + :360-373 on the generator's numbers (float32 like the kernel)."""
    f = np.float32
    key = (seed & M32, (seed >> 32) & M32)
    amp = f(noise) * f(scaling)
    r = philox4x32_10((env, episode, 0, 0x3A2E), key)
    gi = (r[0] * len(goal_xy)) >> 32
    goal = np.array([goal_xy[gi][0] + (f(2) * u01(r[1]) - f(1)) * amp, goal_xy[gi][1] + (f(2) * u01(r[2]) - f(1)) * amp], dtype=f)
    pos, done = goal.copy(), False
    for b in range(1, 33):
        r = philox4x32_10((env, episode, b, 0x3A2E), key)
        for h in range(4):
            ri = (r[h] * len(reset_xy)) >> 32
            pos = np.array(reset_xy[ri], dtype=f)
            d = pos - goal
            if not (np.sqrt(d[0] * d[0] + d[1] * d[1]) <= f(0.5) * f(scaling)):
                done = True
                break
        if done:
            break
    r = philox4x32_10((env, episode, 33, 0x3A2E), key)
    pos = np.array([pos[0] + (f(2) * u01(r[0]) - f(1)) * amp, pos[1] + (f(2) * u01(r[1]) - f(1)) * amp], dtype=f)
    return goal, pos


def test_maze_env_with_in_kernel_resets():
    env = pkg.make_vec("AntMaze_Medium_Diverse_GR-v5", num_envs=6, backend_factory=HostSimBackend, rng_mode="device", max_episode_steps=2)
    o, _ = env.reset(seed=21)
    goal_xy, reset_xy = env._goal_loc.numpy(), env._reset_loc.numpy()
    assert len(goal_xy) >= 2 and len(reset_xy) >= 2            # the _GR maps mark goal and reset cells (maps.py)
    st, _ = env.get_state()
    for i in range(6):
        g, p = py_maze_draw(goal_xy, reset_xy, env.scaling, 0.25, 21, i, 0)
        assert np.array_equal(o["desired_goal"][i].numpy(), g) and np.array_equal(st[i, :2].numpy(), p)
        # the goal is within the noise box of a goal cell, the start within that of a reset cell farther than half a cell away
        assert (np.abs(goal_xy - g).max(axis=1) <= 0.25 * env.scaling + 1e-6).any()
        assert (np.abs(reset_xy - p).max(axis=1) <= 0.25 * env.scaling + 1e-6).any()
        assert not env.cells.is_wall_xy(p) if hasattr(env.cells, "is_wall_xy") else True
    assert torch.equal(st[:, 2:15], env.init_qpos[2:].expand(6, 13))
    g0 = o["desired_goal"].clone()
    for _ in range(3):
        o, *_ = env.step(np.zeros((6, 8), dtype=np.float32))
    assert not torch.equal(o["desired_goal"], g0) and int(env._episode.min()) == 2
    # explicit cells keep the host path (maze_v4.py:313-350)
    o, _ = env.reset(seed=1, options={"goal_cell": np.array([1, 1]), "reset_cell": np.array([1, 2])})
    assert np.abs(o["desired_goal"].numpy() - env.cells.cell_rowcol_to_xy(np.array([1, 1]))).max() <= 0.25 * env.scaling + 1e-6
    pm = pkg.make_vec("PointMaze_UMaze-v3", num_envs=2, backend_factory=HostSimBackend, rng_mode="device")
    o, _ = pm.reset(seed=3)
    st, _ = pm.get_state()
    for i in range(2):
        g, p = py_maze_draw(pm._goal_loc.numpy(), pm._reset_loc.numpy(), pm.scaling, 0.25, 3, i, 0)
        assert np.array_equal(o["desired_goal"][i].numpy(), g) and np.array_equal(st[i, :2].numpy(), p)


def test_hand_env_with_in_kernel_resets():
    """manipulate.py:154-279 in rng_mode="device": start pose (z-rotation / parallel / xyz offset, position noise), settle with the
    on-palm retry, goal from the settled pose -- checked against the reference's formulas on the same Philox numbers."""
    from gymnasium_robotics_b200 import rotations
    from gymnasium_robotics_b200.hand import TARGET_POSITION_RANGE

    f = np.float32
    for env_id, rot in (("HandManipulateBlockRotateZ-v1", "z"), ("HandManipulateBlockRotateParallel-v1", "parallel"),
                        ("HandManipulateBlockFull-v1", "xyz")):
        env = pkg.make_vec(env_id, num_envs=2, backend_factory=HostSimBackend, rng_mode="device")
        o, _ = env.reset(seed=13)
        assert env.reset_attempts >= 1 and int(env._episode.min()) == 1
        st, _ = env.get_state()
        obj = st[:, env._obj].numpy()
        goal = o["desired_goal"].numpy()
        assert (obj[:, 2] > 0.04).all() and np.abs(np.linalg.norm(goal[:, 3:], axis=1) - 1).max() < 1e-6
        par = np.array(rotations.parallel_quats())
        for i in range(2):
            key = (13, 0)
            r, r2, r3 = (philox4x32_10((i, 0, 0x400 + b, 0x4A2D), key) for b in range(3))
            angle = float((f(2) * u01(r[0]) - f(1)) * f(np.pi))
            if rot == "z":
                want = rotations.quat_from_angle_and_axis(angle, np.array([0.0, 0.0, 1.0]))
            elif rot == "parallel":
                zq = rotations.quat_from_angle_and_axis(angle, np.array([0.0, 0.0, 1.0]))
                want = rotations.quat_mul(zq, par[(r[1] * 24) >> 32])
            else:
                axis = np.array([float(f(2) * u01(r2[k]) - f(1)) for k in range(3)])
                want = rotations.quat_from_angle_and_axis(angle, axis)
            assert np.abs(goal[i, 3:] - want / np.linalg.norm(want)).max() < 2e-6, (env_id, i)
            if env.target_position == "random":
                off = np.array([TARGET_POSITION_RANGE[k, 0] + (TARGET_POSITION_RANGE[k, 1] - TARGET_POSITION_RANGE[k, 0]) * float(u01(r3[k]))
                                for k in range(3)])
                assert np.abs(goal[i, :3] - (obj[i, :3] + off)).max() < 2e-6
            else:
                assert np.abs(goal[i, :3] - obj[i, :3]).max() < 1e-7          # "ignore": the goal position is the settled object's
        env2 = pkg.make_vec(env_id, num_envs=2, backend_factory=HostSimBackend, rng_mode="device")
        o2, _ = env2.reset(seed=13)
        assert torch.equal(o["observation"], o2["observation"]) and torch.equal(o["desired_goal"], o2["desired_goal"])


def test_hand_start_pose_draw():
    """One attempt's pose record against the reference's formulas: initial quat * offset, += N(0, 0.005^2) (Box-Muller)."""
    from gymnasium_robotics_b200 import rotations
    from gymnasium_robotics_b200._lib import HandResetC

    L = hostsim.lib()
    par = np.array(rotations.parallel_quats(), dtype=np.float32)
    p = HandResetC()
    p.obj_qadr, p.randomize_rotation, p.randomize_position = 24, 1, 1
    rest = np.zeros(100, dtype=np.float32)
    q0 = np.array([0.3, -0.5, 0.4, 0.7]); q0 /= np.linalg.norm(q0)
    rest[24:27], rest[27:31] = [1.0, 0.87, 0.2], q0
    f = np.float32
    pos = []
    for mode in (1, 2, 3):
        p.rot_mode = mode
        for env in range(60):
            rec = np.full(100, 7.0, dtype=np.float32)
            rec[90:97] = np.arange(7)                                       # the goal must survive
            L.hostsim_hand_pose_record(ctypes.byref(p), par.ctypes.data, 5, env, 1, 2, rest.ctypes.data, 100, 0, 90, 7, rec.ctypes.data)
            assert np.array_equal(rec[90:97], np.arange(7, dtype=np.float32)) and np.array_equal(rec[:24], rest[:24])
            r, r2, r3 = (philox4x32_10((env, 1, 8 + b, 0x4A2D), (5, 0)) for b in range(3))
            angle = float((f(2) * u01(r[0]) - f(1)) * f(np.pi))
            if mode == 1:
                off = rotations.quat_from_angle_and_axis(angle, np.array([0.0, 0.0, 1.0]))
            elif mode == 2:
                off = rotations.quat_mul(rotations.quat_from_angle_and_axis(angle, np.array([0.0, 0.0, 1.0])), par[(r[1] * 24) >> 32].astype(np.float64))
            else:
                off = rotations.quat_from_angle_and_axis(angle, np.array([float(f(2) * u01(r2[k]) - f(1)) for k in range(3)]))
            want = rotations.quat_mul(rest[27:31].astype(np.float64), off)
            assert np.abs(rec[27:31] - want / np.linalg.norm(want)).max() < 2e-6
            u1, u2, u3, u4 = 1 - float(u01(r3[0])), float(u01(r3[1])), 1 - float(u01(r3[2])), float(u01(r3[3]))
            n = 0.005 * np.array([np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * u2), np.sqrt(-2 * np.log(u1)) * np.sin(2 * np.pi * u2),
                                  np.sqrt(-2 * np.log(u3)) * np.cos(2 * np.pi * u4)])
            assert np.abs(rec[24:27] - (rest[24:27] + n)).max() < 1e-6
            pos.append(rec[24:27] - rest[24:27])
    pos = np.array(pos)
    assert 0.003 < pos.std() < 0.007 and abs(pos.mean()) < 0.002          # manipulate.py:200-202: scale 0.005


def test_hand_reach_goal_draw():
    """reach.py:95-121 on the generator's numbers: thumb + one of four fingers meet near the palm; 10 % keep the initial tips."""
    env = pkg.make_vec("HandReach-v3", num_envs=40, backend_factory=HostSimBackend, rng_mode="device")
    o, _ = env.reset(seed=6)
    goals = o["desired_goal"].numpy().reshape(40, 5, 3)
    init = env.initial_goal.numpy().reshape(5, 3)
    meeting0 = env.palm_xpos + np.array([0.0, -0.09, 0.05])
    f = np.float32
    kept = 0
    for i in range(40):
        r = philox4x32_10((i, 0, 0, 0x2EAC4), (6, 0))
        r2 = philox4x32_10((i, 0, 1, 0x2EAC4), (6, 0))
        if u01(r[1]) < f(0.1):
            assert np.array_equal(goals[i], init)
            kept += 1
            continue
        u1, u2, u3, u4 = 1 - float(u01(r2[0])), float(u01(r2[1])), 1 - float(u01(r2[2])), float(u01(r2[3]))
        meet = meeting0 + 0.005 * np.array([np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * u2), np.sqrt(-2 * np.log(u1)) * np.sin(2 * np.pi * u2),
                                            np.sqrt(-2 * np.log(u3)) * np.cos(2 * np.pi * u4)])
        finger = (r[0] * 4) >> 32
        want = init.astype(np.float64).copy()
        for j in (4, finger):
            d = meet - want[j]
            want[j] = meet - 0.005 * d / np.linalg.norm(d)
        assert np.abs(goals[i] - want).max() < 1e-6, i
    assert kept <= 12
    st, _ = env.get_state()
    assert torch.equal(st[:, env._sl["qpos"]], env.initial_qpos.expand(40, -1))
