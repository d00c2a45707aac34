"""The step kernel's task layer (csrc/fetch_task.cuh) on its own, against the fp64 oracle at injected states: what the kernel does
before the first sub-step (the action map) and after the last (observations, goals, rewards, success flags, touch sensors).

Every check runs on the product kernels through the C-ABI (GPU) and on the 32-lane emulation of the build b200sim_create picks
(tests/hostsim `warp`, `warp_wide`).  States are fp32 records; the oracle always runs at those fp32 values.  u = 2^-24, L = the
largest |body position| of the case (at least 1).

1. Refresh (b200sim_refresh: mj_forward + _get_obs) at injected states, every family in its sparse and its dense variant: FetchReach /
   Push / Slide / PickAndPlace, HandReach, HandManipulateBlock / Egg / PenRotate (ignore_z_target_rotation), the four Adroit tasks,
   PointMaze and AntMaze.  States: the oracle's reset state; random joint positions within the ranges with large velocities (free
   bodies spun at 60 rad/s, other dofs ~N(0, 3)) and object orientations uniform on SO(3), w < 0 included; Fetch objects at pitch
   +-pi/2 + {0, 1e-4, 1e-2}; goals at threshold x (1 +- 1e-3) and at exactly 0 distance of the kernel's own achieved goal; for Fetch a
   goal whose fp32 distance IS the threshold; for the Adroit tasks states that put each dense-reward step on each side of its
   threshold.  Compared:
     * entries that copy qpos / qvel (and the Adroit clipped velocities, the door's open flag): bit for bit;
     * positions, relative positions, the Adroit pen's directions: normwise in units of u L (directions u L / length);
     * dt-scaled site velocities: in units of u (|Jp| |qvel| + L |Jr| |qvel|) dt;
     * Euler angles (Fetch object, Adroit hammer): x and z in units of u L / cy, cy = the fp64 sqrt(m22^2 + m12^2) (printed per
       sample, and near gimbal lock the kernel's angles next to the fp64 ones), the pitch in units of u L at any cy;
     * sparse rewards and success flags: equal to the fp64 decision wherever every quantity the rule compares is more than NEAR u
       (its scale) from its threshold; dense rewards there within u times the magnitudes of their terms (the Hand's 2 acos(w) with
       its sensitivity 2 / sqrt(1 - w^2), floored where acos(1 - d) ~ sqrt(2 d) takes over);
     * at the kernel's own fp32 distance (the dense variant's reward is -d bit for bit): the sparse reward -(d > thr) and the
       success flag d < thr, on both sides of the threshold and exactly on it.
   Every compared output must be finite; a NaN error fails its bound.  Not compared: the hammer's touch entry (obs[45]; part 3), the Ant's contact forces (tests/test_ant_info_gpu.py).
2. The action map: one step from an injected state, the stored ctrl and Fetch mocap against the reference's _set_action at the
   pre-step state, for actions uniform in [-3, 3], exactly +-1 and 0, and +-inf in single entries: Hand / Adroit ctrl =
   clip(centre + clip(a) half, lo, hi) within 2 u of the magnitudes and never outside [lo, hi]; Fetch mocap = pose slot + 0.05
   clip(a[:3]) and pose quaternion + (1, 0, 1, 0), finger ctrl = qpos + clip(a[3]) (+ 0 exactly under block_gripper); Ant ctrl == a
   and Point ctrl == clip(a) bit for bit.  Under block_gripper the stored finger qpos are exactly 0 and the step's observation equals
   the refresh observation of the record it stored, bit for bit.
3. Touch sensors alone (tests/devsim STAGE_TOUCH, tests/hostsim touch): touch_observe over the contact records the problem stage
   left (the forces of the warm-start qacc), against an fp64 restatement of oracle.c `sensors()` over the same records, with the
   oracle's site pose at the same qpos: the Hand's sphere and box sites, the hammer's cylinder, at the contact-heavy and random
   states of tests/test_device_problem_gpu.py and at records edited in place (points on, inside and outside each site's surface,
   rays parallel to a box face and to the cylinder axis, rays starting inside or pointing away, the sensor's body as geom2, a world
   geom as the other geom, zero and negative normal force, sensors 32 and up).  A contact whose fp64 hit decision flips under a perturbation of NEAR u L of its point
   or NEAR u of its direction may count either way; every sensor's sum is within u sum |F| of the fp64 sum.  The Boolean touch ids
   report exactly continuous > 0 at the same states.  `ray_hits_site` also runs on its own on site-frame rays (devsim / hostsim
   ray_hits), so that rays exactly along an axis reach the parallel branches a rotated site never gives.  No committed touch model has
   a contact pair with a world geom (g2 < 0): one pair per site type gets g2 = -1 in the model words the harness runs.

Limits are about 4-5x the largest values measured on an H100 80GB HBM3 (700 W) and on the 32-lane emulation (DESIGN.md section 2),
largest over all families, H100 / emulation: positions 2.90 / 2.90 u L, velocities 1.75 / 2.21, Euler angles 1.19 / 1.22,
directions 0.99 / 0.99, dense rewards 2.66 / 2.76; ctrl 0.76 / 0.76 u and mocap 0.59 / 0.59 u (held to the 2 u the action map
allows); touch sums 0.54 / 0.24 u sum |F|.
"""
import copy

import numpy as np
import pytest
import torch

U = 2.0 ** -24
NEAR = 64.0   # decision margin, units of u times the scale of the compared quantity
# limits: 4-5x the largest values measured over all cases (DESIGN.md section 2)
LIM = {"pos": 12.0, "vel": 10.0, "euler": 5.0, "dir": 4.0, "dense": 12.0, "ctrl": 2.0, "mocap": 2.0, "touch": 2.5}
WARP = {False: "warp", True: "warp_wide"}

# (family, sparse id, dense id)
IDS = [("fetch", "FetchReach-v4", "FetchReachDense-v4"), ("fetch", "FetchPush-v4", "FetchPushDense-v4"),
       ("fetch", "FetchSlide-v4", "FetchSlideDense-v4"), ("fetch", "FetchPickAndPlace-v4", "FetchPickAndPlaceDense-v4"),
       ("reach", "HandReach-v3", "HandReachDense-v3"), ("hand", "HandManipulateBlock-v1", "HandManipulateBlockDense-v1"),
       ("hand", "HandManipulateEgg-v1", "HandManipulateEggDense-v1"), ("hand", "HandManipulatePenRotate-v1", "HandManipulatePenRotateDense-v1"),
       ("hammer", "AdroitHandHammerSparse-v2", "AdroitHandHammer-v2"), ("relocate", "AdroitHandRelocateSparse-v2", "AdroitHandRelocate-v2"),
       ("pen", "AdroitHandPenSparse-v2", "AdroitHandPen-v2"), ("door", "AdroitHandDoorSparse-v2", "AdroitHandDoor-v2"),
       ("point", "PointMaze_UMaze-v3", "PointMaze_UMazeDense-v3"), ("ant", "AntMaze_UMaze-v5", "AntMaze_UMazeDense-v5")]


# ------------------------------------------------------------------------------------------------ backends
def _spec(env_id, backend):
    """(model, eq_data, task, env attributes) of an id as its vector env builds them."""
    import gymnasium_robotics_b200 as pkg

    if env_id.startswith("Fetch"):   # (the Fetch env's constructor settles its envs: built from its parts instead)
        from gymnasium_robotics_b200.fetch import FETCH_TASKS, make_task_struct, welded_eq_data
        from gymnasium_robotics_b200.models import load_model

        cfg = FETCH_TASKS[pkg.ENV_IDS[env_id]["task"]]
        m = load_model(cfg["model"])
        return m, welded_eq_data(m), make_task_struct(m, cfg, pkg.ENV_IDS[env_id]["reward_type"]), cfg
    got = {}

    def capture(model, eq, task, n, device):
        got.update(model=model, eq=eq, task=task)
        return _new_backend(backend, model, eq, task, n)
    env = pkg.make_vec(env_id, num_envs=1, backend_factory=capture, rng_mode="numpy", device="cuda:0" if backend == "gpu" else "cpu")
    attrs = {k: getattr(env, k) for k in ("target_position", "target_rotation", "distance_threshold", "rotation_threshold",
                                          "ignore_z_target_rotation", "reward_type") if hasattr(env, k)}
    env.close()
    return got["model"], got["eq"], got["task"], attrs


def _new_backend(backend, model, eq, task, n):
    if backend == "gpu":
        from gymnasium_robotics_b200.fetch import CudaBackend

        return CudaBackend(model, eq, task, n, "cuda:0")
    from tests.hostsim import host_flavor
    from tests.hostsim_backend import HostSimBackend

    return HostSimBackend(model, eq, task, n, "cpu", flavor=WARP[host_flavor(model, task)])


def _launch(be, recs, actions=None):
    """Refresh (actions None) or step of the records [n, stride]: (outputs as float64 numpy, records after the launch)."""
    dev = be.device
    be.state.copy_(torch.as_tensor(np.asarray(recs, np.float32), device=dev))
    out = be.new_outputs()
    if actions is None:
        be.refresh(None, out)
    else:
        be.step(torch.as_tensor(np.asarray(actions, np.float32), device=dev).contiguous(), out)
    o = {k: out[k].double().cpu().numpy() for k in ("obs", "achieved", "desired", "reward", "success")}
    o["obs32"] = out["obs"].cpu().numpy().copy()
    return o, be.state.cpu().numpy().copy()


# ------------------------------------------------------------------------------------------------ the families' oracles
def _oracle(fam, env_id, model, attrs, reward_type):
    if fam == "fetch":
        from oracle.fetch_env import OracleFetchEnv

        return OracleFetchEnv(env_id.split("-")[0].replace("Dense", ""), reward_type=reward_type, model=model)
    if fam == "reach":
        from oracle.hand_env import OracleHandReachEnv

        return OracleHandReachEnv(reward_type=reward_type, model=model)
    if fam == "hand":
        from oracle.hand_env import OracleHandBlockEnv

        return OracleHandBlockEnv(model=model, reward_type=reward_type, **{k: v for k, v in attrs.items() if k != "reward_type"})
    if fam in ("hammer", "relocate", "pen", "door"):
        from oracle import adroit_env

        cls = {"hammer": adroit_env.OracleAdroitHammerEnv, "relocate": adroit_env.OracleAdroitRelocateEnv,
               "pen": adroit_env.OracleAdroitPenEnv, "door": adroit_env.OracleAdroitDoorEnv}[fam]
        o = cls(model, reward_type=reward_type, noslip=False)
        if fam == "pen":   # the two lengths reset_model measures (adroit_pen.py:392-399): rigid, so the model's site offsets
            sp = np.asarray(model.site_pos, np.float64).reshape(-1, 3)
            o.pen_length = float(np.linalg.norm(sp[o.obj_t_site_id] - sp[o.obj_b_site_id]))
            o.tar_length = float(np.linalg.norm(sp[o.tar_t_site_id] - sp[o.tar_b_site_id]))
        return o
    from gymnasium_robotics_b200.maze import MAPS

    if fam == "point":
        from oracle.point_maze_env import OraclePointMazeEnv

        return OraclePointMazeEnv(MAPS["UMaze"], model, reward_type=reward_type)
    from oracle.ant_maze_env import OracleAntMazeEnv

    return OracleAntMazeEnv(MAPS["UMaze"], reward_type=reward_type, model=model, include_cfrc_ext_in_observation=True)


def _record(fam, o, task, lay):
    """The fp32 state record of the oracle env's state (qpos | qvel | warm | ctrl | mocap | pose | goal | per-env body pose)."""
    s, m = o.sim, o.model
    rec = np.zeros(lay["stride"])
    rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
    rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
    rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
    if fam == "fetch":
        rec[lay["mocap"]:lay["mocap"] + 3], rec[lay["mocap"] + 3:lay["mocap"] + 7] = s.mocap_pos[0], s.mocap_quat[0]
        rec[lay["pose"]:lay["pose"] + 3], rec[lay["pose"] + 3:lay["pose"] + 7] = s.site_xpos[o._gripper_frame], o._body_xquat(o._gripper_frame)
    g = o.target_pos if fam == "relocate" else getattr(o, "goal", None)
    if g is not None and fam not in ("hammer", "pen", "door"):
        rec[lay["goal"]:lay["goal"] + len(g)] = g
    if fam in ("hammer", "relocate", "pen", "door"):
        rec[lay["penv"]:lay["penv"] + 3], rec[lay["penv"] + 3:lay["penv"] + 7] = s.body_pos[task.penv_body], s.body_quat[task.penv_body]
    return rec.astype(np.float32)


def _put(fam, o, task, lay, rec):
    """The oracle env at the record's (fp32) state, forwarded."""
    s, m = o.sim, o.model
    r = np.asarray(rec, np.float64)
    s.qpos[:] = r[lay["qpos"]:lay["qpos"] + m.nq]
    s.qvel[:] = r[lay["qvel"]:lay["qvel"] + m.nv]
    s.ctrl[:] = r[lay["ctrl"]:lay["ctrl"] + m.nu]
    if fam == "fetch":
        s.mocap_pos[0], s.mocap_quat[0] = r[lay["mocap"]:lay["mocap"] + 3], r[lay["mocap"] + 3:lay["mocap"] + 7]
    if fam in ("hammer", "relocate", "pen", "door"):
        s.body_pos[task.penv_body], s.body_quat[task.penv_body] = r[lay["penv"]:lay["penv"] + 3], r[lay["penv"] + 3:lay["penv"] + 7]
    ng = int(task.ngoal) if fam != "fetch" else 3
    if fam == "relocate":
        o.target_pos = r[lay["goal"]:lay["goal"] + 3].copy()
    elif fam not in ("hammer", "pen", "door"):
        o.goal = r[lay["goal"]:lay["goal"] + ng].copy()
    s.forward()


def _quat2mat(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _cy(mat):
    return float(np.hypot(mat[2, 2], mat[1, 2]))


def _reference(fam, o, task, lay, rec):
    """fp64 outputs at the record's state and how each is compared: dict(obs, ag, dg, reward, success, groups, ag_kind, dg_kind,
    decisions [(name, q, thr, scale)], rscale, cy)."""
    from gymnasium_robotics_b200 import rotations

    _put(fam, o, task, lay, rec)
    s, m = o.sim, o.model
    L = max(float(np.abs(s.xpos).max()), 1.0)
    av = np.abs(s.qvel)
    r = dict(cy=None)
    if fam == "fetch":
        ob = o._get_obs()
        obs, ag, dg = ob["observation"], ob["achieved_goal"], ob["desired_goal"]
        dt = o.dt

        def vs(site):
            jp, jr = s.jac_site(site)
            return dt * ((np.abs(jp) @ av).max() + L * (np.abs(jr) @ av).max()), dt * (np.abs(jr) @ av).max()
        vg, _ = vs(o._grip_site)
        fv = dt * av[[int(m.jnt_dofadr[j]) for j in o._robot_joints[-2:]]].max()
        if o.has_object:
            vo, wo = vs(o._obj_site)
            cy = _cy(s.site_xmat[o._obj_site].reshape(3, 3))
            r["cy"] = cy
            r["euler"] = (11, 14)
            groups = [(slice(0, 9), "pos", L), (slice(9, 11), "copy", 0), (slice(11, 12), "euler", L / max(cy, 1e-300)),
                      (slice(12, 13), "euler", L), (slice(13, 14), "euler", L / max(cy, 1e-300)), (slice(14, 17), "vel", vo + vg), (slice(17, 20), "vel", wo), (slice(20, 23), "vel", vg), (slice(23, 25), "vel", fv)]
        else:
            groups = [(slice(0, 3), "pos", L), (slice(3, 5), "copy", 0), (slice(5, 8), "vel", vg), (slice(8, 10), "vel", fv)]
        d = float(np.linalg.norm(ag - dg))
        reward, success = float(o.compute_reward(ag, dg, {})), float(o._is_success(ag, dg))
        r.update(ag_kind="pos", dg_kind="copy", decisions=[("d", d, o.distance_threshold, L)], rscale=L)
    elif fam == "reach":
        ob = o._get_obs()
        obs, ag, dg = ob["observation"], ob["achieved_goal"], ob["desired_goal"]
        groups = [(slice(0, 48), "copy", 0), (slice(48, 63), "pos", L)]
        d = float(np.linalg.norm(ag - dg))
        reward, success = float(o.compute_reward(ag, dg, {})), float(o._is_success(ag, dg))
        r.update(ag_kind="pos", dg_kind="copy", decisions=[("d", d, o.distance_threshold, L)], rscale=L)
    elif fam == "hand":
        ob = o._get_obs()
        obs, ag, dg = ob["observation"], ob["achieved_goal"], ob["desired_goal"]
        groups = [(slice(0, 61), "copy", 0)]
        d_pos, d_rot = (float(x) for x in o._goal_distance(ag, dg))
        reward, success = float(o.compute_reward(ag, dg, {})), float(o._is_success(ag, dg))
        # the w of qa * conj(g): its rounding (the sum of |products|, plus the Euler round trip of ignore_z, whose angles are rounded
        # in units of u / cy), through 2 acos(w)
        qa, qg = ag[3:] / np.linalg.norm(ag[3:]), dg[3:]
        sw = float(np.abs(qa * qg).sum()) + 2.0
        if o.ignore_z_target_rotation:
            sw += 1.0 / max(_cy(_quat2mat(ag[3:])), 1e-12) + 1.0 / max(_cy(_quat2mat(dg[3:])), 1e-12)
        w = np.cos(d_rot / 2)
        rs = 2 * sw / max(np.sqrt(max(1 - w * w, 0.0)), np.sqrt(U * sw))
        dec = []
        if o.target_position != "ignore":
            dec.append(("d_pos", d_pos, o.distance_threshold, L))
        if o.target_rotation != "ignore":
            dec.append(("d_rot", d_rot, o.rotation_threshold, rs))
        r.update(ag_kind="copy", dg_kind="copy", decisions=dec, rscale=10 * L + rs)
    elif fam in ("point", "ant"):
        from oracle.maze import compute_reward

        ob = o._get_obs()
        obs, ag, dg = ob["observation"], ob["achieved_goal"], ob["desired_goal"]
        n = len(obs) if fam == "point" else m.nq - 2 + m.nv   # (the Ant's contact forces are not compared here)
        groups = [(slice(0, n), "copy", 0)]
        d = float(np.linalg.norm(ag - dg))
        reward = float(compute_reward(ag, dg, o.reward_type))
        success = float(d <= 0.45)
        r.update(ag_kind="copy", dg_kind="copy", decisions=[("d", d, 0.45, L)], rscale=np.exp(-d) * L + 1.0)
    else:
        obs = o._get_obs()
        reward, ok = o.reward()
        reward, success = float(reward), float(ok)
        nr = m.nq - 6
        if fam == "hammer":
            ag, dg = s.site_xpos[o.target_obj_site_id].copy(), s.site_xpos[o.goal_site_id].copy()
            cy = _cy(_quat2mat(s.xquat[o.obj_body_id]))
            r["cy"] = cy
            r["euler"] = (nr + 12, nr + 15)
            groups = [(slice(0, nr + 6), "copy", 0), (slice(nr + 6, nr + 12), "pos", L), (slice(nr + 12, nr + 13), "euler", L / max(cy, 1e-300)),
                      (slice(nr + 13, nr + 14), "euler", L), (slice(nr + 14, nr + 15), "euler", L / max(cy, 1e-300)),
                      (slice(nr + 15, nr + 18), "pos", L)]
            hamm, head = s.xpos[o.obj_body_id], s.site_xpos[o.tool_site_id]
            gd = float(np.linalg.norm(ag - dg))
            dec = [("hammer z", hamm[2], 0.04, L), ("head z", head[2], 0.04, L), ("goal 0.02", gd, 0.02, L), ("goal 0.01", gd, 0.01, L)]
            r.update(ag_kind="pos", dg_kind="pos", decisions=dec, rscale=11.1 * L + 1e-2 * np.linalg.norm(s.qvel) * m.nv + 102)
        elif fam == "relocate":
            ag, dg = s.xpos[o.obj_body_id].copy(), o.target_pos.copy()
            groups = [(slice(0, nr), "copy", 0), (slice(nr, nr + 9), "pos", L)]
            gd = float(np.linalg.norm(ag - dg))
            dec = [("ball z", ag[2], 0.04, L), ("goal 0.1", gd, 0.1, L), ("goal 0.05", gd, 0.05, L)]
            r.update(ag_kind="pos", dg_kind="copy", decisions=dec, rscale=1.1 * L + 31)
        elif fam == "pen":
            oo, dd = o._orien()
            ag, dg = oo, dd
            ls = L / min(o.pen_length, o.tar_length)
            groups = [(slice(0, nr), "copy", 0), (slice(nr, nr + 3), "pos", L), (slice(nr + 3, nr + 9), "copy", 0),
                      (slice(nr + 9, nr + 15), "dir", ls), (slice(nr + 15, nr + 18), "pos", L), (slice(nr + 18, nr + 21), "dir", ls)]
            pos = s.xpos[o.obj_body_id]
            gd = float(np.linalg.norm(pos - s.site_xpos[o.eps_ball_site_id]))
            sim = float(oo @ dd)
            dec = [("similarity 0.9", sim, 0.9, 2 * ls), ("similarity 0.95", sim, 0.95, 2 * ls), ("goal 0.075", gd, 0.075, L),
                   ("pen z", pos[2], 0.075, L)]
            r.update(ag_kind="dir", dg_kind="dir", decisions=dec, rscale=L + 2 * ls + 65)
        else:   # door: the hinge angle is a copy; the kernel compares it with the fp32 thresholds
            ag, dg = s.site_xpos[o.grasp_site_id].copy(), s.site_xpos[o.handle_site_id].copy()
            nr = m.nq - 3
            groups = [(slice(0, nr + 2), "copy", 0), (slice(nr + 2, nr + 11), "pos", L), (slice(nr + 11, nr + 12), "copy", 0)]
            door = float(s.qpos[o.door_hinge_addrs])
            dec = [(f"door {t}", door, t, t) for t in (0.2, 1.0, 1.35)]
            r.update(ag_kind="pos", dg_kind="pos", decisions=dec,
                     rscale=0.1 * L + 0.1 * (abs(door) + 1.57) ** 2 + 1e-5 * float(s.qvel @ s.qvel) * m.nv + 21)
    r.update(obs=np.asarray(obs, np.float64), ag=np.asarray(ag, np.float64), dg=np.asarray(dg, np.float64), reward=reward,
             success=success, groups=groups, L=L)
    return r


def _note(worst, bad, key, v, where):
    """Record error v of a check (units of u times its scale) and flag it past LIM[key]; a NaN error is flagged and recorded as inf."""
    v = float(v) if v == v else np.inf
    worst[key] = max(worst.get(key, 0.0), v)
    if not v <= LIM[key]:
        bad.append(f"{where}: {key} {v:.1f} u (limit {LIM[key]})")


def _err(kind, got, ref, scale):
    """(error in units of u * scale, exact equality) of one group."""
    if kind == "copy":
        return 0.0, bool(np.array_equal(got, ref))
    d = got - ref
    if kind == "euler":   # angles compare modulo 2 pi
        d = (d + np.pi) % (2 * np.pi) - np.pi
    return float(np.abs(d).max() / (U * max(scale, 1e-30))), True


# ------------------------------------------------------------------------------------------------ states
def _wild_qvel(m, rng):
    qv = rng.normal(0.0, 3.0, m.nv)
    for j in range(m.njnt):
        if int(m.jnt_type[j]) == 0:   # free bodies spun at 60 rad/s
            w = rng.standard_normal(3)
            qv[int(m.jnt_dofadr[j]) + 3:int(m.jnt_dofadr[j]) + 6] = 60.0 * w / np.linalg.norm(w)
    return qv


def _secant(f, x0, target, h):
    """x with f(x) = target (f smooth and monotone near x0)."""
    x1, f0 = x0 + h, f(x0) - target
    f1 = f(x1) - target
    for _ in range(30):
        if f1 == f0 or abs(f1) < 1e-13:
            break
        x0, x1, f0 = x1, x1 - f1 * (x1 - x0) / (f1 - f0), f1
        f1 = f(x1) - target
    return x1


def _states(fam, o, task, lay, base, rng):
    """[(label, record)]: the reset state, random states, object orientations, and the family's threshold states."""
    from gymnasium_robotics_b200 import rotations
    from tests.test_device_kin_gpu import _random_qpos

    m = o.model
    Q, V, G = lay["qpos"], lay["qvel"], lay["goal"]
    out = [("reset", base)]
    free = [int(m.jnt_qposadr[j]) for j in range(m.njnt) if int(m.jnt_type[j]) == 0]
    for k in range(3):
        r = base.copy()
        q = _random_qpos(m, rng)
        for a in free:   # w < 0 in the first case, w > 0 in the second
            q[a + 3:a + 7] *= (-1.0 if k == 0 else 1.0) * np.sign(q[a + 3])
        r[Q:Q + m.nq], r[V:V + m.nv] = q, _wild_qvel(m, rng)
        out.append((f"random {k}", r))
    if fam == "fetch" and free:
        a = free[0]
        for sg in (1, -1):
            for dp in (0.0, 1e-4, 1e-2):
                r = base.copy()
                r[Q + a + 3:Q + a + 7] = rotations.euler2quat(np.array([rng.uniform(-np.pi, np.pi), sg * np.pi / 2 + dp, rng.uniform(-np.pi, np.pi)]))
                if dp == 1e-4:
                    r[V:V + m.nv] = _wild_qvel(m, rng)
                out.append((f"pitch {'+' if sg > 0 else '-'}pi/2 + {dp:g}", r))

    def ref(r):
        return _reference(fam, o, task, lay, np.asarray(r, np.float32).astype(np.float64))

    ng = 3 if fam == "fetch" else int(task.ngoal)
    if fam in ("fetch", "reach", "point", "ant", "relocate"):   # goals at threshold x (1 +- 1e-3)
        thr = {"fetch": 0.05, "reach": 0.01, "point": 0.45, "ant": 0.45, "relocate": 0.1}[fam]
        for src in (base, out[1][1]):
            ag = ref(src)["ag"]
            for f in (1 - 1e-3, 1 + 1e-3) + ((0.5 * (1 - 1e-3), 0.5 * (1 + 1e-3)) if fam == "relocate" else ()):
                v = rng.standard_normal(ng)
                r = src.copy()
                r[G:G + ng] = ag + thr * f * v / np.linalg.norm(v)
                out.append((f"goal at {thr * f:.6g}", r))
    if fam == "hand":
        thr_p, thr_r = o.distance_threshold, o.rotation_threshold
        for src in (base, out[1][1]):
            ag = ref(src)["ag"]
            for f in (1 - 1e-3, 1 + 1e-3):
                v = rng.standard_normal(3)
                r = src.copy()
                r[G:G + 3], r[G + 3:G + 7] = ag[:3] + thr_p * f * v / np.linalg.norm(v), ag[3:]
                out.append((f"goal position at {thr_p * f:.6g}", r))
                ax = np.array([1.0, 0.0, 0.0]) if o.ignore_z_target_rotation else rng.standard_normal(3)
                r = src.copy()
                r[G:G + 3] = ag[:3]
                r[G + 3:G + 7] = rotations.quat_mul(ag[3:], rotations.quat_from_angle_and_axis(thr_r * f, ax / np.linalg.norm(ax)))
                out.append((f"goal rotation at {thr_r * f:.6g}", r))
    if fam in ("hammer", "relocate", "pen", "door"):
        def qadr(name):
            return Q + int(m.jnt_qposadr[m.joint_id(name)])

        def at(r, idx, val):
            r = r.copy()
            r[idx] = val
            return r
        steps = []
        if fam == "hammer":   # hammer and head heights around 0.04 (both raised), the nail's distance around 0.02 / 0.01
            up = _secant(lambda x: min(ref(at(base, qadr("OBJTz"), x))["decisions"][k][1] for k in (0, 1)), float(base[qadr("OBJTz")]), 0.06, 0.01)
            lifted = at(base, qadr("OBJTz"), up)
            for k in (0, 1):
                steps.append((lifted, qadr("OBJTz"), lambda r, k=k: ref(r)["decisions"][k][1], 0.04, 0.01))
            for thr in (0.02, 0.01):
                steps.append((base, qadr("nail_dir"), lambda r: ref(r)["decisions"][2][1], thr, 0.01))
        elif fam == "relocate":
            steps.append((base, qadr("OBJTz"), lambda r: ref(r)["ag"][2], 0.04, 0.01))
        elif fam == "pen":   # the similarity around 0.9 / 0.95 (the target turned towards the pen), the pen height around 0.075
            r0 = ref(base)
            ax = np.cross(r0["dg"], r0["ag"])
            ang = float(np.arctan2(np.linalg.norm(ax), r0["dg"] @ r0["ag"]))
            ax /= np.linalg.norm(ax)

            def turned(x):
                r = base.copy()
                r[lay["penv"] + 3:lay["penv"] + 7] = rotations.quat_mul(rotations.quat_from_angle_and_axis(x, ax),
                                                                         base[lay["penv"] + 3:lay["penv"] + 7].astype(np.float64))
                return r
            for thr in (0.9, 0.95):
                for f in (1 - 1e-3, 1 + 1e-3):
                    x = _secant(lambda x: ref(turned(x))["decisions"][0][1], ang - np.arccos(thr * f), thr * f, 1e-3)
                    out.append((f"similarity at {thr * f:.6g}", turned(x)))
            steps.append((base, qadr("OBJTz"), lambda r: ref(r)["decisions"][3][1], 0.075, 0.01))
        else:   # door hinge around 0.2 / 1.0 / 1.35, and at exactly the fp32 thresholds
            for thr in (0.2, 1.0, 1.35):
                for v in (thr * (1 - 1e-3), thr * (1 + 1e-3), float(np.float32(thr))):
                    out.append((f"door at {v:.8g}", at(base, qadr("door_hinge"), v)))
        for src, idx, f, thr, h in steps:
            for fac in (1 - 1e-3, 1 + 1e-3):
                x = _secant(lambda x: f(at(src, idx, x)), float(src[idx]), thr * fac, h)
                out.append((f"step {thr} x {fac:g}", at(src, idx, x)))
    return [(lb, np.asarray(r, np.float32)) for lb, r in out]


def _own_goals(fam, task, lay, recs, outs, rng):
    """Goals placed from the kernel's own achieved goal: at exactly 0 distance, and (Fetch) at an fp32 distance that is exactly
    distance_threshold under both accumulation orders (fused multiply-add on the device, separate products on the host)."""
    ng = 3 if fam == "fetch" else int(task.ngoal)
    if fam in ("hammer", "pen", "door"):
        return []
    G = lay["goal"]
    new = []
    for e in (0, 1):
        ag = outs["achieved"][e].astype(np.float32)
        r = recs[e].copy()
        r[G:G + ng] = ag
        new.append(("goal = own achieved", r))
        if fam != "fetch":
            continue
        thr = np.float32(task.distance_threshold)
        for _ in range(2000):
            v = rng.standard_normal(3)
            g = (ag + thr * v / np.linalg.norm(v)).astype(np.float32)
            e3 = ag - g
            d_fma = np.float32(0)
            for x in e3:
                d_fma = np.float32(np.float64(x) * np.float64(x) + np.float64(d_fma))   # one rounding per term: fmaf
            d_sep = np.float32(0)
            for x in e3:
                d_sep = np.float32(d_sep + np.float32(x * x))
            if np.sqrt(d_fma) == thr and np.sqrt(d_sep) == thr:
                r = recs[e].copy()
                r[G:G + 3] = g
                new.append(("goal at fp32 distance == threshold", r))
                break
    return new


# ------------------------------------------------------------------------------------------------ 1. refresh
def _check_refresh(fam, o, task, lay, recs, labels, outs, stats, bad, tag):
    worst = stats["worst"]

    def note(key, v, where):
        _note(worst, bad, key, v, f"{tag} [{where}]")
    for e, (lb, rec) in enumerate(zip(labels, recs)):
        rf = _reference(fam, o, task, lay, rec.astype(np.float64))
        got = outs["obs"][e]
        for nm in ("obs", "achieved", "desired", "reward", "success"):
            if not np.isfinite(outs[nm][e]).all():
                bad.append(f"{tag} [{lb}]: {nm} is not finite: {outs[nm][e]}")
        for sl, kind, scale in rf["groups"]:
            v, same = _err(kind, got[sl], rf["obs"][sl], scale)
            if not same:
                bad.append(f"{tag} [{lb}]: observation {sl.start}:{sl.stop} is not a bit-for-bit copy "
                           f"({got[sl][got[sl] != rf['obs'][sl]][:4]} vs {rf['obs'][sl][got[sl] != rf['obs'][sl]][:4]})")
            if kind != "copy":
                note(kind, v, f"{lb}: obs {sl.start}:{sl.stop}")
        if rf["cy"] is not None and not task.reward_dense:   # (once per state: the sparse pass)
            sl = slice(*rf["euler"])
            stats["cy"].append((lb, rf["cy"], got[sl], rf["obs"][sl]))
        for nm, kind in (("achieved", rf["ag_kind"]), ("desired", rf["dg_kind"])):
            ref = rf["ag"] if nm == "achieved" else rf["dg"]
            v, same = _err(kind, outs[nm][e], ref, rf["L"] if kind == "pos" else rf["L"] / 0.1)
            if not same:
                bad.append(f"{tag} [{lb}]: {nm} goal is not a bit-for-bit copy")
            if kind != "copy":
                note(kind, v, f"{lb}: {nm}")
        near = [nm for nm, q, thr, sc in rf["decisions"] if abs(q - thr) <= NEAR * U * sc]
        for nm, q, thr, sc in rf["decisions"]:
            if not near:
                stats["sides"].add((nm, q > thr))
        if near:
            stats["near"].append(f"{lb}: {near}")
            continue
        if task.reward_dense:
            note("dense", abs(outs["reward"][e] - rf["reward"]) / (U * rf["rscale"]), f"{lb}: dense reward {outs['reward'][e]} vs {rf['reward']}")
        elif outs["reward"][e] != np.float32(rf["reward"]):   # (the rewards are float32: the Adroit's -0.1 is -0.1f)
            bad.append(f"{tag} [{lb}]: sparse reward {outs['reward'][e]}, the fp64 rule gives {rf['reward']}")
        if outs["success"][e] != rf["success"]:
            bad.append(f"{tag} [{lb}]: success {outs['success'][e]}, the fp64 rule gives {rf['success']}")
        stats["decided"] += 1


def _refresh_family(backend, fam, sparse_id, dense_id):
    """Both variants of one family at the same states; returns the stats printed and asserted."""
    rng = np.random.default_rng(31)
    stats = dict(worst={}, cy=[], near=[], sides=set(), decided=0, compared=0, boundary=0)
    bad = []
    per = {}
    for env_id in (sparse_id, dense_id):
        model, eq, task, attrs = _spec(env_id, backend)
        rt = "dense" if task.reward_dense else "sparse"
        o = _oracle(fam, env_id, model, attrs if fam == "hand" else {}, rt)
        be0 = _new_backend(backend, model, eq, task, 1)
        lay = be0.layout
        if not per:   # the states are drawn once, from the sparse variant's oracle
            o0 = _oracle(fam, env_id, model, attrs if fam == "hand" else {}, rt)
            o0.reset(seed=5)
            base = _record(fam, o0, task, lay)
            st = _states(fam, o, task, lay, base, rng)
            labels, recs = [s[0] for s in st], np.stack([s[1] for s in st])
            be = _new_backend(backend, model, eq, task, len(recs))
            outs, _ = _launch(be, recs)
            extra = _own_goals(fam, task, lay, recs, outs, rng)
            labels += [s[0] for s in extra]
            recs = np.concatenate([recs, np.stack([s[1] for s in extra])]) if extra else recs
        be = _new_backend(backend, model, eq, task, len(recs))
        outs, _ = _launch(be, recs)
        per[rt] = outs
        _check_refresh(fam, o, task, lay, recs, labels, outs, stats, bad, f"[{backend}] {env_id}")
        stats["compared"] += len(recs)
    # the rule at the kernel's own fp32 distance (goal families whose dense reward is -d): sparse reward -(d > thr), success d < thr
    if fam in ("fetch", "reach"):
        thr = np.float32(task.distance_threshold)
        d = (-per["dense"]["reward"]).astype(np.float32)
        for nm in ("sparse", "dense"):
            if not np.array_equal(per[nm]["success"], (d < thr).astype(np.float64)):
                bad.append(f"[{backend}] {fam} {nm}: success differs from d < {thr} at the kernel's own distance d = {d[per[nm]['success'] != (d < thr)]}")
        if not np.array_equal(per["sparse"]["reward"], -(d > thr).astype(np.float64)):
            bad.append(f"[{backend}] {fam}: sparse reward differs from -(d > {thr}) at the kernel's own distance")
        stats["boundary"] = int((d == thr).sum())
    return stats, bad


def _refresh_check(backend, fam, sparse_id, dense_id):
    stats, bad = _refresh_family(backend, fam, sparse_id, dense_id)
    w = ", ".join(f"{k} {v:.2f}" for k, v in sorted(stats["worst"].items()))
    print(f"\ntask refresh [{backend}] {sparse_id} / {dense_id}: {stats['compared']} cases, {stats['decided']} rule checks; worst (u): {w}")
    if stats["cy"]:
        print("  cy: " + "; ".join(f"{lb} {cy:.3g}" for lb, cy, _, _ in stats["cy"]))
        for lb, cy, g, r in stats["cy"]:
            if cy < 1e-3:   # near gimbal lock only the pitch is bounded (u L); x and z: the fp32 path's against fp64's
                print(f"  Euler angles at cy {cy:.3g} [{lb}]: fp32 kernel {np.array2string(g, precision=7)}, fp64 "
                      f"{np.array2string(r, precision=7)}")
    if fam == "fetch":
        print(f"  fp32 distance exactly at the threshold in {stats['boundary']} cases")
    for s in stats["near"][:8]:
        print(f"  near a threshold (rule not compared): {s}")
    assert not bad, "\n".join(bad[:20])
    # every threshold of the family was seen on both sides, outside the margin
    names = {nm for nm, _ in stats["sides"]}
    one = sorted(nm for nm in names if len({s for n2, s in stats["sides"] if n2 == nm}) < 2)
    assert not one, f"{sparse_id}: thresholds seen on one side only: {one}"
    if fam == "fetch":
        assert stats["boundary"] >= 2, "no case put the fp32 distance exactly on the threshold"


@pytest.mark.gpu
@pytest.mark.parametrize("fam,sparse_id,dense_id", IDS)
def test_task_refresh_on_the_device(fam, sparse_id, dense_id):
    _refresh_check("gpu", fam, sparse_id, dense_id)


@pytest.mark.parametrize("fam,sparse_id,dense_id", IDS)
def test_task_refresh_on_the_32_lane_emulation(fam, sparse_id, dense_id):
    _refresh_check("cpu", fam, sparse_id, dense_id)


# ------------------------------------------------------------------------------------------------ 2. the action map
ACTION_IDS = [("fetch", "FetchReach-v4"), ("fetch", "FetchPush-v4"), ("fetch", "FetchSlide-v4"), ("fetch", "FetchPickAndPlace-v4"),
              ("reach", "HandReach-v3"), ("hand", "HandManipulateBlock-v1"), ("hammer", "AdroitHandHammer-v2"),
              ("relocate", "AdroitHandRelocate-v2"), ("pen", "AdroitHandPen-v2"), ("door", "AdroitHandDoor-v2"),
              ("point", "PointMaze_UMaze-v3"), ("ant", "AntMaze_UMaze-v5")]


def _actions(nact, rng):
    """[(label, action)]: uniform in [-3, 3], exactly +1, -1 and 0, +inf and -inf in single entries."""
    a = [("uniform [-3, 3]", rng.uniform(-3, 3, nact)), ("+1", np.ones(nact)), ("-1", -np.ones(nact)), ("0", np.zeros(nact))]
    for sg in (1, -1):
        v = rng.uniform(-0.5, 0.5, nact)
        v[rng.integers(nact)] = sg * np.inf
        v[-1] = sg * np.inf   # (the Fetch gripper entry)
        a.append((f"{'+' if sg > 0 else '-'}inf entries", v))
    return [(lb, np.asarray(v, np.float32)) for lb, v in a]


def _action_check(backend, fam, env_id):
    rng = np.random.default_rng(41)
    model, eq, task, attrs = _spec(env_id, backend)
    o = _oracle(fam, env_id, model, attrs if fam == "hand" else {}, "sparse" if not task.reward_dense else "dense")
    be1 = _new_backend(backend, model, eq, task, 1)
    lay = be1.layout
    o.reset(seed=9)
    base = _record(fam, o, task, lay)
    nact = int(be1.nact)
    acts = _actions(nact, rng)
    recs = np.stack([base] * len(acts))
    from tests.test_device_kin_gpu import _random_qpos

    for e in range(1, len(recs), 2):   # every other case from a random joint configuration
        recs[e, lay["qpos"]:lay["qpos"] + model.nq] = _random_qpos(model, rng)
    recs = recs.astype(np.float32)
    be = _new_backend(backend, model, eq, task, len(recs))
    outs, after = _launch(be, recs, np.stack([a for _, a in acts]))
    bad, worst = [], {}
    m = model
    C, Q = lay["ctrl"], lay["qpos"]
    for e, (lb, a) in enumerate(acts):
        pre = recs[e].astype(np.float64)
        ctrl = after[e, C:C + m.nu].astype(np.float64)
        ac = np.clip(a.astype(np.float64), -1, 1)
        tag = f"[{backend}] {env_id} [{lb}]"
        if fam in ("hand", "reach", "hammer", "relocate", "pen", "door"):
            cr = np.asarray(m.act_ctrlrange, np.float64).reshape(-1, 2).astype(np.float32).astype(np.float64)
            lo, hi = cr[:, 0], cr[:, 1]
            if fam in ("hand", "reach"):   # the reference's own _set_action at the same pre-step state
                o.sim.ctrl[:] = 0.0
                o._set_action(ac)
                want = np.array(o.sim.ctrl)
            else:                          # adroit_*.py step: act_mean + clip(a) act_rng, clamped to ctrlrange by the actuation
                want = np.clip(o.act_mean + ac * o.act_rng, lo, hi)
            _note(worst, bad, "ctrl", np.abs(ctrl - want).max() / (U * (np.abs(lo) + np.abs(hi)).max()), f"{tag}: ctrl (units of the range)")
            out_of = (after[e, C:C + m.nu] < cr[:, 0].astype(np.float32)) | (after[e, C:C + m.nu] > cr[:, 1].astype(np.float32))
            if out_of.any():
                bad.append(f"{tag}: ctrl outside ctrlrange at actuators {np.nonzero(out_of)[0]}")
        elif fam == "fetch":
            pose = pre[lay["pose"]:lay["pose"] + 7]
            M = lay["mocap"]
            mp, mq = after[e, M:M + 3].astype(np.float64), after[e, M + 3:M + 7].astype(np.float64)
            vp = np.abs(mp - (pose[:3] + 0.05 * ac[:3])).max() / (U * (np.abs(pose[:3]).max() + 0.05))
            vq = np.abs(mq - (pose[3:] + np.array([1.0, 0.0, 1.0, 0.0]))).max() / (U * (np.abs(pose[3:]).max() + 1.0))
            _note(worst, bad, "mocap", vp, f"{tag}: mocap pos (pose slot + 0.05 clip(a))")
            _note(worst, bad, "mocap", vq, f"{tag}: mocap quat (pose quat + (1, 0, 1, 0))")
            g = 0.0 if task.block_gripper else ac[3]
            for i in range(m.nu):
                qa = int(m.jnt_qposadr[int(np.asarray(m.act_trnid).ravel()[i] if np.asarray(m.act_trnid).ndim == 1 else m.act_trnid[i][0])])
                want = pre[Q + qa] + g
                if task.block_gripper and ctrl[i] != want:
                    bad.append(f"{tag}: block_gripper finger ctrl {ctrl[i]} is not qpos {pre[Q + qa]} + 0")
                elif not abs(ctrl[i] - want) <= LIM["ctrl"] * U * (abs(pre[Q + qa]) + 1.0):
                    bad.append(f"{tag}: finger ctrl {i} = {ctrl[i]}, qpos + clip(a[3]) = {want}")
            if task.block_gripper:
                fq = [Q + int(task.finger_qadr[k]) for k in (0, 1)]
                if np.any(after[e, fq] != 0.0):
                    bad.append(f"{tag}: block_gripper left finger qpos {after[e, fq]}")
        elif fam == "ant":
            if not np.array_equal(after[e, C:C + m.nu], a):
                bad.append(f"{tag}: Ant ctrl {after[e, C:C + m.nu]} is not the action {a}")
        else:
            if not np.array_equal(after[e, C:C + m.nu], np.clip(a, -1, 1)):
                bad.append(f"{tag}: Point ctrl {after[e, C:C + m.nu]} is not clip(a)")
    if fam == "fetch" and task.block_gripper:   # the step's observation is the refresh observation of the record it stored
        again, _ = _launch(be, after)
        if not np.array_equal(again["obs32"], outs["obs32"]):
            bad.append(f"[{backend}] {env_id}: the step's observation differs from the refresh observation of its stored record")
    print(f"\naction map [{backend}] {env_id}: worst " + ", ".join(f"{k} {v:.2f} u" for k, v in worst.items()))
    assert not bad, "\n".join(bad[:20])


@pytest.mark.gpu
@pytest.mark.parametrize("fam,env_id", ACTION_IDS)
def test_action_map_on_the_device(fam, env_id):
    _action_check("gpu", fam, env_id)


@pytest.mark.parametrize("fam,env_id", ACTION_IDS)
def test_action_map_on_the_32_lane_emulation(fam, env_id):
    _action_check("cpu", fam, env_id)


# ------------------------------------------------------------------------------------------------ 3. touch sensors
# (committed model, product NVP, per-env body, devsim flavor)
TOUCH = [("hand_block_touch", 30, None, "plain"), ("adroit_hammer", 36, "nail_board", "wide")]
SPHERE, CYLINDER, BOX = 2, 5, 6   # B200_GEOM_*
CNT_NCON = 0


def _ray_hits(tp, size, p, d):
    """oracle.c ray_hits_site in fp64."""
    if tp == SPHERE:
        r, b, c = size[0], p @ d, p @ p - size[0] ** 2
        return bool(c <= 0 or (b * b - c >= 0 and -b >= 0))
    t0, t1 = 0.0, 1e30
    if tp == CYLINDER:
        r, hl = size[0], size[1]
        if abs(d[2]) < 1e-12:
            if abs(p[2]) > hl:
                return False
        else:
            a, b = sorted(((-hl - p[2]) / d[2], (hl - p[2]) / d[2]))
            t0, t1 = max(t0, a), min(t1, b)
            if t0 > t1:
                return False
        A, B, C = d[0] ** 2 + d[1] ** 2, p[0] * d[0] + p[1] * d[1], p[0] ** 2 + p[1] ** 2 - r * r
        if A < 1e-20:
            return bool(C <= 0)
        disc = B * B - A * C
        if disc < 0:
            return False
        sq = np.sqrt(disc)
        return bool(max(t0, (-B - sq) / A) <= min(t1, (-B + sq) / A))
    for k in range(3):
        if abs(d[k]) < 1e-12:
            if abs(p[k]) > size[k]:
                return False
            continue
        a, b = sorted(((-size[k] - p[k]) / d[k], (size[k] - p[k]) / d[k]))
        t0, t1 = max(t0, a), min(t1, b)
        if t0 > t1:
            return False
    return True


class _Tables:
    """The device model's own pair, geom and sensor tables (the kernel's indices)."""

    def __init__(self, sim):
        w = np.asarray(sim.sim.words)
        m = sim.m

        def arr(nm, n, dt=np.int32):
            o = sim.sim.model_offset(nm)
            return w[o:o + n].view(dt).astype(np.int64 if dt == np.int32 else np.float64)
        npair = m.npair
        self.g1, self.g2 = arr("pair_geom1", npair), arr("pair_geom2", npair)
        self.gbody = arr("geom_body", int(max(self.g1.max(), self.g2.max())) + 1)
        ns = m.nsensor
        self.site, self.body, self.type = arr("sensor_site", ns), arr("sensor_body", ns), arr("sensor_type", ns)
        self.size = arr("sensor_size", 3 * ns, np.float32).reshape(ns, 3)
        assert np.array_equal(self.site, np.asarray(m.sensor_site)) and np.array_equal(self.body, np.asarray(m.sensor_body))

    def bodies(self, p):
        return int(self.gbody[self.g1[p]]), (0 if self.g2[p] < 0 else int(self.gbody[self.g2[p]]))


def _contacts(sim, img):
    """The kernel's contact records of an image: [(pair, point, normal, fp64 normal force F0, |F0| rounding scale)]."""
    from tests.test_device_problem_gpu import _con_fields

    lay, o = sim.lay, sim.o
    ncon = int(img[o["counters"]:o["counters"] + 8].view(np.int32)[CNT_NCON])
    out = []
    for i in range(ncon):
        cr = img[o["con"] + i * lay["CON_WORDS"]:o["con"] + (i + 1) * lay["CON_WORDS"]]
        cx = img[o["conx"] + i * lay["CX_WORDS"]:o["conx"] + (i + 1) * lay["CX_WORDS"]]
        dim, _, _, mu = _con_fields(lay, cr)
        D, Uc = float(cr[lay["C_D"]]), cr[lay["C_U"]:lay["C_U"] + lay["NB"]].astype(np.float64)
        if dim == 1:
            f, sc = (-D * Uc[0] if Uc[0] < 0 else 0.0), abs(D * Uc[0])
        else:
            x = [Uc[0] + sg * mu[k] * Uc[k] for k in range(1, dim) for sg in (1, -1)]
            f = sum(-D * v for v in x if v < 0)
            sc = sum(abs(D) * (abs(Uc[0]) + mu[k] * abs(Uc[k])) for k in range(1, dim)) * 2
        out.append((int(cx[lay["CX_PAIR"]:lay["CX_PAIR"] + 1].view(np.int32)[0]), cx[lay["CX_POS"]:lay["CX_POS"] + 3].astype(np.float64),
                    cr[lay["C_W"] + 3:lay["C_W"] + 6].astype(np.float64), f, sc))
    return out


def _touch_reference(tb, orc, cons, L):
    """Per sensor: (fp64 sum over the contacts whose ray hits, sum of the forces of the contacts that may count either way, the
    rounding scale sum |F|, {contact: hit} of the contacts that involve the sensor's body)."""
    res = []
    for k in range(len(tb.site)):
        sp, R = orc.site_xpos[tb.site[k]], orc.site_xmat[tb.site[k]].reshape(3, 3)
        tot, amb, sc, hits = 0.0, 0.0, 0.0, {}
        for i, (p, pos, nrm, f, fs) in enumerate(cons):
            b1, b2 = tb.bodies(p)
            if tb.body[k] not in (b1, b2):
                continue
            sc += abs(f) + fs
            if f <= NEAR * U * fs:   # (an fp32 force this close to 0 may come out either side of it)
                if f > 0:
                    amb += f
                continue
            sg = -1.0 if b2 == tb.body[k] else 1.0
            loc, dl = R.T @ (pos - sp), R.T @ (sg * nrm)
            hit = _ray_hits(tb.type[k], tb.size[k], loc, dl)
            flips = any(_ray_hits(tb.type[k], tb.size[k], loc + e * NEAR * U * L, dl) != hit or
                        _ray_hits(tb.type[k], tb.size[k], loc, dl + e * NEAR * U) != hit for e in np.vstack([np.eye(3), -np.eye(3)]))
            hits[i] = None if flips else hit
            if flips:
                amb += f
            elif hit:
                tot += f
        res.append((tot, amb, sc, hits))
    return res


def _edits(sim, tb, orc, img, world=None):
    """Images with contact 0 replaced by one designed contact on one sensor's site ([(label, image, sensor, expected hit or None)]):
    points inside, outside, on and just off each site type's surface, rays towards, away and parallel, the sensor's body as geom1
    and as geom2, zero and negative normal force, sensors 32 and up.  With `world` ({sensor: pair whose geom2 the tables make a world
    geom}): those sensors only, on those pairs."""
    lay, o = sim.lay, sim.o
    out = []
    ns = len(tb.site)
    pick = sorted(world) if world else sorted({0, ns - 1} | ({int(np.nonzero(tb.type == t)[0][-1]) for t in np.unique(tb.type)}) |
                  ({int(np.nonzero((tb.type == t) & (np.arange(ns) >= 32))[0][0]) for t in np.unique(tb.type[32:])} if ns > 32 else set()))
    cw, cxw = lay["CON_WORDS"], lay["CX_WORDS"]
    dim = int(img[o["con"] + lay["C_DIMGRP"]:o["con"] + lay["C_DIMGRP"] + 1].view(np.int32)[0]) & 0xFF
    for k in pick:
        tp, size = int(tb.type[k]), tb.size[k].astype(np.float64)
        sp, R = orc.site_xpos[tb.site[k]], orc.site_xmat[tb.site[k]].reshape(3, 3)
        ex = np.array([1.0, 0.0, 0.0])
        ez = np.array([0.0, 0.0, 1.0])
        r = size[0]
        if tp == SPHERE:
            geo = [("inside", 0.5 * r * ex, ez, True), ("outside, towards", 2 * r * ex, -ex, True), ("outside, away", 2 * r * ex, ex, False),
                   ("just inside, away", (1 - 1e-3) * r * ex, ex, True), ("just outside, away", (1 + 1e-3) * r * ex, ex, False),
                   ("just outside, tangent", (1 + 1e-3) * r * ex, ez, False), ("on the surface, tangent", r * ex, ez, None)]
        elif tp == BOX:
            h = size
            geo = [("inside", 0.5 * h * np.array([1, -1, 1]), ez, True), ("outside, towards", np.array([2 * h[0], 0, 0]), -ex, True),
                   ("outside, away", np.array([2 * h[0], 0, 0]), ex, False),
                   ("parallel to a face, outside", np.array([2 * h[0], 0.5 * h[1], 0]), np.array([0.0, -1.0, 0.0]), False),
                   ("parallel to a face, inside its slab", np.array([0.5 * h[0], 2 * h[1], 0]), np.array([0.0, -1.0, 0.0]), True),
                   ("just inside a face", np.array([(1 - 1e-3) * h[0], 0, 0]), np.array([0.0, 1.0, 0.0]), True),
                   ("just outside a face", np.array([(1 + 1e-3) * h[0], 0, 0]), np.array([0.0, 1.0, 0.0]), False),
                   ("on a face", np.array([h[0], 0, 0]), np.array([0.0, 1.0, 0.0]), None)]
        else:
            hl = size[1]
            geo = [("beyond an end, along the axis", np.array([0, 0, 2 * hl]), -ez, True),
                   ("outside, towards the axis", np.array([2 * r, 0, 0]), -ex, True), ("outside, away", np.array([2 * r, 0, 0]), ex, False),
                   ("parallel to the axis, outside", np.array([2 * r, 0, 2 * hl]), -ez, False),
                   ("just inside the mantle, along the axis", np.array([(1 - 1e-3) * r, 0, 0]), ez, True),
                   ("just outside the mantle, along the axis", np.array([(1 + 1e-3) * r, 0, 0]), ez, False),
                   ("on the mantle", np.array([r, 0, 0]), ez, None)]
        for flip in ((False,) if world else (False, True)):
            ps = [world[k]] if world else \
                [p for p in range(len(tb.g1)) if tb.bodies(p)[1 if flip else 0] == tb.body[k] and tb.bodies(p)[0 if flip else 1] != tb.body[k]]
            if not ps:
                continue
            for lb, loc, dl, want in geo:
                for force in ("F > 0",) + (("F = 0", "F < 0") if lb.startswith("inside") else ()):
                    im = img.copy()
                    im[o["counters"]:o["counters"] + 1].view(np.int32)[0] = 1
                    cr = im[o["con"]:o["con"] + cw]
                    cx = im[o["conx"]:o["conx"] + cxw]
                    cx[lay["CX_POS"]:lay["CX_POS"] + 3] = sp + R @ loc
                    cx[lay["CX_PAIR"]:lay["CX_PAIR"] + 1].view(np.int32)[0] = ps[0]
                    nrm = R @ dl
                    nrm[np.abs(nrm) < 1e-9] = 0.0   # (a site aligned with the world axes: the ray exactly along its axis)
                    cr[lay["C_W"] + 3:lay["C_W"] + 6] = (-1.0 if flip else 1.0) * nrm
                    cr[lay["C_D"]] = -1.0 if force == "F < 0" else 1.0
                    cr[lay["C_U"]:lay["C_U"] + lay["NB"]] = 0.0
                    cr[lay["C_U"]] = 0.0 if force == "F = 0" else -0.7 / (1 if dim == 1 else 2 * (dim - 1))
                    out.append((f"sensor {k} ({ {SPHERE: 'sphere', BOX: 'box', CYLINDER: 'cylinder'}[tp]}) {lb}, {force}"
                                f"{', its body as geom2' if flip else ''}{', the other geom a world geom' if world else ''}", im, k,
                                want if force == "F > 0" else False))
    return out


def _touch_check(backend, name, nvp, penv, flavor):
    from tests import devsim
    from tests.test_device_problem_gpu import _Sim, _oracle, _states

    m, pb, states = _states(name, penv)
    states = [(lb, st) for lb, mm, st in states if mm is None]
    sim = _Sim(backend, flavor, nvp, m, pb)
    tb = _Tables(sim)

    def touch(imgs):
        if backend == "gpu":
            return sim.sim.run(nvp, devsim.STAGE_TOUCH, imgs)
        vals = []
        for e in range(len(imgs)):
            sim.sim.scratch[:] = imgs[e]
            vals.append(sim.sim.touch())
        return np.stack(vals)
    imgs = np.stack([sim.image(st, pb) for _, st in states])
    sim.run(2, imgs)
    orcs = [_oracle(m, pb, st) for _, st in states]
    cases = [(lb, imgs[e], orcs[e], None, None, tb) for e, (lb, _) in enumerate(states)]
    cases += [(lb, im, orcs[0], k, want, tb) for lb, im, k, want in _edits(sim, tb, orcs[0], imgs[0])]
    got = touch(np.ascontiguousarray(np.stack([c[1] for c in cases]))).astype(np.float64)
    # a contact with a world geom (g2 < 0, b2 = world body 0): no committed touch model has such a pair, so one pair per site type
    # whose geom1 is on the sensor's body gets g2 = -1 in the model words the harness runs (and in the reference's tables)
    world = {}
    for k in sorted({int(np.nonzero(tb.type == t)[0][-1]) for t in np.unique(tb.type)}):
        ps = [p for p in range(len(tb.g1)) if tb.bodies(p)[0] == tb.body[k] and tb.bodies(p)[1] != tb.body[k]]
        if ps:
            world[k] = ps[0]
    live = sim.sim.model_words() if backend == "gpu" else sim.sim.words
    o2 = sim.sim.model_offset("pair_geom2")
    saved = live[o2:o2 + len(tb.g2)].copy()
    tbw = copy.copy(tb)
    tbw.g2 = tb.g2.copy()
    for p in world.values():
        live[o2 + p] = np.uint32(0xFFFFFFFF)
        tbw.g2[p] = -1
    try:
        wcases = [(lb, im, orcs[0], k, want, tbw) for lb, im, k, want in _edits(sim, tbw, orcs[0], imgs[0], world=world)]
        got = np.concatenate([got, touch(np.ascontiguousarray(np.stack([c[1] for c in wcases]))).astype(np.float64)])
    finally:
        live[o2:o2 + len(tb.g2)] = saved
    cases += wcases
    bad, worst, fired, nedit = [], 0.0, 0, 0
    flip_seen, world_seen = set(), set()
    for e, (lb, im, orc, k0, want, tbe) in enumerate(cases):
        L = max(float(np.abs(orc.xpos).max()), 1.0)
        cons = _contacts(sim, im)
        ref = _touch_reference(tbe, orc, cons, L)
        for k, (tot, amb, sc, hits) in enumerate(ref):
            g = got[e, k]
            out = max(tot - g, g - (tot + amb), 0.0) / (U * max(sc, 1e-30)) if np.isfinite(g) else np.inf
            worst = max(worst, out)
            fired += int(g > 0)
            if not out <= LIM["touch"]:
                bad.append(f"[{backend}] {name} [{lb}] sensor {k}: {g} outside the fp64 sum {tot} (+ {amb} of contacts that may count "
                           f"either way) by {out:.1f} u sum |F|")
        if k0 is not None:
            nedit += 1
            h = ref[k0][3].get(0, False)
            if want is not None and h != want:
                bad.append(f"[{backend}] {name} [{lb}]: the designed case's fp64 hit is {h}, not {want} (test construction)")
            if "geom2" in lb and want:
                flip_seen.add(name)
            if "world geom" in lb and want:
                world_seen.add(int(tbe.type[k0]))
    if name == "hand_block_touch":   # the Boolean ids report exactly continuous > 0, through the product refresh at the same states
        vals = {}
        for env_id in ("HandManipulateBlock_ContinuousTouchSensors-v1", "HandManipulateBlock_BooleanTouchSensors-v1"):
            model, eq, task, _ = _spec(env_id, backend)
            be = _new_backend(backend, model, eq, task, len(states))
            lay = be.layout
            recs = np.zeros((len(states), lay["stride"]), np.float32)
            for e, (_, st) in enumerate(states):
                for f, key in (("qpos", "qpos"), ("qvel", "qvel"), ("warm", "qacc"), ("ctrl", "ctrl")):
                    recs[e, lay[f]:lay[f] + len(st[key])] = st[key]
                recs[e, lay["goal"] + 3] = 1.0
            vals[env_id] = _launch(be, recs)[0]["obs"][:, -model.nsensor:]
        cont, boolean = vals.values()
        if not np.array_equal(boolean, (cont > 0).astype(np.float64)):
            bad.append(f"[{backend}] the Boolean touch ids differ from continuous > 0 at {np.argwhere(boolean != (cont > 0))[:5]}")
        fired = int((cont > 0).sum())
    print(f"\ntouch [{backend}] {name}: {len(states)} states, {nedit} edited records ({len(wcases)} with a world geom), {fired} sensor "
          f"readings > 0; worst {worst:.2f} u sum |F|")
    assert not bad, "\n".join(bad[:20])
    assert world_seen == set(np.unique(tb.type).tolist()), f"{name}: world-geom contacts hit sites of types {world_seen} only"
    assert flip_seen, f"{name}: no edited contact hits its site through the flipped normal (the sensor's body as geom2)"


@pytest.mark.gpu
@pytest.mark.parametrize("name,nvp,penv,flavor", TOUCH)
def test_touch_sensors_on_the_device(name, nvp, penv, flavor):
    _touch_check("gpu", name, nvp, penv, flavor)


@pytest.mark.parametrize("name,nvp,penv,flavor", TOUCH)
def test_touch_sensors_on_the_32_lane_emulation(name, nvp, penv, flavor):
    _touch_check("cpu", name, nvp, penv, flavor)


def _site_rays(rng):
    """[(type, size, p [n, 3], d [n, 3])] in the site frame: points inside, on and just off each site type's surface and outside it,
    rays along the exact axes (the parallel-to-a-face and along-the-cylinder-axis branches), diagonal and random."""
    sizes = {SPHERE: [0.005, 0.0, 0.0], BOX: [0.01, 0.006, 0.003], CYLINDER: [0.034, 0.005, 0.0]}   # (the Hand's and the hammer's)
    axes = np.vstack([np.eye(3), -np.eye(3)])
    out = []
    for tp, size in sizes.items():
        ext = np.array([size[0], size[0], size[0]]) if tp == SPHERE else (np.array([size[0], size[0], size[1]]) if tp == CYLINDER else np.array(size))
        ps = [f * ext * s for f in (0.0, 0.5, 1 - 1e-3, 1.0, 1 + 1e-3, 2.0) for s in np.vstack([axes, [[1, 1, 1], [1, -1, 0.5]]])]
        ps += list(rng.uniform(-2.5, 2.5, (16, 3)) * ext)
        ds = list(axes) + [v / np.linalg.norm(v) for v in rng.standard_normal((10, 3))]
        p = np.array([a for a in ps for _ in ds], np.float32)
        d = np.array([b for _ in ps for b in ds], np.float32)
        out.append((tp, np.asarray(size, np.float32), p, d))
    return out


def _ray_check(backend):
    from tests import devsim, hostsim

    rng = np.random.default_rng(53)
    bad, n, amb = [], 0, 0
    for tp, size, p, d in _site_rays(rng):
        got = devsim.ray_hits("plain", tp, size, p, d) if backend == "gpu" else hostsim.ray_hits("warp", tp, size, p, d)
        sz = size.astype(np.float64)
        L = float(np.abs(sz).max())
        for i in range(len(p)):
            pp, dd = p[i].astype(np.float64), d[i].astype(np.float64)
            want = _ray_hits(tp, sz, pp, dd)
            # the decision counts where it is stable under NEAR u L of the point and NEAR u of the direction's non-zero entries
            if any(_ray_hits(tp, sz, pp + e * NEAR * U * L, dd) != want or _ray_hits(tp, sz, pp, dd + e * (dd != 0) * NEAR * U) != want
                   for e in np.vstack([np.eye(3), -np.eye(3), [[1, 1, 1], [-1, -1, -1]]])):
                amb += 1
                continue
            n += 1
            if bool(got[i]) != want:
                bad.append(f"[{backend}] ray_hits_site type {tp}: p {p[i]}, d {d[i]}: {bool(got[i])}, the fp64 test {want}")
    print(f"\nray_hits_site [{backend}]: {n} rays decided as in fp64, {amb} within the margin of a surface")
    assert not bad, "\n".join(bad[:20])


@pytest.mark.gpu
def test_ray_hits_site_on_the_device():
    _ray_check("gpu")


def test_ray_hits_site_on_the_32_lane_emulation():
    _ray_check("cpu")
