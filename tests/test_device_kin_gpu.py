"""The kinematics stage (sim_core.cuh `kinematics`, `com_quantities`, `mass_matrix`) on its own, per product kernel build, against the
fp64 oracle at the same joint positions.

Each committed model runs on the build and NVP its product kernel uses (tests/devsim `stage` op, STAGE_KIN), at the contact-heavy
oracle states of tests/test_device_spd_gpu.py and at random joint positions within the joint ranges.  Both sides get the same fp32
qpos, mocap pose and -- for the Adroit models -- per-env body pose (penv_pos; the oracle's body_pos / body_quat of that body).
Compared, with L = the largest |coordinate| of the case and u = 2^-24:
  * body positions xpos and geom positions geom_xpos in units of u L;
  * body quaternions xquat, up to sign, in units of u;
  * the joint-space inertia M normwise, ||M - M_oracle||_F / ||M_oracle||_F, in units of nv u.
The limits are 4-5x the largest values measured (DESIGN.md section 2).  The GPU half runs the nvcc builds; the CPU half runs the same
cases on the 32-lane emulation (tests/hostsim).
"""
import numpy as np
import pytest

from tests.test_device_collide_gpu import HOST_FLAVOR, device_order

U = 2.0 ** -24
# (committed model, product NVP, per-env body of its task or None)
MODELS = [("antmaze_umaze", 14, None), ("fetch_reach", 15, None), ("fetch_pick_and_place", 21, None), ("fetch_slide", 22, None),
          ("hand_block_touch", 30, None), ("franka_kitchen", 31, None), ("adroit_hammer", 36, "nail_board"),
          ("adroit_relocate", 36, "Object")]
FLAVOR = {14: "plain", 15: "plain", 21: "plain", 22: "plain", 30: "plain", 31: "kitchen_groups", 36: "wide"}
REAL = {"antmaze_umaze": "antmaze", "fetch_reach": "fetch_reach pressed", "fetch_pick_and_place": "fetch grasp",
        "fetch_slide": "fetch_slide", "hand_block_touch": "hand touch", "franka_kitchen": "kitchen pressed",
        "adroit_hammer": "adroit hammer", "adroit_relocate": "adroit relocate"}
NRANDOM = 6
# limits: 4-5x the largest values measured over all cases (DESIGN.md section 2)
POS_C = 16.0      # u L
QUAT_C = 12.0     # u
M_C = 25.0        # nv u


def _random_qpos(m, rng):
    q = np.array(m.qpos0, np.float64)
    rngs = np.asarray(m.jnt_range).reshape(-1, 2)
    for j in range(m.njnt):
        a, t = int(m.jnt_qposadr[j]), int(m.jnt_type[j])
        if t == 0:     # free: a position near the initial one, a random orientation
            q[a:a + 3] += rng.uniform(-0.1, 0.1, 3)
            v = rng.standard_normal(4)
            q[a + 3:a + 7] = v / np.linalg.norm(v)
        elif t == 1:   # ball
            v = rng.standard_normal(4)
            q[a:a + 4] = v / np.linalg.norm(v)
        else:          # slide / hinge
            lo, hi = (rngs[j] if m.jnt_limited[j] else (-np.pi, np.pi))
            q[a] = rng.uniform(lo, hi)
    return q


def _cases(name, penv):
    """(label, oracle sim at the case) for the real state and NRANDOM random joint positions; qpos, mocap and penv rounded to fp32."""
    from gymnasium_robotics_b200.models import load_model
    from oracle.oracle_sim import OracleSim
    from tests.test_device_spd_gpu import _DRIVEN, _contact_state

    m = load_model(name)
    pb = int(m.names["body_map"][penv]) if penv else -1
    label = REAL[name]
    s = _contact_state(label, m) if label in _DRIVEN else None
    if s is None:
        s = OracleSim(m)
        s.step(200)
    out = [(label, s)]
    rng = np.random.default_rng(17)
    for k in range(NRANDOM):
        r = OracleSim(m)
        r.qpos[:] = _random_qpos(m, rng)
        r.mocap_pos[:] = s.mocap_pos
        r.mocap_quat[:] = s.mocap_quat
        if pb > 0:
            r.body_pos[pb] = s.body_pos[pb] + rng.uniform(-0.05, 0.05, 3)
        out.append((f"random qpos {k}", r))
    for _, o in out:
        o.qpos[:] = o.qpos.astype(np.float32)
        o.mocap_pos[:] = o.mocap_pos.astype(np.float32)
        o.mocap_quat[:] = o.mocap_quat.astype(np.float32)
        if pb > 0:
            o.body_pos[pb] = o.body_pos[pb].astype(np.float32)
            o.body_quat[pb] = o.body_quat[pb].astype(np.float32)
        o.forward()
    return m, pb, out


def _run(backend, name, nvp, penv):
    m, pb, cases = _cases(name, penv)
    flavor = FLAVOR[nvp]
    if backend == "gpu":
        from tests import devsim

        sim = devsim.DevModel(flavor, m, penv_body=pb)
        nw = sim.scr_words
    else:
        from tests.hostsim import HostSim

        sim = HostSim(m, penv_body=pb, flavor=HOST_FLAVOR[flavor])
        nw = len(sim.scratch)
    _, _, _, gmap = device_order(m, flavor == "kitchen_groups")
    imgs = np.zeros((len(cases), nw), np.float32)
    for e, (_, o) in enumerate(cases):
        def put(nm, v):
            imgs[e, sim.offset(nm):sim.offset(nm) + len(v)] = v
        put("qpos", o.qpos.ravel())
        if m.nmocap:
            put("mocap_pos", o.mocap_pos.ravel())
            put("mocap_quat", o.mocap_quat.ravel())
        if pb > 0:
            put("penv_pos", np.concatenate([o.body_pos[pb], o.body_quat[pb]]))
    if backend == "gpu":
        sim.run(nvp, devsim.STAGE_KIN, imgs)
    else:
        for e in range(len(cases)):
            sim.scratch[:] = imgs[e]
            sim.kinematics()
            imgs[e] = sim.scratch
    nv, bad, worst = m.nv, [], {"pos": 0.0, "quat": 0.0, "M": 0.0}
    for e, (label, o) in enumerate(cases):
        def get(nm, n):
            return imgs[e, sim.offset(nm):sim.offset(nm) + n].astype(np.float64)
        xpos, xquat = get("xpos", 3 * m.nbody).reshape(-1, 3), get("xquat", 4 * m.nbody).reshape(-1, 4)
        gx = get("geom_xpos", 3 * len(gmap)).reshape(-1, 3)
        ox, oq, og = np.asarray(o.xpos), np.asarray(o.xquat), np.asarray(o.geom_xpos)
        L = max(np.abs(ox).max(), np.abs(og).max(), 1e-3)
        ep = max(np.abs(xpos - ox).max(), max(np.abs(gx[dg] - og[g]).max() for g, dg in gmap.items())) / (U * L)
        eq = np.minimum(np.abs(xquat - oq).max(1), np.abs(xquat + oq).max(1)).max() / U
        P = get("M", nv * (nv + 1) // 2)
        Md = np.zeros((nv, nv))
        Md[np.tril_indices(nv)] = P
        Md = Md + np.tril(Md, -1).T
        Mo = np.asarray(o.M)
        em = np.linalg.norm(Md - Mo) / np.linalg.norm(Mo) / (nv * U)
        worst = {"pos": max(worst["pos"], ep), "quat": max(worst["quat"], eq), "M": max(worst["M"], em)}
        tag = f"{flavor} NVP {nvp} {name} {label}"
        if ep > POS_C:
            bad.append(f"{tag}: xpos / geom_xpos off by {ep:.1f} u L")
        if eq > QUAT_C:
            bad.append(f"{tag}: xquat off by {eq:.1f} u")
        if em > M_C:
            bad.append(f"{tag}: M off by {em:.2f} nv u (normwise)")
    print(f"kinematics [{backend}] {flavor} NVP {nvp} {name}: pos {worst['pos']:.2f} u L, quat {worst['quat']:.2f} u, M {worst['M']:.3f} nv u")
    assert not bad, "\n".join(bad[:20])


@pytest.mark.gpu
@pytest.mark.parametrize("name,nvp,penv", MODELS)
def test_kinematics_on_the_device(name, nvp, penv):
    _run("gpu", name, nvp, penv)


@pytest.mark.parametrize("name,nvp,penv", MODELS)
def test_kinematics_on_the_32_lane_emulation(name, nvp, penv):
    _run("cpu", name, nvp, penv)
