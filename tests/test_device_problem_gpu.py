"""The problem the Newton solver is given, on its own, per product kernel build, against the fp64 oracle: the smooth forces, the
constraint rows (welds, joint and tendon limits, frictionloss, the kitchen's joint equalities, the contacts' pyramid rows), the
implicit Jacobian products J v (rows_begin, rows_from_vec) and J^T f (pass_F), and the Hessian assembly build_H.

Every quantity here is a deterministic function of the injected state, so it has an exact fp64 counterpart; the Newton iterate
itself is only defined up to the solver's tolerance and is not compared.  Each committed model runs on the build and NVP of its
product kernel (tests/devsim STAGE_PROBLEM: every stage forward<NVP> runs up to the first direction solve).  STAGE_JV then runs
rows_from_vec on nv copies of each returned image with the unit vectors e_0 .. e_{nv-1} in `search`: the JV slots read the kernel's
implicit J column by column.

States per model: the contact-heavy oracle state (tests/test_device_spd_gpu.py), random joint positions with large random joint
velocities (free bodies spun at 60 rad/s), a random warm start and controls past both ends of ctrlrange, and every limited joint
driven just past its lower and past its upper side, and the state at rest (frictionloss rows in their quadratic zone).  The models
with frictionloss and tendons (HF: Hand, Adroit, Kitchen) add a copy with jnt_margin raised above half the range, so that both
sides of each joint are active at once; the Hand and Adroit add one with the margins of tendons 32 and up raised (the second 32-lane
chunk of the tendon-limit loop).  The oracle always runs at the fp32-rounded inputs.

Compared, u = 2^-24, L = the largest |coordinate| of the case:
  * fsmooth against qfrc_passive - qfrc_bias + qfrc_actuator per dof, in units of u (|passive_j| + |actuator_j| + |bias_j| +
    ||bias||_inf);
  * dof rows (joint and tendon limits, kitchen joint equalities): dofs, count, order and overflow bit exactly (lower side first,
    joints before tendons; rows past the table's ndr_max dropped and bit 8 set); limit coefficients equal the fp32 oracle +-1 /
    +-tendon coefficient bit for bit;
  * each dof row's D, B and J qacc - aref against the fp64 rule (get_impedance, K, B) evaluated at the kernel's own fp32 distance,
    in units of u times the magnitudes of the terms that enter;
  * the weld rows' and the contacts' J from STAGE_JV against the oracle's efc_J / the fp64 contact row rebuilt with jac_point at the
    kernel's own contact point and frame, normwise in units of u L ||J_row||;
  * the contacts' tangential J qacc - aref (B J qvel + J qacc, no distance term) against the fp64 values; the contacts' D and normal
    row K imp (dist - margin) + B J qvel + J qacc, and the welds' D and J qacc - aref, by the fp64 rule at the oracle's distance /
    residual, the bound carrying the rule's sensitivity to that input times its rounding u L;
  * fcon = J^T f(x) and grad = M qacc - fsmooth - fcon against fp64 sums over the kernel's own rows, and H against
    M + J^T diag(D active) J in fp64 over the kernel's J and recorded activity, componentwise in units of u (|M| + |J|^T D |J|);
  * the contacts' activity bits against the signs of their own stored edge values, the limit rows' against the sign of the fp64
    value where that is far from zero;
  * rows_from_vec writes nothing but the JV slots, make_constraint nothing past the dof-row and weld counts (NaN sentinels), and
    build_H, run again (STAGE_BUILD_H), rebuilds H bit for bit and writes nothing past its nM + 21 kcap words.
Contacts are paired with the oracle's by position and normal, and by their rows where several share a point; where the collision
stage's caps were hit the kept contacts are compared as a subset of the oracle's.
Unlike the collision test, no oracle ensemble is run: every reference is evaluated at the kernel's own fp32 inputs where the
scratch keeps them, and where it does not, the bound carries the sensitivity to the one input the kernel rounds itself.
The limits are 4-5x the largest values measured on the H100 and on the 32-lane emulation (DESIGN.md section 2).
"""
import copy

import numpy as np
import pytest

from tests.test_device_collide_gpu import HOST_FLAVOR
from tests.test_device_kin_gpu import FLAVOR, MODELS, REAL, _random_qpos

U = 2.0 ** -24
SENTINEL = np.uint32(0x7FC0FEED)   # a quiet NaN whose payload no stage writes
NRANDOM = 3
ROW_EQ, ROW_FRICTION, ROW_LIMIT = 0, 1, 2   # oracle.c efc_type
DR_DOF, DR_COEF, DR_D, DR_JAR, DR_JV, DR_DOF2, DR_COEF2, DR_WORDS = range(8)   # dmodel.h
W_W, W_D, W_JAR, W_JV, WELD_WORDS = 0, 36, 42, 48, 56   # dmodel.h
CNT_NCON, CNT_NDR, CNT_NGRP, CNT_NWELD, CNT_OVERFLOW = 0, 1, 2, 4, 6
# limits: 4-5x the largest values measured over all cases (DESIGN.md section 2)
LIM = {"fsmooth": 600.0, "dofrow": 12.0, "weld J": 24.0, "weld x": 12.0, "weld D": 8.0, "contact J": 16.0, "contact x": 3.0,
       "contact n": 6.0, "contact D": 6.0, "fcon": 10.0, "grad": 24.0, "H": 10.0}
PAIR_TOL = 1e-3   # a kept contact and its oracle twin: position + L * normal apart, in units of L


def _impedance(si, pos, margin):
    """oracle.c get_impedance in fp64."""
    si = np.array(si, np.float64)
    si[:2] = np.clip(si[:2], 1e-4, 0.9999)
    si[2] = max(si[2], 0.0)
    si[3] = min(max(si[3], 1e-4), 0.9999)
    si[4] = max(si[4], 1.0)
    if si[0] == si[1] or si[2] <= 1e-15:
        return 0.5 * (si[0] + si[1])
    x = abs((pos - margin) / si[2])
    if x >= 1:
        return si[1]
    if x <= 0:
        return si[0]
    if si[4] == 1:
        y = x
    elif x <= si[3]:
        y = x ** si[4] / si[3] ** (si[4] - 1)
    else:
        y = 1 - (1 - x) ** si[4] / (1 - si[3]) ** (si[4] - 1)
    return si[0] + y * (si[1] - si[0])


def _slope(f, x, si):
    """|df/dx| by a central difference one thousandth of the impedance width wide (the width sets where imp varies)."""
    h = max(1e-3 * float(si[2]), 1e-9)
    return (f(x + h) - f(x - h)) / (2 * h)


def _with_margin(m):
    """A copy of the model whose limited joints and tendons have margins above half their range: both sides of each are active at
    once (past 48 rows on the Hand and Adroit: the table's overflow rule at its cap)."""
    m2 = copy.deepcopy(m)
    if m2.ntendon:
        tr = np.asarray(m2.ten_range, np.float64).reshape(-1, 2)
        m2.ten_margin = 0.6 * (tr[:, 1] - tr[:, 0])
    rng = np.asarray(m2.jnt_range, np.float64).reshape(-1, 2)
    mg = np.array(m2.jnt_margin, np.float64)
    for j in range(m2.njnt):
        if m2.jnt_limited[j] and m2.jnt_type[j] != 0:
            mg[j] = 0.6 * (rng[j, 1] - rng[j, 0])
    m2.jnt_margin = mg
    return m2


def _states(name, penv):
    """(model, penv body, [(label, model copy or None, input dict)]); every input is fp32-representable."""
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
    base = dict(qpos=np.array(s.qpos), qvel=np.array(s.qvel), qacc=np.array(s.qacc), ctrl=np.array(s.ctrl),
                mocap_pos=np.array(s.mocap_pos), mocap_quat=np.array(s.mocap_quat),
                pose=(np.array(s.body_pos[pb]), np.array(s.body_quat[pb])) if pb > 0 else None)
    out = [(label, None, base)]
    rng = np.random.default_rng(23)
    free = [int(m.jnt_dofadr[j]) for j in range(m.njnt) if int(m.jnt_type[j]) == 0]
    cr = np.asarray(m.act_ctrlrange, np.float64).reshape(-1, 2) if m.nu else np.zeros((0, 2))
    jr = np.asarray(m.jnt_range, np.float64).reshape(-1, 2)

    def wild(st):
        st = dict(st)
        st["qvel"] = rng.normal(0.0, 3.0, m.nv)
        for d in free:   # free bodies spun fast: the velocity products of the rotational dofs (dof_pre's free-joint rule)
            w = rng.standard_normal(3)
            st["qvel"][d + 3:d + 6] = 60.0 * w / np.linalg.norm(w)
        st["qacc"] = rng.normal(0.0, 20.0, m.nv)   # pyramid edges on both sides of zero
        w = cr[:, 1] - cr[:, 0]
        side = rng.random(m.nu) < 0.5   # ctrl past one end of ctrlrange or the other
        st["ctrl"] = np.where(side, cr[:, 0] - rng.uniform(0.05, 1.0, m.nu) * w, cr[:, 1] + rng.uniform(0.05, 1.0, m.nu) * w)
        return st

    for k in range(NRANDOM):
        st = dict(base)
        st["qpos"] = _random_qpos(m, rng)
        if pb > 0:
            st["pose"] = (base["pose"][0] + rng.uniform(-0.05, 0.05, 3), base["pose"][1])
        out.append((f"random {k}", None, wild(st)))
    for side, nm in ((0, "lower"), (1, "upper")):   # every limited joint just past one side of its range
        st = dict(base)
        q = np.array(base["qpos"])
        for j in range(m.njnt):
            if m.jnt_limited[j] and int(m.jnt_type[j]) != 0:
                lo, hi = jr[j]
                d = 0.02 * (hi - lo) + 1e-3
                q[int(m.jnt_qposadr[j])] = lo - d if side == 0 else hi + d
        st["qpos"] = q
        out.append((f"every limit {nm}", None, wild(st)))
    st = dict(base)   # at rest: the frictionloss rows in their quadratic zone
    st["qvel"], st["qacc"] = np.zeros(m.nv), np.zeros(m.nv)
    out.append(("rest", None, st))
    if m.ntendon or m.neq and int(m.eq_type[0]) == 2 or np.any(np.asarray(m.dof_frictionloss) > 0):
        mm = _with_margin(m)
        for k in range(2):
            st = dict(base)
            st["qpos"] = _random_qpos(m, rng)
            out.append((f"margin {k}", mm, wild(st)))
    if m.ntendon > 32:   # tendons 32 and up, both sides active: the second 32-lane chunk of the tendon-limit loop
        mt = copy.deepcopy(m)
        tr = np.asarray(mt.ten_range, np.float64).reshape(-1, 2)
        tm = np.array(mt.ten_margin, np.float64)
        tm[32:] = 0.6 * (tr[32:, 1] - tr[32:, 0])
        mt.ten_margin = tm
        out.append(("tendon margin", mt, wild(dict(base))))
    for _, _, st in out:
        for key in ("qpos", "qvel", "qacc", "ctrl", "mocap_pos", "mocap_quat"):
            st[key] = np.asarray(st[key], np.float64).astype(np.float32).astype(np.float64)
        if st["pose"] is not None:
            st["pose"] = tuple(np.asarray(a, np.float32).astype(np.float64) for a in st["pose"])
    return m, pb, out


def _oracle(m, pb, st):
    from oracle.oracle_sim import OracleSim

    o = OracleSim(m)
    o.qpos[:] = st["qpos"]
    o.qvel[:] = st["qvel"]
    o.ctrl[:] = st["ctrl"]
    o.mocap_pos[:] = st["mocap_pos"]
    o.mocap_quat[:] = st["mocap_quat"]
    if pb > 0:
        o.body_pos[pb], o.body_quat[pb] = st["pose"]
    o.forward()
    return o


class _Sim:
    """One model on one backend: the device harness (gpu) or the 32-lane emulation (cpu), batches of scratch images."""

    def __init__(self, backend, flavor, nvp, m, pb):
        self.backend, self.nvp, self.m = backend, nvp, m
        if backend == "gpu":
            from tests import devsim

            self.sim = devsim.DevModel(flavor, m, penv_body=pb)
            self.nw = self.sim.scr_words
        else:
            from tests.hostsim import HostSim

            self.sim = HostSim(m, penv_body=pb, flavor=HOST_FLAVOR[flavor])
            self.nw = len(self.sim.scratch)
        self.o = {k: self.sim.offset(k) for k in ("qpos", "qvel", "qacc", "ctrl", "mocap_pos", "mocap_quat", "M", "fsmooth", "fcon",
                                                  "con", "dofrow", "weld", "group", "counters", "fric", "conx", "H", "grad", "cdof",
                                                  "search", "Ma")}
        lay = self.sim.layout
        self.lay = dict(lay)
        self.lay["C_D"] = lay["C_U"] - 1
        self.lay["NB"] = (lay["C_DIMGRP"] - lay["C_U"]) // 2
        self.lay["C_JV"] = lay["C_U"] + self.lay["NB"]
        o = self.o
        self.ncon_max = (o["dofrow"] - o["con"]) // lay["CON_WORDS"]
        self.ndr_max = (o["weld"] - o["dofrow"]) // DR_WORDS
        self.nfric = (o["conx"] - o["fric"]) // 2
        nv = m.nv
        self.nM = nv * (nv + 1) // 2
        self.kcap = (o["grad"] - o["H"] - self.nM) // 21
        self.mwords = np.asarray(self.sim.words).view(np.float32)

    def marr(self, name, n):
        return self.mwords[self.sim.model_offset(name):self.sim.model_offset(name) + n].astype(np.float64)

    def image(self, st, pb):
        s = np.zeros(self.nw, np.float32)
        o = self.o

        def put(nm, v):
            v = np.asarray(v, np.float32).ravel()
            s[self.sim.offset(nm):self.sim.offset(nm) + len(v)] = v
        put("qpos", st["qpos"]), put("qvel", st["qvel"]), put("qacc", st["qacc"])
        if self.m.nu:
            put("ctrl", st["ctrl"])
        if self.m.nmocap:
            put("mocap_pos", st["mocap_pos"]), put("mocap_quat", st["mocap_quat"])
        if pb > 0:
            put("penv_pos", np.concatenate(st["pose"]))
        # contact, dof-row and weld slots: written only up to their counts.  (The contact slots past CNT_NCON double as the narrow
        # phase's lane slots, dmodel.h s_cslotB, so only the kept records are checked: they must be whole.)
        s.view(np.uint32)[o["con"]:o["weld"] + WELD_WORDS] = SENTINEL
        return s

    def run(self, stage, imgs):
        if self.backend == "gpu":
            self.sim.run(self.nvp, stage, imgs)
            return
        for e in range(len(imgs)):
            self.sim.scratch[:] = imgs[e]
            {2: self.sim.problem, 3: self.sim.jv, 4: self.sim.build_h}[stage](self.nvp)
            imgs[e] = self.sim.scratch


def _rows(sim, img):
    """The kernel's rows of one image as fp64 records."""
    lay, o, m = sim.lay, sim.o, sim.m
    cnt = img[o["counters"]:o["counters"] + 8].view(np.int32)
    ncon, ndr, ngrp, nweld, ovf = (int(cnt[k]) for k in (CNT_NCON, CNT_NDR, CNT_NGRP, CNT_NWELD, CNT_OVERFLOW))
    cw = lay["CON_WORDS"]
    cons = img[o["con"]:o["con"] + ncon * cw].reshape(ncon, cw) if ncon else np.zeros((0, cw), np.float32)
    drs = img[o["dofrow"]:o["dofrow"] + ndr * DR_WORDS].reshape(ndr, DR_WORDS) if ndr else np.zeros((0, DR_WORDS), np.float32)
    welds = img[o["weld"]:o["weld"] + nweld * WELD_WORDS].reshape(nweld, WELD_WORDS)
    return dict(ncon=ncon, ndr=ndr, ngrp=ngrp, nweld=nweld, ovf=ovf, cons=cons.copy(), drs=drs.copy(), welds=welds.copy())


def _con_fields(lay, w):
    dg = int(w[lay["C_DIMGRP"]:lay["C_DIMGRP"] + 1].view(np.int32)[0])
    dim = dg & 0xFF
    mu = [float(w[lay["C_MU"]])] * 3 + [float(w[lay["C_MU"] + 1])] + [float(w[lay["C_MU"] + 2])] * 2 if lay["NB"] == 6 else \
         [float(w[lay["C_MU"]])] * 3 + [float(w[lay["C_MU"] + 1])]
    return dim, (dg >> 8) & 0xFF, (dg >> 16) & 0xFFFF, mu


def _run(backend, name, nvp, penv, stats, flavor):
    m0, pb, states = _states(name, penv)
    sims = {}
    nv = m0.nv
    rec = []
    for label, mm, st in states:
        m = mm if mm is not None else m0
        key = id(mm)
        if key not in sims:
            sims[key] = _Sim(backend, flavor, nvp, m, pb)
        rec.append((label, m, sims[key], st))
    # STAGE_PROBLEM per case, then STAGE_JV on nv copies of each result
    out = []
    for key, sim in sims.items():
        mine = [r for r in rec if r[2] is sim]
        imgs = np.stack([sim.image(st, pb) for _, _, _, st in mine])
        sim.run(2, imgs)
        jv = np.repeat(imgs, nv, axis=0)
        for e in range(len(mine)):
            for k in range(nv):
                jv[e * nv + k, sim.o["search"]:sim.o["search"] + nv] = np.eye(nv, dtype=np.float32)[k]
        before = jv.copy()
        sim.run(3, jv)
        # build_H alone again on the returned images, the H region past its 21 kcap block words filled with sentinels: it must
        # rebuild H bit for bit and leave the sentinels
        hb = imgs.copy()
        h0 = sim.o["H"] + sim.nM + 21 * sim.kcap
        hb.view(np.uint32)[:, h0:sim.o["grad"]] = SENTINEL
        sim.run(4, hb)
        for e, r in enumerate(mine):
            out.append((r, imgs[e], jv[e * nv:(e + 1) * nv], before[e * nv:(e + 1) * nv], hb[e]))
    bad = []
    for (label, m, sim, st), img, jv, jv0, hb in out:
        tag = f"{flavor} NVP {nvp} {name} [{label}]"
        h0, hg = sim.o["H"], sim.o["grad"]
        if np.any(hb.view(np.uint32)[h0:h0 + sim.nM] != img.view(np.uint32)[h0:h0 + sim.nM]):
            bad.append(f"{tag}: build_H run again on the same image gives a different H")
        if np.any(hb.view(np.uint32)[h0 + sim.nM + 21 * sim.kcap:hg] != SENTINEL):
            bad.append(f"{tag}: build_H wrote past its K blocks (H + nM + 21 kcap = {sim.nM + 21 * sim.kcap} .. {hg - h0})")
        _check_case(tag, m, pb, sim, st, img, jv, jv0, stats, bad)
    return bad


def _jv_written(sim, r):
    """Mask of the words rows_from_vec may write: the groups' dV, the contacts' and welds' JV slots, the dof rows' JV, fric[nfric:]."""
    lay, o = sim.lay, sim.o
    w = np.zeros(sim.nw, bool)
    gw = lay["GRP_WORDS"]
    gv = {11: 5, 9: 3}[gw]
    for g in range(r["ngrp"]):
        w[o["group"] + g * gw + gv:o["group"] + g * gw + gv + 6] = True
    for i in range(r["ncon"]):
        w[o["con"] + i * lay["CON_WORDS"] + lay["C_JV"]:o["con"] + i * lay["CON_WORDS"] + lay["C_JV"] + lay["NB"]] = True
    for i in range(r["nweld"]):
        w[o["weld"] + i * WELD_WORDS + W_JV:o["weld"] + i * WELD_WORDS + W_JV + 6] = True
    for i in range(r["ndr"]):
        w[o["dofrow"] + i * DR_WORDS + DR_JV] = True
    w[o["fric"] + sim.nfric:o["fric"] + 2 * sim.nfric] = True
    return w


def _check_case(tag, m, pb, sim, st, img, jv, jv0, stats, bad):
    nv = m.nv
    lay = sim.lay
    orc = _oracle(m, pb, st)
    r = _rows(sim, img)
    qvel, qacc = st["qvel"], st["qacc"]
    L = max(float(np.abs(orc.xpos).max()), 1.0)
    worst = stats["worst"]

    def note(key, v, where):
        worst[key] = max(worst.get(key, 0.0), v)
        if v > LIM[key]:
            bad.append(f"{tag}: {where}: {v:.1f} (limit {LIM[key]})")

    # STAGE_JV writes only the JV slots; everything else must come back bit for bit
    wm = _jv_written(sim, r)
    wm[sim.o["search"]:sim.o["search"] + nv] = False
    ch = np.nonzero(np.any(jv.view(np.uint32)[:, ~wm] != jv0.view(np.uint32)[:, ~wm], axis=0))[0]
    if len(ch):
        bad.append(f"{tag}: rows_from_vec wrote {len(ch)} words outside the JV slots (first at {np.nonzero(~wm)[0][ch[0]]})")
    # the dof-row and weld slots past their counts keep the sentinel
    u32 = img.view(np.uint32)
    recs = u32[sim.o["con"]:sim.o["con"] + r["ncon"] * lay["CON_WORDS"]].reshape(r["ncon"], lay["CON_WORDS"])
    if np.any(recs[:, :lay["C_DIMGRP"] + 1] == SENTINEL):
        bad.append(f"{tag}: a kept contact record is not whole (a word keeps the sentinel)")
    dr_tail = u32[sim.o["dofrow"] + r["ndr"] * DR_WORDS:sim.o["dofrow"] + sim.ndr_max * DR_WORDS]
    if np.any(dr_tail != SENTINEL):
        bad.append(f"{tag}: make_constraint wrote dof-row slots past CNT_NDR = {r['ndr']}")
    if r["nweld"] == 0 and np.any(u32[sim.o["weld"]:sim.o["weld"] + WELD_WORDS] != SENTINEL) or \
            r["nweld"] == 1 and np.any(u32[sim.o["weld"] + np.r_[0:W_JV, W_JV + 6:WELD_WORDS]] == SENTINEL):
        bad.append(f"{tag}: make_constraint wrote the unused weld slot, or left a word of the used one unwritten")

    # ---- smooth forces
    fs = img[sim.o["fsmooth"]:sim.o["fsmooth"] + nv].astype(np.float64)
    fo = np.asarray(orc.qfrc_passive) - np.asarray(orc.qfrc_bias) + np.asarray(orc.qfrc_actuator)
    # per dof: its own passive and actuator terms (single products, rounded in their own units) and the bias in units of the largest
    # bias component (the recursive Newton-Euler sums cancel across the tree)
    scale = np.abs(orc.qfrc_passive) + np.abs(orc.qfrc_actuator) + np.abs(orc.qfrc_bias) + np.abs(orc.qfrc_bias).max()
    note("fsmooth", np.max(np.abs(fs - fo) / (U * np.maximum(scale, 1e-30))), "smooth_forces: fsmooth")

    # ---- kernel J, column by column
    Jc = [np.stack([jv[k, sim.o["con"] + i * lay["CON_WORDS"] + lay["C_JV"]:
                        sim.o["con"] + i * lay["CON_WORDS"] + lay["C_JV"] + lay["NB"]] for k in range(nv)], 1).astype(np.float64)
          for i in range(r["ncon"])]                                   # [NB, nv] per contact
    Jw = [np.stack([jv[k, sim.o["weld"] + i * WELD_WORDS + W_JV:sim.o["weld"] + i * WELD_WORDS + W_JV + 6] for k in range(nv)],
                   1).astype(np.float64) for i in range(r["nweld"])]    # [6, nv] per weld
    Jd = np.stack([jv[k, sim.o["dofrow"] + np.arange(r["ndr"]) * DR_WORDS + DR_JV] for k in range(nv)], 1).astype(np.float64) \
        if r["ndr"] else np.zeros((0, nv))
    Jf = np.stack([jv[k, sim.o["fric"] + sim.nfric:sim.o["fric"] + 2 * sim.nfric] for k in range(nv)], 1).astype(np.float64)
    if sim.nfric and not np.array_equal(Jf, np.eye(nv)):
        bad.append(f"{tag}: rows_from_vec: the frictionloss rows' J is not the identity")

    cn = np.linalg.norm(img[sim.o["cdof"]:sim.o["cdof"] + 6 * nv].astype(np.float64).reshape(nv, 6), axis=1)
    cmax = cn.max()
    otype, oid, oJ = orc.efc("type"), orc.efc("id"), orc.efc("J")
    KBIP, opos, omarg = orc.efc("KBIP"), orc.efc("pos"), orc.efc("margin")
    oaref = orc.efc("aref")
    ox = oJ @ qacc - oaref
    cov = stats["rows"]

    # ---- dof rows: limits (joints, lower side first, then tendons), then the kitchen's joint equalities
    lim = [i for i in range(len(otype)) if otype[i] == ROW_LIMIT]
    eqj = [i for i in range(len(otype)) if otype[i] == ROW_EQ and int(m.eq_type[oid[i]]) == 2]
    want = lim + eqj
    nkeep = min(len(want), sim.ndr_max)
    over = bool(r["ovf"] & 8)
    if r["ndr"] != nkeep or over != (len(want) > sim.ndr_max):
        bad.append(f"{tag}: make_constraint: {r['ndr']} dof rows (overflow bit 8 {over}), the oracle has {len(want)} limit / joint-"
                   f"equality rows and the table holds {sim.ndr_max}")
        return
    if over:
        stats["overflow"].append(f"{tag}: {len(want)} rows, {sim.ndr_max} kept")
    if nkeep == sim.ndr_max and not over:
        stats["full"].append(tag)
    rng_j = np.asarray(m.jnt_range, np.float64).reshape(-1, 2)
    for k, i in enumerate(want[:nkeep]):
        dr = r["drs"][k]
        di = dr.view(np.int32)
        row = np.zeros(nv)
        row[di[DR_DOF]] += float(dr[DR_COEF])
        if di[DR_DOF2] >= 0:
            row[di[DR_DOF2]] += float(dr[DR_COEF2])
        if not np.array_equal(Jd[k], row):
            bad.append(f"{tag}: rows_from_vec: dof row {k} reads back J {Jd[k][Jd[k] != 0]} but its table says {row[row != 0]}")
        kind = "eq" if otype[i] == ROW_EQ else ("tendon" if oid[i] >= m.njnt else "joint")
        oj = oJ[i]
        if kind == "eq":
            d1 = int(m.jnt_dofadr[m.eq_obj1[oid[i]]])
            if di[DR_DOF] != d1 or float(dr[DR_COEF]) != 1.0 or float(dr[DR_D]) >= 0:
                bad.append(f"{tag}: make_constraint: kitchen joint-equality row {k} is not (dof {d1}, 1, two-sided D < 0)")
            nz = [d for d in np.nonzero(oj)[0] if d != d1]
            if nz and (di[DR_DOF2] != nz[0] or abs(dr[DR_COEF2] - oj[nz[0]]) > 64 * U * (abs(oj[nz[0]]) + 1.0)):
                bad.append(f"{tag}: make_constraint: kitchen joint-equality row {k}: -poly' {dr[DR_COEF2]} vs {oj[nz[0]]}")
            cov.add("kitchen joint equality")
        else:
            if not np.array_equal(row, oj.astype(np.float32).astype(np.float64)):
                bad.append(f"{tag}: make_constraint: {kind}-limit row {k} (oracle id {oid[i]}): J {row[row != 0]} at dofs "
                           f"{np.nonzero(row)[0]} vs the oracle's {oj[oj != 0]} at {np.nonzero(oj)[0]}")
                continue
            two = sum(1 for i2 in lim if oid[i2] == oid[i]) == 2
            cov.add("tendon limit" if kind == "tendon" else ("two-sided limit" if two else
                                                             ("lower limit" if oj[np.nonzero(oj)[0][0]] > 0 else "upper limit")))
            if max(abs(di[DR_DOF]), abs(di[DR_DOF2])) >= 32 or oid[i] - (m.njnt if kind == "tendon" else 0) >= 32:
                cov.add("index >= 32")
        # D, B and J qacc - aref by the fp64 rule at the kernel's own fp32 distance
        K, B = KBIP[i, 0], KBIP[i, 1]
        if kind == "joint":
            j = int(oid[i])
            q = np.float32(st["qpos"][int(m.jnt_qposadr[j])])
            lower = oj[int(m.jnt_dofadr[j])] > 0
            dist = float(q - np.float32(rng_j[j, 0])) if lower else float(np.float32(rng_j[j, 1]) - q)
            si, iw, marg = np.ravel(m.jnt_solimp)[5 * j:5 * j + 5], np.ravel(m.dof_invweight0)[int(m.jnt_dofadr[j])], float(np.float32(m.jnt_margin[j]))
            dscale = abs(float(q)) + np.abs(rng_j[j]).max() + abs(marg)
        elif kind == "tendon":
            dist, marg = opos[i], omarg[i]   # the fp32 tendon length is not stored: the oracle's, with the length's rounding
            t = int(oid[i]) - m.njnt
            si, iw = np.ravel(m.ten_solimp)[5 * t:5 * t + 5], np.ravel(m.ten_invweight0)[t]
            dscale = np.abs(oj) @ np.abs(st["qpos"][[int(m.jnt_qposadr[int(m.dof_jnt[d])]) for d in range(nv)]]) + \
                np.abs(np.asarray(m.ten_range).reshape(-1, 2)[t]).max() + abs(marg)
        else:
            dist, marg = opos[i], 0.0
            e = int(oid[i])
            si, iw = np.ravel(m.eq_solimp)[5 * e:5 * e + 5], np.ravel(m.eq_invweight)[2 * e]
            # pos = q1 - q1_0 - poly(q2 - q2_0): the magnitudes of its terms (the residual's rounding)
            data = np.asarray(orc.eq_data[e], np.float64)
            a1, a2 = int(m.jnt_qposadr[m.eq_obj1[e]]), int(m.jnt_qposadr[m.eq_obj2[e]])
            dif = abs(st["qpos"][a2] - m.qpos0[a2])
            dscale = abs(st["qpos"][a1]) + abs(m.qpos0[a1]) + sum(abs(data[p]) * dif ** p for p in range(5)) + \
                (abs(st["qpos"][a2]) + abs(m.qpos0[a2])) * sum(p * abs(data[p]) * dif ** (p - 1) for p in range(1, 5))
        imp = _impedance(si, dist, marg)
        Dref = 1.0 / max((1 - imp) / imp * iw, 1e-15)
        ed = abs(abs(float(dr[DR_D])) - Dref) / (U * Dref * (1 + 1 / (1 - imp)))
        eb = abs(float(dr[DR_JV]) - B) / (U * B)
        xr = K * imp * (dist - marg) + B * (oj @ qvel) + oj @ qacc
        xs = K * imp * dscale + K * abs(dist - marg) + B * (np.abs(oj) @ np.abs(qvel)) + np.abs(oj) @ np.abs(qacc)
        ex = abs(float(dr[DR_JAR]) - xr) / (U * xs)
        note("dofrow", max(ed, eb, ex), f"make_constraint / rows_begin: {kind} row {k}: D {ed:.1f}, B {eb:.1f}, J qacc - aref {ex:.1f} u")
        if kind != "eq" and abs(xr) > 8 * LIM["dofrow"] * U * xs and (float(dr[DR_JAR]) < 0) != (xr < 0):
            bad.append(f"{tag}: rows_begin: {kind} row {k} activity {float(dr[DR_JAR])} vs {xr}")

    # ---- welds: J against efc_J, D and J qacc - aref against the oracle
    wrows = [i for i in range(len(otype)) if otype[i] == ROW_EQ and int(m.eq_type[oid[i]]) == 1]
    if len(wrows) != 6 * r["nweld"]:
        bad.append(f"{tag}: make_constraint: {r['nweld']} welds, the oracle has {len(wrows) // 6}")
        return
    for wi in range(r["nweld"]):
        cov.add("weld")
        w = r["welds"][wi]
        for k in range(6):
            i = wrows[6 * wi + k]
            ej = np.linalg.norm(Jw[wi][k] - oJ[i]) / (U * max(L * np.linalg.norm(oJ[i]), np.linalg.norm(w[W_W + 6 * k:W_W + 6 * k + 6]) * cmax))
            note("weld J", ej, f"make_constraint / rows_from_vec: weld row {k} J")
            # D and aref at the oracle's residual; the kernel's residual is rounded in units of u L, so the bounds carry the
            # sensitivity of D and of K imp r to the residual, times L
            e = int(oid[i])
            si = np.ravel(m.eq_solimp)[5 * e:5 * e + 5]
            iw = np.ravel(m.eq_invweight)[2 * e + (0 if k < 3 else 1)]
            Dfun = (lambda pp: 1.0 / max((1 - _impedance(si, pp, 0.0)) / _impedance(si, pp, 0.0) * iw, 1e-15))
            imp = KBIP[i, 2]
            Dr = Dfun(opos[i])
            note("weld D", abs(float(w[W_D + k]) - Dr) / (U * (Dr * (1 + 1 / (1 - imp)) + abs(_slope(Dfun, opos[i], si)) * L)),
                 f"make_constraint: weld row {k} D")
            K, B = KBIP[i, 0], KBIP[i, 1]
            sens = abs(_slope(lambda pp: K * _impedance(si, pp, 0.0) * pp, opos[i], si))
            xs = K * imp * (abs(opos[i]) + L) + sens * L + \
                (B * np.linalg.norm(oJ[i]) * np.linalg.norm(qvel) + np.linalg.norm(oJ[i]) * np.linalg.norm(qacc)) * L
            note("weld x", abs(float(w[W_JAR + k]) - ox[i]) / (U * xs), f"make_constraint / rows_begin: weld row {k} J qacc - aref")

    # ---- contacts: J at the kernel's own point and frame, the tangential rows' J qacc - aref, activity bits
    ocons = [c for c in orc.contacts() if c["efc_address"] >= 0]
    kc = []
    for w in r["cons"]:
        f = [w[6 * a + 3:6 * a + 6].astype(np.float64) for a in range(3)]
        p = np.asarray(sim.sim.ref, np.float64) + 0.5 * sum(np.cross(f[a], w[6 * a:6 * a + 3].astype(np.float64)) for a in range(3))
        kc.append((p, np.array(f)))
    # Every kept contact is paired with the nearest unused oracle contact by position and normal.  Where the collision stage's caps
    # were hit (overflow bits 2 / 4, tests/test_device_collide_gpu.py) the kept contacts are a subset of the oracle's and are paired
    # the same way; a case whose contacts do not all find their oracle twin (within PAIR_TOL L) counts as skipped.
    # Contacts at one point (several geom pairs of one foot) are told apart by their rows: of the oracle contacts within PAIR_TOL
    # the one whose fp64 rows at the kernel's point and frame come closest to the kernel's J.
    capped = bool(r["ovf"] & 6) and len(ocons) > r["ncon"]
    gb = np.asarray(m.geom_body)
    nefc = len(otype)

    def rows_at(oc, p, F, nb):
        jp1, jr1 = orc.jac_point(int(gb[oc["geom1"]]), p)
        jp2, jr2 = orc.jac_point(int(gb[oc["geom2"]]), p)
        return [F[k] @ (jp2 - jp1) if k < 3 else F[k - 3] @ (jr2 - jr1) for k in range(nb)]

    pairs = []
    if len(ocons) < r["ncon"] or (len(ocons) > r["ncon"] and not capped):
        stats["skipped"].append(f"{tag}: {r['ncon']} contacts, the oracle {len(ocons)}")
    else:
        used = set()
        for ci, (p, F) in enumerate(kc):
            dim = _con_fields(lay, r["cons"][ci])[0]
            nb = 1 if dim == 1 else dim
            near = [j for j in range(len(ocons)) if j not in used and
                    np.linalg.norm(ocons[j]["pos"] - p) + np.linalg.norm(ocons[j]["frame"][0] - F[0]) * L <= PAIR_TOL * L]
            if not near:
                stats["cskip"].append(f"{tag}: kept contact {ci} has no oracle contact within {PAIR_TOL} L")
                continue
            best = min(near, key=lambda j: sum(np.linalg.norm(Jc[ci][k] - rr) for k, rr in enumerate(rows_at(ocons[j], p, F, nb))))
            used.add(best)
            pairs.append((ci, ocons[best]))
        if capped:
            stats["capped"].append(f"{tag}: {r['ncon']} of the oracle's {len(ocons)} contacts kept (overflow {r['ovf'] & 7}), "
                                   f"compared as a subset")
    oD = orc.efc("D")
    for ci, oc in pairs:
        p, F = kc[ci]
        w = r["cons"][ci]
        dim, _, act, mu = _con_fields(lay, w)
        i0 = oc["efc_address"]
        if i0 + max(2 * (dim - 1), 1) > nefc:   # the oracle's own row table (MAXEFC) ran out before this contact's rows
            stats["capped"].append(f"{tag}: contact {ci} not compared: the oracle's own row table is full")
            continue
        if oc["dim"] != dim:
            bad.append(f"{tag}: collision: contact {ci} has condim {dim}, its oracle twin {oc['dim']}")
            continue
        stats["contacts"] += 1
        K, B, imp_o = KBIP[i0, 0], KBIP[i0, 1], KBIP[i0, 2]
        si = np.ravel(m.pair_solimp)[5 * oc["pair"]:5 * oc["pair"] + 5]
        nb = 1 if dim == 1 else dim
        for k, ref in enumerate(rows_at(oc, p, F, nb)):
            sw = _wnorm(w, k)
            ej = np.linalg.norm(Jc[ci][k] - ref) / (U * max(L * np.linalg.norm(ref), sw * cmax))
            note("contact J", ej, f"collision / rows_from_vec: contact {ci} (condim {dim}) base row {k} J")
            # the rounding of B J qvel + J qacc: the group velocity sum cdof v is dotted with the spatial row vector w
            xs = (B * np.abs(ref) @ np.abs(qvel) + np.abs(ref) @ np.abs(qacc)) * L + sw * (B * cn @ np.abs(qvel) + cn @ np.abs(qacc))
            xr = B * (ref @ qvel) + ref @ qacc
            if k >= 1:   # tangential base rows: U = B J qvel + J qacc (no distance term)
                note("contact x", abs(float(w[lay["C_U"] + k]) - xr) / (U * max(xs, 1e-30)),
                     f"rows_begin: contact {ci} base row {k} J qacc - aref")
            else:
                # normal row: U = K imp (dist - margin) + B J qvel + J qacc at the kernel's dist, which the collider rounds in units of
                # u L (the oracle's dist stands for it, with the aref's sensitivity to dist in the bound)
                d_o, mg = opos[i0], omarg[i0]
                kd = K * _impedance(si, d_o, mg) * (d_o - mg)
                sens = abs(_slope(lambda d: K * _impedance(si, d, mg) * (d - mg), d_o, si))
                ns = K * imp_o * (abs(d_o) + abs(mg)) + sens * L + xs
                note("contact n", abs(float(w[lay["C_U"]]) - kd - xr) / (U * ns),
                     f"collision / rows_begin: contact {ci} (condim {dim}) normal row J qacc - aref (K imp (dist - margin) + B J v)")
        # D = 1 / R by the fp64 rule at the oracle's dist: R = (1 - imp) / imp * invweight, the pyramid's 2 mu^2 R0 taken from the
        # oracle's row (the impedance is the only input the kernel computes itself)
        Dfun = (lambda d: oD[i0] * (1 - imp_o) / imp_o * _impedance(si, d, omarg[i0]) / (1 - _impedance(si, d, omarg[i0])))
        Dr = Dfun(opos[i0])
        imp = _impedance(si, opos[i0], omarg[i0])
        dsc = Dr * (1 + 1 / (1 - imp)) + abs(_slope(Dfun, opos[i0], si)) * L
        note("contact D", abs(float(w[lay["C_D"]]) - Dr) / (U * dsc), f"collision: contact {ci} (condim {dim}) D = 1 / R")
        # activity against the oracle's edges where those are far from zero (pyramid rows: + then - per base row k)
        Uc = w[lay["C_U"]:lay["C_U"] + lay["NB"]].astype(np.float64)
        edges = [(0, 0, 1.0)] if dim == 1 else [(2 * k - 2 + s, k, 1 - 2 * s) for k in range(1, dim) for s in (0, 1)]
        for b, k, sg in edges:
            xo = ox[i0 + b]
            thr = 4 * LIM["contact n"] * U * (K * imp_o * (abs(opos[i0]) + L) + abs(_slope(
                lambda d: K * _impedance(si, d, omarg[i0]) * (d - omarg[i0]), opos[i0], si)) * L +
                (B * np.abs(oJ[i0 + b]) @ np.abs(qvel) + np.abs(oJ[i0 + b]) @ np.abs(qacc)) * L * (1 + cmax))
            if abs(xo) > thr and bool((act >> b) & 1) != (xo < 0):
                bad.append(f"{tag}: rows_begin: contact {ci} edge bit {b} is {(act >> b) & 1}, the oracle's edge value {xo}")
    # the contacts' activity bits: the signs of their own stored edges
    for ci, w in enumerate(r["cons"]):
        dim, _, act, mu = _con_fields(lay, w)
        cov.add(f"contact condim {dim}")
        Uc = w[lay["C_U"]:lay["C_U"] + lay["NB"]].astype(np.float64)
        if dim == 1:
            exp = [(0, Uc[0], abs(Uc[0]))]
        else:
            exp = [(2 * k - 2 + s, Uc[0] + (1 - 2 * s) * mu[k] * Uc[k], abs(Uc[0]) + abs(mu[k] * Uc[k]))
                   for k in range(1, dim) for s in (0, 1)]
        for b, x, sc in exp:
            if abs(x) > 4 * U * sc and bool((act >> b) & 1) != (x < 0):
                bad.append(f"{tag}: rows_begin: contact {ci} edge bit {b} is {(act >> b) & 1}, its edge value {x}")

    # ---- J^T f, grad and H over the kernel's own rows
    # (J row, D, active, force, |w|: the norm of the row's spatial vector about `ref`, 0 for the dof and frictionloss rows)
    rows = []
    for ci, w in enumerate(r["cons"]):
        dim, _, act, mu = _con_fields(lay, w)
        D = float(w[lay["C_D"]])
        Uc = w[lay["C_U"]:lay["C_U"] + lay["NB"]].astype(np.float64)
        wn = [_wnorm(w, k) for k in range(max(dim, 1))]
        if dim == 1:
            rows.append((Jc[ci][0], D, bool(act & 1), -D * min(Uc[0], 0.0), wn[0]))
            continue
        for k in range(1, dim):
            for s in (0, 1):
                sg = 1 - 2 * s
                x = Uc[0] + sg * mu[k] * Uc[k]
                rows.append((Jc[ci][0] + sg * mu[k] * Jc[ci][k], D, bool((act >> (2 * k - 2 + s)) & 1), -D * min(x, 0.0),
                             wn[0] + mu[k] * wn[k]))
    for wi in range(r["nweld"]):
        w = r["welds"][wi]
        for k in range(6):
            rows.append((Jw[wi][k], float(w[W_D + k]), True, -float(w[W_D + k]) * float(w[W_JAR + k]),
                         np.linalg.norm(w[W_W + 6 * k:W_W + 6 * k + 6])))
    for k in range(r["ndr"]):
        dr = r["drs"][k]
        D, x = float(dr[DR_D]), float(dr[DR_JAR])
        a = D < 0 or x < 0
        rows.append((Jd[k], abs(D), a, -abs(D) * x if a else 0.0, 0.0))
    fsum = np.zeros(nv)
    if sim.nfric:
        fD, fl = sim.marr("dof_fricD", nv), sim.marr("dof_frictionloss", nv)
        fB = sim.marr("dof_fricB", nv)
        xf = img[sim.o["fric"]:sim.o["fric"] + nv].astype(np.float64)
        for d in range(nv):
            if fD[d] <= 0:
                continue
            quad = abs(xf[d]) * fD[d] < fl[d]
            cov.add("frictionloss quadratic" if quad else "frictionloss linear")
            rows.append((np.eye(nv)[d], fD[d], quad, np.clip(-fD[d] * xf[d], -fl[d], fl[d]), 0.0))
            fsum[d] += fl[d]
            i = [ii for ii in range(len(otype)) if otype[ii] == ROW_FRICTION and oid[ii] == d]
            if i:
                xr = qacc[d] + KBIP[i[0], 1] * qvel[d]
                note("dofrow", abs(xf[d] - xr) / (U * (abs(qacc[d]) + KBIP[i[0], 1] * abs(qvel[d]) + 1e-30)),
                     f"rows_begin: frictionloss row {d} J qacc - aref")
                note("dofrow", abs(fB[d] - KBIP[i[0], 1]) / (U * KBIP[i[0], 1]), f"frictionloss row {d} B")
    Mp = img[sim.o["M"]:sim.o["M"] + sim.nM].astype(np.float64)
    M = np.zeros((nv, nv))
    M[np.tril_indices(nv)] = Mp
    M = M + np.tril(M, -1).T
    fcon = img[sim.o["fcon"]:sim.o["fcon"] + nv].astype(np.float64)
    grad = img[sim.o["grad"]:sim.o["grad"] + nv].astype(np.float64)
    Ma = img[sim.o["Ma"]:sim.o["Ma"] + nv].astype(np.float64)
    # the kernel forms J^T f and J^T D J through the rows' spatial vectors w about `ref` and cdof: an entry J_rj = w_r . cdof_j is
    # rounded in units of |w_r| |cdof_j| (the moment arms cancel only in exact arithmetic)
    fr = sum((J * f for J, _, _, f, _ in rows), np.zeros(nv))
    fa = sum((np.abs(J) * abs(f) + cn * abs(f) * sw for J, _, _, f, sw in rows), np.zeros(nv)) + fsum
    note("fcon", np.max(np.abs(fcon - fr) / (U * (fa + 1e-30))), "pass_F: fcon = J^T f")
    ma_r = M @ qacc
    note("grad", np.max(np.abs(Ma - ma_r) / (U * (np.abs(M) @ np.abs(qacc) + 1e-30))), "mulM: M qacc")
    gs = np.abs(Ma) + np.abs(fs) + np.abs(fcon)
    note("grad", np.max(np.abs(grad - (Ma - fs - fcon)) / (U * (gs + 1e-30))), "newton_check: grad")
    Hr, Hs = M.copy(), np.abs(M)
    for J, D, a, _, sw in rows:
        if a:
            Hr += D * np.outer(J, J)
            Jm = np.abs(J) + cn * sw
            Hs += D * np.outer(Jm, Jm)
    Hp = img[sim.o["H"]:sim.o["H"] + sim.nM].astype(np.float64)
    ti = np.tril_indices(nv)
    eh = np.max(np.abs(Hp - Hr[ti]) / (U * Hs[ti] + 1e-300))
    chunked = r["ngrp"] > sim.kcap
    note("H", eh, f"build_H{' (chunked: ngrp ' + str(r['ngrp']) + ' > kcap ' + str(sim.kcap) + ')' if chunked else ''}")
    stats["ngrp"].append((r["ngrp"], sim.kcap))
    stats["compared"] += 1


def _wnorm(w, k):
    """|w| of base row k of a contact record (translational rows k < 3: W[k]; rotational rows: (W[k - 3][3:6], 0))."""
    return float(np.linalg.norm(w[6 * k:6 * k + 6] if k < 3 else w[6 * (k - 3) + 3:6 * (k - 3) + 6]))


# every row type each build must exercise (the coverage assertion)
NEED = {
    "antmaze_umaze": {"lower limit", "upper limit", "contact condim 3"},
    "fetch_reach": {"weld", "lower limit", "upper limit", "contact condim 3", "contact condim 4"},
    "fetch_pick_and_place": {"weld", "lower limit", "upper limit", "contact condim 3", "contact condim 4"},
    "fetch_slide": {"weld", "lower limit", "upper limit", "contact condim 3", "contact condim 4"},
    "hand_block_touch": {"lower limit", "upper limit", "two-sided limit", "tendon limit", "frictionloss linear",
                         "frictionloss quadratic", "contact condim 1", "contact condim 4", "index >= 32"},
    "franka_kitchen": {"lower limit", "upper limit", "two-sided limit", "kitchen joint equality", "frictionloss linear",
                       "frictionloss quadratic", "contact condim 3", "contact condim 4", "contact condim 6"},
    "adroit_hammer": {"lower limit", "upper limit", "two-sided limit", "tendon limit", "frictionloss linear",
                      "frictionloss quadratic", "contact condim 1", "contact condim 3", "contact condim 4", "index >= 32"},
    "adroit_relocate": {"lower limit", "upper limit", "two-sided limit", "tendon limit", "frictionloss linear",
                        "frictionloss quadratic", "contact condim 1", "contact condim 4", "index >= 32"},
}


# the builds whose states must run build_H chunked (ngrp > kcap) and overflow the dof-row table (bit 8, CNT_NDR == ndr_max)
CHUNKED = {"antmaze_umaze", "fetch_pick_and_place", "fetch_slide", "adroit_hammer"}
OVERFLOW = {"fetch_reach", "fetch_pick_and_place", "fetch_slide", "franka_kitchen", "hand_block_touch", "adroit_hammer", "adroit_relocate"}


# every committed model on its product build, and the kitchen model on the kitchen library without the two-level broad phase too
PARAMS = [(n, v, p, FLAVOR[v]) for n, v, p in MODELS] + [("franka_kitchen", 31, None, "kitchen")]


def _module(backend, name, nvp, penv, flavor):
    stats = dict(worst={}, rows=set(), skipped=[], capped=[], cskip=[], overflow=[], full=[], ngrp=[], compared=0, contacts=0)
    bad = _run(backend, name, nvp, penv, stats, flavor)
    w = ", ".join(f"{k} {v:.2f}" for k, v in sorted(stats["worst"].items()))
    ng = max(stats["ngrp"]) if stats["ngrp"] else (0, 0)
    print(f"\nproblem [{backend}] {flavor} NVP {nvp} {name}: {stats['compared']} cases, {stats['contacts']} contacts "
          f"compared with the oracle's, contacts skipped in "
          f"{len(stats['skipped'])}; max ngrp {ng[0]} (kcap {ng[1]}); rows {sorted(stats['rows'])}")
    print(f"  worst (u): {w}")
    for s in stats["overflow"]:
        print(f"  overflow: {s}")
    for s in stats["full"]:
        print(f"  table full without overflow: {s}")
    for s in stats["capped"]:
        print(f"  contact caps: {s}")
    for s in stats["skipped"] + stats["cskip"]:
        print(f"  skipped: {s}")
    assert not bad, "\n".join(bad[:20])
    missing = NEED[name] - stats["rows"]
    assert not missing, f"{name}: row types no longer exercised: {sorted(missing)}"
    if name in CHUNKED:
        assert max(n for n, _ in stats["ngrp"]) > stats["ngrp"][0][1], f"{name}: build_H never ran chunked (ngrp > kcap)"
    if name in OVERFLOW:
        assert stats["overflow"], f"{name}: no case overflowed the dof-row table"
    if name == "antmaze_umaze":
        assert stats["full"], "antmaze_umaze: no case filled the dof-row table exactly"
    assert len(stats["skipped"]) * 10 <= stats["compared"] and not any(f"[{REAL[name]}]" in s for s in stats["skipped"]), \
        f"{name}: contact sets of {len(stats['skipped'])} cases differ from the oracle's"
    assert len(stats["cskip"]) * 10 <= stats["contacts"], f"{name}: {len(stats['cskip'])} kept contacts have no oracle twin"
    return stats


@pytest.mark.gpu
@pytest.mark.parametrize("name,nvp,penv,flavor", PARAMS)
def test_solver_problem_on_the_device(name, nvp, penv, flavor):
    _module("gpu", name, nvp, penv, flavor)


@pytest.mark.parametrize("name,nvp,penv,flavor", PARAMS)
def test_solver_problem_on_the_32_lane_emulation(name, nvp, penv, flavor):
    _module("cpu", name, nvp, penv, flavor)
