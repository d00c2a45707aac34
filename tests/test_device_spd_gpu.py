"""The register Cholesky (sim_core.cuh `spd_solve<NVP>`) on its own, per product instantiation, against numpy's fp64 solve.

The env-level parity tests see this routine only through the Newton solver, which absorbs a poor search direction as one more
Newton move.  Here each instantiation the product compiles (NVP 14, 15, 21, 22, 30 of b200sim.cu, 31 of the kitchen units, the
bordered 36 of b200sim_wide.cu) solves, for every nv from 1 to NVP (identity padding; nv 33..36 = the border rows):
  * random SPD matrices with a prescribed spectrum, condition number 1, 1e2, 1e4, 1e6;
  * the matrices of the two real solves at contact-heavy states of the committed models (Fetch grasp, Fetch gripper pressed on
    the table, Hand with touch sensors, Kitchen arm pressed on the cabinet, Adroit hammer / relocate, AntMaze, FetchSlide),
    assembled in fp64 from the oracle: the Euler step's M + h diag(damping) and the Newton Hessian H = M + J^T D J over the
    active constraint rows;
each with and without the diagonal term (dadd, hh), out of place (the Euler solve: A = M, work area H) and in place (the Newton
solve: A == work area).  Normwise backward error and forward error are bounded in units of u = 2^-24, and the solve must keep
to its buffers: x past nv, A (out of place) and the work area past the two column buffers of the shared-memory column broadcast
stay bit for bit as they were.

The GPU half runs the nvcc build (tests/devsim: the product's flags, hardware rsqrtf, FMA contraction), one block per case.
The CPU half runs the same cases through the 32-lane emulation (tests/hostsim `warp`, `warp_wide`, `warp_kitchen` flavors):
IEEE arithmetic, but the same lines, the border code of the NVP 36 build included.
"""
import numpy as np
import pytest

U = 2.0 ** -24
NVPS = (14, 15, 21, 22, 30, 31, 36)
HOST_FLAVOR = {31: "warp_kitchen", 36: "warp_wide"}   # the others: "warp"
KAPPAS = (1.0, 1e2, 1e4, 1e6)
GUARD = np.uint32(0x7FEDBEEF)                          # a quiet NaN whose payload the solve never writes

# Limits in units of nv * u (backward error) and kappa * nv * u (forward error), 4-5x the largest value measured over all cases of
# all seven instantiations: on an H100 80GB HBM3 (700 W) 1.32 and 2.63 (NVP 31), on the 32-lane emulation 1.56 and 3.12 (NVP 14, nv = 1:
# a single rounding is already most of nv * u there).  Per instantiation in DESIGN.md section 2.
# The forward bound says nothing once kappa * nv * u * FORWARD_C >= 1 (kappa 1e6 at nv 36: about 26; the real M + hB of the Fetch
# models, with their 1e11 gripper damping, and some Newton Hessians are worse): there the backward bound is the only check that bites.
BACKWARD_C = {"gpu": 6.0, "cpu": 7.0}
FORWARD_C = {"gpu": 12.0, "cpu": 14.0}


def _r4(n):
    return (n + 3) & ~3


def _layout(nvp):
    """(la, lx, lh, col): buffer words of A, x / dadd and the work area, and the words of the two column buffers."""
    na = min(nvp, 32)
    col = 2 * _r4(na)
    nm = nvp * (nvp + 1) // 2
    return _r4(max(nm, col) + 8), _r4(nvp + 4), _r4(col + 8), col


def _pack(A):
    n = A.shape[0]
    return np.concatenate([A[i, :i + 1] for i in range(n)])


def _unpack(p, n):
    A = np.zeros((n, n))
    k = 0
    for i in range(n):
        A[i, :i + 1] = p[k:k + i + 1]
        k += i + 1
    return A + np.tril(A, -1).T


def _random_cases(nvp, seed):
    """(label, nv, A fp32 [nv, nv], dadd fp32 [nv]) for every nv <= nvp and every kappa."""
    rng = np.random.default_rng(seed)
    out = []
    for nv in range(1, nvp + 1):
        for kap in KAPPAS:
            Q, _ = np.linalg.qr(rng.standard_normal((nv, nv)))
            lam = np.logspace(0.0, -np.log10(kap), nv) if nv > 1 else np.ones(1)
            A = ((Q * lam) @ Q.T).astype(np.float32)
            A = (A + A.T) / 2
            out.append((f"random nv={nv} kappa={kap:.0e}", nv, A.astype(np.float32), rng.uniform(0.0, 1.0, nv).astype(np.float32)))
    return out


_REAL = {}
# (label, committed model, the NVP its product kernel uses: b200sim.cu b200sim_create)
REAL_STATES = [("antmaze", "antmaze_umaze", 14), ("fetch_reach pressed", "fetch_reach", 15), ("fetch grasp", "fetch_pick_and_place", 21),
               ("fetch pressed", "fetch_pick_and_place", 21), ("fetch_slide", "fetch_slide", 22), ("hand touch", "hand_block_touch", 30),
               ("kitchen pressed", "franka_kitchen", 31), ("adroit hammer", "adroit_hammer", 36), ("adroit relocate", "adroit_relocate", 36)]
_DRIVEN = {"fetch_reach pressed", "fetch grasp", "fetch pressed", "hand touch", "kitchen pressed", "adroit hammer", "adroit relocate"}


def _contact_state(label, m):
    """The oracle sim of an env driven into a contact-heavy state (the states of tests/test_batch_invariance_gpu.py and
    tests/test_gpu_parity.py): the object between the closing Fetch fingers, the closed gripper driven onto the table, the block on
    the palm of the touch-sensor hand, an arm link pressed onto the kitchen, the Adroit hand with random actions."""
    rng = np.random.default_rng(7)
    if label.startswith("fetch"):
        from tests.parity_util import oracle_env_from_model

        o = oracle_env_from_model("FetchReach" if "reach" in label else "FetchPickAndPlace", m)
        o.reset(seed=300)
        if label == "fetch grasp":
            s = o.sim
            a = m.jnt_qposadr[m.joint_id("object0:joint")]
            s.qpos[a:a + 3] = s.site_xpos[o._grip_site] + np.array([0.002, 0.0, -0.004])
            s.qpos[a + 3:a + 7] = [np.cos(0.025), 0.0, 0.0, np.sin(0.025)]
            for fq in o._finger_q:
                s.qpos[fq] = 0.045
            s.qvel[:] = 0.0
            s.forward()
            for _ in range(4):
                o.step(np.array([0.0, 0.0, 0.0, -1.0]))   # close on the box
        else:
            for _ in range(12):
                o.step(np.array([0.0, 0.0, -1.0, -1.0]))  # closed gripper driven down onto the table (or the object)
        return o.sim
    if label == "hand touch":
        from oracle.hand_env import OracleHandBlockEnv

        o = OracleHandBlockEnv(model=m, touch_get_obs="sensordata")
        o.reset(seed=2)
        for _ in range(3):
            o.step(rng.uniform(-1, 1, m.nu))
        return o.sim
    if label == "kitchen pressed":
        from oracle.kitchen_env import OracleKitchenEnv
        from tests.test_batch_invariance_gpu import KITCHEN_PRESS

        o = OracleKitchenEnv(m)
        o.reset(seed=21)
        for _ in range(6):
            o.step(np.array(KITCHEN_PRESS))
        return o.sim
    from oracle.adroit_env import OracleAdroitHammerEnv, OracleAdroitRelocateEnv

    o = (OracleAdroitHammerEnv if "hammer" in label else OracleAdroitRelocateEnv)(m, noslip=False)
    o.reset(seed=3)
    for _ in range(4):
        o.step(rng.uniform(-1, 1, m.nu))
    return o.sim


def _real_cases(nvp):
    """(label, kind, nv, A fp32, dadd fp32, hh) at a contact state of every committed model whose product kernel is NVP = nvp."""
    if nvp in _REAL:
        return _REAL[nvp]
    from gymnasium_robotics_b200.models import load_model
    from oracle.oracle_sim import OracleSim

    out = []
    for label, name, v in REAL_STATES:
        if v != nvp:
            continue
        m = load_model(name)
        s = _contact_state(label, m) if label in _DRIVEN else None
        if s is None:
            s = OracleSim(m)
            s.step(200)   # from the model's rest pose: the ant on the floor, the FetchSlide puck on the table
        s.forward()
        assert s.ncon > 0 and s.nefc > 0, label
        M = np.array(s.M)
        J, D, f = s.efc("J"), s.efc("D"), s.efc("force")
        act = f != 0
        H = M + (J[act].T * D[act]) @ J[act]
        out.append((f"{label} M+hB", "euler", m.nv, M.astype(np.float32), np.asarray(m.dof_damping, np.float32), np.float32(m.opt[0])))
        out.append((f"{label} H=M+JtDJ ({s.ncon} contacts, {int(act.sum())} active rows)", "newton", m.nv, H.astype(np.float32), None,
                    np.float32(0)))
    _REAL[nvp] = out
    return out


def _solve(backend, nvp, cases, use_dadd, hh, inplace):
    """Run one batch; cases = [(nv, A fp32, b fp32, dadd fp32)].  Returns the buffers before and after."""
    la, lx, lh, _ = _layout(nvp)
    n = len(cases)
    A = np.full((n, la), GUARD, np.uint32).view(np.float32)
    x = np.full((n, lx), GUARD, np.uint32).view(np.float32)
    D = np.full((n, lx), GUARD, np.uint32).view(np.float32)   # a read of dadd past nv would turn the solution into NaN
    H = np.full((n, lh), GUARD, np.uint32).view(np.float32)
    nvs = np.array([c[0] for c in cases], np.int32)
    for e, (nv, Ae, b, d) in enumerate(cases):
        A[e, :nv * (nv + 1) // 2] = _pack(Ae)
        x[e, :nv] = b
        if d is not None:
            D[e, :nv] = d
    before = (A.copy(), x.copy(), H.copy())
    if backend == "gpu":
        from tests import devsim

        devsim.spd(nvp, nvs, A, x, D, hh, H, use_dadd, inplace)
    else:
        from tests import hostsim

        hostsim.spd(HOST_FLAVOR.get(nvp, "warp"), nvp, nvs, A, x, D, hh, H, use_dadd, inplace)
    return before, (A, x, H)


def _same_bits(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _check(backend, nvp, labels, cases, use_dadd, hh, inplace, stats):
    la, lx, lh, col = _layout(nvp)
    (A0, x0, H0), (A1, x1, H1) = _solve(backend, nvp, cases, use_dadd, hh, inplace)
    bad = []
    for e, (label, (nv, Ae, b, d)) in enumerate(zip(labels, cases)):
        tag = f"NVP {nvp} {label} dadd={use_dadd} inplace={inplace}"
        # isolation: x past nv; A untouched out of place; the work area written only inside the two column buffers
        if not _same_bits(x1[e, nv:], x0[e, nv:]):
            bad.append(f"{tag}: x[{nv}:] was written")
        if inplace:
            if not _same_bits(A1[e, col:], A0[e, col:]):
                bad.append(f"{tag}: in-place solve wrote A past its {col} column-buffer words")
        else:
            if not _same_bits(A1[e], A0[e]):
                bad.append(f"{tag}: A was modified")
            if not _same_bits(H1[e, col:], H0[e, col:]):
                bad.append(f"{tag}: the work area was written past its {col} column-buffer words")
        xh = x1[e, :nv].astype(np.float64)
        if not np.isfinite(xh).all():
            bad.append(f"{tag}: non-finite solution")
            continue
        Aeff = Ae.astype(np.float64)
        if use_dadd:
            Aeff = Aeff + np.diag(np.float64(hh) * d.astype(np.float64))
        b64 = b.astype(np.float64)
        xr = np.linalg.solve(Aeff, b64)
        kap = np.linalg.cond(Aeff)
        bwd = np.abs(Aeff @ xh - b64).max() / (np.abs(Aeff).sum(1).max() * np.abs(xh).max() + np.abs(b64).max())
        fwd = np.abs(xh - xr).max() / np.abs(xr).max()
        rb, rf = bwd / (nv * U), fwd / (kap * nv * U)
        stats["bwd"] = max(stats.get("bwd", 0.0), rb)
        stats["fwd"] = max(stats.get("fwd", 0.0), rf)
        if rb > BACKWARD_C[backend]:
            bad.append(f"{tag}: backward error {bwd:.2e} = {rb:.3f} nv u")
        if rf > FORWARD_C[backend]:
            bad.append(f"{tag}: forward error {fwd:.2e} = {rf:.3f} kappa nv u (kappa {kap:.1e})")
    return bad


def _run(backend, nvp):
    stats, bad = {}, []
    rng = np.random.default_rng(1000 + nvp)
    rand = _random_cases(nvp, seed=nvp)
    labels = [r[0] for r in rand]
    for use_dadd in (False, True):
        for inplace in (False, True):
            cases = [(nv, A, rng.standard_normal(nv).astype(np.float32), d) for _, nv, A, d in rand]
            bad += _check(backend, nvp, labels, cases, use_dadd, np.float32(0.01), inplace, stats)
    for label, kind, nv, A, d, hh in _real_cases(nvp):
        b = rng.standard_normal(nv).astype(np.float32)
        if kind == "euler":
            bad += _check(backend, nvp, [label], [(nv, A, b, d)], True, hh, False, stats)
        else:
            bad += _check(backend, nvp, [label], [(nv, A, b, None)], False, hh, True, stats)
    print(f"spd_solve<{nvp}> [{backend}]: max backward error {stats['bwd']:.3f} nv u, max forward error {stats['fwd']:.3f} kappa nv u")
    assert not bad, "\n".join(bad[:20]) + (f"\n... {len(bad)} failures" if len(bad) > 20 else "")


@pytest.mark.gpu
@pytest.mark.parametrize("nvp", NVPS)
def test_register_cholesky_on_the_device(nvp):
    _run("gpu", nvp)


@pytest.mark.parametrize("nvp", NVPS)
def test_register_cholesky_on_the_32_lane_emulation(nvp):
    _run("cpu", nvp)
