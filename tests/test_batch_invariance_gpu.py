"""Batch invariance of the step kernel (run with -m gpu on an H100).

One warp steps one env, but the warps of a block share the staged model, meet at block-wide alignment barriers and run the Newton
loop until the last warp of the block has converged; idle warps (past N, or masked out) run the same control flow and must touch no
memory.  A defect there faults nothing: it makes env i's numbers depend on the envs that share its block.  These tests take K
distinct envs per kernel build (states reached by the product envs themselves, plus contact-heavy ones) and require every
configuration to reproduce the 7-warp launch of the same K envs BIT FOR BIT, for every env: every block size the library
accepts, other batch shapes, other positions and neighbours, masked launches, the classic output arrays.  Comparisons are on the
int32 view of the fp32 outputs (NaN != NaN, -0 == +0 would hide differences).  Every launch writes into a slice of a larger buffer
filled with a NaN sentinel, so a write outside an env's own output columns shows up too.

The last part compares envs placed at block edges, in a partly filled block and in the second wave of the production batch
sizes with the fp64 oracle, against the stated envelopes of tests/test_gpu_parity.py and tests/test_zz_kitchen_gpu.py.

On the host emulation (tests/dryrun_gpu_tests.py) the tests that need the C-ABI are skipped: forcing a block size
(B200SIM_WPB), b200sim_launch_config and the classic output arrays."""
import ctypes

import numpy as np
import pytest
import torch

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.fetch import welded_eq_data
from tests.parity_util import check_envelope, inject_oracle_state, inject_records, oracle_env_from_model, oracle_state_record

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FEDBEEF       # a quiet NaN whose payload no kernel writes
FLAG_SENTINEL = 0xA5
GUARD = 2                   # sentinel rows before row 0 and after row N-1 of every output buffer
TIME_LIMIT = 20             # step counters start at (7 i) % 20, so some envs truncate during the three env-steps
NSTEPS, NRAW = 3, 2         # env-steps per run (a contaminated warm start shows in the later ones); sub-steps of a raw launch

# (case, env id, make_vec kwargs, block sizes b200sim_create accepts for the model): the instantiations of csrc/b200sim.cu
# (B200_FOR_ALL_VARIANTS), b200sim_wide.cu (7, 10, 13, 14) and b200sim_kitchen*.cu (7, 10; 11 with the two-level broad phase) whose
# shared memory (hot_words + WPB * scr_words) fits one block.  A dropped or added instantiation changes this table.
CASES = [
    ("antmaze", "AntMaze_Large-v5", {}, (7, 8, 14, 16, 28)),                       # NVP 14, RK4
    ("pointmaze", "PointMaze_Large-v3", {}, (7, 8, 14, 16, 28)),                   # NVP 14
    ("fetch_reach", "FetchReach-v4", {}, (7, 8, 14, 16, 28)),                      # NVP 15
    ("fetch_pick", "FetchPickAndPlace-v4", {}, (7, 8, 14, 16, 28)),                # NVP 21
    ("fetch_push", "FetchPush-v4", {}, (7, 8, 14, 16, 28)),                        # NVP 21
    ("fetch_slide", "FetchSlide-v4", {}, (7, 8, 14, 16, 28)),                      # NVP 22
    ("hand_touch", "HandManipulateBlock_ContinuousTouchSensors-v1", {}, (7, 14)),  # NVP 30, forward pass on refresh
    ("hand_reach", "HandReach-v3", {}, (7, 14)),                                   # NVP 30
    ("adroit_door", "AdroitHandDoor-v2", {}, (7, 14)),                             # NVP 30
    ("adroit_pen", "AdroitHandPen-v2", {}, (7, 14)),                               # NVP 30
    ("adroit_hammer", "AdroitHandHammer-v2", {}, (7, 10, 13, 14)),                 # wide, forward pass on refresh
    ("adroit_relocate", "AdroitHandRelocate-v2", {}, (7, 10, 13, 14)),             # wide
    ("kitchen_flat", "FrankaKitchen-v1", {"broadphase": "flat"}, (7, 10)),
    ("kitchen_groups", "FrankaKitchen-v1", {}, (7, 10, 11)),
    ("kitchen_hull", "FrankaKitchen-v1", {"mesh_collision": "hull"}, (7, 10, 11)),
]
_CASES = {c[0]: c for c in CASES}
# A PointMaze ball has one wall contact at most and needs one or two Newton moves per env-step, so its blocks mix 1 and 2; the
# NVP 14 build it shares with AntMaze is held to a spread of 2 by the AntMaze case.
MIN_SPREAD = {"pointmaze": 1}
_PREPARED = {}


def _cabi(be):
    return hasattr(be, "L")


def _needs_cabi(be):
    if not _cabi(be):
        pytest.skip("needs the C-ABI (block-size override, launch config, classic outputs)")


def _launch_config(be):
    w, b = ctypes.c_int(), ctypes.c_int()
    assert be.L.b200sim_launch_config(be.h, None, ctypes.byref(w), ctypes.byref(b)) == 0
    return w.value, b.value


def _num_sms(device):
    return torch.cuda.get_device_properties(device).multi_processor_count


def _backend(c, n, wpb, mp):
    """A fresh backend of the case's model and task for n envs; wpb forces the block size (None: the library's choice)."""
    env = c["env"]
    if wpb is None:
        mp.delenv("B200SIM_WPB", raising=False)
    else:
        mp.setenv("B200SIM_WPB", str(wpb))
    if hasattr(env, "broadphase"):
        mp.setenv("B200SIM_KITCHEN_GROUPS", "1" if env.broadphase == "groups" else "0")
    be = type(env.backend)(env.model, c["eq"], env.task, n, env.device)
    be.set_time_limit(TIME_LIMIT, terminate_on_success=True)
    if wpb is not None and _cabi(be):
        assert _launch_config(be)[0] == wpb
    return be


def _outputs(be, n):
    """Packed output rows that are a slice of a sentinel-filled buffer with guard rows; flags pre-filled with a sentinel byte."""
    big = torch.full((n + 2 * GUARD, be.packed_w), SENTINEL, dtype=torch.int32, device=be.device).view(torch.float32)
    p = big[GUARD:GUARD + n]
    no, ng = be.nobs, be.ngoal
    k = no + 2 * ng
    flags = torch.full((2, n), FLAG_SENTINEL, dtype=torch.uint8, device=be.device)
    return dict(big=big, packed=p, obs=p[:, :no], achieved=p[:, no:no + ng], desired=p[:, no + ng:k], reward=p[:, k], success=p[:, k + 1],
                terminated=flags[0].view(torch.bool), truncated=flags[1].view(torch.bool), flags=flags)


def _check_untouched(be, out, n, ncols, mask=None):
    """Guard rows, the columns a launch does not write (pad; the flags after refresh / raw launches) and masked envs' rows still
    hold the sentinel."""
    b = out["big"].view(torch.int32)
    assert bool((b[:GUARD] == SENTINEL).all()) and bool((b[GUARD + n:] == SENTINEL).all()), "a launch wrote outside rows 0..N-1"
    rows = b[GUARD:GUARD + n]
    bad = _differ(rows[:, ncols:], torch.full_like(rows[:, ncols:], SENTINEL))
    assert not bad, f"a launch wrote columns {ncols}.. (pad, or the flags of a refresh / raw launch) of envs {bad[:8]}"
    if mask is not None:
        written = ((rows != SENTINEL).any(1) & ~mask).nonzero().flatten().tolist()
        assert not written, f"masked-out envs {written[:8]} had their output row written"


def _differ(a, b):
    return (a != b).reshape(a.shape[0], -1).any(1).nonzero().flatten().tolist()


def _run_steps(be, S, acts, el0):
    """NSTEPS env-steps of the envs with records S: per step the packed rows, flags and info words; then the records, the step
    counters.  The device overflow counter must grow by the number of info words with overflow bits."""
    n = S.shape[0]
    be.state.copy_(S)
    be.elapsed.copy_(el0)
    out = _outputs(be, n)
    k = be.nobs + 2 * be.ngoal
    info = torch.full((n,), -1, dtype=torch.int32, device=be.device)
    c0 = int(be.overflow_counter[0])
    steps = []
    for a in acts:
        be.step(a, out, info)
        _check_untouched(be, out, n, k + 4)
        steps.append((out["packed"].view(torch.int32).clone(), out["flags"].t().clone(), info.clone()))
    flagged = sum(int(((i >> 16) != 0).sum()) for _, _, i in steps)
    assert int(be.overflow_counter[0]) - c0 == flagged, "device overflow counter != info words with overflow bits"
    return dict(steps=steps, state=be.state.view(torch.int32).clone(), elapsed=be.elapsed.clone())


def _run_masked(be, S, el0, kind, mask):
    """One refresh or raw launch (NRAW sub-steps) of the envs with records S under `mask` (None = all)."""
    n = S.shape[0]
    be.state.copy_(S)
    be.elapsed.copy_(el0)
    out = _outputs(be, n)
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    if kind == "refresh":
        be.refresh(m, out)
    else:
        be.raw_step(NRAW, out, m)
    _check_untouched(be, out, n, be.nobs + 2 * be.ngoal + 2, mask)
    return dict(rows=out["packed"].view(torch.int32).clone(), state=be.state.view(torch.int32).clone(), elapsed=be.elapsed.clone())


def _assert_same(ref, got, src, dst, what):
    """Reference env src[j] must equal env dst[j] of `got` in every output, bit for bit."""
    for t, (r, g) in enumerate(zip(ref["steps"], got["steps"])):
        for name, R, G in zip(("packed row", "flags", "info word"), r, g):
            bad = _differ(R[src], G[dst])
            assert not bad, f"{what}: env-step {t}: {name} of reference envs {src[bad[:8]].tolist()} differs"
    for name in ("state", "elapsed"):
        bad = _differ(ref[name][src], got[name][dst])
        assert not bad, f"{what}: {name} after the steps of reference envs {src[bad[:8]].tolist()} differs"


# ------------------------------------------------------------------------------------------------ the heterogeneous batch (§1)
def _grasp_records(env, count):
    """Fetch states with the object between the open fingers (tests/test_gpu_parity.py::test_fetch_grasp_contact_heavy_parity)."""
    recs = []
    for i in range(count):
        o = oracle_env_from_model(env.task_name, env.model)
        o.reset(seed=300 + i)
        s, m = o.sim, o.model
        a = m.jnt_qposadr[m.joint_id("object0:joint")]
        s.qpos[a:a + 3] = s.site_xpos[o._grip_site] + np.array([0.002 * (i - 1.5), 0.0, -0.004 * (i % 3)])
        yaw = 0.05 * (i - 1.5)
        s.qpos[a + 3:a + 7] = [np.cos(yaw / 2), 0.0, 0.0, np.sin(yaw / 2)]
        for fq in o._finger_q:
            s.qpos[fq] = 0.045
        s.qvel[:] = 0.0
        s.forward()
        recs.append(oracle_state_record(env, o))
    return torch.as_tensor(np.stack(recs), dtype=torch.float32, device=env.device)


KITCHEN_PRESS = (1.0, 1.0, 1.0, -1.0, -1.0, 1.0, -1.0, 0.0, 0.0)   # drives an arm link onto the kitchen (tests/test_mesh_hull.py)


def _press(env, a, t=0):
    """Contact-heavy actions for every third env: the Fetch gripper closed and driven down onto the table (or the object), the
    PointMaze ball pushed against a wall and back (it has no other contact), the Franka arm pressed onto the kitchen."""
    if type(env).__name__ == "FetchVectorEnv":
        a[1::3, 2] = -1.0
        a[1::3, 3] = -1.0
    elif getattr(env, "agent", None) == "point":
        a[1::3] = torch.tensor([1.0 if t % 2 == 0 else -1.0, 0.3], device=a.device)
    elif hasattr(env, "control_targets"):
        a[1::3] = torch.tensor(KITCHEN_PRESS, device=a.device)
    return a


def _prepare(name, mp):
    """K distinct envs of the case (states after a torch-seeded reset and 5..30 random-action env-steps of the product env, each
    env snapshotted after its own number of steps, plus contact-heavy states), distinct actions, and the 7-warp reference."""
    if name in _PREPARED:
        return _PREPARED[name]
    _, env_id, kw, sizes = _CASES[name]
    K = 2 * max(sizes) + 5
    env = pkg.make_vec(env_id, num_envs=K, device="cuda:0", rng_mode="torch", **kw)
    dev = env.device
    env.reset(seed=1234)
    quiet = env.get_state()[0][0].clone()
    g = torch.Generator(device=dev).manual_seed(99)
    nact = env.backend.nact
    snaps = []
    for t in range(30):
        a = _press(env, torch.rand((K, nact), generator=g, device=dev) * 2 - 1)
        env.step(a)
        snaps.append(env.get_state()[0])
    when = [4 + (7 * i) % 26 for i in range(K)]
    S = torch.stack([snaps[when[i]][i] for i in range(K)])
    if getattr(env, "task_name", None) in ("FetchPickAndPlace", "FetchPush"):
        grasp = _grasp_records(env, 4)
        S[4::9] = grasp[torch.arange(len(range(4, K, 9))) % 4]
    acts = []
    for t in range(NSTEPS):
        a = _press(env, torch.rand((K, nact), generator=g, device=dev) * 2 - 1, t + 1)
        if getattr(env, "task_name", None) in ("FetchPickAndPlace", "FetchPush"):
            a[4::9, 3] = -1.0     # keep closing on the object
        if hasattr(env, "control_targets"):
            # the Kitchen's kernel action is the position target the env derives from its last robot observation
            env._last_robot_qpos = S[:, env.backend.layout["qpos"]:env.backend.layout["qpos"] + 9]
            a = env.control_targets(a)
        acts.append(a.contiguous())
    el0 = ((torch.arange(K, device=dev) * 7) % TIME_LIMIT).to(torch.int32)
    c = dict(name=name, env=env, K=K, sizes=sizes, S=S, acts=acts, el0=el0, quiet=quiet,
             eq=welded_eq_data(env.model) if type(env).__name__ == "FetchVectorEnv" else np.zeros((0, 11)))
    be = _backend(c, K, 7, mp)
    c["ref"] = _run_steps(be, S, acts, el0)
    c["ref_masked"] = {kind: _run_masked(be, S, el0, kind, None) for kind in ("refresh", "raw")}
    be.close()
    _PREPARED[name] = c
    return c


@pytest.fixture(params=[c[0] for c in CASES])
def case(request, monkeypatch):
    return _prepare(request.param, monkeypatch)


def test_batch_mixes_newton_iteration_counts(case):
    """The batch exercises the block-uniform Newton loop at every block size: inside at least one block, the iteration counts of
    the info words differ by >= 2, so converged warps idle while a neighbour keeps moving (otherwise the invariance tests below
    would degrade into the identical-env case)."""
    for w in case["sizes"]:
        spread = 0
        for _, _, info in case["ref"]["steps"]:
            it = (info & 0xFFFF).to(torch.int64)
            for b0 in range(0, case["K"], w):
                blk = it[b0:b0 + w]
                spread = max(spread, int(blk.max() - blk.min()))
        assert spread >= MIN_SPREAD.get(case["name"], 2), f"{w}-warp blocks: Newton iteration counts differ by at most {spread} inside a block"


def test_accepted_block_sizes(case, monkeypatch):
    """b200sim_create accepts exactly the block sizes of the table (checked through b200sim_launch_config) and picks 7 warps for
    the K-env batch by default."""
    be = _backend(case, 1, None, monkeypatch)
    _needs_cabi(be)
    be.close()
    accepted = []
    for w in range(1, 29):
        try:
            be = _backend(case, 1, w, monkeypatch)
        except RuntimeError:
            continue
        accepted.append(w)
        be.close()
    assert tuple(accepted) == case["sizes"]
    be = _backend(case, case["K"], None, monkeypatch)
    assert _launch_config(be)[0] == 7
    be.close()


def test_every_block_size_reproduces_the_reference(case, monkeypatch):
    """All K envs, and N = q * W + 1 envs (a tail block with one active warp), at every accepted block size; one env alone; and
    N = SMs * W + 1 envs (a second wave of one env) at the largest block size, the K states repeated."""
    ref, S, acts, el0, K = case["ref"], case["S"], case["acts"], case["el0"], case["K"]
    dev = S.device
    be = _backend(case, 1, 7, monkeypatch)
    _needs_cabi(be)
    got = _run_steps(be, S[:1], [a[:1].contiguous() for a in acts], el0[:1])
    _assert_same(ref, got, torch.arange(1, device=dev), torch.arange(1, device=dev), "N = 1")
    be.close()
    for w in case["sizes"]:
        for n in sorted({K, (K - 1) // w * w + 1}):
            be = _backend(case, n, w, monkeypatch)
            got = _run_steps(be, S[:n], [a[:n].contiguous() for a in acts], el0[:n])
            be.close()
            idx = torch.arange(n, device=dev)
            _assert_same(ref, got, idx, idx, f"{w} warps per block, N = {n}")
    w = max(case["sizes"])
    n = _num_sms(dev) * w + 1
    src = torch.arange(n, device=dev) % K
    be = _backend(case, n, w, monkeypatch)
    assert _launch_config(be)[1] == _num_sms(dev) + 1
    got = _run_steps(be, S[src], [a[src].contiguous() for a in acts], el0[src])
    be.close()
    _assert_same(ref, got, src, torch.arange(n, device=dev), f"{w} warps per block, N = {n} (second wave of one env)")


def test_position_and_neighbours(case, monkeypatch):
    """The K envs reversed, under a fixed permutation, and at an offset inside a larger batch whose other envs alternate between a
    quiescent env and the envs that need the most Newton moves; each env is compared with its reference by identity."""
    ref, S, acts, el0, K = case["ref"], case["S"], case["acts"], case["el0"], case["K"]
    dev = S.device
    perm = torch.randperm(K, generator=torch.Generator().manual_seed(5)).to(dev)
    heavy = torch.argsort((ref["steps"][0][2] & 0xFFFF), descending=True, stable=True)[:4]
    off = max(case["sizes"]) + 3
    n = K + 2 * off
    fill = torch.arange(n, device=dev)
    S_emb = torch.where((fill % 2 == 0)[:, None], case["quiet"][None, :], S[heavy[fill % 4]])
    acts_emb = [torch.where((fill % 2 == 0)[:, None], torch.zeros_like(a[:1]), a[heavy[fill % 4]]) for a in acts]
    el_emb = el0[heavy[fill % 4]].clone()
    S_emb[off:off + K], el_emb[off:off + K] = S, el0
    for a, ae in zip(acts, acts_emb):
        ae[off:off + K] = a
    probe = _backend(case, 1, None, monkeypatch)
    wpbs = [None] + ([max(case["sizes"])] if _cabi(probe) else [])
    probe.close()
    for wpb in wpbs:
        for what, src in (("reversed", torch.arange(K - 1, -1, -1, device=dev)), ("permuted", perm)):
            be = _backend(case, K, wpb, monkeypatch)
            got = _run_steps(be, S[src], [a[src].contiguous() for a in acts], el0[src])
            be.close()
            _assert_same(ref, got, src, torch.arange(K, device=dev), f"{what} (block size {wpb or 'default'})")
        be = _backend(case, n, wpb, monkeypatch)
        got = _run_steps(be, S_emb, [a.contiguous() for a in acts_emb], el_emb)
        be.close()
        _assert_same(ref, got, torch.arange(K, device=dev), torch.arange(off, off + K, device=dev),
                     f"embedded at {off} among quiescent / Newton-heavy envs (block size {wpb or 'default'})")


def _masks(K, w, dev):
    i = torch.arange(K, device=dev)
    return {"alternate": i % 2 == 0, "every other block": (i // w) % 2 == 1, "first env of each block": i % w == 0,
            "last env of each block": i % w == w - 1, "last env of the grid": i == K - 1}


def test_masked_launches_touch_only_their_envs(case, monkeypatch):
    """refresh and raw_step_masked under masks, at every accepted block size: unmasked envs equal an unmasked launch on the same
    records; masked envs keep their state record, output row (sentinel) and step counter bit for bit."""
    S, el0, K, name = case["S"], case["el0"], case["K"], case["name"]
    dev = S.device
    probe = _backend(case, 1, None, monkeypatch)
    wpbs = list(case["sizes"]) if _cabi(probe) else [None]
    probe.close()
    S32 = S.view(torch.int32)
    for wpb in wpbs:
        be = _backend(case, K, wpb, monkeypatch)
        for mname, m in _masks(K, wpb or 7, dev).items():
            for kind in ("refresh", "raw"):
                ref = case["ref_masked"][kind]
                got = _run_masked(be, S, el0, kind, m)
                what = f"{kind}, mask '{mname}', block size {wpb or 'default'}"
                idx = m.nonzero().flatten()
                bad = _differ(ref["rows"][idx], got["rows"][idx]) + _differ(ref["state"][idx], got["state"][idx])
                assert not bad, f"{what}: active envs {idx[bad[:8]].tolist()} differ from the unmasked launch"
                idle = (~m).nonzero().flatten()
                bad = _differ(S32[idle], got["state"][idle])
                assert not bad, f"{what}: masked-out envs {idle[bad[:8]].tolist()} had their state record changed"
                assert torch.equal(got["elapsed"], el0), f"{what}: step counters changed"
                if name == "antmaze" and kind == "refresh":
                    # AntMaze-v5's contact forces after a refresh are +0.0, as after mj_resetData (they once came from
                    # kinematics the refresh never computed, so stale shared memory leaked into the reset observation)
                    assert not bool(got["rows"][idx, 27:105].any()), f"{what}: non-zero contact forces after a refresh"
        be.close()


def test_classic_output_path(case, monkeypatch):
    """b200sim_step with b200sim_set_packed(h, 0): the five output arrays and the byte flags equal the packed columns of the
    reference bit for bit, at 7 warps and at the largest block size."""
    ref, S, acts, el0, K = case["ref"], case["S"], case["acts"], case["el0"], case["K"]
    probe = _backend(case, 1, None, monkeypatch)
    _needs_cabi(probe)
    probe.close()
    no, ng = case["env"].backend.nobs, case["env"].backend.ngoal
    dev = S.device
    for w in sorted({7, max(case["sizes"])}):
        be = _backend(case, K, w, monkeypatch)
        be.L.b200sim_set_packed(be.h, 0)
        be.state.copy_(S)
        be.elapsed.copy_(el0)
        arrs = [torch.full((K, d), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32) for d in (no, ng, ng, 1, 1)]
        flags = torch.full((2, K), FLAG_SENTINEL, dtype=torch.uint8, device=dev)
        info = torch.full((K,), -1, dtype=torch.int32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        for t, a in enumerate(acts):
            rc = be.L.b200sim_step(be.h, a.data_ptr(), *[x.data_ptr() for x in arrs], flags[0].data_ptr(), flags[1].data_ptr(),
                                   info.data_ptr(), stream)
            assert rc == 0, be.L.b200sim_last_error(be.h)
            row, fl, inf = ref["steps"][t]
            got = torch.cat([x.view(torch.int32) for x in arrs], dim=1)
            bad = _differ(row[:, :no + 2 * ng + 2], got)
            assert not bad, f"{w} warps per block, env-step {t}: classic outputs of envs {bad[:8]} differ from the packed row"
            assert torch.equal(flags.t(), fl) and torch.equal(info, inf), f"{w} warps per block, env-step {t}: flags / info differ"
            assert torch.equal(fl.to(torch.float32), row[:, no + 2 * ng + 2:no + 2 * ng + 4].view(torch.float32))
        assert torch.equal(be.state.view(torch.int32), ref["state"]) and torch.equal(be.elapsed, ref["elapsed"])
        be.close()


# ------------------------------------------------------------------------------------- oracle parity at the production sizes (§3)
def _production(env_id, n, case_name, mp, **kw):
    """The production batch with the library's default block size, every env filled with the heterogeneous states of the case,
    and the rows where oracle envs go: first and last warp of a block, both sides of a block boundary, the last (partly filled)
    block, the second wave, the last env.  The oracle envs repeat the seeds and actions of the small-batch parity test in
    tests/test_gpu_parity.py, so its envelope, measured on those samples, applies unchanged."""
    c = _prepare(case_name, mp)
    mp.delenv("B200SIM_WPB", raising=False)
    env = pkg.make_vec(env_id, num_envs=n, device="cuda:0", **kw)
    _needs_cabi(env.backend)
    w, nb = _launch_config(env.backend)
    rows = {3 * w, 4 * w - 1, 9 * w - 1, 9 * w, (nb - 1) * w, n - 1}
    if nb > _num_sms(env.device):
        rows |= {_num_sms(env.device) * w, _num_sms(env.device) * w + w - 1}
    rows = sorted(r for r in rows if r < n)
    fill = c["S"][torch.arange(n, device=c["S"].device) % c["K"]]
    return env, fill, rows


def test_fetch_pick_and_place_4096_parity_at_block_edges(monkeypatch):
    """FetchPickAndPlace, 4096 envs: oracle states injected at block edges and in the second wave, the other envs heterogeneous;
    the envelopes and reward / success rules of tests/test_gpu_parity.py::test_step_parity_from_identical_state."""
    from tests.test_gpu_parity import ENVELOPE

    n, task = 4096, "FetchPickAndPlace"
    env, fill, rows = _production(f"{task}-v4", n, "fetch_pick", monkeypatch, rng_mode="torch")
    env.reset(seed=0)
    env.set_state(fill)
    oracles = [oracle_env_from_model(task, env.model) for _ in rows]
    for i, o in enumerate(oracles):
        o.reset(seed=100 + i % 8)
    rng, g = np.random.default_rng(7), torch.Generator(device=env.device).manual_seed(8)
    free, contact = [], []
    for step in range(12):
        inject_oracle_state(env, oracles, rows=rows)
        a = torch.rand((n, 4), generator=g, device=env.device) * 2 - 1
        ao = rng.uniform(-1, 1, (8, 4)).astype(np.float32)[np.arange(len(rows)) % 8]
        if step >= 6:
            ao[:, 2] = -1.0
            ao[:, 3] = -1.0 if step % 2 else 1.0
        a[rows] = torch.as_tensor(ao, device=env.device)
        o, r, term, trunc, info = env.step(a)
        for i, (row, orc) in enumerate(zip(rows, oracles)):
            oo, orr, _, _, oi = orc.step(ao[i].astype(np.float64))
            got = o["observation"][row].double().cpu().numpy()
            assert np.isfinite(got).all()
            (free if step < 6 else contact).append(np.abs(got - oo["observation"]).max())
            assert not bool(term[row]) and not bool(trunc[row])
            d = np.linalg.norm(oo["achieved_goal"] - oo["desired_goal"])
            if abs(d - 0.05) > 5e-3:
                assert float(r[row]) == float(orr) and float(info["is_success"][row]) == float(oi["is_success"])
    check_envelope(f"fetch_free/{task}@{n}", free, *ENVELOPE[f"fetch_free/{task}"])
    check_envelope(f"fetch_contact/{task}@{n}", contact, *ENVELOPE[f"fetch_contact/{task}"])
    env.close()


def test_hand_touch_2048_parity_at_block_edges(monkeypatch):
    """HandManipulateBlockRotateXYZ_ContinuousTouchSensors, 2048 envs: the touch envelope of
    tests/test_gpu_parity.py::test_hand_touch_sensors_parity at block edges, in the partly filled block and the second wave."""
    from gymnasium_robotics_b200.models import load_model
    from oracle.hand_env import OracleHandBlockEnv
    from tests.test_gpu_parity import ENVELOPE

    n = 2048
    env, fill, rows = _production("HandManipulateBlockRotateXYZ_ContinuousTouchSensors-v1", n, "hand_touch", monkeypatch, rng_mode="torch")
    env.reset(seed=0)
    env.set_state(fill)
    model = load_model("hand_block_touch")
    oracles = [OracleHandBlockEnv(model=model, touch_get_obs="sensordata") for _ in rows]
    for i, o in enumerate(oracles):
        o.reset(seed=60 + i % 4)
    rng, g = np.random.default_rng(6), torch.Generator(device=env.device).manual_seed(8)
    terr, fired_same, fired_total = [], 0, 0
    goal = lambda i, o, rec, lay: rec.__setitem__(slice(lay["goal"], lay["goal"] + 7), o.goal)   # noqa: E731
    for step in range(6):
        env.set_state(inject_records(env, oracles, goal, rows=rows))
        a = torch.rand((n, 20), generator=g, device=env.device) * 2 - 1
        ao = rng.uniform(-1, 1, (4, 20)).astype(np.float32)[np.arange(len(rows)) % 4]
        a[rows] = torch.as_tensor(ao, device=env.device)
        o, *_ = env.step(a)
        for i, (row, orc) in enumerate(zip(rows, oracles)):
            oo, *_ = orc.step(ao[i].astype(np.float64))
            t, ot = o["observation"][row, 61:].double().cpu().numpy(), oo["observation"][61:]
            assert np.isfinite(t).all() and (t >= 0).all()
            terr.append(np.abs(t - ot).max() / max(1.0, ot.max()))
            fired_same += int(((t > 1e-3) == (ot > 1e-3)).sum())
            fired_total += t.size
    check_envelope(f"hand_touch@{n}", terr, *ENVELOPE["hand_touch"])
    assert fired_same >= 0.98 * fired_total
    env.close()


def test_antmaze_1024_parity_at_block_edges(monkeypatch):
    """AntMaze_Large-v5, 1024 envs (one wave of 8-warp blocks on 132 SMs): the envelopes, rewards, success and flags of
    tests/test_gpu_parity.py::test_antmaze_step_parity_from_identical_state."""
    from gymnasium_robotics_b200.maze import MAPS
    from gymnasium_robotics_b200.models import load_model
    from oracle.ant_maze_env import OracleAntMazeEnv
    from tests.test_gpu_parity import ENVELOPE

    n = 1024
    env, fill, rows = _production("AntMaze_Large-v5", n, "antmaze", monkeypatch, rng_mode="torch")
    env.reset(seed=0)
    env.set_state(fill)
    model = load_model("antmaze_large")
    oracles = [OracleAntMazeEnv(MAPS["Large"], model=model, include_cfrc_ext_in_observation=True) for _ in rows]
    for i, o in enumerate(oracles):
        o.reset(seed=20 + i % 8)
    rng, g = np.random.default_rng(2), torch.Generator(device=env.device).manual_seed(8)
    epos, evel, ecf = [], [], []
    goal = lambda i, o, rec, lay: rec.__setitem__(slice(lay["goal"], lay["goal"] + 2), o.goal)   # noqa: E731
    for step in range(12):
        env.set_state(inject_records(env, oracles, goal, rows=rows))
        a = torch.rand((n, 8), generator=g, device=env.device) * 2 - 1
        ao = rng.uniform(-1, 1, (8, 8)).astype(np.float32)[np.arange(len(rows)) % 8]
        a[rows] = torch.as_tensor(ao, device=env.device)
        o, r, te, tr, info = env.step(a)
        for i, (row, orc) in enumerate(zip(rows, oracles)):
            oo, orr, ote, otr, oi = orc.step(ao[i].astype(np.float64))
            d = np.abs(o["observation"][row].double().cpu().numpy() - oo["observation"])
            epos.append(d[:13].max())
            evel.append(d[13:27].max())
            ecf.append(d[27:].max())
            assert float(r[row]) == float(orr) and bool(info["success"][row]) == oi["success"]
            assert bool(te[row]) == bool(ote) and bool(tr[row]) == bool(otr)
    for grp, e in (("pos", epos), ("vel", evel), ("cfrc", ecf)):
        check_envelope(f"antmaze/{grp}@{n}", e, *ENVELOPE[f"antmaze/{grp}"])
    env.close()


def test_adroit_hammer_2048_parity_at_block_edges(monkeypatch):
    """AdroitHandHammer-v2, 2048 envs on the wide build: the envelope and reward / success rules of
    tests/test_gpu_parity.py::test_adroit_hammer_parity."""
    from gymnasium_robotics_b200.models import load_model
    from oracle.adroit_env import OracleAdroitHammerEnv
    from tests.test_gpu_parity import ENVELOPE

    n = 2048
    env, fill, rows = _production("AdroitHandHammer-v2", n, "adroit_hammer", monkeypatch, rng_mode="torch")
    env.reset(seed=0)
    m = load_model("adroit_hammer")
    oracles = [OracleAdroitHammerEnv(m, noslip=False) for _ in rows]
    for i, o in enumerate(oracles):
        o.reset(seed=30 + i % 4)

    def board(i, o, rec, lay):
        rec[lay["penv"]:lay["penv"] + 3] = o.sim.body_pos[o.target_body_id]
        rec[lay["penv"] + 3:lay["penv"] + 7] = np.asarray(m.body_quat).reshape(-1, 4)[o.target_body_id]

    env.backend.state.copy_(fill)
    rng, g = np.random.default_rng(2), torch.Generator(device=env.device).manual_seed(8)
    errs = []
    for step in range(12):
        env.backend.state.copy_(inject_records(env, oracles, board, rows=rows))
        a = torch.rand((n, 26), generator=g, device=env.device) * 2 - 1
        ao = rng.uniform(-1, 1, (4, 26)).astype(np.float32)[np.arange(len(rows)) % 4]
        if step >= 5:
            ao[:, :2] = [-1, -0.5]
        a[rows] = torch.as_tensor(ao, device=env.device)
        o, r, te, tr, info = env.step(a)
        for i, (row, orc) in enumerate(zip(rows, oracles)):
            oo, orr, _, _, oi = orc.step(ao[i].astype(np.float64))
            got = o[row].double().cpu().numpy()
            assert np.isfinite(got).all()
            errs.append(np.abs(got - oo).max())
            assert abs(float(r[row]) - orr) < 1e-3 and bool(info["success"][row]) == bool(oi["success"])
            assert not bool(te[row]) and not bool(tr[row])
    check_envelope(f"adroit_hammer@{n}", errs, *ENVELOPE["adroit_hammer"])
    env.close()


def test_kitchen_2048_parity_at_block_edges(monkeypatch):
    """FrankaKitchen-v1, 2048 envs: seeded envs at block edges, in the partly filled block and the second wave free-run next to
    heterogeneous envs and track oracle envs of the same seeds (tests/test_zz_kitchen_gpu.py::test_kitchen_env_tracks_the_oracle_env)."""
    from oracle.kitchen_env import OracleKitchenEnv
    from tests.test_zz_kitchen_gpu import KITCHEN_ENVELOPE

    n, seed = 2048, 21
    env, fill, rows = _production("FrankaKitchen-v1", n, "kitchen_groups", monkeypatch, rng_mode="numpy")
    obs, _ = env.reset(seed=seed)
    keep = torch.zeros(n, dtype=torch.bool, device=env.device)
    keep[rows] = True
    env.backend.state.copy_(torch.where(keep[:, None], env.backend.state, fill))
    orcs = [OracleKitchenEnv(env.model) for _ in rows]
    for row, o in zip(rows, orcs):
        ob, _ = o.reset(seed=seed + row)
        assert np.abs(obs["observation"][row].cpu().numpy() - ob["observation"]).max() < 1e-5
    rng = np.random.default_rng(2)
    pos_err, vel_err = [], []
    for k in range(4):
        a = rng.uniform(-1, 1, size=(n, 9))
        obs, rew, term, trunc, info = env.step(a)
        for row, o in zip(rows, orcs):
            ob, r, te, tr, _ = o.step(a[row])
            e = np.abs(obs["observation"][row].cpu().numpy() - ob["observation"])
            pos_err.append(max(e[:9].max(), e[18:39].max()))
            vel_err.append(max(e[9:18].max(), e[39:].max()))
            assert float(rew[row]) == r and bool(term[row]) == te and bool(trunc[row]) == tr
    check_envelope(f"kitchen/pos@{n}", pos_err, *KITCHEN_ENVELOPE["kitchen/pos"])
    check_envelope(f"kitchen/vel@{n}", vel_err, *KITCHEN_ENVELOPE["kitchen/vel"])
    env.close()
