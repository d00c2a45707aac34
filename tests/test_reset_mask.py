"""Partial resets, Gymnasium's `reset(options={"reset_mask": mask})`, on the host emulation of the kernel source, for every env class
of the vector-env contract plus AntMaze-v3 (goal redraw) and a maze with `reset_target=True` (goal update).  The rule: a reset of
mask M with seed=x leaves each env of M exactly as a full reset(seed=x) would, and every other env as it was; with seed=None the
envs of M continue their own streams, as an autoreset does."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

from gymnasium_robotics_b200.rollout import RolloutRecorder
from tests.hostsim_backend import HostSimBackend
from tests.hostsim_keys import KeyedHostSimBackend
from tests.test_api_conformance import _leaves, _make
from tests.test_vector_env_contract import CLASSES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = dict(CLASSES, **{"AntMaze_UMaze-v3": {}, "PointMaze_UMaze-v3/reset_target": {"reset_target": True}})
N = 3
M = np.array([True, False, True])
K = 2          # steps before the partial reset
AFTER = 2      # steps after it


def _env(case, rng_mode, **kw):
    kw = dict(CASES.get(case, {}), **kw)
    kw.setdefault("max_episode_steps", 50)
    kw.setdefault("backend_factory", functools.partial(KeyedHostSimBackend, flavor="kitchen") if case.startswith("Franka") else KeyedHostSimBackend)
    return _make(case.split("/")[0], N, rng_mode=rng_mode, autoreset_mode=kw.pop("autoreset_mode", "disabled"), **kw)


def _actions(env, k):
    rng = np.random.default_rng(300 + k)
    return torch.as_tensor(rng.uniform(-1, 1, (env.num_envs, env.single_action_space.shape[0])).astype(np.float32))


def _goal_moves(env):
    return getattr(env, "_goal_update_on", False) or getattr(env, "_goal_redraw_on", False)


def _on_goals(env):
    """Put every goal on its agent, so that the goal update / redraw of the next step acts."""
    if _goal_moves(env):
        st, g = env.backend.state, env._sl["goal"]
        q = env._sl["qpos"].start
        st[:, g] = st[:, q:q + 2]


def _snapshot(env, ret):
    """Everything an env's rows hold after a call: what it returned, the packed row and flags, the record and the step counter."""
    snap = {"ret": list(_leaves(ret)), "packed": env._last["packed"].clone(), "flags": env._last["flags"].clone().t(),
            "state": env.backend.state.clone(), "elapsed": env._elapsed.clone()}
    if env._episode is not None:
        snap["episode"] = env._episode.clone()
    return snap


def _rows(snap, rows):
    out, n = {}, len(rows)
    for k, v in snap.items():
        if k == "ret":
            out.update({"ret" + name: t[rows] for name, t in v if t.dim() and t.shape[0] == n})
        else:
            out[k] = v[rows]
    return out


def _assert_rows_equal(a, b, rows, what=""):
    """The rows of two snapshots are equal bit for bit (floats compared as integer views)."""
    rows = torch.as_tensor(rows).cpu()
    ra, rb = _rows({k: _cpu(v) for k, v in a.items()}, rows), _rows({k: _cpu(v) for k, v in b.items()}, rows)
    assert ra.keys() == rb.keys(), what
    for k in ra:
        x, y = ra[k], rb[k]
        assert x.shape == y.shape, (what, k)
        if x.dtype.is_floating_point:
            x, y = x.contiguous().view(torch.int32 if x.element_size() == 4 else torch.int64), y.contiguous().view(
                torch.int32 if y.element_size() == 4 else torch.int64)
        assert torch.equal(x, y), (what, k)


def _cpu(v):
    return [(name, t.cpu()) for name, t in v] if isinstance(v, list) else v.cpu()


def _steps(env, first, n):
    snaps = []
    for k in range(first, first + n):
        _on_goals(env)
        snaps.append(_snapshot(env, env.step(_actions(env, k))))
    return snaps


def _mask(env):
    return torch.as_tensor(M, device=env.device)


def check_reseed_rule(make, mask, s1=5, s2=11):
    """make(): a fresh env in "disabled" mode.  A: reset(s1), K steps, reset(s2) of `mask`; B: reset(s2); C: A without the partial
    reset.  Through AFTER more steps, A's masked rows are B's and A's other rows are C's, bit for bit."""
    A, B, C = make(), make(), make()
    A.reset(seed=s1), C.reset(seed=s1)
    for k in range(K):
        A.step(_actions(A, k)), C.step(_actions(C, k))
    a = [_snapshot(A, A.reset(seed=s2, options={"reset_mask": mask}))] + _steps(A, K, AFTER)
    b = [_snapshot(B, B.reset(seed=s2))] + _steps(B, K, AFTER)
    c = [_snapshot(C, C._obs_dict(C._last))] + _steps(C, K, AFTER)
    keep = ~torch.as_tensor(mask).cpu()
    for t, (x, y, z) in enumerate(zip(a, b, c)):
        _assert_rows_equal(x, y, mask, what=f"masked rows, call {t}")
        if t:
            _assert_rows_equal(x, z, keep, what=f"other rows, call {t}")
        else:   # (the partial reset returns a reset info, the twin's row is the last step's return)
            _assert_rows_equal({k: v for k, v in x.items() if k != "ret"}, {k: v for k, v in z.items() if k != "ret"}, keep)
    for e in (A, B, C):
        e.close()


def check_autoreset_twin(make, mask):
    """seed=None: the masked envs continue their streams.  make(autoreset_mode) builds an env whose TimeLimit is K.  Twin D runs
    SAME_STEP, so that all its envs are autoreset on step K; the masked rows of A's partial reset after that step are D's rows, and
    so are the masked rows of the step that follows."""
    A, D = make("disabled"), make("same_step")
    A.reset(seed=5), D.reset(seed=5)
    for k in range(K):
        A.step(_actions(A, k)), D.step(_actions(D, k))
    x = _snapshot(A, A.reset(options={"reset_mask": mask})[0])
    y = _snapshot(D, D._obs_dict(D._last))
    c = A.backend.nobs + 2 * A.backend.ngoal + 2
    for snap in (x, y):   # a SAME_STEP autoreset keeps the finished episode's flags in the row; the partial reset clears them
        del snap["flags"]
        snap["packed"][:, c:c + 2] = 0
    _assert_rows_equal(x, y, mask)
    _on_goals(A), _on_goals(D)
    x, y = _snapshot(A, A.step(_actions(A, K))[0]), _snapshot(D, D.step(_actions(D, K))[0])
    for snap in (x, y):
        del snap["flags"], snap["packed"]
    _assert_rows_equal(x, y, mask)
    A.close(), D.close()


@pytest.mark.parametrize("rng_mode", ["numpy", "device"])
@pytest.mark.parametrize("case", CASES)
def test_partial_reseed_equals_a_full_reset_and_leaves_the_others(case, rng_mode):
    check_reseed_rule(lambda: _env(case, rng_mode), M)


@pytest.mark.parametrize("rng_mode", ["numpy", "device"])
@pytest.mark.parametrize("case", CASES)
def test_partial_reset_without_seed_is_an_autoreset_of_the_masked_envs(case, rng_mode):
    check_autoreset_twin(lambda mode: _env(case, rng_mode, max_episode_steps=K, autoreset_mode=mode), torch.as_tensor(M))


# ------------------------------------------------------------------ errors and the state machine
def test_device_reseed_needs_per_env_keys():
    """A backend without set_env_keys draws every env with the batch seed: a partial reset continues the masked envs' streams, but
    one with a seed cannot be expressed and is refused before anything changes."""
    env = _env("FetchPush-v4", "device", backend_factory=HostSimBackend)
    assert env._keys is None
    env.reset(seed=1)
    episode = env._episode.clone()
    with pytest.raises(NotImplementedError, match="set_env_keys"):
        env.reset(seed=2, options={"reset_mask": M})
    assert torch.equal(env._episode, episode)
    env.reset(options={"reset_mask": M})
    assert env._episode.tolist() == [2, 1, 2] and env._elapsed.tolist() == [0, 0, 0]
    env.close()


def test_mask_validation():
    env = _env("FetchReach-v4", "numpy")
    env.reset(seed=0)
    for bad in (np.ones(N, dtype=np.int64), np.ones(N + 1, dtype=bool), np.zeros(N, dtype=bool), torch.ones(N, dtype=torch.uint8),
                torch.ones((N, 1), dtype=torch.bool), [True] * N):
        with pytest.raises(ValueError, match="reset_mask"):
            env.reset(options={"reset_mask": bad})
    env.close()


@pytest.mark.parametrize("rng_mode", ["numpy", "device"])
def test_all_false_torch_mask_is_a_no_op(rng_mode):
    env = _env("FetchPush-v4", rng_mode)
    env.reset(seed=1)
    env.step(_actions(env, 0))
    before = _snapshot(env, env._obs_dict(env._last))
    rngs = [r.bit_generator.state for r in env._np_rngs] if env._np_rngs else None
    obs, info = env.reset(options={"reset_mask": torch.zeros(N, dtype=torch.bool)})
    after = _snapshot(env, obs)
    _assert_rows_equal({k: v for k, v in before.items() if k != "ret"}, {k: v for k, v in after.items() if k != "ret"}, torch.ones(N, dtype=torch.bool))
    assert info == {}
    if rngs is not None:
        assert [r.bit_generator.state for r in env._np_rngs] == rngs
    env.close()


def test_pending_next_step_reset_of_a_masked_env_is_cancelled():
    env = _env("FetchReach-v4", "numpy", max_episode_steps=1, autoreset_mode="next_step")
    env.reset(seed=2)
    _, _, _, tr, _ = env.step(_actions(env, 0))
    assert bool(tr.all())
    obs, _ = env.reset(seed=9, options={"reset_mask": M})
    assert env._needs_reset.tolist() == [False, True, False] and not env._in_phase
    o, r, te, tr, info = env.step(_actions(env, 1))
    # env 1 is reset by this call (reward 0, counter 0); envs 0 and 2 were reset by the mask and take the step
    assert env._elapsed.tolist() == [1, 0, 1] and float(r[1]) == 0.0
    env.close()


def test_full_mask_keeps_the_envs_in_phase():
    env = _env("FetchReach-v4", "numpy", max_episode_steps=2, autoreset_mode="next_step")
    env.reset(seed=2)
    env.step(_actions(env, 0))
    env.reset(options={"reset_mask": np.ones(N, dtype=bool)})
    assert env._in_phase and env._elapsed_ub == 0 and env._elapsed.tolist() == [0] * N
    env.close()


def test_maze_goal_cell_goes_with_the_mask():
    env = _env("PointMaze_UMaze-v3", "device")
    env.reset(seed=3)
    obs0, _ = env.reset(seed=3)
    obs, info = env.reset(options={"reset_mask": _mask(env), "goal_cell": [1, 1]})
    want = torch.as_tensor(env.cells.cell_rowcol_to_xy([1, 1]), dtype=torch.float32)
    d = (obs["desired_goal"] - want).abs().max(dim=1).values
    assert bool((d[M] <= 0.25 * env.scaling + 1e-6).all())              # the cell + the reset noise
    assert torch.equal(obs["desired_goal"][~M], obs0["desired_goal"][~M])
    env.close()


def test_maze_reset_info_masks_are_the_reset_mask():
    env = _env("AntMaze_UMaze-v5/continuing", "numpy", ant_info=True)
    env.reset(seed=3)
    _, info = env.reset(options={"reset_mask": M})
    masks = [k for k in info if k.startswith("_")]
    assert masks and all(torch.equal(info[k], torch.as_tensor(M)) for k in masks)
    env.close()


def test_adroit_initial_state_dict_does_not_combine_with_a_mask():
    env = _env("AdroitHandDoor-v2", "numpy")
    env.reset(seed=0)
    with pytest.raises(ValueError, match="reset_mask"):
        env.reset(options={"reset_mask": M, "initial_state_dict": env.get_env_state()})
    env.close()


def _kitchen(n=N):
    from gymnasium_robotics_b200.kitchen import KitchenVectorEnv
    from gymnasium_robotics_b200.models import load_model

    return KitchenVectorEnv(num_envs=n, backend_factory=functools.partial(KeyedHostSimBackend, flavor="kitchen"), device="cpu",
                            model=load_model("franka_kitchen"), rng_mode="device")


def test_kitchen_state_round_trip_carries_each_envs_key():
    A = _kitchen()
    A.reset(seed=1)
    A.step(_actions(A, 0))
    A.reset(seed=2**63 + 7, options={"reset_mask": np.array([False, True, False])})
    A.reset(seed=-3, options={"reset_mask": np.array([False, False, True])})
    A.step(_actions(A, 1))
    assert len(set(A._keys.tolist())) == 3
    state, elapsed = A.get_state()
    B = _kitchen()
    B.reset(seed=99)
    B.set_state(state, elapsed)
    assert torch.equal(B._keys, A._keys) and torch.equal(B._episode, A._episode)
    for k in range(2, 4):
        oa, ob = A.step(_actions(A, k)), B.step(_actions(B, k))
        for (name, u), (_, v) in zip(_leaves(oa), _leaves(ob)):
            assert torch.equal(u, v), name
    A.close(), B.close()


# ------------------------------------------------------------------ the recorder
def test_recorder_cuts_only_the_masked_episodes():
    env = _env("FetchReach-v4", "numpy")
    rec = RolloutRecorder(env, 16)
    rec.reset(seed=0)
    for k in range(3):
        rec.step(_actions(env, k))
    obs, _ = env.reset(seed=8, options={"reset_mask": M})
    rec.mark_reset(obs, M)
    for k in range(3, 5):
        rec.step(_actions(env, k))
    eps = rec.episodes()
    by_env = {i: [e for e in eps if e["env_index"] == i] for i in range(N)}
    assert [len(by_env[i]) for i in range(N)] == [2, 1, 2]
    for i in (0, 2):
        first, second = by_env[i]
        assert len(first["actions"]) == 3 and bool(first["truncations"][-1]) and not first["truncations"][:-1].any()
        assert np.array_equal(second["observations"]["observation"][0], obs["observation"][i].numpy())
    assert len(by_env[1][0]["actions"]) == 5 and not by_env[1][0]["truncations"].any()
    env.close()


# ------------------------------------------------------------------ sharding
def _run_rank(rank, world, port, n_total, out_q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gymnasium_robotics_b200.fetch import FetchVectorEnv
    from gymnasium_robotics_b200.sharding import gather_step_outputs, local_env_range
    from tests.hostsim_keys import KeyedHostSimBackend

    lo, hi = local_env_range(n_total, rank, world)
    env = FetchVectorEnv("FetchPush", num_envs=hi - lo, backend_factory=KeyedHostSimBackend, rng_mode="device", env_offset=lo,
                         autoreset_mode="disabled")
    out_q.put((rank, _sharded_rollout(env, lo, hi, n_total, gather_step_outputs)))
    dist.barrier()
    dist.destroy_process_group()


def _sharded_rollout(env, lo, hi, n_total, gather):
    tape = np.random.default_rng(0).uniform(-1, 1, (4, n_total, 4)).astype(np.float32)
    mask = (np.arange(n_total) % 3 == 1)[lo:hi]
    env.reset(seed=100)
    res = []
    for t in range(2):
        o, r, *_ = env.step(tape[t, lo:hi])
    o, _ = env.reset(seed=7, options={"reset_mask": torch.as_tensor(mask)})
    res.append(gather(o, torch.zeros(hi - lo)))
    for t in range(2, 4):
        o, r, *_ = env.step(tape[t, lo:hi])
        res.append(gather(o, r))
    return [x.numpy() for x in res]


def test_two_rank_partial_reseed_equals_single_process():
    import torch.multiprocessing as mp

    from gymnasium_robotics_b200.fetch import FetchVectorEnv

    n_total = 4
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_run_rank, args=(r, 2, port, n_total, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    env = FetchVectorEnv("FetchPush", num_envs=n_total, backend_factory=KeyedHostSimBackend, rng_mode="device", autoreset_mode="disabled")

    def gather(o, r):
        return torch.cat([o["observation"], o["achieved_goal"], o["desired_goal"], r[:, None]], 1)

    single = _sharded_rollout(env, 0, n_total, n_total, gather)
    for a, b in zip(got[0], single):
        assert a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))
