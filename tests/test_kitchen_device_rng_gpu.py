"""FrankaKitchen rng_mode="device" on the H100: the observation noise drawn in the kitchen step kernel is invariant to batch shape,
block size and sharding per global env index, equals the host restatement bit for bit, keeps the env within the oracle's
envelope, and makes get_state / set_state a bitwise checkpoint."""
import numpy as np
import pytest
import torch

from tests.test_kitchen_device_rng import restated_obs, restated_uniforms

pytestmark = pytest.mark.gpu
SEED, STEPS, NTOT = 1234, 3, 2048


def _env(n, **kw):
    from gymnasium_robotics_b200 import make_vec

    kw.setdefault("max_episode_steps", 2)   # step 3 is a NEXT_STEP autoreset: the reset's noise is part of every comparison
    return make_vec("FrankaKitchen-v1", num_envs=n, rng_mode="device", **kw)


def _actions(k, lo, hi):
    """Step k's actions of global envs lo..hi-1 (the same whatever the batch that steps them)."""
    a = np.random.default_rng(k).uniform(-1, 1, size=(NTOT, 9)).astype(np.float32)
    return torch.as_tensor(a[lo:hi], device="cuda:0")


def _flat(x):
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in _flat(x[k])]
    if isinstance(x, (tuple, list)):
        return [v for e in x for v in _flat(e)]
    if torch.is_tensor(x):
        x = x.detach().cpu().contiguous()
        return [x.view(torch.int32) if x.dtype == torch.float32 else x]
    return []


def _rollout(env, lo):
    """Reset + STEPS steps; every returned tensor (observation, goals, reward, flags, bookkeeping) per call, on the host."""
    n = env.num_envs
    out = [_flat(env.reset(seed=SEED))]
    for k in range(STEPS):
        out.append(_flat(env.step(_actions(k, lo, lo + n))))
    env.close()
    return out


def _rows(ref, lo, hi):
    return [[t[lo:hi] if t.dim() > 0 and t.shape[0] == NTOT else t for t in call] for call in ref]


def _same(a, b):
    assert len(a) == len(b)
    for ca, cb in zip(a, b):
        assert len(ca) == len(cb)
        for x, y in zip(ca, cb):
            assert x.shape == y.shape and torch.equal(x, y)


@pytest.fixture(scope="module")
def reference():
    return _rollout(_env(NTOT), 0)


@pytest.mark.parametrize("n, lo", [(1, 0), (37, 0), (37, 1000)])
def test_batch_shape_invariance(reference, n, lo):
    _same(_rollout(_env(n, env_offset=lo), lo), _rows(reference, lo, lo + n))


@pytest.mark.parametrize("wpb", [7, 10, 11])
def test_block_size_invariance(reference, wpb, monkeypatch):
    monkeypatch.setenv("B200SIM_WPB", str(wpb))
    env = _env(96)
    import ctypes

    w = ctypes.c_int()
    env.backend.L.b200sim_launch_config(env.backend.h, None, ctypes.byref(w), None)
    assert w.value == wpb
    _same(_rollout(env, 0), _rows(reference, 0, 96))


def test_two_shards_equal_one_batch(reference):
    a, b = _rollout(_env(1024, env_offset=0), 0), _rollout(_env(1024, env_offset=1024), 1024)
    _same(a, _rows(reference, 0, 1024))
    _same(b, _rows(reference, 1024, NTOT))


def _clean(env):
    env.backend.set_obs_noise(None, 0, 0, None)
    out = env.backend.new_outputs()
    env.backend.refresh(None, out)
    env._device_noise()
    return out["obs"].cpu().numpy()


def test_device_noise_equals_the_restatement():
    env = _env(64, max_episode_steps=None, env_offset=3)
    obs, _ = env.reset(seed=99)
    scale = env._noise_scale.cpu().numpy()
    for k in range(3):
        if k:
            obs, *_ = env.step(_actions(k, 0, 64))
        noisy, clean = obs["observation"].cpu().numpy(), _clean(env)
        ep, el = env._episode.cpu().numpy(), env._elapsed.cpu().numpy()
        assert (el == k).all() and (ep == 1).all()
        for i in range(64):
            want = restated_obs(clean[i], scale, 99, 3 + i, int(ep[i]), int(el[i]))
            # noisy - clean in fp64, compared as bit patterns
            assert np.array_equal((noisy[i].astype(np.float64) - clean[i]).view(np.int64), (want.astype(np.float64) - clean[i]).view(np.int64)), (k, i)
    env.close()


class _Replay:
    """np_random stand-in for the oracle: hands out the restated uniforms of (seed, env, episode 1, step t) in draw order."""

    def __init__(self, seed, env):
        self.seed, self.env, self.t, self.buf = seed, env, 0, []

    def uniform(self, low=-1.0, high=1.0, size=None):
        assert (low, high) == (-1.0, 1.0)
        if not self.buf:
            self.buf = list(restated_uniforms(self.seed, self.env, 1, self.t).astype(np.float64))
            self.t += 1
        k = int(np.prod(size))
        out, self.buf = np.array(self.buf[:k]), self.buf[k:]
        return out.reshape(size)


def test_device_env_tracks_the_oracle_with_the_same_noise():
    from oracle.kitchen_env import OracleKitchenEnv
    from tests.parity_util import check_envelope
    from tests.test_zz_kitchen_gpu import KITCHEN_ENVELOPE

    n, seed = 4, 21
    env = _env(n, max_episode_steps=None)
    obs, _ = env.reset(seed=seed)
    orcs = [OracleKitchenEnv(env.model) for _ in range(n)]
    for i, o in enumerate(orcs):
        o.reset()
        o.robot_env.np_random = _Replay(seed, i)
        ob = o._get_obs(o.robot_env.reset_model())      # the reset observation with the injected noise of step 0
        assert np.abs(obs["observation"][i].cpu().numpy() - ob["observation"]).max() < 1e-5
    rng = np.random.default_rng(2)
    pos_err, vel_err = [], []
    for k in range(4):
        a = rng.uniform(-1, 1, size=(n, 9))
        obs, rew, term, trunc, info = env.step(a)
        for i, o in enumerate(orcs):
            ob, r, te, tr, _ = o.step(a[i])
            e = np.abs(obs["observation"][i].cpu().numpy() - ob["observation"])
            pos_err.append(max(e[:9].max(), e[18:39].max()))
            vel_err.append(max(e[9:18].max(), e[39:].max()))
            assert float(rew[i]) == r and bool(term[i]) == te and bool(trunc[i]) == tr
    check_envelope("kitchen/pos", pos_err, *KITCHEN_ENVELOPE["kitchen/pos"])
    check_envelope("kitchen/vel", vel_err, *KITCHEN_ENVELOPE["kitchen/vel"])
    env.close()


def test_checkpoint_round_trip_is_bitwise():
    n = 64
    A = _env(n, max_episode_steps=7)
    A.reset(seed=5)
    for k in range(5):
        A.step(_actions(k, 0, n))
    state, elapsed = A.get_state()
    a_now = _flat(A._obs_dict(A._last)) + _flat([A._todo, A._episode_done, A._episode, A._last_robot_qpos])
    a_ret = [_flat(A.step(_actions(k, 0, n))) for k in range(5, 10)]   # crosses the TimeLimit at 7 and the NEXT_STEP reset
    B = _env(n, max_episode_steps=7)
    b_now = _flat(B.set_state(state, elapsed)) + _flat([B._todo, B._episode_done, B._episode, B._last_robot_qpos])
    _same([a_now], [b_now])
    b_ret = [_flat(B.step(_actions(k, 0, n))) for k in range(5, 10)]
    _same(a_ret, b_ret)
    _same([_flat([A._todo, A._episode_done, A._episode])], [_flat([B._todo, B._episode_done, B._episode])])
    A.close()
    B.close()


def test_obs_noise_entry_point_refuses_other_builds():
    from gymnasium_robotics_b200.fetch import FetchVectorEnv

    env = FetchVectorEnv("FetchReach", num_envs=2)
    scale = torch.zeros(env.backend.nobs, device="cuda:0")
    with pytest.raises(RuntimeError, match="kitchen"):
        env.backend.set_obs_noise(scale, 0, 0, torch.zeros(2, dtype=torch.int32, device="cuda:0"))
    env.close()
