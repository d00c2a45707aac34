"""FrankaKitchen rng_mode="device" on the kitchen-flavor host emulation of the kernel source: the observation noise drawn by
kitchen_observe (csrc/fetch_task.cuh) is Philox4x32-10 over (seed; global env index, episode, step), bit for bit the restatement
below, uniform per entry, and a pure function of the state, so that get_state / set_state checkpoint a Kitchen env."""
import functools

import numpy as np
import pytest
import torch
from scipy import stats

from gymnasium_robotics_b200.kitchen import KitchenVectorEnv
from gymnasium_robotics_b200.models import load_model
from tests import hostsim
from tests.hostsim_backend import HostSimBackend

NOBS = 59
TAG = 0x0B5E


def _philox():
    return hostsim.lib(wide=False).hostsim_philox4x32_10


def restated_uniforms(seed, env, episode, t):
    """Philox4x32-10 (the host build's hostsim_philox4x32_10) at counter (env, episode, (t << 4) | block, 0x0B5E), key (seed low,
    seed high); word w of block b -> entry 4 b + w as 2 (x >> 8) / 2^24 - 1 (exact in fp32)."""
    philox = _philox()
    seed &= 0xFFFFFFFFFFFFFFFF
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32)
    u = np.zeros(60, dtype=np.float32)
    for b in range(15):
        ctr = np.array([env, episode, (t << 4) | b, TAG], dtype=np.uint32)
        r = np.zeros(4, dtype=np.uint32)
        philox(ctr.ctypes.data, key.ctypes.data, r.ctypes.data)
        u[4 * b:4 * b + 4] = ((r >> 8).astype(np.float64) * 2.0 ** -23 - 1.0).astype(np.float32)
    return u[:NOBS]


def restated_obs(clean, scale, seed, env, episode, t):
    """The noisy observation: clean + round(u * scale), both operations rounded to fp32 on their own."""
    noise = restated_uniforms(seed, env, episode, t) * np.asarray(scale, dtype=np.float32)   # fp32 * fp32 -> fp32
    return (np.asarray(clean, dtype=np.float32) + noise).astype(np.float32)


@pytest.fixture(scope="module")
def model():
    return load_model("franka_kitchen")


def _make(model, n, backend=functools.partial(HostSimBackend, flavor="kitchen"), **kw):   # the flat-scan build
    kw.setdefault("rng_mode", "device")
    return KitchenVectorEnv(num_envs=n, backend_factory=backend, device="cpu", model=model, **kw)


def _clean_obs(env):
    """The noise-free observation of the current records (same handle, noise off for one refresh)."""
    env.backend.set_obs_noise(None, 0, 0, None)
    out = env.backend.new_outputs()
    env.backend.refresh(None, out)
    env._device_noise()
    return out["obs"].clone().numpy()


def _check_noise(env, noisy, elapsed=None):
    clean = _clean_obs(env)
    scale = env._noise_scale.numpy()
    el = env._elapsed.numpy() if elapsed is None else elapsed
    for i in range(env.num_envs):
        want = restated_obs(clean[i], scale, env._dev_seed, env.env_offset + i, int(env._episode[i]), int(el[i]))
        got = np.asarray(noisy[i], dtype=np.float32)
        # noisy - clean (fp64) equals the restated noise added in fp32, compared as int32 bit patterns
        assert np.array_equal((got.astype(np.float64) - clean[i]).view(np.int64), (want.astype(np.float64) - clean[i]).view(np.int64)), i
        assert not np.array_equal(got, clean[i])


def test_known_answers_match_the_restatement():
    for seed, env, episode, t in ((0, 0, 0, 0), (7, 3, 1, 0), (2**40 + 12345, 2047, 9, 279), (-3, 1 << 20, 123456, (1 << 28) - 1), (2**64 - 1, 5, 2, 17)):
        out = hostsim.kitchen_noise(seed, env, episode, t)
        want = restated_uniforms(seed, env, episode, t)
        assert np.array_equal(out.view(np.int32), want.view(np.int32)), (seed, env, episode, t)
        assert out.min() >= -1.0 and out.max() < 1.0


def test_noise_at_reset_and_after_steps(model):
    env = _make(model, 3, env_offset=5)
    obs, _ = env.reset(seed=21)
    assert env._episode.tolist() == [1, 1, 1] and env._elapsed.tolist() == [0, 0, 0]
    _check_noise(env, obs["observation"])
    # the next control targets start from the noisy robot qpos
    assert torch.equal(env._last_robot_qpos, obs["observation"][:, :9])
    rng = np.random.default_rng(1)
    for _ in range(2):
        obs, *_ = env.step(torch.as_tensor(rng.uniform(-1, 1, size=(3, 9)), dtype=torch.float32))
        _check_noise(env, obs["observation"])
    # achieved_goal is the true (noise-free) state
    qpos = env.backend.state[:, env._sl["qpos"]]
    assert torch.equal(obs["achieved_goal"]["microwave"][:, 0], qpos[:, 22])
    assert torch.equal(obs["observation"][:, 9 + 22] == qpos[:, 22], torch.zeros(3, dtype=torch.bool))


def test_noise_after_next_step_autoreset(model):
    env = _make(model, 3, max_episode_steps=3)
    env.reset(seed=3)
    # env 1 is one step ahead: its TimeLimit ends first and it alone is reset by the next call (a masked reset)
    state, _ = env.get_state()
    env.set_state(state, torch.tensor([0, 1, 0], dtype=torch.int32))
    a = torch.zeros((3, 9))
    env.step(a)
    _, _, _, trunc, _ = env.step(a)
    assert trunc.tolist() == [False, True, False]
    obs, reward, _, trunc, _ = env.step(a)
    assert env._episode.tolist() == [1, 2, 1] and env._elapsed.tolist() == [3, 0, 3] and float(reward[1]) == 0
    _check_noise(env, obs["observation"])


def test_noise_after_same_step_autoreset(model):
    env = _make(model, 2, max_episode_steps=2, autoreset_mode="same_step")
    env.reset(seed=4)
    a = torch.zeros((2, 9))
    env.step(a)
    obs, _, _, trunc, info = env.step(a)
    assert trunc.all() and env._episode.tolist() == [2, 2] and env._elapsed.tolist() == [0, 0]
    _check_noise(env, obs["observation"])
    # the final observation is the noisy observation of the finished episode's last step: that of an env without autoreset
    ref = _make(model, 2, max_episode_steps=2, autoreset_mode="disabled")
    ref.reset(seed=4)
    ref.step(a)
    last, *_ = ref.step(a)
    assert torch.equal(info["final_obs"]["observation"].view(torch.int32), last["observation"].view(torch.int32))


def test_noise_is_uniform_per_entry_and_independent():
    n = 4000
    u = np.zeros((n, NOBS), np.float32)
    for k in range(n):
        u[k] = hostsim.kitchen_noise(77, k % 500, 1 + k // 2000, (k // 500) % 4 * 70 + 3)
    for j in range(NOBS):
        assert stats.kstest(u[:, j], "uniform", args=(-1.0, 2.0)).pvalue > 1e-4, j
    # robot entries (18) against object entries (41): no correlation beyond sampling noise
    c = np.corrcoef(u.T.astype(np.float64))
    assert np.abs(c[:18, 18:]).max() < 5.0 / np.sqrt(n)
    assert np.abs(c - np.eye(NOBS)).max() < 5.0 / np.sqrt(n)


def test_scaled_noise_is_uniform_on_the_scale(model):
    env = _make(model, 1)
    scale = env._noise_scale.numpy()
    n = 2000
    u = np.zeros((n, NOBS), np.float32)
    for k in range(n):
        u[k] = hostsim.kitchen_noise(5, k, 1, 0)
    noise = u * scale
    for j in (0, 8, 9, 17, 18, 38, 39, 58):
        assert np.abs(noise[:, j]).max() <= scale[j]
        assert stats.kstest(noise[:, j], "uniform", args=(-float(scale[j]), 2.0 * float(scale[j]))).pvalue > 1e-4, j


def _all_arrays(ret):
    """Every tensor of a step's or reset's return value, flattened in a fixed order."""
    out = []
    if isinstance(ret, dict):
        for k in sorted(ret):
            out += _all_arrays(ret[k])
    elif isinstance(ret, (tuple, list)):
        for v in ret:
            out += _all_arrays(v)
    elif torch.is_tensor(ret):
        out.append(ret.clone())
    return out


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.shape == y.shape
        xx, yy = x.contiguous(), y.contiguous()
        if xx.dtype == torch.float32:
            xx, yy = xx.view(torch.int32), yy.view(torch.int32)
        assert torch.equal(xx, yy)


def test_checkpoint_round_trip_is_bitwise(model):
    n, seed = 3, 12
    rng = np.random.default_rng(2)
    acts = [torch.as_tensor(rng.uniform(-1, 1, size=(n, 9)), dtype=torch.float32) for _ in range(10)]
    A = _make(model, n, max_episode_steps=7)
    A.reset(seed=seed)
    for k in range(5):
        A.step(acts[k])
    state, elapsed = A.get_state()
    a_obs = A._obs_dict(A._last)
    a_book = (A._todo.clone(), A._episode_done.clone(), A._episode.clone(), A._last_robot_qpos.clone())
    a_ret = [_all_arrays(A.step(acts[k])) for k in range(5, 10)]   # crosses the TimeLimit at 7 and the NEXT_STEP reset
    B = _make(model, n, max_episode_steps=7)   # fresh: the seed comes with the record
    b_obs = B.set_state(state, elapsed)
    _same(_all_arrays(b_obs), _all_arrays(a_obs))
    _same([B._todo, B._episode_done, B._episode, B._last_robot_qpos], list(a_book))
    b_ret = [_all_arrays(B.step(acts[k])) for k in range(5, 10)]
    for x, y in zip(a_ret, b_ret):
        _same(x, y)
    _same([B._todo, B._episode_done, B._episode], [A._todo, A._episode_done, A._episode])


@pytest.mark.parametrize("rng_mode", ["numpy", "torch"])
def test_set_state_still_raises_with_host_noise(model, rng_mode):
    env = _make(model, 2, rng_mode=rng_mode)
    env.reset(seed=0)
    state, elapsed = env.get_state()
    with pytest.raises(NotImplementedError):
        env.set_state(state, elapsed)


@pytest.mark.parametrize("kind", ["flat", "groups", "hull"])
def test_device_mode_builds_for_every_kitchen_build(kind):
    kw = {"flat": dict(broadphase="flat"), "groups": dict(broadphase="groups"), "hull": dict(mesh_collision="hull")}[kind]
    m = load_model("franka_kitchen_hull" if kind == "hull" else "franka_kitchen")
    env = _make(m, 2, backend=HostSimBackend, **kw)
    assert env.backend.flavor == {"flat": "kitchen", "groups": "kitchen_groups", "hull": "kitchen_hull"}[kind]
    obs, info = env.reset(seed=8)
    assert info["tasks_to_complete"].all()
    _check_noise(env, obs["observation"])
