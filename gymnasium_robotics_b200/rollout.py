"""State serialisation either side of the hot path (SURVEY.md 8f row 4).

* `CtorPickle`: the vector envs pickle the way the reference's envs do through `EzPickle` (e.g. fetch/reach.py:125-147,
  adroit_hammer.py:206-214: the constructor arguments are recorded and the unpickled object is a freshly constructed env;
  simulator state is not part of the pickle -- `get_state/set_state` / `get_env_state/set_env_state` carry that).
* `RolloutRecorder`: steps a vector env and keeps the transitions in preallocated tensors on the env's device (no host
  synchronisation per step), then cuts them into per-env episodes and writes a flat D4RL / Minari-style dump
  (README.md:40 of the reference points at Minari for datasets): `observations`, `actions`, `rewards`, `terminations`,
  `truncations`, `next_observations`, `infos/<success key>`, plus `episode_starts` / `episode_lengths` / `episode_env`.

The recorder understands the three autoreset modes of the vector envs: in `next_step` mode the call after an episode end
is the reset call (its action is ignored and its reward is zero), so that row is dropped from the data and its observation
opens the next episode; in `same_step` mode the last observation of an episode is `info["final_obs"]`; in `disabled` mode
the caller resets and calls `mark_reset()`, with the reset mask when only some envs were reset.
"""
from __future__ import annotations

import functools
import json
import os

import numpy as np
import torch

FORMAT_VERSION = 1


def _rebuild(cls, args, kwargs):
    return cls(*args, **kwargs)


class CtorPickle:
    """Mixin: record the outermost constructor call, pickle as (class, args, kwargs)."""

    def __init_subclass__(cls, **kw):
        super().__init_subclass__(**kw)
        init = cls.__dict__.get("__init__")
        if init is None:
            return

        @functools.wraps(init)
        def wrapped(self, *args, **kwargs):
            if not hasattr(self, "_ctor_call"):  # a subclass constructor got here first: keep the outermost call
                self._ctor_call = (args, dict(kwargs))
                # obs_dtype=torch.float64: observations are cast to the dtype the spaces declare (the reference returns float64,
                # robot_env.py:87-100); default None keeps the kernels' float32 tensors without a copy
                self.obs_dtype = kwargs.get("obs_dtype", None)
            init(self, *args, **kwargs)

        cls.__init__ = wrapped

    def __reduce__(self):
        args, kwargs = getattr(self, "_ctor_call", ((), {}))
        return _rebuild, (type(self), args, kwargs)

    # the rest of gymnasium.vector.VectorEnv's attribute surface that wrappers and training loops touch ([ext] gymnasium >= 1.0
    # vector/vector_env.py: spec, render_mode, closed, unwrapped, np_random, render, close_extras, context manager)
    spec = None
    render_mode = None
    is_vector_env = True

    @property
    def unwrapped(self):
        return self

    @property
    def np_random(self):
        """The per-env generators of rng_mode="numpy" (a list, one `Generator(PCG64)` per env as in the reference), else the torch generator."""
        return getattr(self, "_np_rngs", None) or getattr(self, "_gen", None)

    def _cast_obs(self, obs):
        dt = getattr(self, "obs_dtype", None)
        if dt is None:
            return obs
        return {k: self._cast_obs(v) for k, v in obs.items()} if isinstance(obs, dict) else obs.to(dt)   # (the kitchen's goals nest)

    def render(self):
        return None   # rendering is out of scope for the batched CUDA path (render_mode is always None)

    def close_extras(self, **kwargs):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False


def _flatten_obs(obs, prefix="", out=None):
    """dict (possibly nested, e.g. the kitchen's goal dicts) of [N, ...] tensors -> {"a/b": tensor}; a bare tensor -> {"": t}."""
    out = {} if out is None else out
    if isinstance(obs, dict):
        for k, v in obs.items():
            _flatten_obs(v, f"{prefix}{k}/", out)
    else:
        out[prefix[:-1] if prefix else ""] = obs
    return out


class RolloutRecorder:
    SUCCESS_KEYS = ("is_success", "success")

    def __init__(self, env, capacity_steps: int, env_id: str | None = None):
        self.env, self.capacity, self.env_id = env, int(capacity_steps), env_id
        self.num_envs = env.num_envs
        self.mode = getattr(env, "autoreset_mode", env.metadata.get("autoreset_mode", "next_step"))
        self._buf = None
        self.t = 0

    # ------------------------------------------------------------------ stepping
    def reset(self, *, seed=None, options=None):
        obs, info = self.env.reset(seed=seed, options=options) if options is not None else self.env.reset(seed=seed)
        self._cur = {k: v.clone() for k, v in _flatten_obs(obs).items()}
        self._prev_done = None
        self._seed = seed
        self.t = 0
        return obs, info

    def mark_reset(self, obs, mask=None):
        """`disabled` autoreset: the caller reset (some of) the envs; `obs` is the full batch of current observations (what
        `reset(options={"reset_mask": mask})` returns).  Without `mask` every env continues from `obs`.  With `mask` (bool, [num_envs],
        numpy or torch) only the masked envs' open episodes end here and their rows of `obs` open their next episode; the others
        go on as if nothing happened.  An episode cut this way before it terminated or was truncated gets `truncations=True` on its
        last row: from the agent's side it was cut short."""
        flat = _flatten_obs(obs)
        if mask is None:
            self._cur = {k: v.clone() for k, v in flat.items()}
            return
        dev = next(iter(flat.values())).device
        mask = torch.as_tensor(mask).to(dev, torch.bool)
        if self._buf is not None and self.t > 0:
            b, t = self._buf, self.t - 1
            b["truncations"][t] |= mask & ~b["terminations"][t]
        for k, v in flat.items():
            self._cur[k] = torch.where(mask.reshape((-1,) + (1,) * (v.dim() - 1)), v, self._cur[k])

    def _alloc(self, act, flat):
        T, dev = self.capacity, act.device
        b = {"actions": torch.empty((T,) + tuple(act.shape), dtype=act.dtype, device=dev),
             "rewards": torch.empty((T, self.num_envs), dtype=torch.float32, device=dev),
             "terminations": torch.empty((T, self.num_envs), dtype=torch.bool, device=dev),
             "truncations": torch.empty((T, self.num_envs), dtype=torch.bool, device=dev),
             "success": torch.zeros((T, self.num_envs), dtype=torch.float32, device=dev),
             "skip": torch.zeros((T, self.num_envs), dtype=torch.bool, device=dev)}
        for k, v in flat.items():
            b["obs:" + k] = torch.empty((T,) + tuple(v.shape), dtype=v.dtype, device=dev)
            b["next:" + k] = torch.empty((T,) + tuple(v.shape), dtype=v.dtype, device=dev)
        self._buf = b

    def step(self, actions):
        if self.t >= self.capacity:
            raise RuntimeError(f"RolloutRecorder is full ({self.capacity} steps): call episodes()/save() and clear()")
        obs, reward, terminated, truncated, info = self.env.step(actions)
        flat = _flatten_obs(obs)
        dev = reward.device
        act = torch.as_tensor(np.asarray(actions, dtype=np.float32)) if not torch.is_tensor(actions) else actions
        act = act.to(dev, torch.float32)
        if self._buf is None:
            self._alloc(act, flat)
        b, t = self._buf, self.t
        b["actions"][t] = act
        b["rewards"][t] = reward
        b["terminations"][t] = terminated
        b["truncations"][t] = truncated
        self._success_key = next((k for k in self.SUCCESS_KEYS if k in info), None)
        if self._success_key is not None:
            b["success"][t] = info[self._success_key].to(torch.float32)
        done = terminated | truncated
        final = _flatten_obs(info["final_obs"]) if (self.mode == "same_step" and "final_obs" in info) else None
        fmask = info.get("_final_obs") if final is not None else None
        if final is not None and self._success_key is not None and "final_info" in info and self._success_key in info["final_info"]:
            b["success"][t] = torch.where(fmask, info["final_info"][self._success_key].to(torch.float32), b["success"][t])
        for k, v in flat.items():
            b["obs:" + k][t] = self._cur[k]
            if final is not None:
                m = fmask.reshape((-1,) + (1,) * (v.dim() - 1))
                b["next:" + k][t] = torch.where(m, final[k], v)
            else:
                b["next:" + k][t] = v
        # next_step autoreset: this call reset the envs that were done on the previous one -- not a transition
        if self.mode == "next_step" and self._prev_done is not None:
            b["skip"][t] = self._prev_done
        self._prev_done = done.clone()
        self._cur = {k: v.clone() for k, v in flat.items()}
        self.t += 1
        return obs, reward, terminated, truncated, info

    def clear(self):
        self.t = 0

    # ------------------------------------------------------------------ episodes and files
    def _host(self):
        return {k: v[: self.t].cpu().numpy() for k, v in self._buf.items()} if self._buf is not None else {}

    def episodes(self, include_open: bool = True):
        """List of Minari-style episode dicts (`observations` has one row more than `actions`), env by env, in time order."""
        h = self._host()
        eps = []
        if not h:
            return eps
        okeys = [k[4:] for k in h if k.startswith("obs:")]
        for i in range(self.num_envs):
            keep = np.nonzero(~h["skip"][:, i])[0]
            done = (h["terminations"][keep, i] | h["truncations"][keep, i])
            start = 0
            ends = list(np.nonzero(done)[0] + 1)
            if include_open and (not ends or ends[-1] < len(keep)):
                ends.append(len(keep))
            for e in ends:
                rows = keep[start:e]
                if len(rows) == 0:
                    continue
                obs = {k: np.concatenate([h["obs:" + k][rows, i], h["next:" + k][rows[-1:], i]], axis=0) for k in okeys}
                eps.append({"env_index": i, "observations": obs[""] if okeys == [""] else obs, "actions": h["actions"][rows, i],
                            "rewards": h["rewards"][rows, i], "terminations": h["terminations"][rows, i],
                            "truncations": h["truncations"][rows, i], "infos": {self._success_key or "success": h["success"][rows, i]}})
                start = e
        return eps

    def save(self, path: str, include_open: bool = True):
        """Write `<path>.npz` (flat arrays + episode index) and `<path>.json` (metadata)."""
        eps = self.episodes(include_open)
        flat, starts, lengths, envs = {}, [], [], []
        n = 0
        for ep in eps:
            L = len(ep["actions"])
            starts.append(n); lengths.append(L); envs.append(ep["env_index"])
            n += L
        def cat(fn):
            return np.concatenate([fn(ep) for ep in eps], axis=0) if eps else np.zeros((0,))
        obs_is_dict = bool(eps) and isinstance(eps[0]["observations"], dict)
        keys = list(eps[0]["observations"].keys()) if obs_is_dict else [""]
        for k in keys:
            get = (lambda ep, k=k: ep["observations"][k]) if obs_is_dict else (lambda ep: ep["observations"])
            name = ("/" + k) if k else ""
            flat["observations" + name] = cat(lambda ep: get(ep)[:-1])
            flat["next_observations" + name] = cat(lambda ep: get(ep)[1:])
        for k in ("actions", "rewards", "terminations", "truncations"):
            flat[k] = cat(lambda ep, k=k: ep[k])
        skey = self._success_key or "success"
        flat["infos/" + skey] = cat(lambda ep: ep["infos"][skey])
        flat["episode_starts"] = np.asarray(starts, dtype=np.int64)
        flat["episode_lengths"] = np.asarray(lengths, dtype=np.int64)
        flat["episode_env"] = np.asarray(envs, dtype=np.int64)
        os.makedirs(os.path.dirname(os.path.abspath(path)) or ".", exist_ok=True)
        np.savez_compressed(path + ".npz", **flat)
        ctor = getattr(self.env, "_ctor_call", ((), {}))
        meta = {"format_version": FORMAT_VERSION, "env_id": self.env_id, "env_class": type(self.env).__name__, "num_envs": self.num_envs,
                "autoreset_mode": self.mode, "seed": self._seed if isinstance(self._seed, (int, type(None))) else list(self._seed),
                "total_steps": int(n), "total_episodes": len(eps), "max_episode_steps": getattr(self.env, "max_episode_steps", None),
                "ctor_kwargs": {k: v for k, v in ctor[1].items() if isinstance(v, (int, float, str, bool, type(None)))},
                "observation_keys": keys, "action_shape": list(flat["actions"].shape[1:]), "success_key": skey}
        with open(path + ".json", "w") as f:
            json.dump(meta, f, indent=1)
        return meta


def load_rollout(path: str):
    """Inverse of `RolloutRecorder.save`: (metadata, list of episode dicts)."""
    with open(path + ".json") as f:
        meta = json.load(f)
    z = np.load(path + ".npz")
    keys = meta["observation_keys"]
    eps = []
    for s, L, i in zip(z["episode_starts"], z["episode_lengths"], z["episode_env"]):
        sl = slice(int(s), int(s + L))
        obs = {}
        for k in keys:
            name = ("/" + k) if k else ""
            obs[k] = np.concatenate([z["observations" + name][sl], z["next_observations" + name][int(s + L) - 1: int(s + L)]], axis=0)
        eps.append({"env_index": int(i), "observations": obs[""] if keys == [""] else obs, "actions": z["actions"][sl],
                    "rewards": z["rewards"][sl], "terminations": z["terminations"][sl], "truncations": z["truncations"][sl],
                    "infos": {meta["success_key"]: z["infos/" + meta["success_key"]][sl]}})
    return meta, eps
