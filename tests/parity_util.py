"""Helpers shared by the parity tests, smoke() and the bench's CPU-baseline leg (the only allowed oracle users)."""
from __future__ import annotations

import numpy as np
import torch

from oracle.fetch_env import OracleFetchEnv


def oracle_env_from_model(task, model, reward_type="sparse"):
    """Oracle env built from an already compiled model (so nothing reads /root/reference at run time)."""
    return OracleFetchEnv(task, reward_type=reward_type, model=model)


def oracle_state_record(env, orc):
    """One fp32 state record (layout of include/b200sim.h) from the oracle env's current fp64 state."""
    lay = env.backend.layout
    m = env.model
    rec = np.zeros(lay["stride"], dtype=np.float64)
    s = orc.sim
    rec[lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
    rec[lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
    rec[lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
    rec[lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
    rec[lay["mocap"]:lay["mocap"] + 3] = s.mocap_pos[0]
    rec[lay["mocap"] + 3:lay["mocap"] + 7] = s.mocap_quat[0]
    rec[lay["pose"]:lay["pose"] + 3] = s.site_xpos[orc._gripper_frame]
    rec[lay["pose"] + 3:lay["pose"] + 7] = orc._body_xquat(orc._gripper_frame)
    rec[lay["goal"]:lay["goal"] + 3] = orc.goal
    return rec


def inject_oracle_state(env, oracles, rows=None):
    """Oracle i's state into env row rows[i] (default: row i for every env of the batch); the other rows keep their records."""
    recs = torch.as_tensor(np.stack([oracle_state_record(env, o) for o in oracles]), dtype=torch.float32).to(env.backend.state.device)
    rows = slice(None) if rows is None else torch.as_tensor(rows, device=env.backend.state.device)
    st = env.backend.state.clone()
    st[rows] = recs
    obs = env.set_state(st)
    # set_state refreshes derived data, which re-anchors the stored "pose of the welded body as of the last forward
    # pass" to the injected qpos; the oracle's value is one sub-step stale (SURVEY.md Appendix C.1/C.3): restore it
    lay = env.backend.layout
    env.backend.state[rows, lay["pose"]:lay["pose"] + 7] = recs[:, lay["pose"]:lay["pose"] + 7]
    return obs


def oracle_obs_vector(obs):
    return np.asarray(obs["observation"], dtype=np.float64)


# ------------------------------------------------------------------------------------------------ stated tolerance envelopes
PARITY_STATS = {}   # name -> dict(n, p50, p99, max): written to $B200_PARITY_STATS at session end (tests/conftest.py)


def check_envelope(name, errs, p50, p99, mx):
    """The fp32-vs-fp64 error distribution of one observation group of one env family against its STATED envelope: median, 99th
    percentile and maximum are all asserted (no share of the samples is exempt).  `errs`: one value per (env, env-step) sample =
    max |obs_gpu - obs_oracle| over the entries of the group."""
    e = np.asarray(errs, dtype=np.float64).ravel()
    assert e.size > 0 and np.isfinite(e).all(), f"{name}: non-finite error samples"
    st = dict(n=int(e.size), p50=float(np.quantile(e, 0.5)), p99=float(np.quantile(e, 0.99)), max=float(e.max()),
              limit=dict(p50=p50, p99=p99, max=mx))
    PARITY_STATS[name] = st
    print(f"parity[{name}]: n={st['n']} p50={st['p50']:.2e} p99={st['p99']:.2e} max={st['max']:.2e}   (envelope {p50:.0e} / {p99:.0e} / {mx:.0e})")
    assert st["p50"] <= p50 and st["p99"] <= p99 and st["max"] <= mx, f"{name}: {st} outside its envelope"


def inject_records(env, oracles, extra=None, rows=None):
    """State records (qpos | qvel | warm start | ctrl [| goal] [| per-env body pose]) from oracle envs that expose `.sim` (families
    without a mocap weld: Shadow Hand, Adroit, mazes).  `extra(i, oracle, rec, lay)` fills family-specific slots.  Without `rows`
    the result holds one record per oracle; with `rows` it is the env's whole state with oracle i's record in row rows[i]."""
    lay, m = env.backend.layout, env.model
    rec = np.zeros((len(oracles), lay["stride"]))
    for i, o in enumerate(oracles):
        s = o.sim
        rec[i, lay["qpos"]:lay["qpos"] + m.nq] = s.qpos
        rec[i, lay["qvel"]:lay["qvel"] + m.nv] = s.qvel
        rec[i, lay["warm"]:lay["warm"] + m.nv] = s.qacc_warmstart
        rec[i, lay["ctrl"]:lay["ctrl"] + m.nu] = s.ctrl
        if extra is not None:
            extra(i, o, rec[i], lay)
    recs = torch.as_tensor(rec, dtype=torch.float32, device=env.backend.state.device)
    if rows is None:
        return recs
    st = env.backend.state.clone()
    st[torch.as_tensor(rows, device=st.device)] = recs
    return st
