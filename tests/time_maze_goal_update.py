"""Time the goal update of continuing maze tasks (reset_target=True) at AntMaze_Large-v5 x 1024 and PointMaze_Large-v3 x 4096:
b200sim_step on one handle with the update kernel on and off (alternating blocks, CUDA events around each step), and env.step end
to end in rng_mode "device" (update kernel) against "torch" (the host loop over the succeeding envs).  Before every timed step,
outside the timed window, every goal is set to the agent's position, so every env succeeds and is redrawn.  Prints one JSON line
with the card, its power limit and clocks.
    python tests/time_maze_goal_update.py [--steps 20] [--blocks 4] [out.json]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

CASES = (("AntMaze_Large-v5", 1024), ("PointMaze_Large-v3", 4096))


def _card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))
    except (OSError, IndexError):
        return {}


def _all_succeed(env):
    st = env.backend.state
    q, g = env._sl["qpos"].start, env._sl["goal"]
    st[:, g] = st[:, q:q + 2]


def _timed(fn, env, steps):
    """Mean ms of fn() over `steps` calls, each after _all_succeed (not timed)."""
    total = 0.0
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(steps):
        _all_succeed(env)
        torch.cuda.synchronize()
        t0.record()
        fn()
        t1.record()
        t1.synchronize()
        total += t0.elapsed_time(t1)
    return total / steps


def _case(env_id, n, steps, blocks):
    from gymnasium_robotics_b200 import make_vec
    from gymnasium_robotics_b200.maze import NOISE

    g = torch.Generator(device="cuda").manual_seed(7)
    dev = make_vec(env_id, num_envs=n, rng_mode="device", reset_target=True, max_episode_steps=None)
    nact = dev.single_action_space.shape[0]
    acts = [(torch.rand((n, nact), generator=g, device="cuda") * 2 - 1) for _ in range(8)]
    dev.reset(seed=0)
    be, out = dev.backend, dev.backend.new_outputs()
    on_args = (dev._goal_loc, dev.scaling, NOISE, dev._dev_seed, dev.env_offset, dev._episode)
    k = [0]

    def step():
        be.step(acts[k[0] % len(acts)], out)
        k[0] += 1

    res = {"on": [], "off": []}
    for block in range(-1, blocks):   # block -1: warm-up of both
        for mode in ("on", "off"):
            be.set_goal_update(*on_args) if mode == "on" else be.set_goal_update(None, 0, 0, 0, 0, None)
            ms = _timed(step, dev, steps if block >= 0 else 3)
            if block >= 0:
                res[mode].append(ms)
    be.set_goal_update(*on_args)
    dev.reset(seed=0)
    _timed(lambda: dev.step(acts[0]), dev, 3)
    e2e_dev = _timed(lambda: dev.step(acts[1]), dev, steps)
    dev.close()
    host = make_vec(env_id, num_envs=n, rng_mode="torch", reset_target=True, max_episode_steps=None)
    host.reset(seed=0)
    _timed(lambda: host.step(acts[0]), host, 3)
    e2e_host = _timed(lambda: host.step(acts[1]), host, steps)
    host.close()
    med = lambda v: sorted(v)[len(v) // 2]
    return {"env": env_id, "envs": n, "step_ms_update_on": res["on"], "step_ms_update_off": res["off"],
            "step_ms_median_on": med(res["on"]), "step_ms_median_off": med(res["off"]),
            "env_step_ms_device_rng": e2e_dev, "env_step_ms_torch_rng_host_loop": e2e_host}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("out", nargs="?")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    rows = {"cases": [_case(e, n, a.steps, a.blocks) for e, n in CASES], "card": _card()}
    text = json.dumps(rows)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
