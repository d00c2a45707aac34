"""Time AntMaze-v3's goal redraw at AntMaze_Large-v3 x 1024: b200sim_step on a v3 handle (rng_mode="device": the step kernel of the
ant build, then the redraw kernel) against b200sim_step on an AntMaze_Large-v4 handle with ant_info=True (the same ant build, no
redraw), in alternating blocks with CUDA events around each step; and env.step end to end in the device and torch modes.  Before
every timed step, outside the timed window, every goal is set to the ant's position, so every env succeeds and is redrawn.  Prints one
JSON line with the card, its power limit and clocks.
    python tests/time_antmaze_v3.py [--steps 20] [--blocks 4] [out.json]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tests.time_maze_goal_update import _card, _timed  # noqa: E402

N = 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("out", nargs="?")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from gymnasium_robotics_b200 import make_vec

    g = torch.Generator(device="cuda").manual_seed(7)
    acts = [(torch.rand((N, 8), generator=g, device="cuda") * 2 - 1) for _ in range(8)]
    envs = {"v3_redraw": make_vec("AntMaze_Large-v3", num_envs=N, rng_mode="device", max_episode_steps=None),
            "v4_ant_info": make_vec("AntMaze_Large-v4", num_envs=N, rng_mode="device", max_episode_steps=None, ant_info=True)}
    steppers = {}
    for name, env in envs.items():
        env.reset(seed=0)
        out, k = env.backend.new_outputs(), [0]

        def step(env=env, out=out, k=k):
            env.backend.step(acts[k[0] % len(acts)], out)
            k[0] += 1
        steppers[name] = step
    res = {name: [] for name in envs}
    for block in range(-1, a.blocks):   # block -1: warm-up of both
        for name, env in envs.items():
            ms = _timed(steppers[name], env, a.steps if block >= 0 else 3)
            if block >= 0:
                res[name].append(ms)
    for env in envs.values():
        env.close()
    e2e = {}
    for mode in ("device", "torch"):
        env = make_vec("AntMaze_Large-v3", num_envs=N, rng_mode=mode, max_episode_steps=None)
        env.reset(seed=0)
        _timed(lambda: env.step(acts[0]), env, 3)
        e2e[mode] = _timed(lambda: env.step(acts[1]), env, a.steps)
        env.close()
    med = lambda v: sorted(v)[len(v) // 2]
    rows = {"env": "AntMaze_Large-v3", "envs": N, "step_ms_v3_redraw": res["v3_redraw"], "step_ms_v4_ant_info": res["v4_ant_info"],
            "step_ms_median_v3_redraw": med(res["v3_redraw"]), "step_ms_median_v4_ant_info": med(res["v4_ant_info"]),
            "env_step_ms_device_rng": e2e["device"], "env_step_ms_torch_rng": e2e["torch"], "card": _card()}
    text = json.dumps(rows)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
