"""Time the Ant's per-step info (ant_info=True) at AntMaze_Large-v5 x 1024: the step launch (b200sim_step) of a handle with the info on
(the ant kernel build) against one with it off (the plain build), in alternating blocks, CUDA events around each block.  Prints one
JSON line with the card, its power limit and clocks.
    python tests/time_ant_info.py [--steps 50] [--blocks 6] [out.json]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def _card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))
    except (OSError, IndexError):
        return {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("out", nargs="?")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ant_info.py measures the GPU: no CUDA device")
    import gymnasium_robotics_b200 as pkg

    n = 1024
    envs = {on: pkg.make_vec("AntMaze_Large-v5", num_envs=n, device="cuda:0", rng_mode="device", ant_info=on) for on in (False, True)}
    g = torch.Generator(device="cuda:0").manual_seed(0)
    acts = [torch.rand((n, 8), generator=g, device="cuda:0") * 2 - 1 for _ in range(args.steps)]
    outs = {}
    for on, env in envs.items():
        env.reset(seed=0)
        outs[on] = env.backend.new_outputs()
        if on:
            env._new_ant_rows()
        for a in acts[:10]:      # warm-up: module load, the ants land
            env.backend.step(a, outs[on])
    torch.cuda.synchronize()
    times = {False: [], True: []}
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for b in range(args.blocks):
        for on in ((False, True) if b % 2 == 0 else (True, False)):
            env = envs[on]
            t0.record()
            for a in acts:
                env.backend.step(a, outs[on])
            t1.record()
            t1.synchronize()
            times[on].append(t0.elapsed_time(t1) / len(acts))
    res = dict(case="AntMaze_Large-v5 x 1024, b200sim_step", card=_card(), steps_per_block=args.steps, blocks=args.blocks,
               info_off_ms=sorted(times[False]), info_on_ms=sorted(times[True]),
               median_off_ms=sorted(times[False])[len(times[False]) // 2], median_on_ms=sorted(times[True])[len(times[True]) // 2])
    line = json.dumps(res, default=str)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
