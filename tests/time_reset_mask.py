"""Time partial resets in rng_mode="device": `env.reset(options={"reset_mask": m})` for 1 % and 50 % of the envs (a random device
mask, seed=None and seed=7) against a full `env.reset()`, at FetchPickAndPlace-v4 x 4096 and FrankaKitchen-v1 x 2048 (the bench
sizes).  Host clock around each call, which ends in a device synchronise; the median of `--reps` calls after two warm-up calls.
Prints one JSON line with the card, its power limit and clocks.
    python tests/time_reset_mask.py [--reps 20] [out.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

CASES = (("FetchPickAndPlace-v4", 4096), ("FrankaKitchen-v1", 2048))


def _card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))
    except (OSError, IndexError):
        return {}


def _median_ms(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


def _case(env_id, n, reps):
    from gymnasium_robotics_b200 import make_vec

    env = make_vec(env_id, num_envs=n, rng_mode="device", autoreset_mode="disabled")
    env.reset(seed=0)
    g = torch.Generator(device="cuda").manual_seed(1)
    row = {"env": env_id, "envs": n, "full_reset_ms": _median_ms(lambda: env.reset(), reps)}
    for frac in (0.01, 0.5):
        m = torch.rand(n, generator=g, device="cuda") < frac
        pct = int(frac * 100)
        row[f"partial_{pct}pct_ms"] = _median_ms(lambda: env.reset(options={"reset_mask": m}), reps)
        row[f"partial_{pct}pct_seeded_ms"] = _median_ms(lambda: env.reset(seed=7, options={"reset_mask": m}), reps)
    env.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("out", nargs="?")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    rows = {"cases": [_case(e, n, a.reps) for e, n in CASES], "card": _card()}
    text = json.dumps(rows)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
