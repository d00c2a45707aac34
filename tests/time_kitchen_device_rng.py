"""Time the FrankaKitchen-v1 step with the observation noise drawn in the kitchen step kernel (rng_mode="device") at 2048 envs:
the step kernel alone with the noise on and off (same handle, alternating blocks of launches, CUDA events), and env.step end to
end in rng_mode "device" against "torch" (host-drawn noise).  Prints one JSON line with the card, its power limit and clocks.
    python tests/time_kitchen_device_rng.py [--envs 2048] [--launches 30] [--blocks 4]"""
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


def _kernel_ms(env, acts, launches, noise):
    be = env.backend
    if noise:
        env._device_noise()
    else:
        be.set_obs_noise(None, 0, 0, None)
    out = be.new_outputs()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for k in range(launches):
        be.step(acts[k % len(acts)], out)
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / launches


def _env_ms(env, acts, steps):
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for k in range(steps):
        env.step(acts[k % len(acts)])
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    from gymnasium_robotics_b200 import make_vec

    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=2048)
    ap.add_argument("--launches", type=int, default=30)
    ap.add_argument("--blocks", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    n = a.envs
    g = torch.Generator(device="cuda").manual_seed(7)
    raw = [(torch.rand((n, 9), generator=g, device="cuda") * 2 - 1) for _ in range(8)]
    dev = make_vec("FrankaKitchen-v1", num_envs=n, rng_mode="device", max_episode_steps=None)
    dev.reset(seed=0)
    # the kernel's input is the position target env.step derives from the last noisy robot pose
    acts = [dev.control_targets(x) for x in raw]
    for noise in (True, False):
        _kernel_ms(dev, acts, 3, noise)   # warm-up of both branches
    on, off = [], []
    for _ in range(a.blocks):
        on.append(_kernel_ms(dev, acts, a.launches, True))
        off.append(_kernel_ms(dev, acts, a.launches, False))
    dev._device_noise()
    dev.reset(seed=0)
    _env_ms(dev, raw, 3)
    e2e_dev = _env_ms(dev, raw, a.launches)
    dev.close()
    host = make_vec("FrankaKitchen-v1", num_envs=n, rng_mode="torch", max_episode_steps=None)
    host.reset(seed=0)
    _env_ms(host, raw, 3)
    e2e_host = _env_ms(host, raw, a.launches)
    host.close()
    print(json.dumps({"envs": n, "kernel_ms_noise_on": on, "kernel_ms_noise_off": off,
                      "kernel_ms_median_on": sorted(on)[len(on) // 2], "kernel_ms_median_off": sorted(off)[len(off) // 2],
                      "env_step_ms_device_rng": e2e_dev, "env_step_ms_torch_rng": e2e_host, "card": _card()}))


if __name__ == "__main__":
    main()
