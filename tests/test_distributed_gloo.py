"""world_size-2 gloo test of the multi-GPU path (SURVEY.md 8e): envs shard by contiguous index range, seeds follow the
global env index, and the optional all_gather of step outputs reproduces the single-process batch bit for bit."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(rank, world, port, n_total, steps, out_q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gymnasium_robotics_b200.fetch import FetchVectorEnv
    from gymnasium_robotics_b200.sharding import env_seeds, gather_step_outputs, local_env_range
    from tests.hostsim_backend import HostSimBackend

    lo, hi = local_env_range(n_total, rank, world)
    env = FetchVectorEnv("FetchReach", num_envs=hi - lo, backend_factory=HostSimBackend, rng_mode="numpy")
    env.reset(seed=env_seeds(100, rank, world, n_total))
    tape = np.random.default_rng(0).uniform(-1, 1, (steps, n_total, 4)).astype(np.float32)
    for t in range(steps):
        o, r, *_ = env.step(tape[t, lo:hi])
    g = gather_step_outputs(o, r)
    if rank == 0:
        out_q.put(g.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_shards_equal_single_process():
    from gymnasium_robotics_b200.sharding import local_env_range

    assert local_env_range(4096, 3, 8) == (1536, 2048) and local_env_range(10, 3, 4) == (9, 10)
    n_total, steps = 4, 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_run, args=(r, 2, port, n_total, steps, q)) for r in range(2)]
    for p in procs:
        p.start()
    gathered = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    # single process, same global seeds and actions
    from gymnasium_robotics_b200.fetch import FetchVectorEnv
    from tests.hostsim_backend import HostSimBackend

    env = FetchVectorEnv("FetchReach", num_envs=n_total, backend_factory=HostSimBackend, rng_mode="numpy")
    env.reset(seed=list(range(100, 100 + n_total)))
    tape = np.random.default_rng(0).uniform(-1, 1, (steps, n_total, 4)).astype(np.float32)
    for t in range(steps):
        o, r, *_ = env.step(tape[t])
    single = torch.cat([o["observation"], o["achieved_goal"], o["desired_goal"], r[:, None]], 1).numpy()
    assert gathered.shape == single.shape and np.array_equal(gathered, single)


def _run_mixed(rank, world, port, n_local, steps, out_q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import gymnasium_robotics_b200 as pkg
    from gymnasium_robotics_b200.sharding import gather_mixed_outputs, mixed_batch_assignment
    from tests.hostsim_backend import HostSimBackend

    env_id = mixed_batch_assignment(["AdroitHandHammer-v2", "AdroitHandRelocate-v2"], world)[rank]
    env = pkg.make_vec(env_id, num_envs=n_local, backend_factory=HostSimBackend, rng_mode="numpy")
    env.reset(seed=[7 + rank * n_local + i for i in range(n_local)])
    rng = np.random.default_rng(rank)
    for _ in range(steps):
        o, r, *_ = env.step(rng.uniform(-1, 1, (n_local, env.single_action_space.shape[0])).astype(np.float32))
    g = gather_mixed_outputs(o, r, width=46)
    if rank == 0:
        out_q.put((g.numpy(), o.numpy(), r.numpy()))
    dist.barrier()
    dist.destroy_process_group()


def test_mixed_batch_whole_ranks_per_model():
    """BASELINE config 5 shape: heterogeneous models on one node, whole ranks per model (here Hammer on rank 0 and
    Relocate on rank 1 -- Kitchen is not on the CUDA path yet), observations gathered zero-padded to the widest one."""
    from gymnasium_robotics_b200.sharding import mixed_batch_assignment

    assert mixed_batch_assignment(["a", "b"], 4) == ["a", "a", "b", "b"] and mixed_batch_assignment(["a", "b"], 3) == ["a", "a", "b"]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_run_mixed, args=(r, 2, port, 2, 2, q)) for r in range(2)]
    for p in procs:
        p.start()
    g, o0, r0 = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert g.shape == (4, 47)
    assert np.array_equal(g[:2, :46], o0) and np.array_equal(g[:2, 46], r0)      # rank 0: hammer, 46 wide
    assert np.all(g[2:, 39:46] == 0) and np.isfinite(g).all() and np.abs(g[2:, :39]).max() > 0   # rank 1: relocate, 39 wide, padded


def _run_packed(rank, world, port, n_total, steps, out_q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gymnasium_robotics_b200.fetch import FetchVectorEnv
    from gymnasium_robotics_b200.sharding import PackedGather, env_seeds, local_env_range
    from tests.hostsim_backend import HostSimBackend

    lo, hi = local_env_range(n_total, rank, world)
    env = FetchVectorEnv("FetchPush", num_envs=hi - lo, backend_factory=HostSimBackend, rng_mode="numpy", max_episode_steps=2)
    env.reset(seed=env_seeds(100, rank, world, n_total))
    gather = PackedGather(hi - lo, env.backend.packed_w, "cpu")
    tape = np.random.default_rng(0).uniform(-1, 1, (steps, n_total, 4)).astype(np.float32)
    rows = []
    for t in range(steps):
        env.step(tape[t, lo:hi])
        gather.launch(env._last["packed"])       # the packed rows of this step (flags included), every step
        rows.append(gather.wait().clone())
    if rank == 0:
        out_q.put(torch.stack(rows).numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_packed_rows_gathered_from_two_ranks_equal_one_process():
    """sharding.PackedGather (the optional all-gather of SURVEY.md 8e) on the packed step rows: two ranks' gathered rows -- obs,
    goals, reward, success AND the kernel's terminated / truncated flags -- equal the single-process batch bit for bit, on the step
    that crosses the TimeLimit too."""
    n_total, steps = 4, 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_run_packed, args=(r, 2, port, n_total, steps, q)) for r in range(2)]
    for p in procs:
        p.start()
    gathered = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    from gymnasium_robotics_b200.fetch import FetchVectorEnv
    from tests.hostsim_backend import HostSimBackend

    env = FetchVectorEnv("FetchPush", num_envs=n_total, backend_factory=HostSimBackend, rng_mode="numpy", max_episode_steps=2)
    env.reset(seed=list(range(100, 100 + n_total)))
    tape = np.random.default_rng(0).uniform(-1, 1, (steps, n_total, 4)).astype(np.float32)
    for t in range(steps):
        env.step(tape[t])
        single = env._last["packed"].numpy()
        assert gathered[t].shape == single.shape and np.array_equal(gathered[t], single), t
        k = env.backend.nobs + 6
        assert np.all(single[:, k + 3] == (1.0 if t == 1 else 0.0))      # truncated flag of the TimeLimit (2 steps), NEXT_STEP reset after it
