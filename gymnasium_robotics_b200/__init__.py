"""gymnasium_robotics_b200: batched CUDA simulator (H100, sm_90a) behind the Gymnasium-Robotics env API (hot path only).

Drop-in boundary mirrored from the reference registry (gymnasium_robotics/__init__.py:12-80): the same env ids and
kwargs, constructed as batched vector envs.  `make_vec(id, num_envs=N)` works without gymnasium; when gymnasium is
importable the ids are also registered with a `vector_entry_point` so that
`gymnasium.make_vec(id, num_envs=N, vectorization_mode="vector_entry_point")` builds the CUDA env.
"""
from __future__ import annotations

import os

__version__ = "0.1.0"

# id -> (task, reward_type, max_episode_steps); only the new-binding versions (-v4) of the reference are mirrored,
# the mujoco_py (-v1) ids are out of scope (SURVEY.md section 2, rows 3/11/12)
ENV_IDS = {"FrankaKitchen-v1": dict(kitchen=True, max_episode_steps=280)}   # __init__.py:1117-1121
for _task in ("FetchReach", "FetchPush", "FetchSlide", "FetchPickAndPlace"):
    for _rt, _suffix in (("sparse", ""), ("dense", "Dense")):
        ENV_IDS[f"{_task}{_suffix}-v4"] = dict(task=_task, reward_type=_rt, max_episode_steps=50)
# AntMaze: the reference registers v3/v4/v5 x sparse/dense (__init__.py:838-958), all three are mirrored
for _maze, _steps in (("UMaze", 700), ("Open", 700), ("Open_Diverse_G", 700), ("Open_Diverse_GR", 700), ("Medium", 1000),
                      ("Medium_Diverse_G", 1000), ("Medium_Diverse_GR", 1000), ("Large", 1000), ("Large_Diverse_G", 1000),
                      ("Large_Diverse_GR", 1000)):
    for _rt, _suffix in (("sparse", ""), ("dense", "Dense")):
        # -v5 wraps Gymnasium's Ant-v5 with its defaults: the observation carries the clipped per-body contact forces,
        # (105,) = 27 + 13 x 6 (envs/maze/ant_maze_v5.py:99, 132-134, 249-255)
        ENV_IDS[f"AntMaze_{_maze}{_suffix}-v5"] = dict(maze=_maze, reward_type=_rt, max_episode_steps=_steps, include_cfrc_ext_in_observation=True)
        # -v4 (envs/maze/ant_maze_v4.py) is the same class on Gymnasium's Ant-v4 (use_contact_forces defaults to False there): the
        # same ant.xml, frame_skip and maze_v4 logic with the (27,) observation
        ENV_IDS[f"AntMaze_{_maze}{_suffix}-v4"] = dict(maze=_maze, reward_type=_rt, max_episode_steps=_steps)
        # -v3 (envs/maze/ant_maze_v3.py) wraps Gymnasium's Ant-v4 too, with the older task logic of envs/maze/maze.py (maze_version=3)
        ENV_IDS[f"AntMaze_{_maze}{_suffix}-v3"] = dict(maze=_maze, reward_type=_rt, max_episode_steps=_steps, maze_version=3)
# PointMaze-v3 (__init__.py:960-1080)
for _maze, _steps in (("UMaze", 300), ("Open", 300), ("Open_Diverse_G", 300), ("Open_Diverse_GR", 300), ("Medium", 600),
                      ("Medium_Diverse_G", 600), ("Medium_Diverse_GR", 600), ("Large", 800), ("Large_Diverse_G", 800),
                      ("Large_Diverse_GR", 800)):
    for _rt, _suffix in (("sparse", ""), ("dense", "Dense")):
        ENV_IDS[f"PointMaze_{_maze}{_suffix}-v3"] = dict(maze=_maze, agent="point", reward_type=_rt, max_episode_steps=_steps)
# Shadow-Hand block manipulation, new-binding ids (-v1; __init__.py:105-395); touch-sensor variants are "next"
for _task in ("HandManipulateBlockRotateZ", "HandManipulateBlockRotateParallel", "HandManipulateBlockRotateXYZ",
              "HandManipulateBlockFull", "HandManipulateBlock", "HandManipulateEggRotate", "HandManipulateEggFull",
              "HandManipulateEgg", "HandManipulatePenRotate", "HandManipulatePenFull",
              "HandManipulatePen"):
    for _rt, _suffix in (("sparse", ""), ("dense", "Dense")):
        ENV_IDS[f"{_task}{_suffix}-v1"] = dict(hand_task=_task, reward_type=_rt, max_episode_steps=100)
        # 92 touch sensors appended to the observation (__init__.py:122-170 and siblings)
        ENV_IDS[f"{_task}_BooleanTouchSensors{_suffix}-v1"] = dict(hand_task=_task, reward_type=_rt, max_episode_steps=100,
                                                                  touch_get_obs="boolean")
        ENV_IDS[f"{_task}_ContinuousTouchSensors{_suffix}-v1"] = dict(hand_task=_task, reward_type=_rt, max_episode_steps=100,
                                                                     touch_get_obs="sensordata")
# HandReach, new-binding version (__init__.py:90-95)
for _rt, _suffix in (("sparse", ""), ("dense", "Dense")):
    ENV_IDS[f"HandReach{_suffix}-v3"] = dict(hand_task="HandReach", reward_type=_rt, max_episode_steps=50)
# Adroit hand (__init__.py:1082-1101): dense reward is the plain id, `Sparse` the suffix; max_episode_steps = 200
for _rt, _suffix in (("dense", ""), ("sparse", "Sparse")):
    ENV_IDS[f"AdroitHandHammer{_suffix}-v2"] = dict(adroit_task="AdroitHandHammer", reward_type=_rt, max_episode_steps=200)
    ENV_IDS[f"AdroitHandRelocate{_suffix}-v2"] = dict(adroit_task="AdroitHandRelocate", reward_type=_rt, max_episode_steps=200)
    ENV_IDS[f"AdroitHandDoor{_suffix}-v2"] = dict(adroit_task="AdroitHandDoor", reward_type=_rt, max_episode_steps=200)
    ENV_IDS[f"AdroitHandPen{_suffix}-v2"] = dict(adroit_task="AdroitHandPen", reward_type=_rt, max_episode_steps=200)


def _ant_version(env_id):
    """The Ant an AntMaze id wraps: Ant-v5 (-v5), Ant-v4 (-v4 and -v3, ant_maze_v3.py:7)."""
    return 4 if env_id.endswith("-v3") else int(env_id[-1])


def make_vec(env_id: str, num_envs: int = 1, **kwargs):
    """Batched replacement for `gym.make_vec(env_id, num_envs=...)` (reference ids, e.g. "FetchPickAndPlace-v4")."""
    if env_id.startswith("FrankaKitchen"):
        # kernel build csrc/b200sim_kitchen*.cu (joint-equality rows, condim 6, two-level broad phase); validated on the GPU against
        # the oracle env and the host emulation (tests/test_zz_kitchen_gpu.py)
        if env_id != "FrankaKitchen-v1":
            raise KeyError(f"{env_id!r}: the reference registers FrankaKitchen-v1 only")
        kwargs.pop("experimental", None)   # accepted and ignored: the id was opt-in while the build was unvalidated
        from .kitchen import KitchenVectorEnv

        return KitchenVectorEnv(num_envs=num_envs, **kwargs)
    if env_id not in ENV_IDS:
        raise KeyError(f"{env_id!r} is not provided by the CUDA path yet; available: {sorted(ENV_IDS)}")
    spec = dict(ENV_IDS[env_id])
    spec.update(kwargs)
    if env_id.startswith("AntMaze_"):
        spec["ant_version"] = _ant_version(env_id)
    if "maze" in spec:
        from .maze import MazeVectorEnv

        return MazeVectorEnv(num_envs=num_envs, **spec)
    if "hand_task" in spec:
        from .hand import make_hand_vec

        return make_hand_vec(spec.pop("hand_task"), num_envs=num_envs, **spec)
    if "adroit_task" in spec:
        from .adroit import make_adroit_vec

        return make_adroit_vec(spec.pop("adroit_task"), num_envs=num_envs, **spec)
    from .fetch import FetchVectorEnv

    return FetchVectorEnv(num_envs=num_envs, **spec)


def _vector_entry_point(task, **kwargs):
    from .fetch import FetchVectorEnv

    return FetchVectorEnv(task=task, **kwargs)


def register_envs():
    """Register the ids with gymnasium (no-op when gymnasium is not installed)."""
    try:
        import gymnasium  # noqa: F401
        from gymnasium.envs.registration import register, registry
    except Exception:  # noqa: BLE001
        return False
    for env_id, spec in ENV_IDS.items():
        if env_id in registry:
            continue
        ep = "gymnasium_robotics_b200.maze:MazeVectorEnv" if "maze" in spec else \
            ("gymnasium_robotics_b200.hand:make_hand_vec" if "hand_task" in spec else
             ("gymnasium_robotics_b200.adroit:make_adroit_vec" if "adroit_task" in spec else
              ("gymnasium_robotics_b200.kitchen:KitchenVectorEnv" if "kitchen" in spec else "gymnasium_robotics_b200.fetch:FetchVectorEnv")))
        kw = dict(spec)
        kw.pop("kitchen", None)
        if "hand_task" in kw:
            kw["task"] = kw.pop("hand_task")
        if "adroit_task" in kw:
            kw["task"] = kw.pop("adroit_task")
        if env_id.startswith("AntMaze_"):
            kw["ant_version"] = _ant_version(env_id)
        register(id=env_id, vector_entry_point=ep, kwargs=kw)
    return True
