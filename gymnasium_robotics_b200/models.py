"""Compiled model store.

The reference's MJCF/STL assets are not redistributed; `build_models()` compiles them (when B200SIM_REFERENCE_ASSETS names the
reference checkout's ``gymnasium_robotics/envs/assets``) into constant-table blobs under ``gymnasium_robotics_b200/models/``,
which are committed: they are what ships and what the library loads.
"""
from __future__ import annotations

import os

from .mjcf import Model, compile_mjcf, replace_maze_walls

_HERE = os.path.dirname(os.path.abspath(__file__))
MODEL_DIR = os.path.join(_HERE, "models")
REFERENCE_ASSETS = os.environ.get("B200SIM_REFERENCE_ASSETS", "")

# model name -> MJCF path relative to the reference's assets directory
MODEL_SOURCES = {
    "fetch_reach": "fetch/reach.xml",
    "fetch_push": "fetch/push.xml",
    "fetch_slide": "fetch/slide.xml",
    "fetch_pick_and_place": "fetch/pick_and_place.xml",
    "hand_block": "hand/manipulate_block.xml",
    "hand_block_touch": "hand/manipulate_block_touch_sensors.xml",   # + 92 touch sensors
    "hand_reach": "hand/reach.xml",
    "adroit_hammer": "adroit_hand/adroit_hammer.xml",
    "adroit_relocate": "adroit_hand/adroit_relocate.xml",
    "adroit_pen": "adroit_hand/adroit_pen.xml",
    "adroit_door": "adroit_hand/adroit_door.xml",
    # Franka Kitchen: compiles (mesh-derived link inertias, 5 joint equalities, condim-6 pairs, 3 708 candidate pairs) and runs
    # in the oracle; the CUDA builder refuses it loudly (DESIGN.md section 7)
    "franka_kitchen": "kitchen_franka/kitchen_assets/kitchen_env_model.xml",
    "hand_egg": "hand/manipulate_egg.xml",
    "hand_egg_touch": "hand/manipulate_egg_touch_sensors.xml",
    "hand_pen": "hand/manipulate_pen.xml",
    "hand_pen_touch": "hand/manipulate_pen_touch_sensors.xml",
}
# compile-time edits: the Hand's visual-only `target` free body (contype 0, never observed) is not simulated
# and only the sensors the envs read are kept ("robot0:TS_*", manipulate_touch_sensors.py:66-79)
_HAND = {"drop_bodies": ["target"], "sensor_prefix": "robot0:TS_"}
# Adroit hammer: the unused mocap body is dropped (its weld is commented out, adroit_assets.xml:92-94); nail_board stays a
# runtime body because reset_model redraws its height per episode (adroit_hammer.py:372-378); only the sensor the env reads
_ADROIT_HAMMER = {"drop_bodies": ["vive_tracker"], "keep_bodies": ["nail_board"], "sensor_prefix": "S_nail"}
# relocate: no sensor is observed (the 21 "Tch_*" touch sensors of the hand model are never read by the env)
_ADROIT_RELOCATE = {"drop_bodies": ["vive_tracker"], "sensor_prefix": "<none>"}
# pen: the static `target` pen (a colliding cylinder whose body_quat is redrawn per episode, adroit_pen.py:379-384) stays a runtime body
_ADROIT_PEN = {"drop_bodies": ["vive_tracker"], "keep_bodies": ["target"], "sensor_prefix": "<none>"}
# door: the static door `frame` is redrawn per episode (adroit_door.py:359-371)
_ADROIT_DOOR = {"drop_bodies": ["vive_tracker"], "keep_bodies": ["frame"], "sensor_prefix": "<none>"}
MODEL_OVERRIDES = {"adroit_door": _ADROIT_DOOR, "adroit_hammer": _ADROIT_HAMMER, "adroit_relocate": _ADROIT_RELOCATE, "adroit_pen": _ADROIT_PEN, "hand_block": _HAND, "hand_block_touch": _HAND, "hand_pen": _HAND, "hand_pen_touch": _HAND, "hand_egg": _HAND, "hand_egg_touch": _HAND, "hand_reach": {"sensor_prefix": "robot0:TS_"}}


# models compiled a second time with hull vertex tables for their mesh geoms (mjcf.py compile_mjcf(mesh_hull=True)): blob name -> source
# model; served by the hull build of the library (csrc/b200sim_kitchen_hull.cu), opt-in through `mesh_collision="hull"`
MODEL_HULL = {"franka_kitchen_hull": "franka_kitchen"}


# maze models: in-tree legacy twin of Gymnasium's ant.xml (Gymnasium itself is un-vendored) + generated wall boxes
ANT_XML = "../mujoco/assets/ant.xml"
POINT_XML = "point/point.xml"
MAZE_MODELS = {f"{a}maze_{k.lower()}": (a, k) for a in ("ant", "point") for k in ("Open", "UMaze", "Medium", "Large")}


def compile_maze_model(agent, maze_map):
    """Compile agent + maze walls (restating Maze.make_maze, maze_v4.py:148-242); needs the reference assets.  Generates the
    committed maze blobs; the envs build custom layouts with `build_maze_model`."""
    from .maze import AGENTS
    from .mjcf import make_maze_xml

    xml = os.path.normpath(os.path.join(REFERENCE_ASSETS, ANT_XML if agent == "ant" else POINT_XML))
    root, grid = make_maze_xml(xml, maze_map, AGENTS[agent]["scaling"], AGENTS[agent]["height"])
    return compile_mjcf(xml, root=root, grid=grid)


def build_maze_model(agent, maze_map):
    """The model of `agent` ("ant" or "point") in the layout `maze_map`, equal to `compile_maze_model(agent, maze_map)` but
    built from the committed U-maze blob of the same agent (`mjcf.replace_maze_walls`), so it needs no reference assets."""
    from .maze import AGENTS

    cfg = AGENTS[agent]
    return replace_maze_walls(load_model(f"{agent}maze_umaze"), maze_map, cfg["scaling"], cfg["height"])


def build_models(force: bool = False):
    """(Re)compile every model blob from the reference's assets, if they are available."""
    if not os.path.isdir(REFERENCE_ASSETS):
        return []
    os.makedirs(MODEL_DIR, exist_ok=True)
    built = []
    for name, rel in MODEL_SOURCES.items():
        out = os.path.join(MODEL_DIR, name + ".b200m")
        if os.path.exists(out) and not force:
            continue
        blob = compile_mjcf(os.path.join(REFERENCE_ASSETS, rel), overrides=MODEL_OVERRIDES.get(name)).to_blob()
        with open(out, "wb") as f:
            f.write(blob)
        built.append(out)
    for name, src in MODEL_HULL.items():
        out = os.path.join(MODEL_DIR, name + ".b200m")
        if os.path.exists(out) and not force:
            continue
        blob = compile_mjcf(os.path.join(REFERENCE_ASSETS, MODEL_SOURCES[src]), overrides=MODEL_OVERRIDES.get(src), mesh_hull=True).to_blob()
        with open(out, "wb") as f:
            f.write(blob)
        built.append(out)
    build_franka_config(force)
    from .maze import MAPS

    for name, (agent, key) in MAZE_MODELS.items():
        out = os.path.join(MODEL_DIR, name + ".b200m")
        if os.path.exists(out) and not force:
            continue
        with open(out, "wb") as f:
            f.write(compile_maze_model(agent, MAPS[key]).to_blob())
        built.append(out)
    return built


def build_franka_config(force: bool = False):
    """Per-dof position / velocity bounds and observation-noise amplitudes of franka_config.xml (read by FrankaRobot at
    construction, envs/franka_kitchen/franka_env.py:172-202) as a committed JSON next to the model blobs."""
    import json
    import xml.etree.ElementTree as ET

    out = os.path.join(MODEL_DIR, "franka_config.json")
    src = os.path.join(REFERENCE_ASSETS, "kitchen_franka", "franka_assets", "franka_config.xml")
    if (os.path.exists(out) and not force) or not os.path.exists(src):
        return out
    root = ET.parse(src).getroot()
    cfg = {"name": root.get("name"), "pos_bound": [], "vel_bound": [], "pos_noise_amp": [], "vel_noise_amp": []}
    i = 0
    while root.find(f"qpos{i}") is not None:
        n = root.find(f"qpos{i}")
        cfg["pos_bound"].append([float(x) for x in n.get("pos_bound").split()])
        cfg["vel_bound"].append([float(x) for x in n.get("vel_bound").split()])
        cfg["pos_noise_amp"].append(float(n.get("pos_noise_amp").split()[0]))
        cfg["vel_noise_amp"].append(float(n.get("vel_noise_amp").split()[0]))
        i += 1
    with open(out, "w") as f:
        json.dump(cfg, f, indent=0)
    return out


def load_franka_config():
    import json

    path = os.path.join(MODEL_DIR, "franka_config.json")
    if not os.path.exists(path):
        build_franka_config()
    return json.load(open(path))


def load_model(name: str) -> Model:
    path = os.path.join(MODEL_DIR, name + ".b200m")
    if not os.path.exists(path):
        build_models()
    if not os.path.exists(path):
        raise FileNotFoundError(f"compiled model {path} is missing and the reference assets are not available to build it")
    with open(path, "rb") as f:
        return Model.from_blob(f.read())
