"""Writes tests/golden/fetch_fixture.json from the reference's Fetch MJCF (B200SIM_REFERENCE_ASSETS = the reference checkout's
gymnasium_robotics/envs/assets): the numbers tests/test_model_compiler.py reads from the XML text and from a fresh compile of
fetch/pick_and_place.xml, so that those tests run without the reference checkout.
  subtree_mass: sum of the <inertial mass=...> entries of each robot body's subtree (fetch/robot.xml)
  gripper_link_inertial_pos: <inertial pos> of robot0:gripper_link (fetch/robot.xml)
  M0_upper: the upper triangle (numpy.triu_indices order) of the compiler's dense mass matrix at qpos0, summed on the unfused
  MJCF tree"""
import json
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from gymnasium_robotics_b200.mjcf import compile_mjcf  # noqa: E402
from tests.test_model_compiler import _xml_subtree_masses  # noqa: E402

ASSETS = os.environ["B200SIM_REFERENCE_ASSETS"]
robot = os.path.join(ASSETS, "fetch", "robot.xml")
sub = _xml_subtree_masses(robot)
g = next(b for b in ET.parse(robot).getroot().iter("body") if b.get("name") == "robot0:gripper_link")
m = compile_mjcf(os.path.join(ASSETS, "fetch", "pick_and_place.xml"))
out = {"subtree_mass": {k: sub[k] for k in ("robot0:base_link", "robot0:torso_lift_link")},
       "gripper_link_inertial_pos": [float(x) for x in g.find("inertial").get("pos").split()],
       "M0_upper": [float(x) for x in m._full_arrays["M0"][np.triu_indices(m.nv)]]}
with open(os.path.join(HERE, "fetch_fixture.json"), "w") as f:
    json.dump(out, f, separators=(",", ":"))
    f.write("\n")
