"""Support-map narrow phase for mesh geoms (compile_mjcf(mesh_hull=True), kernel builds with -DB200_HULL): the fp32 emulation of the
kernel source (1-lane and 32-lane) against the fp64 oracle on scenes whose moving body is a mesh -- dropped onto a plane (plane-hull: the
deepest vertices), onto a fixed box and against a capsule (portal refinement on the hull's support function)."""
import numpy as np
import pytest

from gymnasium_robotics_b200.mjcf import compile_mjcf
from oracle.oracle_sim import OracleSim
from tests.hostsim import HostSim

# a wedge-like convex polytope (no symmetry: the support vertex is unique in almost every direction)
VERTS = "-0.06 -0.04 -0.03  0.06 -0.04 -0.03  0.06 0.04 -0.03  -0.06 0.04 -0.03  -0.03 -0.02 0.04  0.04 -0.02 0.04  0.04 0.03 0.04  -0.03 0.03 0.04  0 0 0"
SCENE = """
<mujoco><option timestep="0.002"/>
<asset><mesh name="wedge" vertex="{verts}"/></asset>
<worldbody>
  {floor}
  <body name="w" pos="0 0 0.12" euler="12 -7 25">
    <freejoint/>
    <inertial pos="0 0 0" mass="0.4" diaginertia="0.0004 0.0006 0.0008"/>
    <geom name="wg" type="mesh" mesh="wedge" friction="0.8 0.005 0.0001"/>
  </body>
  {extra}
</worldbody></mujoco>"""
CASES = {
    "plane": ('<geom name="floor" type="plane" size="1 1 0.1"/>', ""),
    "box": ("", '<body name="t" pos="0.01 0.0 0.0"><geom type="box" size="0.2 0.2 0.05"/></body>'),
    "capsule": ('<geom name="floor" type="plane" size="1 1 0.1"/>',
                '<body name="c" pos="0.02 0 0.03"><geom type="capsule" size="0.02 0.15" euler="90 0 0"/></body>'),
}


@pytest.mark.parametrize("flavor", ["kitchen_hull", "warp_kitchen_hull"])
@pytest.mark.parametrize("case", list(CASES))
def test_hull_scenes_track_the_oracle(mjcf_file, case, flavor):
    floor, extra = CASES[case]
    model = compile_mjcf(mjcf_file(SCENE.format(verts=VERTS, floor=floor, extra=extra)), mesh_hull=True)
    assert 7 in model.geom_type.tolist() and model.hull_vert.shape == (8, 3)        # the interior point is not a hull vertex
    orc, hs = OracleSim(model), HostSim(model, ref=(0.0, 0.0, 0.1), flavor=flavor)
    hs.qpos[:] = orc.qpos
    hs.qvel[:] = 0
    hs.qacc[:] = 0
    contacts = 0
    for k in range(12):
        orc.step(25)
        hs.step(25)
        contacts = max(contacts, orc.ncon)
        # falling, hitting, tumbling: positions to 0.3 mm, the quaternion to 3e-3 (an impact on one vertex amplifies round-off)
        assert np.abs(hs.qpos[:3] - orc.qpos[:3]).max() < 3e-4, (k, hs.qpos, orc.qpos)
        assert np.abs(hs.qpos[3:7] - orc.qpos[3:7]).max() < 3e-3, (k, hs.qpos, orc.qpos)
    assert contacts >= 1 and float(orc.qpos[2]) > 0.0           # it landed on something and did not fall through


def test_box_proxy_models_are_refused_by_nothing_and_mesh_models_by_the_plain_builds(mjcf_file):
    """A model compiled with mesh_hull carries MESH geoms: the builds without -DB200_HULL refuse it loudly instead of treating the
    vertex table as a box."""
    floor, extra = CASES["plane"]
    model = compile_mjcf(mjcf_file(SCENE.format(verts=VERTS, floor=floor, extra=extra)), mesh_hull=True)
    with pytest.raises(Exception):
        HostSim(model, ref=(0.0, 0.0, 0.1), flavor="kitchen_groups")
    proxy = compile_mjcf(mjcf_file(SCENE.format(verts=VERTS, floor=floor, extra=extra)))      # default: box proxy, no vertex table
    assert 7 not in proxy.geom_type.tolist() and proxy.hull_vert.size == 0
    HostSim(proxy, ref=(0.0, 0.0, 0.1), flavor="kitchen_groups")


# ---------------------------------------------------------------------------------------------------------------
# FrankaKitchen-v1 with mesh_collision="hull": the env on the hull emulation against the oracle env on the same hull model
def test_kitchen_hull_env_tracks_the_oracle_env():
    import torch

    from gymnasium_robotics_b200.kitchen import KitchenVectorEnv
    from gymnasium_robotics_b200.models import load_model
    from oracle.kitchen_env import OracleKitchenEnv
    from tests.hostsim_backend import HostSimBackend

    model = load_model("franka_kitchen_hull")
    gh = np.asarray(model.geom_hull).reshape(-1, 2)
    assert int((np.asarray(model.geom_type) == 7).sum()) == 9 and gh[:, 1].max() == 32 and model.hull_vert.shape == (288, 3)
    # the hull of every link lies inside its box proxy and reaches it on all six faces (bounding box of the same vertices)
    for g in np.nonzero(gh[:, 1])[0]:
        v = model.hull_vert[gh[g, 0]: gh[g, 0] + gh[g, 1]]
        assert np.all(np.abs(v) <= model.geom_size[g] + 1e-9) and np.allclose(np.abs(v).max(axis=0), model.geom_size[g], atol=1e-9)
    n, seed = 2, 31
    env = KitchenVectorEnv(num_envs=n, backend_factory=HostSimBackend, device="cpu", rng_mode="numpy", model=model, mesh_collision="hull")
    obs, _ = env.reset(seed=seed)
    orcs = [OracleKitchenEnv(model) for _ in range(n)]
    for i, o in enumerate(orcs):
        ob, _ = o.reset(seed=seed + i)
        assert np.abs(obs["observation"][i].numpy() - ob["observation"]).max() < 1e-5
    rng = np.random.default_rng(4)
    for k in range(3):
        a = rng.uniform(-1, 1, size=(n, 9))
        obs, rew, term, trunc, info = env.step(a)
        for i, o in enumerate(orcs):
            ob, r, te, tr, _ = o.step(a[i])
            e = np.abs(obs["observation"][i].numpy() - ob["observation"])
            assert max(e[:9].max(), e[18:39].max()) < 2e-5 and e.max() < 2e-3, (k, i, e.max())
            assert float(rew[i]) == r and bool(term[i]) == te
    env.close()


def test_kitchen_hull_contact_phase_matches_the_oracle():
    """The contact case: a constant action drives the arm until a link's hull touches the kitchen (oracle: a contact with a MESH geom from
    env-step 7 on); the env on the hull emulation keeps tracking the oracle env through the touch."""
    from gymnasium_robotics_b200.kitchen import KitchenVectorEnv
    from gymnasium_robotics_b200.models import load_model
    from oracle.kitchen_env import OracleKitchenEnv
    from tests.hostsim_backend import HostSimBackend

    model = load_model("franka_kitchen_hull")
    env = KitchenVectorEnv(num_envs=1, backend_factory=HostSimBackend, device="cpu", rng_mode="numpy", model=model, mesh_collision="hull")
    env.reset(seed=1)
    orc = OracleKitchenEnv(model)
    orc.reset(seed=1)
    a = np.array([[1.0, 1.0, 1.0, -1.0, -1.0, 1.0, -1.0, 0.0, 0.0]])
    mesh_contact_steps = 0
    for k in range(12):
        obs, rew, term, trunc, info = env.step(a)
        ob, r, te, tr, _ = orc.step(a[0])
        e = np.abs(obs["observation"][0].numpy() - ob["observation"])
        hit = any(model.geom_type[int(c["geom1"])] == 7 or (int(c["geom2"]) >= 0 and model.geom_type[int(c["geom2"])] == 7) for c in orc.sim.contacts())
        mesh_contact_steps += int(hit)
        assert max(e[:9].max(), e[18:39].max()) < (2e-5 if mesh_contact_steps == 0 else 5e-4), (k, e[:9].max(), e[18:39].max())
        assert float(rew[0]) == r
    assert mesh_contact_steps >= 4, "no hull geom came into contact: the test would not exercise the hull narrow phase"
    env.close()
