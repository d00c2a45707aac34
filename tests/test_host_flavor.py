"""The host emulation picks its flavor as b200sim_create picks its kernel build (tests.hostsim.host_flavor): for every registered id and
the Kitchen and AntMaze variants, the derived flavor accepts the model and lays out the device model and the per-env scratch as the
flavor the tests named by hand before (Kitchen: "kitchen_hull" for the hull model, "kitchen" for the flat scan; an ant-build maze task:
"ant"; else the plain or, above 32 dofs, the wide flavor).  The one exception is the default FrankaKitchen-v1, which the old table ran on
the flat-scan layout although the library runs it on the two-level broad phase: its named flavor here is "kitchen_groups"."""
import pytest

import gymnasium_robotics_b200 as pkg
from gymnasium_robotics_b200.fetch import reference_point
from tests.hostsim import HostSim, host_flavor

VARIANTS = [("FrankaKitchen-v1", dict(broadphase="flat")), ("FrankaKitchen-v1", dict(mesh_collision="hull")),
            ("AntMaze_UMaze-v5", dict(ant_info=True)), ("AntMaze_Large-v4", dict(use_contact_forces=True))]
CASES = [(env_id, {}) for env_id in sorted(pkg.ENV_IDS)] + VARIANTS


class _Captured(Exception):
    pass


def _backend_args(env_id, kw):
    """The backend factory's arguments of an id, and the flavor derived inside the factory call (where KitchenVectorEnv sets the broad
    phase), without building the env."""
    got = {}

    def factory(model, eq_data, task, num_envs, device):
        got.update(model=model, eq_data=eq_data, task=task, flavor=host_flavor(model, task))
        raise _Captured

    with pytest.raises(_Captured):
        pkg.make_vec(env_id, num_envs=1, backend_factory=factory, **kw)
    return got


def _words(model, eq_data, task, flavor):
    penv = int(task.penv_body) if task.kind in (4, 5, 6, 7) else -1
    s = HostSim(model, eq_data=eq_data if len(eq_data) else None, ref=reference_point(task), penv_body=penv, flavor=flavor)
    return int(s._L.hostsim_hot_words(s._h)), int(s._L.hostsim_scr_words(s._h))


@pytest.mark.parametrize("env_id,kw", CASES, ids=[env_id + "".join(f"-{k}={v}" for k, v in kw.items()) for env_id, kw in CASES])
def test_derived_flavor_lays_the_model_out_as_the_named_one(env_id, kw):
    a = _backend_args(env_id, kw)
    model, task = a["model"], a["task"]
    if env_id.startswith("Franka"):
        named = "kitchen_hull" if kw.get("mesh_collision") == "hull" else "kitchen" if kw.get("broadphase") == "flat" else "kitchen_groups"
    elif task.kind == 1 and task.touch_mode >= 2:
        named = "ant"
    else:
        named = model.nv > 32
    derived = _words(model, a["eq_data"], task, a["flavor"])   # (HostSim raises when hostsim_create refuses the model)
    assert derived == _words(model, a["eq_data"], task, named), (a["flavor"], named)
