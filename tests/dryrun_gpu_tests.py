"""Pre-flight for GPU test files on a machine without a GPU: rewrites `device="cuda"` -> "cpu" in a temporary copy and routes `make_vec`
to the host emulation backends, then runs pytest on the copies.  It checks the tests' own logic and API usage (shapes, layouts, launch
counts, the expected draws), not the CUDA kernels.  Only tests that build their envs through `make_vec` can be routed; a test that
constructs a `*VectorEnv` or a `CudaBackend` directly hits the product path's loud "no CPU fallback" error here, as it should.
    python tests/dryrun_gpu_tests.py tests/test_reset_device_gpu.py tests/test_rollout_gpu.py tests/test_zz_kitchen_gpu.py"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = '''
import gymnasium_robotics_b200 as _p
from tests.hostsim_backend import HostSimBackend


def make_vec(env_id, num_envs=1, **kw):
    if env_id.startswith("Franka"):
        kw.setdefault("device", "cpu")
    kw.setdefault("backend_factory", HostSimBackend)
    return _p.make_vec(env_id, num_envs=num_envs, **kw)
'''

if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        open(os.path.join(tmp, "gpu_dryrun_shim.py"), "w").write(SHIM)
        # the session hooks of tests/conftest.py (marker registration, B200_PARITY_STATS dump) apply to the copies too
        open(os.path.join(tmp, "conftest.py"), "w").write(open(os.path.join(ROOT, "tests", "conftest.py")).read())
        os.makedirs(os.path.join(tmp, "golden"), exist_ok=True)
        for f in os.listdir(os.path.join(ROOT, "tests", "golden")):
            if f.endswith((".json", ".b200m", ".npz")):
                os.symlink(os.path.join(ROOT, "tests", "golden", f), os.path.join(tmp, "golden", f))
        names = []
        for path in sys.argv[1:]:
            s = open(path).read()
            for a, b in (('device="cuda"', 'device="cpu"'), (".cuda()", ".cpu()"), ('"cuda:0"', '"cpu"'), ("pytestmark = pytest.mark.gpu", "pytestmark = []"),
                         (".is_cuda", ".is_cpu"), ("import gymnasium_robotics_b200 as pkg", "import gpu_dryrun_shim as pkg"),
                         ("from gymnasium_robotics_b200 import make_vec", "from gpu_dryrun_shim import make_vec"),
                         ("from gymnasium_robotics_b200.fetch import CudaBackend", "from tests.hostsim_backend import HostSimBackend as CudaBackend"),
                         ("ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))", f'ROOT = "{ROOT}"')):
                s = s.replace(a, b)
            names.append(os.path.join(tmp, os.path.basename(path)))
            open(names[-1], "w").write(s)
        env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + tmp)
        sys.exit(subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-rxX"] + sys.argv[1:0] + names +
                                (["-k", os.environ["DRYRUN_K"]] if os.environ.get("DRYRUN_K") else []), cwd=tmp, env=env).returncode)
