"""Build library variants for A/B timing on the GPU box (experiments): python tests/build_variants.py name[:srcdir][:extra flags] ...
Each variant is compiled from `srcdir` (default: this checkout) into build/variants/lib<name>.so, with this checkout's library
nvcc flags.  A `srcdir` from before the experiment-only build knobs were removed needs, among the extra flags, the two defines that
its own _lib.NVCC_FLAGS carried: without them it compiles without block-wide barriers and with the shuffle Cholesky, which is not
the library that checkout shipped."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gymnasium_robotics_b200 import _lib  # noqa: E402

BASE = [f for f in _lib.NVCC_FLAGS if f != "-shared"]
NAMES = ("b200sim", "b200sim_wide", "b200sim_kitchen", "b200sim_kitchen_groups", "b200sim_kitchen_hull")


def build(name, src, extra):
    out = os.path.join(ROOT, "build", "variants", f"lib{name}.so")
    objs, procs = [], []
    only = os.environ.get("B200_VARIANT_ONLY")            # e.g. "b200sim": compile that unit only ...
    reuse = os.environ.get("B200_VARIANT_REUSE")          # ... and link the other units' objects of an earlier variant
    for n in NAMES:
        if only and n != only:
            objs.append(os.path.join("/tmp", f"var_{reuse}_{n}.o"))
            continue
        o = os.path.join("/tmp", f"var_{name}_{n}.o")
        objs.append(o)
        procs.append(subprocess.Popen(["nvcc"] + BASE + extra + ["-c", "-o", o, os.path.join(src, "gymnasium_robotics_b200", "csrc", n + ".cu")],
                                      stdout=subprocess.DEVNULL, stderr=subprocess.PIPE))
    for p in procs:
        _, err = p.communicate()
        if p.returncode:
            sys.exit(err.decode()[-3000:])
    subprocess.check_call(["nvcc", "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", out] + objs)
    print("built", out, flush=True)


if __name__ == "__main__":
    os.makedirs(os.path.join(ROOT, "build", "variants"), exist_ok=True)
    for spec in sys.argv[1:]:
        parts = spec.split(":")
        build(parts[0], parts[1] if len(parts) > 1 and parts[1] else ROOT, parts[2].split() if len(parts) > 2 else [])
