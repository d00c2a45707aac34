"""Local-memory traffic of the 32-warp Fetch step kernel (no GPU needed: nvcc cross-compiles, nvdisasm reads the cubin).

A 1024-thread block of `fetch_kernel<32, 21>` (the FetchPickAndPlace headline batch) gets 64 registers per thread and leaves
only ~25 KB of the SM's L1 beside its shared memory, so every LDL / STL of the kernel is an L2 round trip.  The driver loops
(the sub-step loop and forward()'s Newton loop, inlined into the entry function) used to keep the env's scratch pointer on
the stack and reload it after every one of the ~50 noinline stage calls of a sub-step.  This test compiles b200sim.cu with
the library's flags and pins the local-memory instructions of the entry function (the LDLs that directly follow a stage
call, and the totals) and of the collision stage.
"""
import os
import re
import shutil
import subprocess

import pytest

from gymnasium_robotics_b200 import _lib

KERNEL = "_Z12fetch_kernelILi32ELi21EEvPKj9FetchTaskiii6StepIO"
TOOLS = ("nvcc", "nvdisasm")


def _tool(name):
    cuda = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return shutil.which(name) or (cuda if os.path.exists(cuda) else None)


pytestmark = pytest.mark.skipif(any(_tool(t) is None for t in TOOLS), reason="needs nvcc and nvdisasm (CUDA toolkit)")


def _function_name(label):
    """`$<kernel>$<mangled internal function>` -> the function's plain name (internal functions are cloned per kernel)."""
    mangled = label[len(KERNEL) + 2:]
    m = re.match(r"_ZN(\d+)", mangled)   # _ZN<len><anonymous namespace of the translation unit><len><name>...
    if m:
        rest = mangled[m.end() + int(m.group(1)):]
    else:
        rest = mangled[len("_Z"):] if mangled.startswith("_Z") else mangled
    n = re.match(r"(\d+)", rest)
    return rest[n.end():n.end() + int(n.group(1))] if n else mangled


def sass_by_function(text):
    """nvdisasm listing -> {function: [instruction lines]} for KERNEL; its entry function is 'ENTRY'."""
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"^(\$?[\w$.]+):\s*$", line)
        if m and not m.group(1).startswith((".L_", ".text.")):
            lab = m.group(1)
            cur = "ENTRY" if lab == KERNEL else (_function_name(lab) if lab.startswith("$" + KERNEL + "$") else None)
            if cur is not None:
                out.setdefault(cur, [])
            continue
        if cur is not None and re.match(r"^\s*/\*[0-9a-f]{4,}\*/", line):
            out[cur].append(line)
    return out


def count(lines, op):
    return sum(1 for l in lines if re.search(r"\b%s\b" % op, l))


def reloads_after_calls(lines, window=11):
    """LDLs within `window` instructions after a CALL: values the caller kept on the stack across that call."""
    return sum(count(lines[i + 1:i + 1 + window], "LDL") for i, l in enumerate(lines) if re.search(r"\bCALL\b", l))


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    d = tmp_path_factory.mktemp("local_memory")
    cubin = str(d / "b200sim.cubin")
    flags = [f for f in _lib.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    src = os.path.join(os.path.dirname(_lib.__file__), "csrc", "b200sim.cu")
    subprocess.check_call([_tool("nvcc")] + flags + ["-cubin", "-o", cubin, src])
    text = subprocess.run([_tool("nvdisasm"), "-c", cubin], check=True, capture_output=True, text=True).stdout
    funcs = sass_by_function(text)
    assert "ENTRY" in funcs and "collision" in funcs, "fetch_kernel<32, 21> or its collision stage not found in the listing"
    print("\nfunction               LDL   STL  CALL")
    for name, lines in funcs.items():
        if count(lines, "LDL") or count(lines, "STL") or name == "ENTRY":
            print(f"{name:22s} {count(lines, 'LDL'):4d}  {count(lines, 'STL'):4d}  {count(lines, 'CALL'):4d}")
    return funcs


def test_driver_loops_do_not_reload_state_after_stage_calls(sass):
    # before: 91 LDLs within 11 instructions of the entry's 52 stage calls (the scratch pointer and a flag word after nearly
    # every call); what is left is the flag word of the sub-step loop and the RK4 / observation paths
    entry = sass["ENTRY"]
    assert reloads_after_calls(entry) <= 27


def test_entry_local_memory_bound(sass):
    # before: 250 LDL / 43 STL in the entry function
    entry = sass["ENTRY"]
    assert count(entry, "LDL") <= 155
    assert count(entry, "STL") <= 37


def test_collision_local_memory_bound(sass):
    # each lane's narrow-phase result (ContactOut, 29 words) is still on the stack: pinned so that it does not grow
    coll = sass["collision"]
    assert count(coll, "LDL") <= 97
    assert count(coll, "STL") <= 184
