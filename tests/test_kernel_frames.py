"""Per-thread stack frames of the planning kernels, read from the built library with cuobjdump (no GPU needed).

A struct kernel parameter (LatDev alone is 424 bytes) whose address reaches an out-of-line device function is copied
into every thread's local memory at kernel entry unless it is declared __grid_constant__; for a 10 000-scenario tick
that is ~136 MB of local stores in k_plan. A run-time indexed local array (k_plan's action-set table before it was
packed into one integer) adds 24 - 40 bytes. The bounds are the frames of the current build (CUDA 12.9, sm_90a, DESIGN.md
section 5: 40 bytes of them are the float64 sin / cos slow path); they fail as soon as either comes back."""
import os
import re
import shutil
import subprocess

import pytest

# k_plan<ZONE, STATE, DENSE> -> bytes (with the parameter copy: 616 - 680, with the unpacked table: 176 - 208)
K_PLAN_MAX_STACK = {(False, False): 136,   # first tick (the benchmarked kernel)
                    (True, False): 168,    # first tick with blocked zones
                    (False, True): 184,    # stateful tick
                    (True, True): 184}
K_STARTPOS_MAX_STACK = 40  # bytes; with the parameter copy 464


def _cuobjdump():
    # on PATH, next to the nvcc that builds the library, or in the CUDA toolkit
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    dirs = ([os.path.dirname(nvcc)] if nvcc else []) + [os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")]
    return shutil.which("cuobjdump") or shutil.which("cuobjdump", path=os.pathsep.join(dirs))


def _stack_frames():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    lib = capi.build_library()
    out = subprocess.run([tool, "--dump-resource-usage", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, check=True).stdout
    frames, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
        m = re.search(r"STACK:(\d+)", line)
        if m and fn:
            frames[fn] = int(m.group(1))
            fn = None
    return frames


def test_plan_kernels_keep_their_parameters_out_of_local_memory():
    frames = _stack_frames()
    plan = {f: s for f, s in frames.items() if f.startswith("_Z6k_planI")}
    assert len(plan) == 8, sorted(frames)
    for f, s in plan.items():
        zone, state = (b == "1" for b in re.match(r"_Z6k_planILb(\d)ELb(\d)E", f).groups())
        assert s <= K_PLAN_MAX_STACK[(zone, state)], (f, s)
    startpos = [s for f, s in frames.items() if f.startswith("_Z10k_startpos")]
    assert len(startpos) == 1, sorted(frames)
    assert startpos[0] <= K_STARTPOS_MAX_STACK, startpos
