"""debug (GPU box): build library variants with extra -D flags and time the tick kernels.
usage: python tools/gpu_tune.py l216 "-DVR_P=8" "-DVR_P=16" ..."""
import os, subprocess, sys, json
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
if len(sys.argv) > 2 and sys.argv[1] == "--child":
    import ctypes as C
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.LIB_PATH = sys.argv[2]
    tag = sys.argv[3]
    import torch, bench
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    from tools.workload import timed_ms
    pl = BatchPlanner(bench.get_lattice(tag), device="cuda:0")
    pl.set_vel_params(**bench.vel_kwargs())
    pl.stage_scenarios(bench.make_batch(tag, int(os.environ.get("TUNE_BATCH", "10000")))); pl.upload(); pl.set_startpos()
    def timed(fn, steps=10):
        return sum(timed_ms(fn) for _ in range(steps)) / steps
    for _ in range(3): pl.tick()
    res = {"tick_ms": timed(pl.tick)}
    for stage, name in {1: "k_plan", 2: "k_path", 3: "k_vel"}.items():
        def one(stage=stage):
            capi.check(pl.lib, pl.lib.ltpl_launch_stage(stage, pl.handle, C.byref(pl.params), C.byref(pl.dims), C.byref(pl.buf), pl.stream), name)
        one(); res[name] = timed(one)
    if os.environ.get("TUNE_VEL"):
        import numpy as np
        from graphbasedlocaltrajectoryplanner_b200.scenarios import make_velocity_microbench
        from graphbasedlocaltrajectoryplanner_b200.velprofile import velprofile_batch_device
        mb = make_velocity_microbench(100000, 500)
        d = {k: torch.from_numpy(np.ascontiguousarray(mb[k])).cuda() for k in ("kappa", "el", "v_start", "v_end")}
        vx = torch.empty_like(d["kappa"]); ax = torch.empty_like(d["kappa"])
        pl.set_vel_params(vel_max=60.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=bench.ax_max_machines(), safety_d=30.0)
        vp = lambda: velprofile_batch_device(pl, d["kappa"], d["el"], d["v_start"], d["v_end"], vx, ax)
        vp(); res["velprofile_ms"] = timed(vp, 5)
    bench.emit(res)
    sys.exit(0)
from graphbasedlocaltrajectoryplanner_b200 import capi
tag = sys.argv[1]
for i, flags in enumerate(sys.argv[2:] or [""]):
    lib = "/tmp/libltpl_var%d.so" % i
    subprocess.check_call(["nvcc"] + capi.NVCC_FLAGS + flags.split() + ["-I" + capi.INCLUDE_DIR, "-o", lib, os.path.join(capi.CSRC_DIR, "ltpl_api.cu")])
    out = subprocess.run([sys.executable, __file__, "--child", lib, tag], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[-1]
    print("%-40s %s" % (flags, out))
