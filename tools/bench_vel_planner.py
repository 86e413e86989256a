"""The stand-alone velocity planner (ltpl_vel_plan_batch) on 100 000 paths x 500 points of make_velocity_microbench:
  old       ltpl_velprofile_batch, the dense constant-friction entry (bench.py's velprofile_100k_x_500)
  const     VelocityPlanner.calc_vel_profile with a friction tuple (the same kernel instance as `old`)
  per_point VelocityPlanner.calc_vel_profile with loc_gg [N][P][2]
  ragged    VelocityPlanner.calc_vel_profile with lengths drawn from [250, 500] (constant friction)
  brake     VelocityPlanner.calc_vel_brake_em with a friction tuple
Device-event time of one call, the L2 flushed before each (a 256 MB write), after two warm-up calls per variant; the
rounds alternate the variants, and each variant reports the median and the spread over rounds.  Algorithmic bytes from
the shapes: 32 B per live point in float64 (kappa, el in; vx, ax out), + 16 B with per-point friction; GB/s against
them, beside NVIDIA's data-sheet HBM3 figure for the H100 SXM (3.35 TB/s, not a measured value).
Prints one JSON line with the card and its power limit.

    python tools/bench_vel_planner.py [--paths 100000] [--points 500] [--rounds 7]
"""
import argparse
import ctypes as C
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from graphbasedlocaltrajectoryplanner_b200 import capi  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import make_velocity_microbench  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner  # noqa: E402
from tools.workload import card  # noqa: E402

DATASHEET_HBM_GBPS = 3350.0
AXM = [[0.0, 7.0], [30.0, 5.0], [60.0, 3.0], [100.0, 2.5]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=100000)
    ap.add_argument("--points", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    n, p = a.paths, a.points
    mb = make_velocity_microbench(n, p)
    d = {k: torch.from_numpy(np.ascontiguousarray(mb[k])).to(dev) for k in ("kappa", "el", "v_start", "v_end")}
    s = np.cumsum(mb["el"], axis=1) - mb["el"]
    gg = torch.from_numpy(np.stack((4.5 + 0.5 * np.sin(s / 50.0), 5.0 + 0.5 * np.cos(s / 70.0)), axis=-1)).to(dev)
    n_pts = torch.from_numpy(np.random.default_rng(1).integers(p // 2, p + 1, size=n).astype(np.int32)).to(dev)
    vx = torch.empty((n, p), dtype=torch.float64, device=dev)
    ax = torch.empty_like(vx)
    vp = VelocityPlanner(device=dev)
    vp.update_dyn_parameters(vel_max=60.0, gg_scale=1.0, ax_max_machines=AXM)
    lib = vp.lib
    prm = capi.Params.from_buffer_copy(vp.params)
    prm.gg_ax, prm.gg_ay = 5.0, 5.0
    vb = capi.VelBatch()
    vb.n_paths, vb.n_points = n, p
    vb.kappa, vb.el, vb.v_start, vb.v_end = d["kappa"].data_ptr(), d["el"].data_ptr(), d["v_start"].data_ptr(), \
        d["v_end"].data_ptr()
    vb.vx, vb.ax = vx.data_ptr(), ax.data_ptr()

    def old():
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        capi.check(lib, lib.ltpl_velprofile_batch(C.byref(prm), C.byref(vb), st), "ltpl_velprofile_batch")

    args = (d["kappa"], d["el"])
    live = float(n) * p
    variants = {
        "old": (old, 32 * live),
        "const": (lambda: vp.calc_vel_profile(*args, (5.0, 5.0), d["v_start"], d["v_end"], out=(vx, ax)), 32 * live),
        "per_point": (lambda: vp.calc_vel_profile(*args, gg, d["v_start"], d["v_end"], out=(vx, ax)), 48 * live),
        "ragged": (lambda: vp.calc_vel_profile(*args, (5.0, 5.0), d["v_start"], d["v_end"], n_pts=n_pts,
                                               out=(vx, ax)), 32 * float(n_pts.sum().item())),
        "brake": (lambda: vp.calc_vel_brake_em(*args, (5.0, 5.0), d["v_start"], out=(vx, ax)), 32 * live),
    }
    flush = torch.empty(64 * 2 ** 20, dtype=torch.float32, device=dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        flush.fill_(1.0)
        ev0.record()
        fn()
        ev1.record()
        ev1.synchronize()
        return ev0.elapsed_time(ev1)

    for fn, _ in variants.values():
        fn()
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, (fn, _) in variants.items():
            ms[k].append(timed(fn))
    res = {}
    for k, (_, nbytes) in variants.items():
        med = float(np.median(ms[k]))
        res[k] = {"ms_median": round(med, 4), "ms_min": round(min(ms[k]), 4), "ms_max": round(max(ms[k]), 4),
                  "algorithmic_GB": round(nbytes / 1e9, 3), "GBps": round(nbytes / med / 1e6, 1),
                  "share_of_datasheet_hbm": round(nbytes / med / 1e6 / DATASHEET_HBM_GBPS, 3)}
    print(json.dumps({"bench": "vel_planner", "paths": n, "points": p, "rounds": a.rounds, "card": card(),
                      "datasheet_hbm_GBps": DATASHEET_HBM_GBPS, "variants": res}))


if __name__ == "__main__":
    main()
