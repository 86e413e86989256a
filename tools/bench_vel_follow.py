"""Follow-mode velocity profiles (ltpl_vel_follow_batch) on 100 000 paths x 500 points of make_velocity_microbench, with
follow scalars drawn from a fixed seed (opponents near random points of the Monteblanco race line, 795 points):
  profile       VelocityPlanner.calc_vel_profile on the same paths (constant friction), for comparison
  follow        VelocityPlanner.calc_vel_profile_follow, constant friction, PD controller
  follow_pdtan  the same with the PDtan controller
  follow_gg     calc_vel_profile_follow with loc_gg [N][P][2]
Device-event time of one call, the L2 flushed before each (a 256 MB write), after two warm-up calls per variant; the
rounds alternate the variants, and each variant reports the median and the spread over rounds, and its ratio to
`profile`.  Prints one JSON line with the card and its power limit.

    python tools/bench_vel_follow.py [--paths 100000] [--points 500] [--rounds 7]
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from graphbasedlocaltrajectoryplanner_b200.lattice import build_lattice  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import make_velocity_microbench  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner  # noqa: E402
from tools.workload import card  # noqa: E402

AXM = [[0.0, 7.0], [30.0, 5.0], [60.0, 3.0], [100.0, 2.5]]
PD = {"c_p": 1.25, "k_d": 0.025, "k_p": 0.2}
PDTAN = {"c_p": 1.15, "k_d": 0.025, "k_p": 0.2, "tan_w": 15.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=100000)
    ap.add_argument("--points", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    n, p = a.paths, a.points
    lat = build_lattice(os.path.join(REPO, "inputs", "traj_ltpl_cl", "traj_ltpl_cl_monteblanco.csv"),
                        os.path.join(REPO, "params", "ltpl_config_offline.ini"))
    glob_rl = np.asarray(lat.glob_rl, dtype=np.float64)
    mb = make_velocity_microbench(n, p)
    rng = np.random.default_rng(2024)
    j = rng.integers(0, glob_rl.shape[0] - 1, size=n)
    v_start = mb["v_start"] * 1.5
    h = dict(kappa=mb["kappa"], el=mb["el"], v_start=v_start, v_end=mb["v_end"],
             v_ego=v_start + rng.uniform(-2.0, 2.0, size=n), v_obj=rng.uniform(0.0, 50.0, size=n),
             safety_d=rng.uniform(5.0, 40.0, size=n), obj_dist=rng.uniform(0.0, 250.0, size=n),
             obj_pos=glob_rl[j, 1:3] + rng.uniform(-3.0, 3.0, size=(n, 2)))
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in h.items()}
    s = np.cumsum(mb["el"], axis=1) - mb["el"]
    gg = torch.from_numpy(np.stack((4.5 + 0.5 * np.sin(s / 50.0), 5.0 + 0.5 * np.cos(s / 70.0)), axis=-1)).to(dev)
    vx = torch.empty((n, p), dtype=torch.float64, device=dev)
    ax = torch.empty_like(vx)
    tc = torch.empty(n, dtype=torch.bool, device=dev)
    vb = torch.empty(n, dtype=torch.bool, device=dev)
    planners = {}
    for name, ctype, cp in (("pd", "PD", PD), ("pdtan", "PDtan", PDTAN)):
        vp = VelocityPlanner(device=dev, len_veh=float(lat.veh_length), follow_control_type=ctype,
                             follow_control_params=cp, glob_rl=glob_rl)
        vp.update_dyn_parameters(vel_max=60.0, gg_scale=1.0, ax_max_machines=AXM)
        planners[name] = vp
    fargs = (d["v_start"], d["v_ego"], d["v_obj"], d["safety_d"], d["obj_dist"], d["obj_pos"])
    pd, pdt = planners["pd"], planners["pdtan"]
    variants = {
        "profile": lambda: pd.calc_vel_profile(d["kappa"], d["el"], (5.0, 5.0), d["v_start"], d["v_end"],
                                               out=(vx, ax)),
        "follow": lambda: pd.calc_vel_profile_follow(d["kappa"], d["el"], (5.0, 5.0), *fargs, out=(vx, ax, tc, vb)),
        "follow_pdtan": lambda: pdt.calc_vel_profile_follow(d["kappa"], d["el"], (5.0, 5.0), *fargs,
                                                            out=(vx, ax, tc, vb)),
        "follow_gg": lambda: pd.calc_vel_profile_follow(d["kappa"], d["el"], gg, *fargs, out=(vx, ax, tc, vb)),
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

    for fn in variants.values():
        fn()
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, fn in variants.items():
            ms[k].append(timed(fn))
    base = float(np.median(ms["profile"]))
    res = {}
    for k in variants:
        med = float(np.median(ms[k]))
        res[k] = {"ms_median": round(med, 4), "ms_min": round(min(ms[k]), 4), "ms_max": round(max(ms[k]), 4),
                  "x_profile": round(med / base, 2)}
    follow_share = {k: float(v.float().mean().item()) for k, v in (("too_close", tc), ("vel_bound", vb))}
    print(json.dumps({"bench": "vel_follow", "paths": n, "points": p, "rounds": a.rounds, "race_line_points":
                      int(glob_rl.shape[0] - 1), "card": card(), "variants": res, "last_call_flag_share": follow_share}))


if __name__ == "__main__":
    main()
