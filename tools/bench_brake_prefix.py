"""Brake prefixes to a lowered vel_max (ltpl_brake_prefix_batch) on 100 000 paths x 500 points of
make_velocity_microbench, vel_max 30 m/s, a course of 4 points per path, beside calc_vel_brake_em on the same paths:
  brake_em        VelocityPlanner.calc_vel_brake_em from the braking set's vel_plan (a full brake profile per path)
  prefix_0        check_brake_prefix with no path braking (vel_plan <= vel_max + 0.1: the course copy and zeros)
  prefix_50       half of the paths braking (vel_plan in [40, 70] m/s), every other one
  prefix_100      every path braking
each with constant friction and with loc_gg [N][P][2] (suffix _gg).  Device-event time of one call, the L2 flushed
before each (a 256 MB write), after two warm-up calls per variant; the rounds alternate the variants, and each variant
reports the median and the spread over rounds, and its ratio to brake_em of the same friction.  Prints one JSON line
with the card and its power limit, and the mean pref_idx of each braking set.

    python tools/bench_brake_prefix.py [--paths 100000] [--points 500] [--rounds 7]
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from graphbasedlocaltrajectoryplanner_b200.scenarios import make_velocity_microbench  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner  # noqa: E402
from tools.workload import card  # noqa: E402

AXM = [[0.0, 7.0], [30.0, 5.0], [60.0, 3.0], [100.0, 2.5]]
VEL_MAX, COURSE = 30.0, 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", type=int, default=100000)
    ap.add_argument("--points", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    n, p = a.paths, a.points
    mb = make_velocity_microbench(n, p)
    rng = np.random.default_rng(2025)
    fast = rng.uniform(40.0, 70.0, size=n)
    slow = rng.uniform(0.0, VEL_MAX, size=n)
    plans = {"0": slow, "50": np.where(np.arange(n) % 2 == 0, fast, slow), "100": fast}
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in plans.items()}
    kappa = torch.from_numpy(mb["kappa"]).to(dev)
    el = torch.from_numpy(mb["el"]).to(dev)
    course = torch.from_numpy(rng.uniform(10.0, 60.0, size=(n, COURSE))).to(dev)
    s = np.cumsum(mb["el"], axis=1) - mb["el"]
    gg = torch.from_numpy(np.stack((4.5 + 0.5 * np.sin(s / 50.0), 5.0 + 0.5 * np.cos(s / 70.0)), axis=-1)).to(dev)
    vp = VelocityPlanner(device=dev)
    vp.update_dyn_parameters(vel_max=VEL_MAX, gg_scale=0.9, ax_max_machines=AXM)
    old = torch.full((n,), 1.0, dtype=torch.float64, device=dev)
    vx = torch.empty((n, p), dtype=torch.float64, device=dev)
    ax = torch.empty_like(vx)
    out = (torch.empty((n, COURSE + p - 1), dtype=torch.float64, device=dev),
           torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
           torch.empty(n, dtype=torch.float64, device=dev))
    variants = {}
    for suffix, fr in (("", (5.0, 5.0)), ("_gg", gg)):
        variants["brake_em" + suffix] = lambda fr=fr: vp.calc_vel_brake_em(kappa, el, fr, d["100"], out=(vx, ax))
        for share in ("0", "50", "100"):
            variants["prefix_%s%s" % (share, suffix)] = lambda fr=fr, share=share: vp.check_brake_prefix(
                d[share], course, kappa, el, fr, old, out=out)
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
    pref_mean = {}
    for share in ("50", "100"):
        vp.check_brake_prefix(d[share], course, kappa, el, (5.0, 5.0), old, out=out)
        pref_mean[share] = float(out[2].double().mean().item())
    ms = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, fn in variants.items():
            ms[k].append(timed(fn))
    res = {}
    for k in variants:
        med = float(np.median(ms[k]))
        base = float(np.median(ms["brake_em" + ("_gg" if k.endswith("_gg") else "")]))
        res[k] = {"ms_median": round(med, 4), "ms_min": round(min(ms[k]), 4), "ms_max": round(max(ms[k]), 4),
                  "x_brake_em": round(med / base, 2)}
    print(json.dumps({"bench": "brake_prefix", "paths": n, "points": p, "course": COURSE, "vel_max": VEL_MAX,
                      "rounds": a.rounds, "card": card(), "variants": res, "mean_pref_idx": pref_mean}))


if __name__ == "__main__":
    main()
