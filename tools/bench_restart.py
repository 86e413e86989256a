"""Cost of restarts inside the stateful tick: bench.py's 8-tick closed loop (10 000 scenarios on the ~200 x 11 lattice,
a vehicle dummy advancing every scenario 0.1 s on its first kept trajectory) with CUDA events around every next_tick.
Every tick is timed in the same loop with restart=None and with a restart mask of the chosen fraction (the masked
scenarios re-anchored at their position estimate, half of them with the start pose of another scenario), alternating
per round, from the same recorded state (two planners fed identically).  Prints one JSON line: device ms per tick of
both variants, the card and its power limit.

    python tools/bench_restart.py --restart-frac F [--rounds 5]      (F = 0: an all-zero mask)
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner, read_online_config  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch  # noqa: E402
from tools.workload import card, closed_loop_step, timed_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--restart-frac", type=float, required=True, help="share of the batch restarted per tick (0 .. 1)")
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of the 8-tick replay")
    args = ap.parse_args()
    if not 0.0 <= args.restart_frac <= 1.0:
        sys.exit("--restart-frac must lie in [0, 1]")
    device = torch.device("cuda:0")
    lat = bench.get_lattice("l216")
    sc = bench.make_batch("l216", args.batch)
    online = read_online_config(bench.ONLINE_INI)
    B, n_loop, dt = sc.size, 8, 0.1
    rng = np.random.default_rng(bench.SEED + 17)
    masks = [rng.random(B) < args.restart_frac for _ in range(n_loop)]
    planners = {}
    for key in ("none", "mask"):
        pl = BatchPlanner(lat, online=online, device=device, stateful=True)
        pl.set_vel_params(**bench.vel_kwargs())
        planners[key] = pl

    def first_tick(pl):
        pl.stage_scenarios(sc)
        pl.upload()
        pl.set_startpos()
        pl.tick()

    # record the loop once (driven by the planner without restarts): inputs of every tick
    pl = planners["none"]
    first_tick(pl)
    rec = []
    pos, vel = sc.pos.copy(), sc.vel.copy()
    for k in range(n_loop):
        p_new, v_new, sel, ok, head = closed_loop_step(pl.fetch("traj_row", "traj_len", "action_id", "traj"), dt)
        pos, vel = np.where(ok[:, None], p_new, pos), np.where(ok, v_new, vel)
        heading, vel_start = sc.heading.copy(), sc.vel.copy()
        m = masks[k]
        heading[m & ok] = head[m & ok]
        vel_start[m] = vel[m]
        rpos = pos.copy()
        other = rng.permutation(B)
        jump = m & (rng.random(B) < 0.5)
        rpos[jump], heading[jump], vel_start[jump] = sc.pos[other][jump], sc.heading[other][jump], sc.vel[other][jump]
        rec.append((rpos, heading, vel_start, vel.copy(), sel, m))
        pl.next_tick(ScenarioBatch(rpos, heading, vel_start, sc.n_obj, sc.obj), sel, 2.0 * dt, vel_est=vel)
    torch.cuda.synchronize(device)

    times = {"none": [], "mask": []}
    for r in range(args.rounds):
        order = ("none", "mask") if r % 2 == 0 else ("mask", "none")
        for key in order:
            pl = planners[key]
            first_tick(pl)
            for rpos, heading, vel_start, vel_e, sel, m in rec:
                sck = ScenarioBatch(rpos, heading, vel_start, sc.n_obj, sc.obj)
                times[key].append(timed_ms(lambda: pl.next_tick(sck, sel, 2.0 * dt, vel_est=vel_e,
                                                                restart=m if key == "mask" else None)))
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({"tool": "bench_restart", "card": card(), "batch": B, "ticks": n_loop, "rounds": args.rounds,
                      "restart_frac": args.restart_frac, "restarted_per_tick": float(np.mean([m.sum() for m in masks])),
                      "ms_per_tick_median": {"restart_none": med["none"], "restart_mask": med["mask"]},
                      "ms_per_tick_mean": {"restart_none": float(np.mean(times["none"])),
                                           "restart_mask": float(np.mean(times["mask"]))},
                      "note": "device time of one next_tick (CUDA events, L2 flushed before every tick), both variants "
                              "alternating on the same recorded inputs"}))


if __name__ == "__main__":
    main()
