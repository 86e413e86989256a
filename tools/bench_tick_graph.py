"""Eager device ticks against ticks replayed from CUDA graphs (BatchPlanner.capture_tick / capture_next_tick): bench.py's
8-tick closed loop on the ~200 x 11 lattice (a vehicle dummy advancing every scenario 0.1 s on its first kept
trajectory), recorded once, then replayed from the same per-tick device tensors two ways: eager tick() / next_tick(),
and copy_ into graph.inputs + replay() (the copies count in its time).  Every round replays the first tick and the 8
stateful ticks of both variants, alternating which goes first, after one warm-up round.  Each call is timed from the
host (wall: call until the device is idle) and with CUDA events (device), L2 flushed before it.  Prints one JSON line
per batch size with the medians, whether both variants gave the same bytes, the card and its power limit.

    python tools/bench_tick_graph.py [--rounds 5] [--batch 256 2000 10000]
"""
import argparse
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner, read_online_config  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch  # noqa: E402
from tools.workload import card, closed_loop_step, timed_ms  # noqa: E402

RESULTS = ("action_id", "traj_len", "traj_id", "status", "sc_flags", "path_len", "em_info", "trim")


def timed(fn):
    """(wall ms, device ms) of fn(): wall = host clock from the call until the device is idle"""
    box = {}

    def run():
        box["t0"] = time.perf_counter()
        fn()
    dev = timed_ms(run)
    return 1e3 * (time.perf_counter() - box["t0"]), dev


def results(pl):
    """the last tick's per-path results and the compact export rows in path order"""
    f = pl.fetch(*RESULTS, "traj_row", "traj")
    rows = np.where(f["traj_row"][..., None, None] >= 0, f["traj"][np.maximum(f["traj_row"], 0)], 0.0)
    return [f[k] for k in RESULTS] + [rows]


def run_batch(lat, online, n, rounds, device):
    sc = bench.make_batch("l216", n)
    n_loop, dt = 8, 0.1
    planners = {}
    for key in ("record", "eager", "graph"):
        pl = BatchPlanner(lat, online=online, device=device, stateful=True)
        pl.set_vel_params(**bench.vel_kwargs())
        planners[key] = pl

    # record the loop once: the device inputs of every tick
    pl = planners.pop("record")
    d0 = sc.to_device(device)
    pl.stage_scenarios(d0)
    pl.set_startpos()
    pl.tick()
    ticks = []
    pos, vel = sc.pos.copy(), sc.vel.copy()
    for _ in range(n_loop):
        p_new, v_new, sel, ok, _ = closed_loop_step(pl.fetch("traj_row", "traj_len", "action_id", "traj"), dt)
        pos, vel = np.where(ok[:, None], p_new, pos), np.where(ok, v_new, vel)
        dsc = ScenarioBatch(pos.copy(), sc.heading, sc.vel, sc.n_obj, sc.obj).to_device(device)
        ticks.append((dsc, torch.as_tensor(sel, device=device), torch.as_tensor(vel, device=device)))
        pl.next_tick(dsc, ticks[-1][1], 2.0 * dt, vel_est=ticks[-1][2])
    del pl

    def eager_first(pl):
        pl.stage_scenarios(d0)
        pl.set_startpos()
        pl.tick()

    # the graphs: a first tick, and a stateful tick captured behind it; the eager planner plans the same first tick,
    # so that both count their trajectory ids alike
    pg = planners["graph"]
    first = pg.capture_tick(d0)
    first.replay()
    nxt = pg.capture_next_tick(ticks[0][0], ticks[0][1], 2.0 * dt, vel_est=ticks[0][2])
    eager_first(planners["eager"])

    def graph_first(_):
        first.inputs.copy_(d0)
        first.replay()

    def eager_next(pl, dsc, sel, vel_e):
        pl.next_tick(dsc, sel, 2.0 * dt, vel_est=vel_e)

    def graph_next(_, dsc, sel, vel_e):
        nxt.inputs.copy_(dsc, sel, vel_est=vel_e)
        nxt.replay()

    calls = {"eager": (eager_first, eager_next), "graph": (graph_first, graph_next)}
    times = {k: {"first_wall": [], "first_dev": [], "next_wall": [], "next_dev": []} for k in planners}
    same = True
    for r in range(rounds + 1):   # round 0 warms up every shape and is not kept
        for key in (("eager", "graph") if r % 2 == 0 else ("graph", "eager")):
            pl, (f_first, f_next) = planners[key], calls[key]
            w, d = timed(lambda: f_first(pl))
            if r:
                times[key]["first_wall"].append(w)
                times[key]["first_dev"].append(d)
            for dsc, sel, vel_e in ticks:
                w, d = timed(lambda: f_next(pl, dsc, sel, vel_e))
                if r:
                    times[key]["next_wall"].append(w)
                    times[key]["next_dev"].append(d)
        same = same and all(np.array_equal(a, b) for a, b in zip(results(planners["eager"]),
                                                                  results(planners["graph"])))
    for g in (first, nxt):
        g.close()
    med = {k: {m: round(float(np.median(v)), 4) for m, v in t.items()} for k, t in times.items()}
    return {"batch": n, "same_results": bool(same),
            "ms_median": {k: {"next_tick_wall": v["next_wall"], "next_tick_device": v["next_dev"],
                              "first_tick_wall": v["first_wall"], "first_tick_device": v["first_dev"]}
                          for k, v in med.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[256, 2000, 10000])
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of the replay")
    args = ap.parse_args()
    device = torch.device("cuda:0")
    lat = bench.get_lattice("l216")
    online = read_online_config(bench.ONLINE_INI)
    out = [run_batch(lat, online, n, args.rounds, device) for n in args.batch]
    print(json.dumps({"tool": "bench_tick_graph", "card": card(), "lattice": "l216", "ticks": 8, "rounds": args.rounds,
                      "same_results": all(o["same_results"] for o in out), "batches": out,
                      "note": "wall: host clock from the call until the device is idle; device: CUDA events around "
                              "the call; first tick = k_stage + set_startpos + tick; graph = copy_ into graph.inputs "
                              "+ replay(); same_results: byte equality of both variants after every round"}))


if __name__ == "__main__":
    main()
