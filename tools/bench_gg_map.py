"""Cost of location dependent friction from a friction map, on bench.py's 10 000-scenario batch on the ~200 x 11 lattice
(l216).  Measured alternately in one call, with CUDA events (L2 flushed before every call):
  - device ms per first tick() with the constant gg tuple, with gg planes uploaded once beforehand (the velocity kernel's
    local_gg variant without k_gg_map), with a 1 m map (~11.5 MB, fits in L2) and with a 0.25 m map (~184 MB, larger
    than L2), both over a box around the whole Monteblanco track;
  - wall ms of the round trip the map replaces: calc_paths -> fetch of the paths -> NumPy evaluation of the 1 m map ->
    set_local_gg_planes -> calc_vel_profile (host clock, ends in a device synchronise);
  - device ms per next_tick() of bench's 8-tick closed loop (every scenario drives 0.1 s along its first kept
    trajectory), without and with the 1 m map.  Each variant replays the loop recorded on a planner of its own kind
    (the map changes the kept trajectories, so the two loops drive the vehicles differently).
Prints one JSON line (stdout) with the card and its power limit.

    python tools/bench_gg_map.py [--rounds 5]
"""
import argparse
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
from tests import gg_map_ref as M  # noqa: E402
from tools.workload import card, closed_loop_step, timed_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of every variant")
    args = ap.parse_args()
    device = torch.device("cuda:0")
    lat = bench.get_lattice("l216")
    sc = bench.make_batch("l216", args.batch)
    online = read_online_config(bench.ONLINE_INI)
    maps = {"map_1m": (1.0, M.surface_map(1.0)), "map_0.25m": (0.25, M.surface_map(0.25))}

    def planner(key, stateful=False):
        pl = BatchPlanner(lat, online=online, device=device, stateful=stateful)
        pl.set_vel_params(**bench.vel_kwargs())
        if key in maps:
            cell, (ax, ay) = maps[key]
            pl.set_gg_map(ax, ay, M.BOX_X0, M.BOX_Y0, cell)
        pl.stage_scenarios(sc)
        pl.upload()
        pl.set_startpos()
        return pl

    first = {k: planner(k) for k in ("const", "planes", "map_1m", "map_0.25m", "round_trip")}
    cell, (ax1, ay1) = maps["map_1m"]
    first["planes"].calc_paths()   # planes of the 1 m map along the batch's paths; every later tick() reads them
    first["planes"].set_local_gg_planes(*M.planes_along(first["planes"], ax1, ay1, M.BOX_X0, M.BOX_Y0, cell))

    def round_trip(pl):
        pl.calc_paths()
        pl.set_local_gg_planes(*M.planes_along(pl, ax1, ay1, M.BOX_X0, M.BOX_Y0, cell))
        pl.calc_vel_profile()
        torch.cuda.synchronize(device)

    for key, pl in first.items():   # warm-up: every shape once
        round_trip(pl) if key == "round_trip" else pl.tick()
    torch.cuda.synchronize(device)

    # the closed loop of each variant, recorded once on a planner of that variant: inputs of every tick
    n_loop, dt = 8, 0.1
    rec = {}
    for key in ("const", "map_1m"):
        pl = planner(key, stateful=True)
        pl.tick()
        rec[key] = []
        pos, vel = sc.pos.copy(), sc.vel.copy()
        for k in range(n_loop):
            p_new, v_new, sel, ok, _ = closed_loop_step(pl.fetch("traj_row", "traj_len", "action_id", "traj"), dt)
            pos, vel = np.where(ok[:, None], p_new, pos), np.where(ok, v_new, vel)
            rec[key].append((pos.copy(), vel.copy(), sel))
            pl.next_tick(ScenarioBatch(pos.copy(), sc.heading, sc.vel, sc.n_obj, sc.obj), sel, 2.0 * dt, vel_est=vel)
    torch.cuda.synchronize(device)
    loop = {k: planner(k, stateful=True) for k in rec}

    t_first = {k: [] for k in first}
    t_loop = {k: [] for k in loop}
    for r in range(args.rounds):
        keys = list(first) if r % 2 == 0 else list(first)[::-1]
        for key in keys:
            p = first[key]
            if key == "round_trip":
                timed_ms(lambda: None)   # same L2 flush and idle device as the timed variants
                t0 = time.perf_counter()
                round_trip(p)
                t_first[key].append(1e3 * (time.perf_counter() - t0))
            else:
                t_first[key].append(timed_ms(p.tick))
        for key in (("const", "map_1m") if r % 2 == 0 else ("map_1m", "const")):
            p = loop[key]
            p.stage_scenarios(sc)
            p.upload()
            p.set_startpos()
            p.tick()
            for rpos, v, sel in rec[key]:
                sck = ScenarioBatch(rpos, sc.heading, sc.vel, sc.n_obj, sc.obj)
                t_loop[key].append(timed_ms(lambda: p.next_tick(sck, sel, 2.0 * dt, vel_est=v)))
    med = lambda v: float(np.median(v))   # noqa: E731
    bench.emit({
        "tool": "bench_gg_map", "card": card(), "batch": sc.size, "lattice": "l216", "rounds": args.rounds,
        "map_vertices": {k: list(m[1][0].shape[::-1]) for k, m in maps.items()},
        "map_mb": {k: round(m[1][0].size * 16 / 1e6, 1) for k, m in maps.items()},
        "tick_device_ms_median": {k: med(t_first[k]) for k in ("const", "planes", "map_1m", "map_0.25m")},
        "round_trip_wall_ms_median": med(t_first["round_trip"]),
        "next_tick_device_ms_median": {k: med(v) for k, v in t_loop.items()},
        "next_tick_ticks": n_loop,
        "note": "tick / next_tick: CUDA events, L2 flushed before every call; round trip: host clock around calc_paths "
                "-> fetch -> NumPy (1 m map) -> set_local_gg_planes -> calc_vel_profile -> synchronise; next_tick: each variant "
                "on the closed loop recorded on its own planner"})


if __name__ == "__main__":
    main()
