"""Location dependent friction between the two halves of a stateful tick, three ways: bench.py's 8-tick closed loop on
the ~200 x 11 lattice (a vehicle dummy advancing every scenario 0.1 s on its first kept trajectory) with the friction
field of tests/helpers.local_gg_field evaluated along every planned path, recorded once, then replayed from the same
per-tick device tensors as
  (a) host:   next_calc_paths -> fetch of the path planes -> NumPy field -> set_local_gg_planes(NumPy) ->
              next_calc_vel_profile (the round trip a caller without device planes makes);
  (b) device: next_calc_paths -> torch field on device_results()["path"] -> set_local_gg_planes(tensors) ->
              next_calc_vel_profile;
  (c) graph:  (b) from a SplitTickGraph: paths_inputs.copy_ -> replay_paths -> torch field into vel_inputs ->
              replay_vel_profile (the copies count in its time).
Every round runs an untimed first tick and the 8 stateful ticks of each variant, in a rotating order, after one
warm-up round.  Each stateful tick is timed from the host (wall: call until the device is idle) and with CUDA events
(device), L2 flushed before it.  (b) and (c) must give the same bytes after every round.  Prints one JSON line with
the medians per batch size, the card and its power limit.

    python tools/bench_split_tick.py [--rounds 3] [--batch 2000 10000]
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
from graphbasedlocaltrajectoryplanner_b200.planner import NSLOT, BatchPlanner, read_online_config  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch  # noqa: E402
from tests.helpers import local_gg_field  # noqa: E402
from tools.workload import card, closed_loop_step, timed_ms  # noqa: E402

RESULTS = ("action_id", "traj_len", "traj_id", "status", "sc_flags", "path_len", "em_info", "trim")
VARIANTS = ("host", "device", "graph")
T_CONST = 0.2


def timed(fn):
    """(wall ms, device ms) of fn(): wall = host clock from the call until the device is idle"""
    box = {}

    def run():
        box["t0"] = time.perf_counter()
        fn()
    dev = timed_ms(run)
    return 1e3 * (time.perf_counter() - box["t0"]), dev


def results(pl):
    """the last tick's per-path results, the memory records and the compact export rows in path order"""
    f = pl.fetch(*RESULTS, "traj_row", "traj")
    rows = np.where(f["traj_row"][..., None, None] >= 0, f["traj"][np.maximum(f["traj_row"], 0)], 0.0)
    mem = [pl._state[k].cpu().numpy() for k in ("st_info", "vel_plan", "course", "zone_s0")]
    return [f[k] for k in RESULTS] + mem + [rows]


def field_torch(path, batch):
    """local_gg_field by torch along the path planes [5][NSLOT * B][p_max]: (ax, ay) [NSLOT][B][p_max]"""
    x, y = path[0], path[1]
    ax = 4.2 + 1.1 * torch.sin(0.011 * x + 0.5)
    ay = 4.6 + 0.9 * torch.cos(0.013 * y - 0.3)
    return ax.view(NSLOT, batch, -1), ay.view(NSLOT, batch, -1)


def field_host(pl):
    """the round trip: the path planes fetched (a synchronisation), local_gg_field in NumPy"""
    path = pl.fetch("path")["path"]
    gg = local_gg_field(np.column_stack((path[0].ravel(), path[1].ravel())))
    shape = (NSLOT, pl.dims.batch, path.shape[2])
    return gg[:, 0].reshape(shape), gg[:, 1].reshape(shape)


def run_batch(lat, online, n, rounds, device):
    sc = bench.make_batch("l216", n)
    n_loop, dt = 8, 0.1
    planners = {}
    for key in ("record",) + VARIANTS:
        pl = BatchPlanner(lat, online=online, device=device, stateful=True)
        pl.set_vel_params(**bench.vel_kwargs())
        planners[key] = pl
    d0 = sc.to_device(device)

    def first(pl):
        pl.stage_scenarios(d0)
        pl.set_startpos()
        pl.calc_paths()
        pl.set_local_gg_planes(*field_torch(pl.device_results()["path"], n))
        pl.calc_vel_profile()

    def device_tick(pl, dsc, sel, pos, vel):
        pl.next_calc_paths(dsc, sel, T_CONST)
        pl.set_local_gg_planes(*field_torch(pl.device_results()["path"], n))
        pl.next_calc_vel_profile(pos_est=pos, vel_est=vel)

    def host_tick(pl, dsc, sel, pos, vel):
        pl.next_calc_paths(dsc, sel, T_CONST)
        pl.set_local_gg_planes(*field_host(pl))
        pl.next_calc_vel_profile(pos_est=pos, vel_est=vel)

    # record the loop once with the device variant: the device inputs of every tick
    pl = planners.pop("record")
    first(pl)
    ticks = []
    pos, vel = sc.pos.copy(), sc.vel.copy()
    for _ in range(n_loop):
        p_new, v_new, sel, ok, _ = closed_loop_step(pl.fetch("traj_row", "traj_len", "action_id", "traj"), dt)
        pos, vel = np.where(ok[:, None], p_new, pos), np.where(ok, v_new, vel)
        dsc = ScenarioBatch(pos.copy(), sc.heading, sc.vel, sc.n_obj, sc.obj).to_device(device)
        ticks.append((dsc, torch.as_tensor(sel, device=device), dsc.pos, torch.as_tensor(vel, device=device)))
        device_tick(pl, *ticks[-1])
    del pl

    pg = planners["graph"]
    first(pg)
    ones = torch.ones((NSLOT, n, pg.dims.p_max), dtype=torch.float64, device=device)
    dsc, sel, pos, vel = ticks[0]
    graph = pg.capture_next_split_tick(dsc, sel, T_CONST, vel_est=vel, pos_est=pos, local_gg=(ones, ones.clone()))
    for key in ("host", "device"):   # the same first tick, so that every variant counts its trajectory ids alike
        first(planners[key])

    def graph_tick(_, dsc, sel, pos, vel):
        graph.paths_inputs.copy_(dsc, sel)
        graph.replay_paths()
        graph.vel_inputs.copy_(pos, vel, field_torch(pg.device_results()["path"], n))
        graph.replay_vel_profile()

    calls = {"host": host_tick, "device": device_tick, "graph": graph_tick}
    times = {k: {"wall": [], "dev": []} for k in VARIANTS}
    same = True
    for r in range(rounds + 1):   # round 0 warms up every shape and is not kept
        for key in VARIANTS[r % 3:] + VARIANTS[:r % 3]:
            pl = planners[key]
            first(pl)
            torch.cuda.synchronize()
            for tick in ticks:
                w, d = timed(lambda: calls[key](pl, *tick))
                if r:
                    times[key]["wall"].append(w)
                    times[key]["dev"].append(d)
        same = same and all(np.array_equal(a, b) for a, b in zip(results(planners["device"]),
                                                                  results(planners["graph"])))
    graph.close()
    med = {k: {"split_tick_wall": round(float(np.median(t["wall"])), 4),
               "split_tick_device": round(float(np.median(t["dev"])), 4)} for k, t in times.items()}
    return {"batch": n, "same_results_device_graph": bool(same), "p_max": int(planners["host"].dims.p_max),
            "ms_median": med}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[2000, 10000])
    ap.add_argument("--rounds", type=int, default=3, help="rounds of the replay after the warm-up round")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_split_tick.py needs a CUDA device")
    device = torch.device("cuda:0")
    lat = bench.get_lattice("l216")
    online = read_online_config(bench.ONLINE_INI)
    out = [run_batch(lat, online, n, args.rounds, device) for n in args.batch]
    print(json.dumps({"tool": "bench_split_tick", "card": card(), "lattice": "l216", "ticks": 8,
                      "rounds": args.rounds, "same_results_device_graph": all(o["same_results_device_graph"]
                                                                              for o in out),
                      "batches": out,
                      "note": "per stateful tick; wall: host clock from the call until the device is idle; device: "
                              "CUDA events around the call; host = fetch paths + NumPy field + uploaded planes; "
                              "device = torch field + device planes; graph = device from SplitTickGraph replays"}))


if __name__ == "__main__":
    main()
