"""Cost of host staging in the tick: bench.py's 8-tick closed loop (10 000 scenarios on the ~200 x 11 lattice, a vehicle
dummy advancing every scenario 0.1 s on its first kept trajectory), planned once from host ScenarioBatches and once
from the same batches uploaded beforehand as DeviceScenarioBatches (sel_action and vel_est as device tensors too).
The loop is recorded once; every round replays the first tick() (set_startpos + tick) and the 8 next_ticks of both
variants, alternating which goes first.  Each call is timed from the host (wall: call until the device is idle) and
with CUDA events (device), L2 flushed before it.  Prints one JSON line with the medians, the card and its power limit.

    python tools/bench_device_inputs.py [--rounds 5] [--batch 10000]
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
from tools.workload import card, closed_loop_step  # noqa: E402

_FLUSH = []


def timed(fn):
    """(wall ms, device ms) of fn(): L2 flushed and the device idle before; wall = host clock from the call until the
    device has finished, device = CUDA events on the current stream around the call"""
    if not _FLUSH:
        _FLUSH.append(torch.empty(256 << 20, dtype=torch.uint8, device="cuda"))
    _FLUSH[0].fill_(1)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0 = time.perf_counter()
    e0.record(stream)
    fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - w0), e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of the replay")
    args = ap.parse_args()
    device = torch.device("cuda:0")
    lat = bench.get_lattice("l216")
    sc = bench.make_batch("l216", args.batch)
    online = read_online_config(bench.ONLINE_INI)
    n_loop, dt = 8, 0.1
    planners = {}
    for key in ("host", "device"):
        pl = BatchPlanner(lat, online=online, device=device, stateful=True)
        pl.set_vel_params(**bench.vel_kwargs())
        planners[key] = pl

    # record the loop once on the host planner: the inputs of every tick
    pl = planners["host"]
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.tick()
    rec = []
    pos, vel = sc.pos.copy(), sc.vel.copy()
    for _ in range(n_loop):
        p_new, v_new, sel, ok, _ = closed_loop_step(pl.fetch("traj_row", "traj_len", "action_id", "traj"), dt)
        pos, vel = np.where(ok[:, None], p_new, pos), np.where(ok, v_new, vel)
        rec.append((ScenarioBatch(pos.copy(), sc.heading, sc.vel, sc.n_obj, sc.obj), sel, vel.copy()))
        pl.next_tick(rec[-1][0], sel, 2.0 * dt, vel_est=vel)
    torch.cuda.synchronize(device)
    inputs = {"host": (sc, rec),
              "device": (sc.to_device(device), [(s.to_device(device), torch.as_tensor(a, device=device),
                                                 torch.as_tensor(v, device=device)) for s, a, v in rec])}

    def first_tick(pl, sc0):
        pl.stage_scenarios(sc0)
        pl.upload()
        pl.set_startpos()
        pl.tick()

    times = {k: {"first_wall": [], "first_dev": [], "next_wall": [], "next_dev": []} for k in planners}
    for r in range(args.rounds + 1):   # round 0 warms up every shape and is not kept
        for key in (("host", "device") if r % 2 == 0 else ("device", "host")):
            pl, (sc0, ticks) = planners[key], inputs[key]
            w, d = timed(lambda: first_tick(pl, sc0))
            if r:
                times[key]["first_wall"].append(w)
                times[key]["first_dev"].append(d)
            for sck, sel, vel_e in ticks:
                w, d = timed(lambda: pl.next_tick(sck, sel, 2.0 * dt, vel_est=vel_e))
                if r:
                    times[key]["next_wall"].append(w)
                    times[key]["next_dev"].append(d)
    same = all(np.array_equal(a, b) for a, b in zip(planners["host"].fetch("traj_len", "action_id").values(),
                                                    planners["device"].fetch("traj_len", "action_id").values()))
    med = {k: {m: round(float(np.median(v)), 4) for m, v in t.items()} for k, t in times.items()}
    print(json.dumps({"tool": "bench_device_inputs", "card": card(), "batch": sc.size, "lattice": "l216",
                      "ticks": n_loop, "rounds": args.rounds, "same_results": bool(same),
                      "ms_median": {k: {"next_tick_wall": v["next_wall"], "next_tick_device": v["next_dev"],
                                        "first_tick_wall": v["first_wall"], "first_tick_device": v["first_dev"]}
                                    for k, v in med.items()},
                      "note": "wall: host clock from the call until the device is idle (host staging included); "
                              "device: CUDA events around the call; first tick = stage + set_startpos + tick; "
                              "device inputs uploaded before the timed loop"}))


if __name__ == "__main__":
    main()
