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
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner, read_online_config  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


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

    def advance(pl):   # position / velocity estimate after dt on the first kept trajectory of every scenario
        f = pl.fetch("traj_row", "traj_len", "action_id", "traj")
        rows, acts = f["traj_row"], f["action_id"]
        slot = np.argmax(rows >= 0, axis=0)
        b = np.arange(B)
        ok = rows[slot, b] >= 0
        tr = f["traj"][np.where(ok, rows[slot, b], 0)].astype(np.float64)
        n = np.maximum(f["traj_len"][slot, b], 2)
        s_t = tr[:, 0, 0] + np.maximum(tr[:, 0, 5] * dt + 0.5 * tr[:, 0, 6] * dt ** 2, 0.0)
        valid = np.arange(tr.shape[1])[None, :] < n[:, None]
        i0 = np.clip((np.where(valid, tr[:, :, 0], np.inf) <= s_t[:, None]).sum(axis=1) - 1, 0, n - 2)
        s0, s1 = tr[b, i0, 0], tr[b, i0 + 1, 0]
        w = np.clip((s_t - s0) / np.maximum(s1 - s0, 1e-9), 0.0, 1.0)
        lerp = lambda c: tr[b, i0, c] * (1 - w) + tr[b, i0 + 1, c] * w   # noqa: E731
        return np.column_stack((lerp(1), lerp(2))), lerp(5), np.where(ok, acts[slot, b], 0).astype(np.int32), ok, \
            tr[b, i0, 3]

    # record the loop once (driven by the planner without restarts): inputs of every tick
    pl = planners["none"]
    first_tick(pl)
    rec = []
    pos, vel = sc.pos.copy(), sc.vel.copy()
    for k in range(n_loop):
        p_new, v_new, sel, ok, head = advance(pl)
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

    stream = torch.cuda.current_stream(device)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=device)
    times = {"none": [], "mask": []}
    for r in range(args.rounds):
        order = ("none", "mask") if r % 2 == 0 else ("mask", "none")
        for key in order:
            pl = planners[key]
            first_tick(pl)
            for rpos, heading, vel_start, vel_e, sel, m in rec:
                sck = ScenarioBatch(rpos, heading, vel_start, sc.n_obj, sc.obj)
                flush.fill_(1)
                torch.cuda.synchronize(device)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                pl.next_tick(sck, sel, 2.0 * dt, vel_est=vel_e, restart=m if key == "mask" else None)
                e1.record(stream)
                torch.cuda.synchronize(device)
                times[key].append(e0.elapsed_time(e1))
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
