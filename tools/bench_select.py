"""The trajectory each scenario takes, selected on the device (BatchPlanner.select) against the same pick on the host or
in torch code.  Two measurements on the ~200 x 11 lattice (l216) with bench.py's batch:
  (a) e2e: plan_stream over the same host ScenarioBatch, ms per step, without prefer (every kept trajectory and, with
      incl_emerg_traj, every emergency trajectory downloaded; the host picks) and with prefer (k_select + the
      fixed-size download of the selected rows), incl_emerg_traj off and on.  Rounds alternate the two variants after
      one warm-up round; D2H bytes per step from the buffer sizes.  The selected rows of one tick are checked against
      the host pick from the full download of the same tick.
  (b) closed loop: a first tick and 8 stateful ticks replayed from capture_next_tick(..., "selected", prefer=P) (the
      pick inside the graph) against the same loop replayed from capture_next_tick with a static sel_action that torch
      code fills from device_results() between replays; a vehicle dummy on the device drives every scenario to row 1
      of its selected trajectory.  Results, memory and selected rows must be byte-equal after every tick of the checked
      round; the timed rounds alternate the variants.
Prints one JSON line with the medians, the byte counts, the card and its power limit.

    python tools/bench_select.py [--batch 10000] [--steps 40] [--rounds 3]
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
from graphbasedlocaltrajectoryplanner_b200.planner import PREFER_IDS, BatchPlanner, read_online_config  # noqa: E402
from tests.select_ref import select_ref  # noqa: E402
from tools.workload import card  # noqa: E402

ORDER = ["left", "straight", "follow", "right"]
T_CONST = 0.2


def feed(sc, n):
    for _ in range(n):
        yield sc


def stream_ms(pl, sc, steps, prefer):
    """ms per step of plan_stream over `steps` copies of sc (wall clock until the last result is on the host)"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rows = 0
    for out in pl.plan_stream(feed(sc, steps), prefer=prefer):
        rows += int(out.get("n_rows", 0))
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps, rows / steps


def check_one_tick(pl, sc, names):
    """one tick: the full download, then select + download_selected of the same tick; the selected rows must be the
    host pick's rows of the full download, byte for byte"""
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.tick()
    full = {k: (v.clone() if hasattr(v, "clone") else v) for k, v in pl.download().items()}
    pl.select(names)
    out = pl.download_selected()
    ids = np.array([[PREFER_IDS[a] for a in names]])
    act, info = select_ref(*(full[k].numpy() for k in ("action_id", "traj_row", "traj_len", "traj_id", "em_info")),
                           full["incl_emerg_traj"], ids)
    rows = np.where(info[:, 1, None, None] >= 0, full["traj"].numpy()[np.maximum(info[:, 1], 0)], 0.0)
    return bool(np.array_equal(out["sel_info"].numpy(), info) and np.array_equal(out["sel_traj"].numpy(), rows))


def run_e2e(lat, online, sc, args, emerg):
    pl = BatchPlanner(lat, online=online, device="cuda:0")
    pl.set_vel_params(**dict(bench.vel_kwargs(), incl_emerg_traj=emerg))
    names = (["emergency"] if emerg else []) + ORDER
    same = check_one_tick(pl, sc, names)
    times = {"full": [], "selected": []}
    rows = 0.0
    for r in range(args.rounds + 1):   # round 0 warms up both variants and is not kept
        for key in (("full", "selected") if r % 2 == 0 else ("selected", "full")):
            ms, n = stream_ms(pl, sc, args.steps, names if key == "selected" else None)
            if key == "full":
                rows = n
            if r:
                times[key].append(ms)
    B, NE = pl.dims.batch, pl.dims.n_export
    meta = pl.d2h_bytes(0)
    return {"incl_emerg_traj": emerg, "selected_rows_equal_host_pick": same,
            "ms_per_step_median": {k: round(float(np.median(v)), 4) for k, v in times.items()},
            "ms_per_step_all": {k: [round(x, 4) for x in v] for k, v in times.items()},
            "rows_per_step_full": rows,
            "d2h_bytes_per_step": {"full": pl.d2h_bytes(int(round(rows))), "selected": meta + B * 16 + B * NE * 28}}


def torch_pick(pl, prefer_ids, emerg, sel_out):
    """the selection in torch code on device_results(): the first action of prefer_ids (one list) the tick returned;
    writes the actions into sel_out, returns (sel_info [B][4], rows [B][n_export][7]) as k_select gives them"""
    r = pl.device_results()
    act, row, tl, tid, em = r["action_id"], r["traj_row"], r["traj_len"], r["traj_id"], pl.t["em_info"]
    B = act.shape[1]
    kept = row >= 0
    info = torch.tensor([-1, -1, 0, -1], dtype=torch.int32, device=act.device).repeat(B, 1)
    for a in reversed(prefer_ids):   # the first listed action wins: apply the list back to front
        if a == 4:
            if not emerg:
                continue
            hit = kept.any(0) & (em[:, 0] >= 0)
            cand = torch.stack((torch.full_like(em[:, 0], 4), em[:, 0], em[:, 1], em[:, 2]), dim=1)
        else:
            slot_hit = (act == a) & kept
            hit = slot_hit.any(0)
            s = slot_hit.int().argmax(0)
            pick = lambda x: x.gather(0, s[None])[0]   # noqa: E731
            cand = torch.stack((torch.full_like(s, a, dtype=torch.int32), pick(row), pick(tl), pick(tid)), dim=1)
        info = torch.where(hit[:, None], cand.int(), info)
    sel_out.copy_(info[:, 0])
    rows = r["traj"][info[:, 1].clamp(min=0).long()] * (info[:, 1] >= 0)[:, None, None]
    return info, rows


def results(pl, info, rows):
    f = pl.fetch("action_id", "traj_len", "traj_id", "status", "sc_flags", "path_len", "em_info", "trim", "traj_row",
                 "traj")
    # the compact row of a trajectory is unspecified and holds older bytes behind its length: compare without both
    out = [f[k] for k in ("action_id", "traj_len", "traj_id", "status", "sc_flags", "path_len", "trim")]
    out.append(f["em_info"][:, 1:])
    exp = np.where(f["traj_row"][..., None, None] >= 0, f["traj"][np.maximum(f["traj_row"], 0)], 0.0)
    exp[np.arange(exp.shape[2])[None, None, :] >= f["traj_len"][..., None]] = 0.0
    out.append(exp)
    out += [pl._state[k].cpu().numpy() for k in ("st_info", "vel_plan", "course")]
    info, rows = info.cpu().numpy(), rows.cpu().numpy().copy()
    rows[np.arange(rows.shape[1])[None, :] >= info[:, 2:3]] = 0.0
    return out + [info[:, [0, 2, 3]], rows]


def run_loop(lat, online, sc, args):
    """(b): per tick ms of the two graph-replayed closed loops, and whether they agree byte for byte"""
    dev = torch.device("cuda:0")
    names = ["emergency"] + ORDER
    ids = [PREFER_IDS[a] for a in names]
    d0 = sc.to_device(dev)
    B = sc.size
    t_const = torch.full((B,), T_CONST, dtype=torch.float64, device=dev)
    prefer = torch.as_tensor([ids], dtype=torch.int32, device=dev).expand(B, len(ids))   # one list, stride 0
    loops = {}
    for key in ("in_graph", "torch_pick"):
        pl = BatchPlanner(lat, online=online, device=dev, stateful=True)
        pl.set_vel_params(**dict(bench.vel_kwargs(), incl_emerg_traj=True))
        pl.capture_tick(d0).close()   # ids from the device counter, as in the replays
        loops[key] = dict(pl=pl, state=None)

    def first(key):
        lp = loops[key]
        pl = lp["pl"]
        pl.stage_scenarios(d0)
        pl.set_startpos()
        pl.tick()
        lp["pos"], lp["vel"] = d0.pos.clone(), d0.vel.clone()
        if key == "in_graph":
            s = pl.select(prefer)
            lp["info"], lp["rows"] = s["sel_info"], s["sel_traj"]
        else:
            if "sel" not in lp:
                lp["sel"] = torch.zeros(B, dtype=torch.int32, device=dev)
            lp["info"], lp["rows"] = torch_pick(pl, ids, True, lp["sel"])

    for key in loops:
        first(key)
    lp = loops["in_graph"]
    lp["graph"] = lp["pl"].capture_next_tick(d0, "selected", t_const, vel_est=d0.vel, prefer=prefer)
    lp = loops["torch_pick"]
    lp["graph"] = lp["pl"].capture_next_tick(d0, lp["sel"], t_const, vel_est=d0.vel)
    lp["sel"] = lp["graph"].inputs.sel_action   # the pick goes straight into the graph's input

    def tick(key):
        lp = loops[key]
        ok = lp["info"][:, :1] >= 0
        lp["pos"] = torch.where(ok, lp["rows"][:, 1, 1:3].double(), lp["pos"])
        lp["vel"] = torch.where(ok[:, 0], lp["rows"][:, 1, 5].double(), lp["vel"])
        g = lp["graph"]
        g.inputs.sc.pos.copy_(lp["pos"])
        g.inputs.vel_est.copy_(lp["vel"])
        g.replay()
        if key == "torch_pick":
            lp["info"], lp["rows"] = torch_pick(lp["pl"], ids, True, g.inputs.sel_action)

    same = True
    times = {k: [] for k in loops}
    for r in range(args.rounds + 2):   # round 0 checks every tick, round 1 warms up; neither is timed
        for key in (("in_graph", "torch_pick") if r % 2 == 0 else ("torch_pick", "in_graph")):
            first(key)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for k in range(8):
                tick(key)
                if r == 0:
                    loops[key]["res_%d" % k] = results(loops[key]["pl"], loops[key]["info"], loops[key]["rows"])
            torch.cuda.synchronize()
            if r >= 2:
                times[key].append(1e3 * (time.perf_counter() - t0) / 8)
        if r == 0:
            for k in range(8):
                a, b = loops["in_graph"]["res_%d" % k], loops["torch_pick"]["res_%d" % k]
                same = same and all(np.array_equal(x, y) for x, y in zip(a, b))
    for lp in loops.values():
        lp["graph"].close()
    return {"batch": B, "same_results_every_tick": bool(same),
            "ms_per_tick_median": {k: round(float(np.median(v)), 4) for k, v in times.items()},
            "ms_per_tick_all": {k: [round(x, 4) for x in v] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=40, help="plan_stream steps per timed round")
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds per variant")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_select.py needs a CUDA device")
    lat = bench.get_lattice("l216")
    online = read_online_config(bench.ONLINE_INI)
    sc = bench.make_batch("l216", args.batch)
    e2e = [run_e2e(lat, online, sc, args, emerg) for emerg in (False, True)]
    loop = run_loop(lat, online, sc, args)
    print(json.dumps({"tool": "bench_select", "card": card(), "lattice": "l216", "batch": args.batch,
                      "steps": args.steps, "rounds": args.rounds, "e2e": e2e, "closed_loop_8_ticks": loop,
                      "note": "e2e: plan_stream wall ms per step, full = every kept row downloaded, selected = "
                              "k_select + B rows of n_export x 7 fp32; closed loop: wall ms per replayed stateful tick "
                              "incl. the device vehicle dummy, in_graph = k_select recorded in the graph, torch_pick = "
                              "the same pick in torch code between replays"}))


if __name__ == "__main__":
    main()
