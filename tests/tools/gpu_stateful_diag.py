"""GPU diagnostic: bench.py's stateful closed loop on the bench workload; per tick the scenarios that get flagged
LTPL_SC_STATE_FALLBACK / LTPL_SC_CAPACITY for the first time, by reason code (bits 8..10 of sc_flags), and for a few of
them what the session oracle (the reference's behaviour) does with the same inputs.

    python tests/tools/gpu_stateful_diag.py [--batch 10000] [--ticks 8] [--show 10] > gpurun_out/stateful_diag.txt
"""
import argparse
import collections
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import bench  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200 import capi  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner, read_online_config  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch  # noqa: E402
from tools.workload import closed_loop_step  # noqa: E402


class _Clk(object):
    def __init__(self):
        self.t = 100.0

    def __call__(self):
        return self.t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--ticks", type=int, default=8)
    ap.add_argument("--show", type=int, default=10)
    ap.add_argument("--tag", default="l216")
    a = ap.parse_args()
    device = torch.device("cuda:0")
    lat = bench.get_lattice(a.tag)
    sc = bench.make_batch(a.tag, a.batch, seed=bench.SEED)
    pl = BatchPlanner(lat, online=read_online_config(bench.ONLINE_INI), device=device, stateful=True)
    pl.set_vel_params(**bench.vel_kwargs())
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.tick()
    dt = 0.1
    pos_e, vel_e = sc.pos.copy(), sc.vel.copy()
    rec_in = []
    seen = np.zeros(a.batch, dtype=bool)
    shown = collections.Counter()
    names = {v: k for k, v in capi.ACTION_NAMES.items()}
    inv = capi.ACTION_NAMES
    for k in range(1, a.ticks + 1):
        prev = pl.fetch("traj_row", "traj_len", "action_id", "traj", "status")
        p_new, v_new, sel_a, ok, _ = closed_loop_step(prev, dt)
        pos_e, vel_e = np.where(ok[:, None], p_new, pos_e), np.where(ok, v_new, vel_e)
        rec_in.append((pos_e.copy(), vel_e.copy(), sel_a))
        pl.next_tick(ScenarioBatch(pos_e.copy(), sc.heading, sc.vel, sc.n_obj, sc.obj), sel_a, 2.0 * dt, vel_est=vel_e)
        torch.cuda.synchronize(device)
        f = pl.fetch("sc_flags", "action_id", "traj_len", "status")
        flags = f["sc_flags"]
        new = (flags != 0) & ~seen
        seen |= flags != 0
        reason = (flags & capi.SC_REASON_MASK) >> capi.SC_REASON_SHIFT
        hist = collections.Counter()
        for b in np.nonzero(new)[0]:
            hist[("capacity" if flags[b] & capi.SC_CAPACITY else "reason%d" % reason[b])] += 1
        print("tick %d: newly flagged %d %s; no trajectory before this tick: %d" % (
            k, int(new.sum()), dict(hist), int((~ok & ~(seen & ~new)).sum())))
        for b in np.nonzero(new)[0]:
            key = "capacity" if flags[b] & capi.SC_CAPACITY else "reason%d" % reason[b]
            if shown[key] >= a.show:
                continue
            shown[key] += 1
            print("  scenario %d (%s): executed %s; last tick actions %s rows %s status %s; this tick actions %s status %s" % (
                b, key, inv.get(int(sel_a[b]), sel_a[b]), prev["action_id"][:, b].tolist(), prev["traj_len"][:, b].tolist(),
                prev["status"][:, b].tolist(), f["action_id"][:, b].tolist(), f["status"][:, b].tolist()))
            try:   # what the reference does with the same inputs (session oracle = test infrastructure)
                from oracle.ltpl_oracle import OracleLTPL
                from oracle.ltpl_session import OracleSession
                clk = _Clk()
                ses = OracleSession(OracleLTPL(lat), clock=clk)
                ses.set_startpos(sc.pos[b], sc.heading[b], sc.vel[b])
                ol = sc.object_list(int(b))
                clk.t += dt
                ses.calc_paths("straight", ol)
                traj, _ = ses.calc_vel_profile(sc.pos[b], float(sc.vel[b]), **bench.vel_kwargs())
                for kk in range(k):
                    clk.t += dt
                    p_k, v_k, s_k = rec_in[kk]
                    had = sorted(traj)
                    paths = ses.calc_paths(inv[int(s_k[b])], ol)
                    bk = ses.backup is not None
                    traj, _ = ses.calc_vel_profile(p_k[b], float(v_k[b]), **bench.vel_kwargs())
                    if kk == k - 1:
                        print("    oracle tick %d: had %s, executed %s, backup %s -> paths %s traj %s rows %s vx0 %s" % (
                            kk + 1, had, inv[int(s_k[b])], bk, sorted(paths), sorted(traj),
                            [traj[x][0].shape[0] for x in sorted(traj)],
                            ["%.3f" % traj[x][0][0, 5] for x in sorted(traj)]))
            except Exception as e:   # noqa: BLE001
                print("    oracle: %s: %s" % (type(e).__name__, str(e)[:200]))


if __name__ == "__main__":
    main()
