"""CPU diagnostic (not part of the product): replay bench.py's stateful closed loop (8 ticks, 0.1 s, the vehicle dummy on
the first kept trajectory) through the session ORACLE on a sample of the bench workload and count which branches of the
reference's iterative memory occur -- in particular those the device flags LTPL_SC_STATE_FALLBACK (DESIGN.md section 11).

    python tests/tools/cpu_stateful_diag.py [--n 400] [--tag l216] [--procs 8]
"""
import argparse
import collections
import os
import sys
from multiprocessing import Pool

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import bench  # noqa: E402
from tools.workload import step_along  # noqa: E402


class _Clk(object):
    def __init__(self):
        self.t = 100.0

    def __call__(self):
        return self.t


def _run(args):
    tag, lo, hi, n_total, seed = args
    from oracle.ltpl_oracle import OracleLTPL
    from oracle.ltpl_session import OracleSession
    lat = bench.get_lattice(tag)
    sc = bench.make_batch(tag, n_total, seed=seed)
    out = []
    vel = bench.vel_kwargs()
    for b in range(lo, hi):
        clk = _Clk()
        ses = OracleSession(OracleLTPL(lat), clock=clk)
        ev = []
        if ses.set_startpos(sc.pos[b], sc.heading[b], sc.vel[b]):
            out.append((b, ["tick0:out_of_track"]))
            continue
        pos_e, vel_e, sel = sc.pos[b].copy(), float(sc.vel[b]), "straight"
        ol = sc.object_list(b)
        for k in range(9):
            clk.t += 0.1
            try:
                st_before = ses.start_node
                m_path = ses.m_path
                exists = m_path is not None and sel in m_path
                rows = (ses.m_bp[sel][0].shape[0] if (ses.m_bp is not None and sel in ses.m_bp) else -1)
                if k > 0 and not (exists and rows > 2):
                    ev.append("tick%d:invalid_last(sel=%s,exists=%s,rows=%d)" % (k, sel, exists, rows))
                paths = ses.calc_paths(sel, ol)
                if not paths:
                    ev.append("tick%d:no_paths" % k)
                had_backup = ses.backup is not None
                traj, ids = ses.calc_vel_profile(pos_e, vel_e, **vel)
                if not traj:
                    ev.append("tick%d:no_traj" % k)
                    break
                # did the backup brake trigger?  (session keeps no flag: detect through the memory path identity)
                order = [a for a in ("follow", "straight", "left", "right") if a in traj and len(traj[a])]
                if not order:
                    ev.append("tick%d:no_traj" % k)
                    break
                sel = order[0]
                t = traj[sel][0]
                if t.shape[0] <= 2:
                    ev.append("tick%d:short_traj(%d)" % (k, t.shape[0]))
                p, v, _ = step_along(t[None], [t.shape[0]], 0.1)
                pos_e, vel_e = p[0], v[0]
            except Exception as e:   # noqa: BLE001
                ev.append("tick%d:exception(%s: %s)" % (k, type(e).__name__, str(e)[:80]))
                break
        out.append((b, ev))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=400)
    ap.add_argument("--tag", default="l216")
    ap.add_argument("--procs", type=int, default=8)
    ap.add_argument("--batch", type=int, default=10000)
    a = ap.parse_args()
    chunks = np.linspace(0, a.n, a.procs + 1).astype(int)
    jobs = [(a.tag, int(chunks[i]), int(chunks[i + 1]), a.batch, bench.SEED)
            for i in range(a.procs)]
    with Pool(a.procs) as p:
        res = [r for part in p.map(_run, jobs) for r in part]
    cnt = collections.Counter()
    for b, ev in res:
        for e in ev:
            cnt[e.split(":", 1)[1].split("(")[0]] += 1
    print("scenarios %d; events %s" % (len(res), dict(cnt)))
    for b, ev in res:
        if ev:
            print(b, ev[:4])


if __name__ == "__main__":
    main()
