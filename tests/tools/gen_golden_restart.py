"""Golden vectors of restarts inside a closed loop: `Graph_LTPL.set_startpos` called on a LIVE instance of the unmodified
reference (OTH:161-179, 204: reinit_iterative_memory; the next calc_paths is a first tick with the forced 'straight'),
made on the shims of oracle/gen_golden.py with its scripted clock.  Writes exactly two files and nothing else under the
repository:

  tests/golden/ticks_multitick_restart_default.npz   12 x 10 closed-loop ticks, default lattice
  tests/golden/ticks_multitick_restart_l216.npz      12 x 10 closed-loop ticks, ~200 x 11 lattice

Every sequence starts with set_startpos + a first tick.  Restarts (`restart[q, k]`, kind in `rs_kind`):
  1 (a) re-anchoring at the current position estimate (heading of the driven trajectory there, velocity estimate)
  2 (b) a jump to a seeded new start elsewhere on the track with another start velocity
  3 (c) a pose off the track, 4 (c) a pose with a wrong heading: rejected, the sequence is not planned until the valid
        restart one or two ticks later
Schedule: every sequence restarts at ticks 3 and 7; the odd sequences execute the 'emergency' trajectory of ticks 1 and
2 (so the restart at tick 3 follows an executed 'emergency'), the grip drops (gg_scale 0.45) at tick 6 in every
sequence (brake on the backup plan right before the restart at tick 7), and the objects make the sequences execute
'follow', 'left' and 'right'.  The emergency trajectory is on.

Per tick the fixture holds the inputs of a batched replay -- pos / heading / vel (the new pose and start velocity at a
restart, else the position estimate and the pose of the latest set_startpos), sel (executed action, 4 = 'emergency'),
vel_est, objects, gg_scale, dt of the scripted clock and the t_const the reference used (0 where it took no constant
segment) -- and the outputs (node sequences, trajectories, ids; `planned` = the reference planned this tick).
The calculation-time buffer of the reference survives set_startpos (OTH:62 is not reset); it starts empty in every
sequence (each sequence stands for a fresh instance).

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_restart
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

N_SEQ, N_TICKS = 12, 10
RESTART_TICKS = (3, 7)
EM_TICKS = (1, 2)          # odd sequences execute the emergency trajectory of these ticks
GG_DROP = (6, 0.45)        # tick, gg_scale
PMAX, HMAX = 115, 60
KIND_A, KIND_B, KIND_OFF, KIND_HEAD = 1, 2, 3, 4


class CountingClock(GG.ScriptedClock):
    """the scripted clock; counts the calls, so that the branch calc_paths took is known (OTH:353-354: two calls when
    a constant segment of the last trajectory is kept, OTH:395: one otherwise)"""

    def __init__(self):
        super().__init__()
        self.calls = 0

    def time(self):
        self.calls += 1
        return self.t


def heading_on(traj, pos):
    """psi of the trajectory row nearest to pos (the re-anchoring heading)"""
    i = int(np.argmin(np.hypot(traj[:, 1] - pos[0], traj[:, 2] - pos[1])))
    return float(traj[i, 3])


def restart_fixture(ltpl, track, vel_kwargs, seed):
    import graph_ltpl.online_graph.src.OnlineTrajectoryHandler as oth_mod
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_scenarios
    clock = CountingClock()
    real_time = oth_mod.time
    oth_mod.time = clock
    try:
        sc = make_scenarios(track, N_SEQ, seed=seed, n_obj_min=1, n_obj_max=3)
        jumps = make_scenarios(track, 2 * N_SEQ, seed=seed + 7, n_obj_min=0, n_obj_max=0)
        rng = np.random.default_rng(seed + 1)
        prefer = (("right", "left", "straight", "follow"), ("follow", "straight", "left", "right"),
                  ("left", "straight", "follow", "right"))
        K = sc.obj.shape[1]
        f64 = lambda *s: np.zeros((N_SEQ, N_TICKS) + s)   # noqa: E731
        i32 = lambda *s: np.zeros((N_SEQ, N_TICKS) + s, dtype=np.int32)   # noqa: E731
        out = dict(dt=f64(), sel=i32(), pos=f64(2), heading=f64(), vel=f64(), vel_est=f64(), obj=f64(K, 5),
                   restart=i32(), rs_kind=i32(), t_const=f64(), planned=i32(), rejected=i32(),
                   gg_scale=np.ones((N_SEQ, N_TICKS)),
                   traj=f64(4, PMAX, 7), traj_len=i32(4), traj_id=np.full((N_SEQ, N_TICKS, 4), -1, dtype=np.int32),
                   nodes=np.full((N_SEQ, N_TICKS, 4, HMAX, 2), -1, dtype=np.int32), nodes_len=i32(4),
                   path_len=i32(4), em_traj=f64(PMAX, 7), em_len=i32())
        n_jump = 0
        for q in range(N_SEQ):
            oth = None
            objs = sc.obj[q, :int(sc.n_obj[q])].copy()
            pose = (np.array(sc.pos[q]), float(sc.heading[q]), float(sc.vel[q]))   # of the latest set_startpos
            pos_est, vel_est, sel, traj_set, drive = pose[0].copy(), pose[2], "straight", None, "straight"
            order = prefer[q % len(prefer)]
            planning = False                        # the last set_startpos was accepted and the loop is alive
            valid_at = None                         # tick of the valid restart after a rejected one
            for k in range(N_TICKS):
                dt = float(rng.uniform(0.04, 0.16))
                clock.t += dt
                for j in range(objs.shape[0]):      # opponents keep heading and speed
                    objs[j, 0] -= np.sin(objs[j, 2]) * objs[j, 3] * dt
                    objs[j, 1] += np.cos(objs[j, 2]) * objs[j, 3] * dt
                if planning and traj_set is not None:
                    pos_est, vel_est = advance_on_traj_safe(traj_set[drive][0], dt, pos_est, vel_est)
                kind = 0
                if k == 0:
                    kind = -1                       # the initial set_startpos (not a restart)
                elif k in RESTART_TICKS:
                    if k == RESTART_TICKS[0] and q % 4 == 2:
                        kind = KIND_OFF if q % 8 == 2 else KIND_HEAD
                        valid_at = k + (1 if q % 8 == 2 else 2)
                    elif k == RESTART_TICKS[0]:
                        kind = KIND_B if q % 4 == 1 else KIND_A
                    else:
                        kind = KIND_B if q % 2 == 0 else KIND_A
                elif k == valid_at:
                    kind = KIND_B
                if kind == KIND_A and not planning:
                    kind = KIND_B                   # nothing to re-anchor on
                if kind == -1:
                    pose = (np.array(sc.pos[q]), float(sc.heading[q]), float(sc.vel[q]))
                elif kind == KIND_A:
                    pose = (pos_est.copy(), heading_on(traj_set[drive][0], pos_est), float(vel_est))
                elif kind == KIND_B:
                    j = n_jump % jumps.size
                    n_jump += 1
                    pose = (np.array(jumps.pos[j]), float(jumps.heading[j]), float(jumps.vel[j]))
                elif kind == KIND_OFF:              # 40 m to the side of the track
                    h = float(pose[1])
                    pose = (pos_est + 40.0 * np.array([np.cos(h), np.sin(h)]), h, float(vel_est))
                elif kind == KIND_HEAD:             # facing backwards
                    h = float(np.arctan2(np.sin(pose[1] + np.pi), np.cos(pose[1] + np.pi)))
                    pose = (pos_est.copy(), h, float(vel_est))
                if kind != 0:
                    pos_est, vel_est = pose[0].copy(), pose[2]
                out['dt'][q, k] = dt
                out['sel'][q, k] = 4 if sel == 'emergency' else GG.ACTIONS.index(sel)
                out['pos'][q, k], out['heading'][q, k], out['vel'][q, k] = pos_est, pose[1], pose[2]
                out['vel_est'][q, k] = vel_est
                out['obj'][q, k, :objs.shape[0]] = objs
                out['restart'][q, k] = int(kind > 0)
                out['rs_kind'][q, k] = max(kind, 0)
                if kind != 0:
                    rejected = ltpl.set_startpos(pos_est=np.array(pose[0]), heading_est=float(pose[1]),
                                                 vel_est=float(pose[2]))
                    out['rejected'][q, k] = int(rejected)
                    planning = not rejected
                    if oth is None:
                        oth = ltpl._Graph_LTPL__oth
                        oth._OnlineTrajectoryHandler__calc_buffer = []    # a fresh instance per sequence
                        ltpl._Graph_LTPL__obj_zone = []
                        ltpl._Graph_LTPL__obj_list_handler._ObjectListInterface__object_zones = []
                    traj_set = None
                if not planning:
                    continue
                ol = [{'id': j + 1, 'type': 'physical', 'X': float(o[0]), 'Y': float(o[1]), 'theta': float(o[2]),
                       'v': float(o[3]), 'length': float(o[4]), 'width': 2.5} for j, o in enumerate(objs)]
                clock.calls = 0
                paths = ltpl.calc_paths(prev_action_id=sel, object_list=ol)
                if clock.calls == 2:                # OTH:351-375: the t_const the reference used
                    buf = oth._OnlineTrajectoryHandler__calc_buffer
                    out['t_const'][q, k] = min(float(np.sum(buf) / len(buf))
                                               * oth._OnlineTrajectoryHandler__calc_time_safety, 0.5)
                nodes = oth._OnlineTrajectoryHandler__last_action_set_nodes
                for a, act in enumerate(GG.ACTIONS):
                    if act in paths and len(paths[act]) and np.size(paths[act][0]):
                        out['path_len'][q, k, a] = paths[act][0].shape[0]
                        nd = [[-1 if v is None else int(v) for v in pair] for pair in nodes[act][0]]
                        out['nodes'][q, k, a, :len(nd)] = nd
                        out['nodes_len'][q, k, a] = len(nd)
                vk = dict(vel_kwargs)
                if k == GG_DROP[0]:
                    vk['gg_scale'] = GG_DROP[1]
                out['gg_scale'][q, k] = vk.get('gg_scale', 1.0)
                traj_set, ids, _ = ltpl.calc_vel_profile(pos_est=pos_est, vel_est=vel_est, **vk)
                out['planned'][q, k] = 1
                for a, act in enumerate(GG.ACTIONS):
                    if act in traj_set and len(traj_set[act]):
                        t = traj_set[act][0]
                        out['traj'][q, k, a, :t.shape[0]] = t
                        out['traj_len'][q, k, a] = t.shape[0]
                        out['traj_id'][q, k, a] = ids[act]
                if 'emergency' in traj_set:
                    t = traj_set['emergency'][0]
                    out['em_traj'][q, k, :t.shape[0]] = t
                    out['em_len'][q, k] = t.shape[0]
                cand = [a for a in order if a in traj_set and len(traj_set[a])]
                if not cand:
                    planning, traj_set = False, None
                    continue
                sel = cand[0]
                if q % 2 == 1 and k in EM_TICKS and 'emergency' in traj_set:
                    sel = 'emergency'
                drive = sel
        out.update(ax_max_machines=vel_kwargs['ax_max_machines'], sc_n_obj=sc.n_obj)
        return out
    finally:
        oth_mod.time = real_time


def advance_on_traj_safe(traj, dt, pos_est, vel_est):
    """the vehicle dummy of oracle/gen_golden.py; a trajectory of one row leaves the vehicle where it is"""
    if traj.shape[0] < 2:
        return pos_est, vel_est
    return GG.advance_on_traj(traj, dt)


def coverage(f):
    """restart counts per kind and per situation before the restart (what the tick before executed)"""
    r = f['restart'] > 0
    prev_sel = np.zeros_like(f['sel'])
    prev_sel[:, 1:] = f['sel'][:, 1:]            # sel of tick k = the action executed since tick k - 1
    out = {"restarts": int(r.sum()), "rejected": int((r & (f['rejected'] > 0)).sum())}
    for kind, name in ((KIND_A, "a"), (KIND_B, "b"), (KIND_OFF, "c_off_track"), (KIND_HEAD, "c_heading")):
        out[name] = int((f['rs_kind'] == kind).sum())
    planned_before = np.zeros_like(r)
    planned_before[:, 1:] = f['planned'][:, :-1] > 0
    for code, name in ((1, "after_follow"), (2, "after_left"), (3, "after_right"), (4, "after_emergency")):
        out[name] = int((r & planned_before & (prev_sel == code)).sum())
    drop = np.zeros_like(r)
    drop[:, 1:] = f['gg_scale'][:, :-1] < 1.0
    out["after_grip_drop"] = int((r & planned_before & drop).sum())
    # a valid restart one or two ticks after a rejected one
    ok = 0
    for q, k in zip(*np.nonzero(r & (f['rejected'] > 0))):
        ok += int(any(k + d < f['restart'].shape[1] and f['restart'][q, k + d] and not f['rejected'][q, k + d]
                      for d in (1, 2)))
    out["valid_after_rejected"] = ok
    return out


def main():
    graph_ltpl = GG.load_reference()
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    track = Track(GG.REF + "/inputs/traj_ltpl_cl/traj_ltpl_cl_monteblanco.csv")
    vel_kwargs = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
                      safety_d=30.0, incl_emerg_traj=True)
    for tag, overrides, seed in (("default", {}, 5151), ("l216", {"lat_resolution": 1.0, "lon_straight_step": 12.0},
                                                          5252)):
        ltpl, _ = GG.make_ltpl(graph_ltpl, tag, overrides)
        f = restart_fixture(ltpl, track, vel_kwargs, seed)
        print("[restart %s] %d planned ticks; coverage %s" % (tag, int(f['planned'].sum()), coverage(f)))
        np.savez_compressed(os.path.join(GG.GOLDEN, 'ticks_multitick_restart_%s.npz' % tag), **f)


if __name__ == "__main__":
    main()
