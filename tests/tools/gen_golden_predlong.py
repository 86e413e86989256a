"""Golden vectors of objects with LONG 'prediction' arrays (OLI:117-119; GLNT:169-189 turns every point into one obstacle
disc, the LAST one decides the object's layer -- quirk q14), made by running the UNMODIFIED reference on the shims of
oracle/gen_golden.py.  Writes exactly one file and nothing else under the repository:

  tests/golden/ticks_predlong.npz   first ticks; sub-sets '<set>__<name>' (read through tests/helpers.py):
                                      default  default lattice, 48 scenarios
                                      l216     ~216 x 11 lattice (lat_resolution 1.0, lon_straight_step 12.0), 32
                                      open     last ~400 m of the open track (points past the track end), 32

1-5 objects per scenario; per object 0-80 prediction points at 0.1 s (constant velocity plus a lateral drift, so that
long arrays leave the planning range and the track), about one object in seven without the key (built-in 0.2 s point).
Most scenarios hold more than 32 discs (on-track objects + their points), some more than 128.

What the discs decide is kept whole: which actions exist, their node sequences and node indices, the reduced-horizon
flags, the closest object, and of every trajectory its length, id and the columns vx, ax of the whole profile (the
follow-mode profile depends on the closest object).  Paths and the other trajectory columns are functions of the node
sequences, pinned by the other first-tick fixtures, so only their lengths are kept here.  The prediction points are
rounded to float32-representable values before the reference sees them and stored as float32, without loss.

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_predlong
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

SETS = (
    # name, lattice tag, offline overrides, scenarios, seed
    ("default", "default", {}, 48, 8101),
    ("l216", "l216", {"lat_resolution": 1.0, "lon_straight_step": 12.0}, 32, 8102),
    ("open", "open", {}, 32, 8103),
)
K_PRED = 80
COLS = (5, 6)   # vx, ax of a trajectory row
KEEP = ('out_of_track', 'start_node', 'closest_obj_index', 'path_len', 'nodes', 'nodes_len', 'node_idx', 'red_len',
        'traj', 'traj_len', 'traj_id')
DT = 0.1


def add_predictions(sc, rng):
    """constant velocity along the heading plus a lateral drift (m/s) per object; about 1 in 7 objects has no key."""
    n, k = sc.obj.shape[0], sc.obj.shape[1]
    sc.pred = np.zeros((n, k, K_PRED, 2))
    sc.n_pred = np.full((n, k), -1, dtype=np.int32)
    for b in range(n):
        for j in range(int(sc.n_obj[b])):
            if rng.random() < 0.15:
                continue
            m = int(rng.integers(0, 8)) if rng.random() < 0.1 else int(rng.integers(16, K_PRED + 1))
            x, y, th, v, _ = sc.obj[b, j]
            drift = rng.uniform(-1.5, 1.5)
            t = DT * np.arange(1, m + 1)
            sc.pred[b, j, :m, 0] = x - np.sin(th) * v * t + np.cos(th) * drift * t
            sc.pred[b, j, :m, 1] = y + np.cos(th) * v * t + np.sin(th) * drift * t
            sc.n_pred[b, j] = m
    sc.pred = sc.pred.astype(np.float32).astype(np.float64)   # exactly what the fixture stores
    return sc


def disc_counts(sc):
    """discs per scenario if every object is on the track: its position + its points (1 for the built-in point)."""
    per = 1 + np.where(sc.n_pred < 0, 1, sc.n_pred)
    live = np.arange(sc.obj.shape[1])[None, :] < sc.n_obj[:, None]
    return (per * live).sum(axis=1).astype(np.int32)


def main():
    graph_ltpl = GG.load_reference()
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    open_csv = os.path.join(REPO, "inputs", "traj_ltpl_cl", "traj_ltpl_cl_monteblanco_open.csv")   # committed
    vel_kwargs = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
                      safety_d=30.0, incl_emerg_traj=False)
    out = {}
    for name, tag, overrides, n, seed in SETS:
        is_open = tag == "open"
        ltpl, _ = GG.make_ltpl(graph_ltpl, tag, overrides, csv=open_csv if is_open else None)
        track = Track(open_csv if is_open else GG.REF + "/inputs/traj_ltpl_cl/traj_ltpl_cl_monteblanco.csv")
        sc = make_scenarios(track, n, seed=seed, n_obj_min=1, n_obj_max=5,
                            s_min=(track.length - 400.0) if is_open else 0.0,
                            s_max=(track.length - 8.0) if is_open else None)
        sc = add_predictions(sc, np.random.default_rng(seed + 1))
        recs = [GG.run_tick(ltpl, sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(b), vel_kwargs, full=True)
                for b in range(sc.size)]
        pk = GG.pack_ticks(recs)
        tmax = max(int(pk['traj_len'].max()), 1)
        pk = {k: pk[k] for k in KEEP}
        pk['traj'] = pk['traj'][:, :, :tmax][..., COLS]
        pk.update(sc_pos=sc.pos, sc_heading=sc.heading, sc_vel=sc.vel, sc_n_obj=sc.n_obj, sc_obj=sc.obj,
                  sc_pred=sc.pred.astype(np.float32), sc_n_pred=sc.n_pred, n_disc=disc_counts(sc), lattice=np.array(tag))
        out.update({"%s__%s" % (name, k): v for k, v in pk.items()})
        nd = pk['n_disc']
        print("[predlong %s] discs: > 32 in %d / %d, > 128 in %d, max %d; closest object %d; action paths %s" % (
            name, int((nd > 32).sum()), n, int((nd > 128).sum()), int(nd.max()), int((pk['closest_obj_index'] >= 0).sum()),
            {a: int((pk['path_len'][:, i] > 0).sum()) for i, a in enumerate(GG.ACTIONS)}))
    out["ax_max_machines"] = vel_kwargs['ax_max_machines']
    np.savez_compressed(os.path.join(GG.GOLDEN, 'ticks_predlong.npz'), **out)


if __name__ == "__main__":
    main()
