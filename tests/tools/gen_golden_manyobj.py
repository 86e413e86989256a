"""Golden vectors of LONG object lists (OLI:96-141: every 'physical' entry is tested against the track bounds, the
on-track ones become the vehicle list in list order), made by running the UNMODIFIED reference on the shims of
oracle/gen_golden.py.  Writes exactly one file and nothing else under the repository:

  tests/golden/ticks_manyobj.npz   first ticks; sub-sets '<set>__<name>' (read through tests/helpers.py):
                                     default  default lattice, 48 scenarios
                                     l216     ~216 x 11 lattice (lat_resolution 1.0, lon_straight_step 12.0), 32
                                     open     last ~400 m of the open track (points past the track end), 32

17-64 objects per scenario: 10-40 of them on the track, 20-600 m ahead (a crowded field, partly beyond the planning
range), the rest beyond the track bounds, interleaved in the list, so that an object's vehicle index differs from its slot.  About a
third of the objects carry a 'prediction' array of 0-20 points at 0.1 s.  In about a quarter of the scenarios the last
on-track object stands beside the ego vehicle, so that it lies beside the constant path segment (MOPG:86-104).

What the objects decide is kept whole: which actions exist, their node sequences and node indices, the reduced-horizon
flags, the closest object, and of every trajectory its length, id and the columns vx, ax of the whole profile.  Objects
and prediction points are rounded to float32-representable values before the reference sees them and stored as float32,
without loss.

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_manyobj
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

SETS = (
    # name, lattice tag, offline overrides, scenarios, seed
    ("default", "default", {}, 48, 8201),
    ("l216", "l216", {"lat_resolution": 1.0, "lon_straight_step": 12.0}, 32, 8202),
    ("open", "open", {}, 32, 8203),
)
K_OBJ = 64
K_PRED = 20
COLS = (5, 6)   # vx, ax of a trajectory row
KEEP = ('out_of_track', 'start_node', 'closest_obj_index', 'path_len', 'nodes', 'nodes_len', 'node_idx', 'red_len',
        'traj', 'traj_len', 'traj_id')
DT = 0.1


def f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def object_field(track, sc, b, rng):
    """object rows (X, Y, theta, v, length), prediction counts (-1: no key) and points of scenario b of the batch sc."""
    n_obj = int(rng.integers(17, K_OBJ + 1))
    n_on = int(rng.integers(10, min(40, n_obj) + 1))
    # arc length of the ego vehicle: the nearest race-line point
    d2 = np.sum((track.raceline - sc.pos[b]) ** 2, axis=1)
    s_e = float(track.s[int(np.argmin(d2))])
    beside = rng.random() < 0.25 and n_on >= 31
    ds = rng.uniform(20.0, 600.0, size=n_obj)
    if beside:   # the last on-track object next to the ego vehicle: beside the constant path segment
        ds[n_on - 1] = rng.uniform(1.0, 6.0)
    rows = np.zeros((n_obj, 5))
    for j in range(n_obj):
        ref, nv, wl, wr, psi, vrl = track.frame(np.array([s_e + ds[j]]))
        ref, nv, wl, wr, psi, vrl = ref[0], nv[0], float(wl[0]), float(wr[0]), float(psi[0]), float(vrl[0])
        if j < n_on:
            u = rng.uniform(0.0, 1.0)
            if beside and j == n_on - 1:
                u = 0.0 if rng.random() < 0.5 else 1.0
            d = -(wl - 1.4) + u * ((wr - 1.4) + (wl - 1.4))
        else:   # 3-20 m beyond the left or the right bound
            d = -(wl + rng.uniform(3.0, 20.0)) if rng.random() < 0.5 else wr + rng.uniform(3.0, 20.0)
        rows[j, 0:2] = ref + nv * d
        rows[j, 2] = psi
        rows[j, 3] = rng.uniform(0.0, 0.5) * vrl
        rows[j, 4] = 5.0
    order = rng.permutation(n_obj)   # on-track and off-track objects interleaved
    rows = f32(rows[order])
    n_pred = np.full(n_obj, -1, dtype=np.int32)
    pred = np.zeros((n_obj, K_PRED, 2))
    for j in range(n_obj):
        if rng.random() < 1.0 / 3.0:
            m = int(rng.integers(0, K_PRED + 1))
            x, y, th, v, _ = rows[j]
            drift = rng.uniform(-1.0, 1.0)
            t = DT * np.arange(1, m + 1)
            pred[j, :m, 0] = x - np.sin(th) * v * t + np.cos(th) * drift * t
            pred[j, :m, 1] = y + np.cos(th) * v * t + np.sin(th) * drift * t
            n_pred[j] = m
    return rows, n_pred, f32(pred)


def object_list(rows, n_pred, pred):
    out = []
    for k in range(rows.shape[0]):
        x, y, th, v, ln = (float(a) for a in rows[k])
        out.append({'id': k + 1, 'type': 'physical', 'X': x, 'Y': y, 'theta': th, 'v': v, 'length': ln, 'width': 2.5})
        if n_pred[k] >= 0:
            out[-1]['prediction'] = pred[k, :int(n_pred[k])].copy()
    return out


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
        sc = make_scenarios(track, n, seed=seed, n_obj_min=0, n_obj_max=0, k_max=1,
                            s_min=(track.length - 400.0) if is_open else 0.0,
                            s_max=(track.length - 8.0) if is_open else None)
        rng = np.random.default_rng(seed + 1)
        obj = np.zeros((n, K_OBJ, 5), dtype=np.float32)
        n_obj = np.zeros(n, dtype=np.int32)
        n_pred = np.full((n, K_OBJ), -1, dtype=np.int32)
        pred = np.zeros((n, K_OBJ, K_PRED, 2), dtype=np.float32)
        recs = []
        for b in range(n):
            rows, npd, pts = object_field(track, sc, b, rng)
            k = rows.shape[0]
            obj[b, :k], n_obj[b], n_pred[b, :k], pred[b, :k] = rows, k, npd, pts
            recs.append(GG.run_tick(ltpl, sc.pos[b], sc.heading[b], sc.vel[b], object_list(rows, npd, pts), vel_kwargs,
                                    full=True))
        pk = GG.pack_ticks(recs)
        tmax = max(int(pk['traj_len'].max()), 1)
        pk = {k: pk[k] for k in KEEP}
        pk['traj'] = pk['traj'][:, :, :tmax][..., COLS]
        pk.update(sc_pos=sc.pos, sc_heading=sc.heading, sc_vel=sc.vel, sc_n_obj=n_obj, sc_obj=obj, sc_pred=pred,
                  sc_n_pred=n_pred, lattice=np.array(tag))
        out.update({"%s__%s" % (name, k): v for k, v in pk.items()})
        coi = pk['closest_obj_index']
        print("[manyobj %s] objects %d-%d; closest object %d (vehicle index >= 16: %d); action paths %s" % (
            name, int(n_obj.min()), int(n_obj.max()), int((coi >= 0).sum()), int((coi >= 16).sum()),
            {a: int((pk['path_len'][:, i] > 0).sum()) for i, a in enumerate(GG.ACTIONS)}))
    out["ax_max_machines"] = vel_kwargs['ax_max_machines']
    np.savez_compressed(os.path.join(GG.GOLDEN, 'ticks_manyobj.npz'), **out)


if __name__ == "__main__":
    main()
