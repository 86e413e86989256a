"""Golden vectors of velocity smoothing ([SMOOTHING] filt_window_width > 1, tph.conv_filt on every kept profile,
OTH:926-941 / 986-1004), made by running the UNMODIFIED reference on the shims of oracle/gen_golden.py with a copy of its
online ini in which only filt_window_width is changed.  Writes exactly two files and nothing else under the repository:

  tests/golden/ticks_smooth.npz                   first ticks, emergency trajectory on; sub-sets '<set>__<name>':
                                                  w3_default, w7_default (default lattice), w5_open (last ~400 m of
                                                  the open track: reduced horizons ending in the zero tail)
  tests/golden/ticks_multitick_smooth_default.npz 12 x 8 closed-loop ticks at window 5, emergency trajectory on, grip
                                                  drop on the odd sequences (smoothed backup brake and vel_course seam)

Smoothing changes only the vx / ax columns of a trajectory, so the first-tick file keeps of every trajectory these two
columns (whole profile, before the export cut) and of the emergency trajectory its exported rows; paths and the other
columns are pinned at window 1 by the other fixtures, the node sequences and row counts are kept here as well.

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_smooth
"""
import os
import re
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

SETS = (
    # name, filt_window_width, lattice tag, objects per scenario, seed
    ("w3_default", 3, "default", (1, 3), 6301),
    ("w7_default", 7, "default", (0, 3), 6302),
    ("w5_open", 5, "open", (0, 3), 6303),
)
COLS = (5, 6)             # vx, ax of a trajectory row
N_EXPORT = 115            # EXPORT.nmbr_export_points of the shipped online ini


def make_ltpl(graph_ltpl, tag, window, csv=None):
    """reference instance on the shipped offline ini and the shipped online ini with filt_window_width = window."""
    ini = '/tmp/golden_offline_%s.ini' % tag
    GG.write_offline_ini(ini, {})
    txt = open(GG.REF + "/params/ltpl_config_online.ini").read()
    pat = re.compile(r"^filt_window_width=.*$", re.M)
    assert len(pat.findall(txt)) == 1
    online = '/tmp/golden_online_%s_filt%d.ini' % (tag, window)
    open(online, 'w').write(pat.sub("filt_window_width=%d" % window, txt))
    path_dict = {'globtraj_input_path': csv or (GG.REF + "/inputs/traj_ltpl_cl/traj_ltpl_cl_monteblanco.csv"),
                 'graph_store_path': "/tmp/golden_graph_%s.pckl" % tag,
                 'ltpl_offline_param_path': ini,
                 'ltpl_online_param_path': online}
    ltpl = graph_ltpl.Graph_LTPL.Graph_LTPL(path_dict=path_dict, visual_mode=False, log_to_file=False)
    t0 = time.time()
    ltpl.graph_init()
    print("[%s, window %d] reference graph_init: %.1f s" % (tag, window, time.time() - t0))
    return ltpl


def first_tick_set(ltpl, track, n, n_obj, seed, is_open, vel_kwargs):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_scenarios
    sc = make_scenarios(track, n, seed=seed, n_obj_min=n_obj[0], n_obj_max=n_obj[1],
                        s_min=(track.length - 400.0) if is_open else 0.0, s_max=(track.length - 8.0) if is_open else None)
    recs = [GG.run_tick(ltpl, sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(b), vel_kwargs, full=True)
            for b in range(sc.size)]
    pk = GG.pack_ticks(recs)
    em = np.zeros((n, N_EXPORT, len(COLS)))
    em_len, em_id = np.zeros(n, dtype=np.int32), np.full(n, -1, dtype=np.int32)
    for i, r in enumerate(recs):
        if 'traj' in r and 'emergency' in r['traj']:
            t = r['traj']['emergency'][0]
            em[i, :min(t.shape[0], N_EXPORT)] = t[:N_EXPORT, COLS]
            em_len[i] = t.shape[0]
            em_id[i] = r['ids']['emergency']
    tmax = max(int(pk['traj_len'].max()), 1)
    return dict(out_of_track=pk['out_of_track'], path_len=pk['path_len'], nodes=pk['nodes'], nodes_len=pk['nodes_len'],
                red_len=pk['red_len'], traj=pk['traj'][:, :, :tmax][..., COLS], traj_len=pk['traj_len'],
                traj_id=pk['traj_id'], em_traj=em, em_len=em_len, em_id=em_id, sc_pos=sc.pos, sc_heading=sc.heading,
                sc_vel=sc.vel, sc_n_obj=sc.n_obj, sc_obj=sc.obj)


def main():
    graph_ltpl = GG.load_reference()
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    track = Track(GG.REF + "/inputs/traj_ltpl_cl/traj_ltpl_cl_monteblanco.csv")
    open_csv = os.path.join(REPO, "inputs", "traj_ltpl_cl", "traj_ltpl_cl_monteblanco_open.csv")   # committed
    vel_kwargs = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
                      safety_d=30.0, incl_emerg_traj=True)
    out = {}
    for name, w, tag, n_obj, seed in SETS:
        is_open = tag == "open"
        ltpl = make_ltpl(graph_ltpl, tag, w, csv=open_csv if is_open else None)
        st = first_tick_set(ltpl, Track(open_csv) if is_open else track, 32, n_obj, seed, is_open, vel_kwargs)
        st.update(filt_window=np.int32(w), lattice=np.array(tag))
        out.update({"%s__%s" % (name, k): v for k, v in st.items()})
        print("[smooth %s] trajectories %s; reduced %d; emergency %d; out of track %d" % (
            name, {a: int((st['traj_len'][:, i] > 0).sum()) for i, a in enumerate(GG.ACTIONS)},
            int(st['red_len'].sum()), int((st['em_len'] > 0).sum()), int(st['out_of_track'].sum())))
    out["ax_max_machines"] = vel_kwargs['ax_max_machines']
    np.savez_compressed(os.path.join(GG.GOLDEN, 'ticks_smooth.npz'), **out)

    ltpl = make_ltpl(graph_ltpl, "default", 5)
    mt = GG.multitick_fixture(graph_ltpl, ltpl, track, 12, 8, vel_kwargs, seed=2727, gg_drop=(3, 0.45), n_obj=(0, 3))
    mt['filt_window'] = np.int32(5)
    np.savez_compressed(os.path.join(GG.GOLDEN, 'ticks_multitick_smooth_default.npz'), **mt)


if __name__ == "__main__":
    main()
