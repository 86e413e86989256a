"""Velocity smoothing on the device ([SMOOTHING] filt_window_width > 1, k_smooth in csrc/ltpl_smooth.cuh) against golden
vectors of the unmodified reference (tests/golden/ticks_smooth.npz, ticks_multitick_smooth_default.npz), through the
Graph_LTPL facade with an online ini that sets the window, and on the full 10 000-scenario batch."""
import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,windows", [("w3_default", 1), ("w7_default", 3), ("w5_open", 4)])
def test_smoothed_first_tick_matches_reference_golden(name, windows):
    """node sequences, whole smoothed profiles (f64 planes), the fp32 export rows k_smooth rewrites, and the emergency
    trajectory."""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    g = H.golden("ticks_smooth.npz")
    sub = H._Sub(g, name)
    pl = D.planner(H.lattice_for(str(sub["lattice"])), windows, online=dict(filt_window_width=int(sub["filt_window"])),
                   ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True)
    n = sub["sc_pos"].shape[0]
    sc = ScenarioBatch.from_object_lists(sub["sc_pos"], sub["sc_heading"], sub["sc_vel"],
                                         [H.object_list(sub, b) for b in range(n)], k_max=3)
    D.first_tick(pl, sc)
    recs = pl.records()
    n_traj = sum(H.compare_first_tick(recs[b], sub, b, ctx=name + " gpu", exported=True, emergency=True)
                 for b in range(n))
    assert n_traj >= n


def _replay_multitick(g, windows):
    """the closed-loop sequences of a multi-tick fixture as one batch on a stateful planner at the fixture's window."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    n_seq, n_ticks = g["dt"].shape
    pl = D.planner(H.lattice_for("default"), windows, stateful=True,
                   online=dict(filt_window_width=int(g.g["filt_window"])), ax_max_machines=g["ax_max_machines"],
                   incl_emerg_traj=True)
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)])
    fails, compared = [], 0
    alive = np.ones(n_seq, dtype=bool)
    for k in range(n_ticks):
        sc = ScenarioBatch(g["pos_est"][:, k].copy(), g["sc_heading"].copy(), g["sc_vel"].copy(), g["sc_n_obj"].copy(),
                           g["obj"][:, k].copy())
        assert len(set(g["gg_scale"][:, k].tolist())) == 1
        pl.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True,
                          **dict(D.VEL, gg_scale=float(g["gg_scale"][0, k])))
        if k == 0:
            D.first_tick(pl, sc, vel_est=g["vel_est"][:, k])
        else:
            pl.next_tick(sc, sel_action=g["sel"][:, k], t_const=tc[:, k - 1], vel_est=g["vel_est"][:, k])
        recs = pl.records()
        for q in range(n_seq):
            if not alive[q] or k >= int(g["n_done"][q]):
                continue
            ctx = "sequence %d tick %d (%d windows)" % (q, k, windows)
            rec = recs[q]
            try:
                assert not rec["out_of_track"] and "error" not in rec and not (rec["flags"] & capi.SC_STATE_FALLBACK), \
                    ctx + " flags %d" % rec["flags"]
                compared += D.compare_multitick_row(rec, g, q, k, ctx, True)
            except AssertionError as e:
                fails.append(str(e)[:400])
                alive[q] = False            # later ticks of this sequence depend on this one
    assert not fails, "%d sequences diverged (%d trajectories matched before):\n%s" % (len(fails), compared,
                                                                                      "\n".join(fails[:8]))
    return compared


@pytest.mark.parametrize("group,windows", [(0, 1), (0, 4), (1, 2), (1, 3)])
def test_smoothed_next_tick_matches_reference_sequences(group, windows):
    """window 5, emergency trajectory on; group 1 (the odd sequences) loses grip from tick 3 on, so the brake on the backup
    plan behind vel_course is smoothed across the seam.  gg_scale is a per-batch parameter: the groups run apart."""
    g = D.Rows(H.golden("ticks_multitick_smooth_default.npz"), np.arange(group, 12, 2))
    assert _replay_multitick(g, windows) > 30


def test_facade_with_smoothing_ini_replays_reference_sequences(tmp_path):
    """Graph_LTPL reads filt_window_width = 5 from its online ini and replays three recorded sequences."""
    g = H.golden("ticks_multitick_smooth_default.npz")
    txt = open(H.ONLINE_INI).read()
    assert txt.count("filt_window_width=1\n") == 1
    ini = tmp_path / "online_w5.ini"
    ini.write_text(txt.replace("filt_window_width=1\n", "filt_window_width=%d\n" % int(g["filt_window"])))
    seqs = (0, 3, 6)                                       # sequences without the grip drop (one gg_scale per call)
    assert D.replay_facade(D.facade(tmp_path, ini), g, seqs, True) > 20


def _smoothed_tick(lat, sc, axm, w, windows):
    pl = D.planner(lat, windows, online=dict(filt_window_width=w), ax_max_machines=axm, incl_emerg_traj=True)
    D.first_tick(pl, sc)
    f = pl.fetch("status", "path_len", "traj_len", "traj_row", "traj", "s_vx_ax", "em_info")
    rows = D.export_rows(f, cut=True)                     # behind the export cut: unspecified
    ne = f["traj"].shape[1]
    em = np.zeros((rows.shape[1], ne, 7), dtype=np.float32)
    has_em = f["em_info"][:, 0] >= 0
    em[has_em] = f["traj"][f["em_info"][has_em, 0]]
    em[np.arange(ne)[None, :] >= f["em_info"][:, 1:2]] = 0.0
    return pl, dict(status=f["status"], path_len=f["path_len"], traj_len=f["traj_len"], rows=rows, em=em,
                    em_len=f["em_info"][:, 1].copy(), s_vx_ax=f["s_vx_ax"])


def test_full_batch_smoothing():
    """10 000 seeded scenarios on the ~200 x 11 lattice at window 5: bit-identical for 1, 4 and 5 scenario windows; equal
    to conv_filt of the SAME batch's unsmoothed (window 1) profiles, to float64 rounding, because nothing upstream of
    the filter depends on it in a first tick; the emergency trajectory is unchanged; the oracle agrees on a sample."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    from oracle.ltpl_oracle import OracleLTPL
    from oracle.tph_port import conv_filt
    axm = H.golden("ticks_l216.npz")["ax_max_machines"]
    lat = H.lattice_for("l216")
    B, w = 10000, 5
    sc = make_scenarios(Track(H.TRACK_CSV), B, seed=4242, n_obj_min=1, n_obj_max=3)
    pl, r5 = _smoothed_tick(lat, sc, axm, w, 4)
    for windows in (1, 5):
        other = _smoothed_tick(lat, sc, axm, w, windows)[1]
        for k in r5:
            assert np.array_equal(r5[k], other[k]), "'%s' differs between 4 and %d scenario windows" % (k, windows)
    r1 = _smoothed_tick(lat, sc, axm, 1, 4)[1]
    for k in ("status", "path_len", "traj_len", "em", "em_len"):
        assert np.array_equal(r5[k], r1[k]), "'%s' depends on the window" % k
    valid = (r5["status"].reshape(-1) & capi.ST_TRAJ_VALID) != 0
    assert valid.sum() > B
    s, v1, v5, a5 = r1["s_vx_ax"][0], r1["s_vx_ax"][1], r5["s_vx_ax"][1], r5["s_vx_ax"][2]
    n_path = r5["path_len"].reshape(-1)
    changed = 0
    for q in np.nonzero(valid)[0]:
        n = int(n_path[q])
        vf = conv_filt(signal=v1[q, :n], filt_window=w, closed=False)
        af = np.append((vf[1:] ** 2 - vf[:-1] ** 2) / (2 * np.diff(s[q, :n])), 0.0)
        af[:-1][np.isclose(vf[:-1], 0.0) & np.isclose(af[:-1], 0.0)] = -5.0
        assert v5[q, 0] == v1[q, 0], "path %d: row 0 changed" % q
        assert np.allclose(v5[q, :n], vf, rtol=1e-12, atol=1e-12), "path %d: vx != conv_filt(vx of window 1)" % q
        assert np.allclose(a5[q, :n], af, rtol=1e-9, atol=1e-9), "path %d: ax != calc_ax_profile(smoothed vx)" % q
        changed += int(not np.array_equal(v5[q, :n], v1[q, :n]))
    assert changed > valid.sum() // 2
    # the exported vx / ax columns are the fp32 image of the smoothed planes
    ok = r5["traj_len"] > 0
    for s_ in range(ok.shape[0]):
        for b in np.nonzero(ok[s_])[0][:200]:
            q, tl = s_ * B + b, int(r5["traj_len"][s_, b])
            assert np.array_equal(r5["rows"][s_, b, :tl, 5], v5[q, :tl].astype(np.float32))
            assert np.array_equal(r5["rows"][s_, b, :tl, 6], a5[q, :tl].astype(np.float32))

    pick = np.sort(np.random.default_rng(4243).choice(B, size=48, replace=False))
    D.assert_sample_matches_oracle(pl, OracleLTPL(lat, online=dict(filt_window_width=w)), sc, pick,
                                   dict(D.VEL, ax_max_machines=axm, incl_emerg_traj=True), "l216 w5", emergency=True)
