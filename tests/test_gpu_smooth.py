"""Velocity smoothing on the device ([SMOOTHING] filt_window_width > 1, k_smooth in csrc/ltpl_smooth.cuh) against golden
vectors of the unmodified reference (tests/golden/ticks_smooth.npz, ticks_multitick_smooth_default.npz), through the
Graph_LTPL facade with an online ini that sets the window, and on the full 10 000-scenario batch."""
import numpy as np
import pytest

from tests import helpers as H
from tests.smooth_golden import compare_smooth_record
from tests.test_gpu_multitick import _Rows, _t_const

pytestmark = pytest.mark.gpu

VEL = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)
EXPORT_COLS = ("s", "x", "y", "psi", "kappa", "vx", "ax")


@pytest.mark.parametrize("name,windows", [("w3_default", 1), ("w7_default", 3), ("w5_open", 4)])
def test_smoothed_first_tick_matches_reference_golden(name, windows):
    """node sequences, whole smoothed profiles (f64 planes), the fp32 export rows k_smooth rewrites, and the emergency
    trajectory."""
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    g = H.golden("ticks_smooth.npz")
    sub = H._Sub(g, name)
    w = int(sub["filt_window"])
    pl = BatchPlanner(H.lattice_for(str(sub["lattice"])), online=dict(filt_window_width=w), device="cuda:0")
    pl.set_subbatches(windows)
    pl.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True, **VEL)
    n = sub["sc_pos"].shape[0]
    sc = ScenarioBatch.from_object_lists(sub["sc_pos"], sub["sc_heading"], sub["sc_vel"],
                                         [H.object_list(sub, b) for b in range(n)], k_max=3)
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.tick()
    recs = pl.records()
    n_traj = sum(compare_smooth_record(recs[b], sub, b, ctx=name + " gpu", exported=True) for b in range(n))
    assert n_traj >= n


def _replay_multitick(g, windows):
    """the closed-loop sequences of a multi-tick fixture as one batch on a stateful planner at the fixture's window."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    n_seq, n_ticks = g["dt"].shape
    pl = BatchPlanner(H.lattice_for("default"), online=dict(filt_window_width=int(g.g["filt_window"])),
                      device="cuda:0", stateful=True)
    pl.set_subbatches(windows)
    tc = np.array([_t_const(g["dt"][q, 1:]) for q in range(n_seq)])
    fails, compared = [], 0
    alive = np.ones(n_seq, dtype=bool)
    for k in range(n_ticks):
        sc = ScenarioBatch(g["pos_est"][:, k].copy(), g["sc_heading"].copy(), g["sc_vel"].copy(), g["sc_n_obj"].copy(),
                           g["obj"][:, k].copy())
        assert len(set(g["gg_scale"][:, k].tolist())) == 1
        pl.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True,
                          **dict(VEL, gg_scale=float(g["gg_scale"][0, k])))
        if k == 0:
            pl.stage_scenarios(sc, vel_est=g["vel_est"][:, k])
            pl.upload()
            pl.set_startpos()
            pl.tick()
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
                for a, act in enumerate(H.ACTIONS):
                    n_want = int(g["path_len"][q, k, a])
                    assert (act in rec["paths"]) == (n_want > 0), ctx + " path " + act
                    if n_want and not rec["tie"].get(act):
                        nd = [[-1 if v is None else int(v) for v in p] for p in rec["nodes"][act][0]]
                        assert nd == g["nodes"][q, k, a, :int(g["nodes_len"][q, k, a])].tolist(), ctx + " nodes " + act
                    t_want = int(g["traj_len"][q, k, a])
                    assert (act in rec["traj"]) == (t_want > 0), ctx + " trajectory " + act
                    if t_want:
                        assert rec["traj"][act][0].shape[0] == t_want, ctx + " rows " + act
                        H.assert_close("traj[%s]" % act, rec["traj"][act][0], g["traj"][q, k, a, :t_want], EXPORT_COLS,
                                       ctx)
                        compared += 1
                n_em = min(int(g["em_len"][q, k]), 115)
                assert ("emergency" in rec["traj"]) == (n_em > 0), ctx + " emergency presence"
                if n_em:
                    H.assert_close("traj[emergency]", rec["traj"]["emergency"][0], g["em_traj"][q, k, :n_em],
                                   EXPORT_COLS, ctx, w_rel=H.W_REL_BRAKE)
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
    g = _Rows(H.golden("ticks_multitick_smooth_default.npz"), np.arange(group, 12, 2))
    assert _replay_multitick(g, windows) > 30


def test_facade_with_smoothing_ini_replays_reference_sequences(tmp_path):
    """Graph_LTPL reads filt_window_width = 5 from its online ini and replays three recorded sequences."""
    from graphbasedlocaltrajectoryplanner_b200.Graph_LTPL import Graph_LTPL
    g = H.golden("ticks_multitick_smooth_default.npz")
    txt = open(H.ONLINE_INI).read()
    assert txt.count("filt_window_width=1\n") == 1
    ini = tmp_path / "online_w5.ini"
    ini.write_text(txt.replace("filt_window_width=1\n", "filt_window_width=%d\n" % int(g["filt_window"])))
    pd = {'globtraj_input_path': H.TRACK_CSV, 'graph_store_path': str(tmp_path / "lattice.npz"),
          'ltpl_offline_param_path': H.OFFLINE_INI, 'ltpl_online_param_path': str(ini)}
    ltpl = Graph_LTPL(path_dict=pd, visual_mode=False, log_to_file=False, device="cuda:0")
    ltpl.graph_init()

    class Clk(object):
        t = 10.0

        def __call__(self):
            return self.t
    clk = Clk()
    ltpl.clock = clk
    compared = 0
    for q in (0, 3, 6):                                    # sequences without the grip drop (one gg_scale per call)
        assert ltpl.set_startpos(pos_est=g["sc_pos"][q], heading_est=g["sc_heading"][q], vel_est=g["sc_vel"][q]) is False
        n_obj = int(g["sc_n_obj"][q])
        for k in range(int(g["n_done"][q])):
            clk.t += float(g["dt"][q, k])
            ol = [{'id': j + 1, 'type': 'physical', 'X': float(o[0]), 'Y': float(o[1]), 'theta': float(o[2]),
                   'v': float(o[3]), 'length': float(o[4]), 'width': 2.5} for j, o in enumerate(g["obj"][q, k, :n_obj])]
            paths = ltpl.calc_paths(prev_action_id=(H.ACTIONS + ("emergency",))[int(g["sel"][q, k])], object_list=ol)
            traj, ids, _ = ltpl.calc_vel_profile(pos_est=g["pos_est"][q, k], vel_est=float(g["vel_est"][q, k]),
                                                 ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True,
                                                 **dict(VEL, gg_scale=float(g["gg_scale"][q, k])))
            ctx = "facade sequence %d tick %d" % (q, k)
            for a, act in enumerate(H.ACTIONS):
                assert (act in paths) == (int(g["path_len"][q, k, a]) > 0), ctx + " paths " + act
                t_want = int(g["traj_len"][q, k, a])
                assert (act in traj) == (t_want > 0), ctx + " trajectories " + act
                if t_want:
                    H.assert_close("traj[%s]" % act, traj[act][0], g["traj"][q, k, a, :t_want], EXPORT_COLS, ctx)
                    compared += 1
            if int(g["em_len"][q, k]):
                H.assert_close("traj[emergency]", traj["emergency"][0], g["em_traj"][q, k, :int(g["em_len"][q, k])],
                               EXPORT_COLS, ctx, w_rel=H.W_REL_BRAKE)
    assert compared > 20


def _first_tick(lat, sc, axm, w, windows):
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    pl = BatchPlanner(lat, online=dict(filt_window_width=w), device="cuda:0")
    pl.set_subbatches(windows)
    pl.set_vel_params(ax_max_machines=axm, incl_emerg_traj=True, **VEL)
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.tick()
    f = pl.fetch("status", "path_len", "traj_len", "traj_row", "traj", "s_vx_ax", "em_info")
    ok = f["traj_row"] >= 0
    ne = f["traj"].shape[1]
    rows = np.zeros(ok.shape + (ne, 7), dtype=np.float32)
    rows[ok] = f["traj"][f["traj_row"][ok]]
    rows[np.arange(ne)[None, None, :] >= f["traj_len"][..., None]] = 0.0   # behind the export cut: unspecified
    em = np.zeros((ok.shape[1], ne, 7), dtype=np.float32)
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
    pl, r5 = _first_tick(lat, sc, axm, w, 4)
    for windows in (1, 5):
        other = _first_tick(lat, sc, axm, w, windows)[1]
        for k in r5:
            assert np.array_equal(r5[k], other[k]), "'%s' differs between 4 and %d scenario windows" % (k, windows)
    r1 = _first_tick(lat, sc, axm, 1, 4)[1]
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

    rng = np.random.default_rng(4243)
    pick = np.sort(rng.choice(B, size=48, replace=False))
    recs = pl.records(indices=pick.tolist())
    orc = OracleLTPL(lat, online=dict(filt_window_width=w))
    vk = dict(ax_max_machines=axm, incl_emerg_traj=True, **VEL)
    fails = []
    for rec, b in zip(recs, pick):
        want = orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(int(b)), vk)
        ctx = "l216 w5 scenario %d of %d" % (b, B)
        try:
            em_g = em_w = None
            if not rec["out_of_track"]:                   # records() lists 'emergency' with the exported rows only
                em_g = rec["traj"].pop("emergency", None)
                rec["ids"].pop("emergency", None)
            if not want["out_of_track"]:
                em_w = want["traj"].pop("emergency", None)
                want["traj_full"].pop("emergency", None)
                want["ids"].pop("emergency", None)
            H.compare_records(rec, want, ctx=ctx)
            assert (em_g is None) == (em_w is None), ctx + " emergency presence"
            if em_w is not None:
                H.assert_close("traj[emergency]", em_g[0], em_w[0], EXPORT_COLS, ctx, w_rel=H.W_REL_BRAKE)
        except AssertionError as e:
            fails.append(str(e).split("\n")[0][:300])
    assert not fails, "%d/48 sampled scenarios differ from the oracle:\n%s" % (len(fails), "\n".join(fails[:8]))
