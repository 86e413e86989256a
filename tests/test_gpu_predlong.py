"""Objects with long 'prediction' arrays on the device: k_plan visits a scenario's obstacle discs in chunks of 32, so a
scenario may hold any number of them.  Against golden vectors of the unmodified reference (tests/golden/ticks_predlong.npz),
the oracle on seeded batches with exact disc counts around the chunk size, the stateful oracle in a closed loop, and
against the device itself (results of a scenario do not depend on the batch's prediction capacity, sub-batch,
permutation or scenario windows)."""
import numpy as np
import pytest

from tests import helpers as H
from tests.predlong_golden import IDX, compare_predlong_record, subset

pytestmark = pytest.mark.gpu

VEL = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)


def _axm():
    return H.golden("ticks_predlong.npz")["ax_max_machines"]


def _planner(lat, windows=4, stateful=False):
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    pl = BatchPlanner(lat, device="cuda:0", stateful=stateful)
    pl.set_subbatches(windows)
    pl.set_vel_params(ax_max_machines=_axm(), **VEL)
    return pl


def _first_tick(pl, sc):
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.tick()


def _snapshot(pl):
    """H.tick_snapshot without the emergency entries: these ticks do not compute the emergency trajectory."""
    snap = H.tick_snapshot(pl)
    del snap["em_len"], snap["em_rows"]
    return snap


def _cv_pred(sc, n_points, dt=0.1, drift=0.0, rng=None):
    """n_points[b, k] constant-velocity points (plus a lateral drift) for object k of scenario b; -1: no key."""
    kp = max(1, int(np.max(n_points)))
    sc.pred = np.zeros(sc.obj.shape[:2] + (kp, 2))
    sc.n_pred = np.asarray(n_points, dtype=np.int32).copy()
    for b in range(sc.size):
        for k in range(int(sc.n_obj[b])):
            m = int(sc.n_pred[b, k])
            x, y, th, v, _ = sc.obj[b, k]
            dr = drift if rng is None else rng.uniform(-drift, drift)
            t = dt * np.arange(1, max(m, 0) + 1)
            sc.pred[b, k, :len(t), 0] = x - np.sin(th) * v * t + np.cos(th) * dr * t
            sc.pred[b, k, :len(t), 1] = y + np.cos(th) * v * t + np.sin(th) * dr * t
    return sc


@pytest.mark.parametrize("name,windows", [("default", 1), ("default", 3), ("l216", 2), ("open", 4)])
def test_long_predictions_match_reference_golden(name, windows):
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    sub = subset(name)
    n = sub["sc_pos"].shape[0]
    sc = ScenarioBatch.from_object_lists(sub["sc_pos"], sub["sc_heading"], sub["sc_vel"],
                                         [H.object_list(sub, b) for b in range(n)], k_max=5)
    assert sc.pred is not None and np.array_equal(sc.n_pred, sub["sc_n_pred"]) and sc.pred.shape[2] <= 80
    pl = _planner(H.lattice_for(str(sub["lattice"])), windows)
    _first_tick(pl, sc)
    recs = pl.records()
    for b in range(n):
        assert not (recs[b]["flags"] & capi.SC_CAPACITY), "scenario %d (%d discs) flagged" % (b, int(sub["n_disc"][b]))
        compare_predlong_record(recs[b], sub, b, ctx="predlong gpu " + name, exported=True)


def test_facade_plans_a_60_point_prediction(tmp_path):
    """Graph_LTPL with one 60-point prediction per object no longer raises and returns the golden result."""
    from graphbasedlocaltrajectoryplanner_b200.Graph_LTPL import Graph_LTPL
    sub = subset("default")
    pd = {'globtraj_input_path': H.TRACK_CSV, 'graph_store_path': str(tmp_path / "lattice.npz"),
          'ltpl_offline_param_path': H.OFFLINE_INI, 'ltpl_online_param_path': H.ONLINE_INI}
    ltpl = Graph_LTPL(path_dict=pd, visual_mode=False, log_to_file=False, device="cuda:0")
    ltpl.graph_init()
    done = 0
    for b in range(sub["sc_pos"].shape[0]):
        if bool(sub["out_of_track"][b]) or int(sub["sc_n_pred"][b].max()) < 60 or int(sub["n_disc"][b]) <= 32:
            continue
        ol = H.object_list(sub, b)
        assert ltpl.set_startpos(pos_est=sub["sc_pos"][b], heading_est=sub["sc_heading"][b],
                                 vel_est=sub["sc_vel"][b]) is False
        paths = ltpl.calc_paths(prev_action_id="straight", object_list=ol)
        traj, _, _ = ltpl.calc_vel_profile(pos_est=sub["sc_pos"][b], vel_est=float(sub["sc_vel"][b]),
                                           ax_max_machines=_axm(), **VEL)
        for a, act in enumerate(H.ACTIONS):
            assert (act in paths) == (int(sub["path_len"][b, a]) > 0), "facade scenario %d %s" % (b, act)
            t_want = int(sub["traj_len"][b, a])
            assert (act in traj) == (t_want > 0), "facade scenario %d trajectory %s" % (b, act)
            if t_want:
                assert traj[act][0].shape[0] == min(t_want, 115), "facade scenario %d rows %s" % (b, act)
                H.assert_close("traj[%s]" % act, traj[act][0][:, IDX], sub["traj"][b, a, :min(t_want, 115)],
                               ("vx", "ax"), "facade scenario %d" % b)
        done += 1
        if done == 4:
            break
    assert done == 4


@pytest.mark.parametrize("zone", [False, True])
def test_exact_disc_counts_match_oracle(zone):
    """every scenario holds exactly 31, 32, 33, 64, 65 or 200 discs (if all its objects are on the track): one, two or
    seven chunks, a vehicle cut by a chunk boundary; with a blocked zone on every other scenario: k_plan<1, ..>."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    from oracle.gen_golden import make_zone
    from oracle.ltpl_oracle import OracleLTPL
    lat = H.lattice_for("default")
    counts = (31, 32, 33, 64, 65, 200)
    sc = make_scenarios(Track(H.TRACK_CSV), 96, seed=9301 + int(zone), n_obj_min=3, n_obj_max=3)
    npts = np.full((sc.size, 3), -1)
    for b in range(sc.size):
        total = counts[b % len(counts)]
        # three vehicles: position + built-in point, then two arrays sharing the rest (the last vehicle's discs cross
        # disc 32 for 33, 64 and 65 discs)
        rest = total - 4
        npts[b] = (-1, rest // 2, rest - rest // 2)
        assert 2 + (1 + npts[b, 1]) + (1 + npts[b, 2]) == total
    sc = _cv_pred(sc, npts, drift=0.8, rng=np.random.default_rng(9303))
    zones = None
    if zone:
        rng = np.random.default_rng(9304)
        zones = [{"z%d" % b: make_zone(lat, rng, sc.pos[b])} if b % 2 == 0 else None for b in range(sc.size)]
        sc.set_zones(zones)
    pl = _planner(lat, 3)
    _first_tick(pl, sc)
    recs = pl.records()
    orc = OracleLTPL(lat)
    vk = dict(VEL, ax_max_machines=_axm())
    n_obj_closest = 0
    for b in range(sc.size):
        assert not (recs[b]["flags"] & capi.SC_CAPACITY), "scenario %d flagged" % b
        want = orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(b), vk,
                        blocked_zones=None if zones is None else zones[b])
        H.compare_records(recs[b], want, ctx="%d discs scenario %d" % (counts[b % len(counts)], b))
        n_obj_closest += int(want.get("closest_obj_index") is not None) if not want["out_of_track"] else 0
    assert n_obj_closest > 10


def test_short_scenarios_ignore_the_prediction_capacity():
    """a scenario with <= 32 discs gives byte-identical results whether the batch's prediction arrays hold 0 or 80 points
    (the same scenarios, once without any 'prediction' key and once beside scenarios with 80-point arrays)."""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    lat = H.lattice_for("default")
    sc = make_scenarios(Track(H.TRACK_CSV), 256, seed=9401, n_obj_min=1, n_obj_max=3)
    pl = _planner(lat, 4)
    _first_tick(pl, sc)
    assert pl.dims.k_pred == 0
    plain = _snapshot(pl)
    npts = np.full((sc.size, 3), -1)
    npts[1::2, :] = 80                                         # odd scenarios: 80-point arrays (> 32 discs)
    sc2 = _cv_pred(sc.subset(np.arange(sc.size)), npts)
    pl2 = _planner(lat, 4)
    _first_tick(pl2, sc2)
    assert pl2.dims.k_pred == 80
    long_ = _snapshot(pl2)
    even = np.arange(0, sc.size, 2)
    for k in plain:
        a, b = plain[k], long_[k]
        if a.ndim >= 2 and a.shape[0] == 3 and a.shape[1] == sc.size:   # [NSLOT][B] ...
            assert np.array_equal(a[:, even], b[:, even]), k
        else:
            assert np.array_equal(a[even], b[even]), k


def test_full_batch_long_predictions_invariance():
    """10 000 scenarios on the ~200 x 11 lattice, 3 objects x 50 points each (151 discs if all are on the track): results
    do not depend on the scenario windows, on the sub-batch or on the order of the batch; a sample agrees with the
    oracle."""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    from oracle.ltpl_oracle import OracleLTPL
    lat = H.lattice_for("l216")
    B = 10000
    sc = make_scenarios(Track(H.TRACK_CSV), B, seed=9501, n_obj_min=3, n_obj_max=3)
    sc = _cv_pred(sc, np.full((B, 3), 50), drift=1.0, rng=np.random.default_rng(9502))
    pl = _planner(lat, 4)
    _first_tick(pl, sc)
    ref = _snapshot(pl)

    def cols(snap, idx):   # scenario-major view of a snapshot restricted to scenarios idx
        return {k: (v[:, idx] if (v.ndim >= 2 and v.shape[0] == 3 and v.shape[1] == B) else v[idx]) for k, v in snap.items()}

    for windows in (1, 3):
        pw = _planner(lat, windows)
        _first_tick(pw, sc)
        got = _snapshot(pw)
        for k in ref:
            assert np.array_equal(ref[k], got[k]), "'%s' differs between 4 and %d scenario windows" % (k, windows)
    perm = np.random.default_rng(9503).permutation(B)
    pp = _planner(lat, 4)
    _first_tick(pp, sc.subset(perm))
    got = _snapshot(pp)
    inv = np.argsort(perm)
    for k in ref:
        g = got[k]
        g = g[:, inv] if (g.ndim >= 2 and g.shape[0] == 3 and g.shape[1] == B) else g[inv]
        assert np.array_equal(ref[k], g), "'%s' depends on the order of the batch" % k
    part = np.arange(1000, 1700)
    ps_ = _planner(lat, 2)
    _first_tick(ps_, sc.subset(part))
    got, want = _snapshot(ps_), cols(ref, part)
    for k in want:
        assert np.array_equal(want[k], got[k]), "'%s' differs in a sub-batch" % k
    pick = np.sort(np.random.default_rng(9504).choice(B, size=48, replace=False))
    recs = pl.records(indices=pick.tolist())
    orc = OracleLTPL(lat)
    vk = dict(VEL, ax_max_machines=_axm())
    fails = []
    for rec, b in zip(recs, pick):
        want = orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(int(b)), vk)
        try:
            H.compare_records(rec, want, ctx="l216 50-point scenario %d" % b)
        except AssertionError as e:
            fails.append(str(e).split("\n")[0][:300])
    assert not fails, "%d/48 sampled scenarios differ from the oracle:\n%s" % (len(fails), "\n".join(fails[:8]))


def test_closed_loop_long_predictions_match_session_oracle():
    """64 sequences x 8 stateful ticks on the default lattice; moving opponents carry a 40-80 point prediction each tick;
    the stateful oracle replays the same inputs."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch, Track, make_scenarios
    from oracle.gen_golden import advance_on_traj
    from oracle.ltpl_oracle import OracleLTPL
    from oracle.ltpl_session import OracleSession
    lat = H.lattice_for("default")
    n_seq, n_ticks = 64, 8
    sc0 = make_scenarios(Track(H.TRACK_CSV), n_seq, seed=9601, n_obj_min=1, n_obj_max=3)
    rng = np.random.default_rng(9602)
    npts = rng.integers(40, 81, size=(n_seq, sc0.obj.shape[1]))
    prefer = (("right", "left", "straight", "follow"), ("follow", "straight", "left", "right"))
    pl = _planner(lat, 3, stateful=True)

    class Clk(object):
        def __init__(self):
            self.t = 50.0

        def __call__(self):
            return self.t
    clks = [Clk() for _ in range(n_seq)]
    ses = [OracleSession(OracleLTPL(lat), clock=clks[q]) for q in range(n_seq)]
    objs = sc0.obj.copy()
    pos_est, vel_est = sc0.pos.copy(), sc0.vel.copy()
    sel = ["straight"] * n_seq
    cbuf = [[] for _ in range(n_seq)]
    alive = np.ones(n_seq, dtype=bool)
    last_traj = [None] * n_seq
    vel = dict(VEL, ax_max_machines=_axm())
    fails, ticks_ok = [], 0
    for k in range(n_ticks):
        dts = rng.uniform(0.04, 0.16, size=n_seq)
        tcs = np.zeros(n_seq)
        for q in range(n_seq):
            dt = float(dts[q])
            clks[q].t += dt
            for j in range(int(sc0.n_obj[q])):
                objs[q, j, 0] -= np.sin(objs[q, j, 2]) * objs[q, j, 3] * dt
                objs[q, j, 1] += np.cos(objs[q, j, 2]) * objs[q, j, 3] * dt
            if k > 0:
                if last_traj[q] is not None:
                    pos_est[q], vel_est[q] = advance_on_traj(last_traj[q], dt)
                if len(cbuf[q]) >= 5:
                    cbuf[q].pop(0)
                cbuf[q].append(dt)
                tcs[q] = min(float(np.sum(cbuf[q]) / len(cbuf[q])) * 2.0, 0.5)
        sc = ScenarioBatch(pos_est.copy(), sc0.heading.copy(), sc0.vel.copy(), sc0.n_obj.copy(), objs.copy())
        sc = _cv_pred(sc, npts, drift=0.6)
        if k == 0:
            pl.stage_scenarios(sc, vel_est=vel_est)
            pl.upload()
            pl.set_startpos()
            pl.tick()
        else:
            pl.next_tick(sc, sel_action=[H.ACTIONS.index(a) for a in sel], t_const=tcs, vel_est=vel_est)
        recs = pl.records()
        for q in range(n_seq):
            if not alive[q]:
                continue
            rec = recs[q]
            ctx = "sequence %d tick %d (sel %s)" % (q, k, sel[q])
            if rec["out_of_track"] or (rec["flags"] & (capi.SC_STATE_FALLBACK | capi.SC_BRAKE_PREFIX)):
                alive[q] = False
                continue
            try:
                if k == 0:
                    assert ses[q].set_startpos(sc.pos[q], sc.heading[q], sc.vel[q]) is False
                paths = ses[q].calc_paths(sel[q], sc.object_list(q))
                traj, _ = ses[q].calc_vel_profile(sc.pos[q], float(vel_est[q]), **vel)
            except Exception:   # noqa: BLE001  (e.g. the reference's own brake-prefix failure)
                alive[q] = False
                continue
            try:
                assert not (rec["flags"] & capi.SC_CAPACITY), ctx + " flagged"
                assert sorted(rec["paths"]) == sorted(paths), "%s: paths %s vs %s" % (ctx, sorted(rec["paths"]),
                                                                                   sorted(paths))
                for act in paths:
                    if ses[q].tie.get(act) or rec["tie"].get(act):
                        continue
                    nd = [[-1 if v is None else int(v) for v in p] for p in rec["nodes"][act][0]]
                    want = [[-1 if v is None else int(v) for v in p] for p in ses[q].m_nodes[act][0]] \
                        if act in ses[q].m_nodes else None
                    assert want is None or nd == want, "%s: nodes of %s" % (ctx, act)
                assert sorted(rec["traj"]) == sorted(traj), ctx + " trajectory set"
                for act in traj:
                    H.assert_close("traj[%s]" % act, rec["traj"][act][0], traj[act][0],
                                   ("s", "x", "y", "psi", "kappa", "vx", "ax"), ctx)
                ticks_ok += 1
            except AssertionError as e:
                fails.append(str(e).split("\n")[0][:400])
                alive[q] = False
                continue
            cand = [a for a in prefer[(q + k) % len(prefer)] if a in rec["traj"]]
            if not cand:
                alive[q] = False
                continue
            sel[q] = cand[0]
            last_traj[q] = rec["traj"][sel[q]][0]
    assert not fails, "%d sequences diverged (%d ticks matched):\n%s" % (len(fails), ticks_ok, "\n".join(fails[:8]))
    assert ticks_ok > n_seq * n_ticks // 2, ticks_ok
