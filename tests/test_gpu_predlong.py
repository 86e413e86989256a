"""Objects with long 'prediction' arrays on the device: k_plan visits a scenario's obstacle discs in chunks of 32, so a
scenario may hold any number of them.  Against golden vectors of the unmodified reference (tests/golden/ticks_predlong.npz),
the oracle on seeded batches with exact disc counts around the chunk size, the stateful oracle in a closed loop, and
against the device itself (results of a scenario do not depend on the batch's prediction capacity, sub-batch,
permutation or scenario windows)."""
import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H

pytestmark = pytest.mark.gpu


def _vk():
    return dict(D.VEL, ax_max_machines=H.golden("ticks_predlong.npz")["ax_max_machines"])


def _subset(name):
    return H._Sub(H.golden("ticks_predlong.npz"), name, upcast=True)


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
    sub = _subset(name)
    n = sub["sc_pos"].shape[0]
    sc = ScenarioBatch.from_object_lists(sub["sc_pos"], sub["sc_heading"], sub["sc_vel"],
                                         [H.object_list(sub, b) for b in range(n)], k_max=5)
    assert sc.pred is not None and np.array_equal(sc.n_pred, sub["sc_n_pred"]) and sc.pred.shape[2] <= 80
    pl = D.planner(H.lattice_for(str(sub["lattice"])), windows, **_vk())
    D.first_tick(pl, sc)
    recs = pl.records()
    for b in range(n):
        assert not (recs[b]["flags"] & capi.SC_CAPACITY), "scenario %d (%d discs) flagged" % (b, int(sub["n_disc"][b]))
        H.compare_first_tick(recs[b], sub, b, ctx="predlong gpu " + name, exported=True)


def test_facade_plans_a_60_point_prediction(tmp_path):
    """Graph_LTPL with one 60-point prediction per object no longer raises and returns the golden result."""
    sub = _subset("default")
    ltpl = D.facade(tmp_path)
    done = 0
    for b in range(sub["sc_pos"].shape[0]):
        if bool(sub["out_of_track"][b]) or int(sub["sc_n_pred"][b].max()) < 60 or int(sub["n_disc"][b]) <= 32:
            continue
        ol = H.object_list(sub, b)
        assert ltpl.set_startpos(pos_est=sub["sc_pos"][b], heading_est=sub["sc_heading"][b],
                                 vel_est=sub["sc_vel"][b]) is False
        paths = ltpl.calc_paths(prev_action_id="straight", object_list=ol)
        traj, _, _ = ltpl.calc_vel_profile(pos_est=sub["sc_pos"][b], vel_est=float(sub["sc_vel"][b]), **_vk())
        for a, act in enumerate(H.ACTIONS):
            assert (act in paths) == (int(sub["path_len"][b, a]) > 0), "facade scenario %d %s" % (b, act)
            t_want = int(sub["traj_len"][b, a])
            assert (act in traj) == (t_want > 0), "facade scenario %d trajectory %s" % (b, act)
            if t_want:
                n_rows = min(t_want, H.N_EXPORT)
                assert traj[act][0].shape[0] == n_rows, "facade scenario %d rows %s" % (b, act)
                H.assert_close("traj[%s]" % act, traj[act][0][:, H.VA_IDX], sub["traj"][b, a, :n_rows], H.VA_COLS,
                               "facade scenario %d" % b)
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
    pl = D.planner(lat, 3, **_vk())
    D.first_tick(pl, sc)
    recs = pl.records()
    orc = OracleLTPL(lat)
    vk = _vk()
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
    pl = D.planner(lat, 4, **_vk())
    D.first_tick(pl, sc)
    assert pl.dims.k_pred == 0
    plain = D.tick_snapshot(pl, emergency=False)
    npts = np.full((sc.size, 3), -1)
    npts[1::2, :] = 80                                         # odd scenarios: 80-point arrays (> 32 discs)
    sc2 = _cv_pred(sc.subset(np.arange(sc.size)), npts)
    pl2 = D.planner(lat, 4, **_vk())
    D.first_tick(pl2, sc2)
    assert pl2.dims.k_pred == 80
    even = np.arange(0, sc.size, 2)
    plain, long_ = D.take(plain, even), D.take(D.tick_snapshot(pl2, emergency=False), even)
    for k in plain:
        assert np.array_equal(plain[k], long_[k]), k


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
    pl = D.assert_batch_invariance(lat, sc, np.random.default_rng(9503).permutation(B), np.arange(1000, 1700), **_vk())
    pick = np.sort(np.random.default_rng(9504).choice(B, size=48, replace=False))
    D.assert_sample_matches_oracle(pl, OracleLTPL(lat), sc, pick, _vk(), "l216 50-point")


def test_closed_loop_long_predictions_match_session_oracle():
    """64 sequences x 8 stateful ticks on the default lattice; moving opponents carry a 40-80 point prediction each tick;
    the stateful oracle replays the same inputs."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    lat = H.lattice_for("default")
    n_seq, n_ticks = 64, 8
    sc0 = make_scenarios(Track(H.TRACK_CSV), n_seq, seed=9601, n_obj_min=1, n_obj_max=3)
    rng = np.random.default_rng(9602)
    npts = rng.integers(40, 81, size=(n_seq, sc0.obj.shape[1]))
    prefer = (("right", "left", "straight", "follow"), ("follow", "straight", "left", "right"))
    n = D.closed_loop_vs_session(D.planner(lat, 3, stateful=True, **_vk()), lat, sc0, rng, _vk(), prefer,
                                 capi.SC_STATE_FALLBACK | capi.SC_BRAKE_PREFIX,
                                 batch=lambda sc: _cv_pred(sc, npts, drift=0.6), n_ticks=n_ticks)
    assert n["capacity"] == 0, "%d compared ticks flagged SC_CAPACITY" % n["capacity"]
    assert n["ticks"] > n_seq * n_ticks // 2, n
