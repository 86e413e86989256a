"""Long object lists on the device: k_plan's object stage visits the object slots in chunks of 32 and keeps one record
per on-track object in shared memory, so a scenario may list any number of objects up to that memory's bound.  Against
golden vectors of the unmodified reference (tests/golden/ticks_manyobj.npz), the oracle on seeded batches with exact
object counts around the chunk size, the stateful oracle in a closed loop, and against the device itself (results do not
depend on the batch's object capacity, sub-batch, permutation or scenario windows)."""
import ctypes as C

import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H

pytestmark = pytest.mark.gpu


def vel_kwargs():
    return dict(D.VEL, ax_max_machines=H.golden("ticks_manyobj.npz")["ax_max_machines"])


def _field(tag, B, n_obj, seed, off_frac=0.4, pred_frac=0.0, k_max=None, ahead=(20.0, 500.0)):
    """B scenarios with n_obj[b] objects (an int: the same for all) 20-500 m ahead: a share off_frac of them 3-15 m
    beyond the left or right track bound, interleaved with the others; a share pred_frac carries a 'prediction' array
    of 0-12 points."""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    track = Track(H.track_csv_for(tag))
    n_obj = np.broadcast_to(np.asarray(n_obj, dtype=np.int32), (B,)).copy()
    K = int(n_obj.max() if k_max is None else k_max)
    sc = make_scenarios(track, B, seed=seed, n_obj_min=0, n_obj_max=0, k_max=1)
    s_e = np.random.default_rng(seed).uniform(0.0, track.length, size=B)   # make_scenarios' first draw: the ego's s
    rng = np.random.default_rng(seed + 1)
    obj = np.zeros((B, K, 5))
    for j in range(int(n_obj.max())):
        ref, nv, wl, wr, psi, vrl = track.frame(s_e + rng.uniform(ahead[0], ahead[1], size=B))
        d_in = -(wl - 1.4) + rng.uniform(0.0, 1.0, size=B) * ((wr - 1.4) + (wl - 1.4))
        d_out = np.where(rng.random(B) < 0.5, -(wl + rng.uniform(3.0, 15.0, size=B)), wr + rng.uniform(3.0, 15.0, size=B))
        d = np.where(rng.random(B) < off_frac, d_out, d_in)
        obj[:, j, 0:2] = ref + nv * d[:, None]
        obj[:, j, 2] = psi
        obj[:, j, 3] = rng.uniform(0.0, 0.5, size=B) * vrl
        obj[:, j, 4] = 5.0
    obj[np.arange(K)[None, :] >= n_obj[:, None]] = 0.0
    sc.n_obj, sc.obj = n_obj, obj
    if pred_frac > 0.0:
        npts = np.where(rng.random((B, K)) < pred_frac, rng.integers(0, 13, size=(B, K)), -1)
        npts[np.arange(K)[None, :] >= n_obj[:, None]] = -1
        sc.n_pred = npts.astype(np.int32)
        sc.pred = np.zeros((B, K, 12, 2))
        t = 0.1 * np.arange(1, 13)
        x, y, th, v = obj[..., 0:1], obj[..., 1:2], obj[..., 2:3], obj[..., 3:4]
        sc.pred[..., 0] = x - np.sin(th) * v * t + np.cos(th) * 0.5 * t
        sc.pred[..., 1] = y + np.cos(th) * v * t + np.sin(th) * 0.5 * t
    return sc


@pytest.mark.parametrize("name,windows", [("default", 1), ("default", 3), ("l216", 2), ("open", 4)])
def test_many_objects_match_reference_golden(name, windows):
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    sub = H._Sub(H.golden("ticks_manyobj.npz"), name, upcast=True)
    n = sub["sc_pos"].shape[0]
    sc = ScenarioBatch.from_object_lists(sub["sc_pos"], sub["sc_heading"], sub["sc_vel"],
                                         [H.object_list(sub, b) for b in range(n)])
    assert sc.obj.shape[1] > 32
    pl = D.planner(H.lattice_for(str(sub["lattice"])), windows, **vel_kwargs())
    D.first_tick(pl, sc)
    assert pl.dims.k_obj == sc.obj.shape[1]
    recs = pl.records()
    for b in range(n):
        assert not (recs[b]["flags"] & capi.SC_CAPACITY), "scenario %d flagged" % b
        H.compare_first_tick(recs[b], sub, b, ctx="manyobj gpu " + name, exported=True)


def test_facade_plans_a_40_entry_list(tmp_path):
    """Graph_LTPL with 40 entries: on-track and off-track 'physical' objects and non-'physical' entries, interleaved;
    the facade drops the non-'physical' ones on the host, the device the off-track ones."""
    from oracle.ltpl_oracle import OracleLTPL
    sc = _field("default", 6, 32, seed=7101, off_frac=0.4, pred_frac=0.3)
    ltpl = D.facade(tmp_path)
    orc = OracleLTPL(H.lattice_for("default"))
    vk = vel_kwargs()
    done = 0
    for b in range(sc.size):
        ol = sc.object_list(b)
        for i in range(8):   # 8 entries of other types between the objects
            ol.insert(4 * i + 1, {'id': 100 + i, 'type': 'static' if i % 2 else 'unknown', 'X': ol[0]['X'],
                                  'Y': ol[0]['Y'], 'theta': 0.0, 'v': 0.0, 'length': 50.0})
        assert len(ol) == 40
        want = orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], ol, vk)
        if want["out_of_track"]:
            continue
        assert ltpl.set_startpos(pos_est=sc.pos[b], heading_est=sc.heading[b], vel_est=sc.vel[b]) is False
        paths = ltpl.calc_paths(prev_action_id="straight", object_list=ol)
        traj, _, _ = ltpl.calc_vel_profile(pos_est=sc.pos[b], vel_est=float(sc.vel[b]), **vk)
        ctx = "facade scenario %d" % b
        assert sorted(paths) == sorted(want["paths"]), "%s: %s vs %s" % (ctx, sorted(paths), sorted(want["paths"]))
        assert sorted(traj) == sorted(want["traj"]), ctx + " trajectory set"
        for act in traj:
            if want["tie"].get(act):
                continue
            H.assert_close("traj[%s]" % act, traj[act][0], want["traj"][act][0][:115],
                           ("s", "x", "y", "psi", "kappa", "vx", "ax"), ctx)
        done += 1
    assert done >= 4


@pytest.mark.parametrize("zone,pred", [(False, False), (True, False), (False, True), (True, True)])
def test_exact_object_counts_match_oracle(zone, pred):
    """scenarios with exactly 16, 17, 30, 31, 32, 33, 64, 65 or 200 objects: one to seven chunks of the object stage; in
    half of them every object is on the track (30 / 31 vehicles end the first s-coordinate round), in the other half
    40 % are beyond the bounds; with a blocked zone on every other scenario (k_plan<1, ..>) and with prediction arrays."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from oracle.gen_golden import make_zone
    from oracle.ltpl_oracle import OracleLTPL
    lat = H.lattice_for("default")
    counts = (16, 17, 30, 31, 32, 33, 64, 65, 200)
    B = 2 * len(counts) * 2
    n_obj = np.array([counts[b % len(counts)] for b in range(B)])
    seed = 7201 + 2 * int(zone) + int(pred)
    sc_on = _field("default", B // 2, n_obj[:B // 2], seed, off_frac=0.0, pred_frac=0.3 if pred else 0.0, k_max=200)
    sc_mix = _field("default", B // 2, n_obj[B // 2:], seed + 50, off_frac=0.4, pred_frac=0.3 if pred else 0.0,
                    k_max=200)
    sc = sc_on.subset(np.arange(B // 2))
    for k in ("pos", "heading", "vel", "n_obj", "obj") + (("pred", "n_pred") if pred else ()):
        setattr(sc, k, np.concatenate((getattr(sc_on, k), getattr(sc_mix, k))))
    zones = None
    if zone:
        rng = np.random.default_rng(seed + 7)
        zones = [{"z%d" % b: make_zone(lat, rng, sc.pos[b])} if b % 2 == 0 else None for b in range(sc.size)]
        sc.set_zones(zones)
    pl = D.planner(lat, 3, **vel_kwargs())
    D.first_tick(pl, sc)
    assert pl.dims.k_obj == 200
    recs = pl.records()
    orc = OracleLTPL(lat)
    vk = vel_kwargs()
    n_closest = 0
    for b in range(sc.size):
        assert not (recs[b]["flags"] & capi.SC_CAPACITY), "scenario %d flagged" % b
        want = orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(b), vk,
                        blocked_zones=None if zones is None else zones[b])
        H.compare_records(recs[b], want, ctx="%d objects scenario %d" % (n_obj[b], b))
        n_closest += int(not want["out_of_track"] and want.get("closest_obj_index") is not None)
    assert n_closest > B // 2


def test_short_lists_ignore_the_object_capacity():
    """a scenario with <= 16 objects gives byte-identical results whether the batch's object capacity is 16 or 200 (the
    same scenarios, once alone and once beside scenarios with 200 objects)."""
    lat = H.lattice_for("default")
    sc = _field("default", 256, np.random.default_rng(7301).integers(0, 17, size=256), seed=7302, pred_frac=0.3,
                k_max=16)
    pl = D.planner(lat, 4, **vel_kwargs())
    D.first_tick(pl, sc)
    assert pl.dims.k_obj == 16
    plain = D.tick_snapshot(pl, emergency=False)
    big = _field("default", 256, 200, seed=7303, pred_frac=0.3)
    sc2 = sc.subset(np.arange(sc.size))
    K = 200
    sc2.obj = np.zeros((256, K, 5))
    sc2.obj[:, :16] = sc.obj
    sc2.n_pred = np.full((256, K), -1, dtype=np.int32)
    sc2.n_pred[:, :16] = sc.n_pred
    sc2.pred = np.zeros((256, K, 12, 2))
    sc2.pred[:, :16] = sc.pred
    odd = np.arange(1, 256, 2)
    for k in ("pos", "heading", "vel", "n_obj", "obj", "n_pred", "pred"):
        getattr(sc2, k)[odd] = getattr(big, k)[odd]
    pl2 = D.planner(lat, 4, **vel_kwargs())
    D.first_tick(pl2, sc2)
    assert pl2.dims.k_obj == 200
    even = np.arange(0, 256, 2)
    plain, wide = D.take(plain, even), D.take(D.tick_snapshot(pl2, emergency=False), even)
    for k in plain:
        assert np.array_equal(plain[k], wide[k]), k


def test_full_batch_many_objects_invariance():
    """10 000 scenarios on the ~200 x 11 lattice with 48 objects each (about 60 % on the track): results do not depend on
    the scenario windows, on the sub-batch or on the order of the batch; a sample agrees with the oracle."""
    from oracle.ltpl_oracle import OracleLTPL
    lat = H.lattice_for("l216")
    B = 10000
    sc = _field("l216", B, 48, seed=7401, pred_frac=0.2)
    pl = D.assert_batch_invariance(lat, sc, np.random.default_rng(7402).permutation(B), np.arange(3000, 3700),
                                   **vel_kwargs())
    pick = np.sort(np.random.default_rng(7403).choice(B, size=48, replace=False))
    D.assert_sample_matches_oracle(pl, OracleLTPL(lat), sc, pick, vel_kwargs(), "l216 48-object")


def test_object_count_beyond_the_bound_is_refused():
    """dims.k_obj above ltpl_max_objects: every tick call returns an error naming the cause and launches nothing; the
    next tick with a valid k_obj on the same handle plans as usual; the planner refuses such a batch with ValueError."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from oracle.ltpl_oracle import OracleLTPL
    lat = H.lattice_for("default")
    pl = D.planner(lat, 2, **vel_kwargs())
    sc = _field("default", 32, 20, seed=7501)
    D.first_tick(pl, sc)
    before = D.tick_snapshot(pl, emergency=False)
    bound = pl.max_objects
    assert bound == int(pl.lib.ltpl_max_objects(C.byref(pl.header), int(pl.dims.h_max))) and bound >= 500
    k_keep = pl.dims.k_obj
    pl.dims.k_obj = bound + 1
    n0 = pl.launch_count()
    for fn in ("ltpl_calc_paths_batch", "ltpl_tick_batch", "ltpl_calc_vel_profile_batch", "ltpl_set_startpos_batch"):
        rc = getattr(pl.lib, fn)(pl.handle, C.byref(pl.params), C.byref(pl.dims), C.byref(pl.buf), pl.stream)
        assert rc != 0, fn
        assert b"too many object slots" in pl.lib.ltpl_last_error(), pl.lib.ltpl_last_error()
    assert pl.launch_count() == n0
    pl.dims.k_obj = k_keep
    D.first_tick(pl, sc)
    assert all(np.array_equal(before[k], v) for k, v in D.tick_snapshot(pl, emergency=False).items())
    recs = pl.records(indices=list(range(8)))
    orc = OracleLTPL(lat)
    for b, rec in enumerate(recs):
        H.compare_records(rec, orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(b), vel_kwargs()),
                          ctx="after the refusal, scenario %d" % b)
    wide = _field("default", 32, bound + 1, seed=7502, ahead=(20.0, 30.0))
    with pytest.raises(ValueError, match="at most %d" % bound):
        pl.stage_scenarios(wide)
    assert pl.dims.k_obj == k_keep and capi.ABI_VERSION == pl.lib.ltpl_version()


def test_closed_loop_many_objects_match_session_oracle():
    """64 sequences x 8 stateful ticks on the default lattice with 20-40 moving objects each (on and off the track, a
    quarter with prediction arrays); the stateful oracle replays the same inputs."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    lat = H.lattice_for("default")
    n_seq, n_ticks = 64, 8
    rng = np.random.default_rng(7602)
    sc0 = _field("default", n_seq, rng.integers(20, 41, size=n_seq), seed=7601, pred_frac=0.25, k_max=40)
    prefer = (("right", "left", "straight", "follow"), ("follow", "straight", "left", "right"))
    n = D.closed_loop_vs_session(D.planner(lat, 3, stateful=True, **vel_kwargs()), lat, sc0, rng, vel_kwargs(), prefer,
                                 capi.SC_STATE_FALLBACK | capi.SC_BRAKE_PREFIX, n_ticks=n_ticks)
    assert n["capacity"] == 0, "%d compared ticks flagged SC_CAPACITY" % n["capacity"]
    assert n["ticks"] > n_seq * n_ticks // 2, n
