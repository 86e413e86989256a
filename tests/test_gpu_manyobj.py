"""Long object lists on the device: k_plan's object stage visits the object slots in chunks of 32 and keeps one record
per on-track object in shared memory, so a scenario may list any number of objects up to that memory's bound.  Against
golden vectors of the unmodified reference (tests/golden/ticks_manyobj.npz), the oracle on seeded batches with exact
object counts around the chunk size, the stateful oracle in a closed loop, and against the device itself (results do not
depend on the batch's object capacity, sub-batch, permutation or scenario windows)."""
import ctypes as C

import numpy as np
import pytest

from tests import helpers as H
from tests.manyobj_golden import VEL, compare_predlong_record, subset, vel_kwargs

pytestmark = pytest.mark.gpu


def _planner(lat, windows=4, stateful=False):
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    pl = BatchPlanner(lat, device="cuda:0", stateful=stateful)
    pl.set_subbatches(windows)
    pl.set_vel_params(ax_max_machines=vel_kwargs()["ax_max_machines"], **VEL)
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
    sub = subset(name)
    n = sub["sc_pos"].shape[0]
    sc = ScenarioBatch.from_object_lists(sub["sc_pos"], sub["sc_heading"], sub["sc_vel"],
                                         [H.object_list(sub, b) for b in range(n)])
    assert sc.obj.shape[1] > 32
    pl = _planner(H.lattice_for(str(sub["lattice"])), windows)
    _first_tick(pl, sc)
    assert pl.dims.k_obj == sc.obj.shape[1]
    recs = pl.records()
    for b in range(n):
        assert not (recs[b]["flags"] & capi.SC_CAPACITY), "scenario %d flagged" % b
        compare_predlong_record(recs[b], sub, b, ctx="manyobj gpu " + name, exported=True)


def test_facade_plans_a_40_entry_list(tmp_path):
    """Graph_LTPL with 40 entries: on-track and off-track 'physical' objects and non-'physical' entries, interleaved;
    the facade drops the non-'physical' ones on the host, the device the off-track ones."""
    from graphbasedlocaltrajectoryplanner_b200.Graph_LTPL import Graph_LTPL
    from oracle.ltpl_oracle import OracleLTPL
    sc = _field("default", 6, 32, seed=7101, off_frac=0.4, pred_frac=0.3)
    pd = {'globtraj_input_path': H.TRACK_CSV, 'graph_store_path': str(tmp_path / "lattice.npz"),
          'ltpl_offline_param_path': H.OFFLINE_INI, 'ltpl_online_param_path': H.ONLINE_INI}
    ltpl = Graph_LTPL(path_dict=pd, visual_mode=False, log_to_file=False, device="cuda:0")
    ltpl.graph_init()
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
    pl = _planner(lat, 3)
    _first_tick(pl, sc)
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
    pl = _planner(lat, 4)
    _first_tick(pl, sc)
    assert pl.dims.k_obj == 16
    plain = _snapshot(pl)
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
    pl2 = _planner(lat, 4)
    _first_tick(pl2, sc2)
    assert pl2.dims.k_obj == 200
    wide = _snapshot(pl2)
    even = np.arange(0, 256, 2)
    for k in plain:
        a, b = plain[k], wide[k]
        if a.ndim >= 2 and a.shape[0] == 3 and a.shape[1] == sc.size:   # [NSLOT][B] ...
            assert np.array_equal(a[:, even], b[:, even]), k
        else:
            assert np.array_equal(a[even], b[even]), k


def test_full_batch_many_objects_invariance():
    """10 000 scenarios on the ~200 x 11 lattice with 48 objects each (about 60 % on the track): results do not depend on
    the scenario windows, on the sub-batch or on the order of the batch; a sample agrees with the oracle."""
    from oracle.ltpl_oracle import OracleLTPL
    lat = H.lattice_for("l216")
    B = 10000
    sc = _field("l216", B, 48, seed=7401, pred_frac=0.2)
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
    perm = np.random.default_rng(7402).permutation(B)
    pp = _planner(lat, 4)
    _first_tick(pp, sc.subset(perm))
    got = _snapshot(pp)
    inv = np.argsort(perm)
    for k in ref:
        g = got[k]
        g = g[:, inv] if (g.ndim >= 2 and g.shape[0] == 3 and g.shape[1] == B) else g[inv]
        assert np.array_equal(ref[k], g), "'%s' depends on the order of the batch" % k
    part = np.arange(3000, 3700)
    ps_ = _planner(lat, 2)
    _first_tick(ps_, sc.subset(part))
    got, want = _snapshot(ps_), cols(ref, part)
    for k in want:
        assert np.array_equal(want[k], got[k]), "'%s' differs in a sub-batch" % k
    pick = np.sort(np.random.default_rng(7403).choice(B, size=48, replace=False))
    recs = pl.records(indices=pick.tolist())
    orc = OracleLTPL(lat)
    vk = vel_kwargs()
    fails = []
    for rec, b in zip(recs, pick):
        want = orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(int(b)), vk)
        try:
            H.compare_records(rec, want, ctx="l216 48-object scenario %d" % b)
        except AssertionError as e:
            fails.append(str(e).split("\n")[0][:300])
    assert not fails, "%d/48 sampled scenarios differ from the oracle:\n%s" % (len(fails), "\n".join(fails[:8]))


def test_object_count_beyond_the_bound_is_refused():
    """dims.k_obj above ltpl_max_objects: every tick call returns an error naming the cause and launches nothing; the
    next tick with a valid k_obj on the same handle plans as usual; the planner refuses such a batch with ValueError."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from oracle.ltpl_oracle import OracleLTPL
    lat = H.lattice_for("default")
    pl = _planner(lat, 2)
    sc = _field("default", 32, 20, seed=7501)
    _first_tick(pl, sc)
    before = _snapshot(pl)
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
    _first_tick(pl, sc)
    assert all(np.array_equal(before[k], v) for k, v in _snapshot(pl).items())
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
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    from oracle.gen_golden import advance_on_traj
    from oracle.ltpl_oracle import OracleLTPL
    from oracle.ltpl_session import OracleSession
    lat = H.lattice_for("default")
    n_seq, n_ticks = 64, 8
    rng = np.random.default_rng(7602)
    sc0 = _field("default", n_seq, rng.integers(20, 41, size=n_seq), seed=7601, pred_frac=0.25, k_max=40)
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
    vel = vel_kwargs()
    fails, ticks_ok = [], 0
    for k in range(n_ticks):
        dts = rng.uniform(0.04, 0.16, size=n_seq)
        tcs = np.zeros(n_seq)
        for q in range(n_seq):
            dt = float(dts[q])
            clks[q].t += dt
            m = int(sc0.n_obj[q])
            objs[q, :m, 0] -= np.sin(objs[q, :m, 2]) * objs[q, :m, 3] * dt
            objs[q, :m, 1] += np.cos(objs[q, :m, 2]) * objs[q, :m, 3] * dt
            if k > 0:
                if last_traj[q] is not None:
                    pos_est[q], vel_est[q] = advance_on_traj(last_traj[q], dt)
                if len(cbuf[q]) >= 5:
                    cbuf[q].pop(0)
                cbuf[q].append(dt)
                tcs[q] = min(float(np.sum(cbuf[q]) / len(cbuf[q])) * 2.0, 0.5)
        sc = ScenarioBatch(pos_est.copy(), sc0.heading.copy(), sc0.vel.copy(), sc0.n_obj.copy(), objs.copy(),
                           pred=sc0.pred, n_pred=sc0.n_pred)
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
