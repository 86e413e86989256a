"""The planner's float64 decisions at their exact boundaries, on the device (tests/golden/ticks_knife_edge.npz,
tests/knife_edge.py): every flip pair, exact tie and equality of the fixture gives the reference's decision, and the
+-4 ulps around every flip pair give the oracle's; the in-track test of the ego (k_startpos) and of an object (k_plan's
chunk_objects, in the first and the second object chunk) agree on shared points.  First ticks on the default, "216 x 11"
and open lattices, with 1 and 4 scenario windows."""
import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H
from tests import knife_edge as K

pytestmark = pytest.mark.gpu

SETS = ("default", "l216", "open")
VEL = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)


def _axm():
    return H.golden("ticks_manyobj.npz")["ax_max_machines"]


def _batch(scen):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    pos = np.array([s[0] for s in scen], dtype=np.float64).reshape(-1, 2)
    hd = np.array([s[1] for s in scen], dtype=np.float64)
    return ScenarioBatch.from_object_lists(pos, hd, np.full(len(scen), 10.0), [s[2] for s in scen])


def _axis_window(pair, axis):
    """the flip pair and +-4 ulps around it along its axis"""
    return [K.at(pair[0], axis, v) for v in K.window(pair[0][axis], K.W + 1)[1:]]


@pytest.mark.parametrize("tag", SETS)
def test_ego_decisions_at_the_boundary(tag):
    """k_startpos: in-track test (F1), nearest node -> start node (F2, incl. exact ties: the lower global index), heading
    test (F3); fixture points against the reference's decisions, the windows against the oracle's."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    g = K.golden_set(tag)
    orc = K.oracle_for(tag)
    L = orc.lat.num_layers
    scen, want_flag, want_start, ctx = [], [], [], []

    def add(pos, heading, flag, start, what):
        scen.append((pos, heading, []))
        want_flag.append(flag)
        want_start.append(start)
        ctx.append(what)
    for k, pair in enumerate(g["f1_p"]):
        for j, p in enumerate(pair):
            add(p, 0.0, 0 if g["f1_in"][k, j] else capi.SC_OUT_OF_TRACK, None, "F1 pair %d" % k)
        for p in _axis_window(pair, int(g["f1_axis"][k])):
            add(p, 0.0, 0 if K.in_track(orc, p) else capi.SC_OUT_OF_TRACK, None, "F1 window %d" % k)
    start = lambda lay: (lay + 2) % (L - 1)   # noqa: E731
    for k, pair in enumerate(g["f2_p"]):
        for j, p in enumerate(pair):
            add(p, None, None, start(int(g["f2_layer"][k, j])), "F2 pair %d" % k)
        for p in _axis_window(pair, int(g["f2_axis"][k])):
            add(p, None, None, start(K.start_layer_of(orc, p)) if K.in_track(orc, p) else -1, "F2 window %d" % k)
    for k, p in enumerate(g["f2_tie_p"]):
        add(p, None, None, start(int(g["f2_tie_layer"][k])), "F2 tie %d" % k)
    for k in range(g["f3_h"].shape[0]):
        pos, psi = K.ego_pose(orc, int(g["f3_layer"][k]))
        for j, h in enumerate(g["f3_h"][k]):
            add(pos, h, 0 if g["f3_ok"][k, j] else capi.SC_HEADING_MISMATCH, None, "F3 pair %d" % k)
        for h in K.window(g["f3_h"][k, 0]):
            add(pos, h, 0 if K.heading_ok(orc, h, psi) else capi.SC_HEADING_MISMATCH, None, "F3 window %d" % k)
    scen = [(p, 0.0 if h is None else h, o) for p, h, o in scen]
    pl = D.planner(orc.lat, 1, ax_max_machines=_axm())
    pl.stage_scenarios(_batch(scen))
    pl.upload()
    pl.set_startpos()
    f = pl.fetch("sc_flags", "start_node")
    bad = []
    for b in range(len(scen)):
        # F1 sees the in-track bit (its egos keep heading 0), F3 the heading bit
        fl = int(f["sc_flags"][b]) & (capi.SC_OUT_OF_TRACK if ctx[b].startswith("F1") else capi.SC_HEADING_MISMATCH)
        if want_flag[b] is not None and fl != want_flag[b]:
            bad.append("%s: flags %d, want %d" % (ctx[b], fl, want_flag[b]))
        if want_start[b] is not None and int(f["start_node"][b, 0]) != want_start[b]:
            bad.append("%s: start layer %d, want %d" % (ctx[b], int(f["start_node"][b, 0]), want_start[b]))
    assert not bad, "%s: %d/%d decisions differ:\n%s" % (tag, len(bad), len(scen), "\n".join(bad[:12]))


def _object_scenarios(g, orc):
    """F1' (one object; the same behind 33 off-track objects), F4 (two objects), F7 (one object): scenario tuples and
    the expected closest object / cobj_start (None: not checked)"""
    scen, want_co, want_cs, ctx = [], [], [], []
    for k, pair in enumerate(g["f1_p"]):
        pts = list(zip(pair, g["f1_in"][k])) + [(p, K.in_track(orc, p)) for p in _axis_window(pair, int(g["f1_axis"][k]))]
        for j, (p, inside) in enumerate(pts):
            for chunk2 in ((False, True) if j < 2 else (False,)):
                s = K.f1_scenario(orc, p, chunk2)
                if s is not None:
                    scen.append(s)
                    want_co.append(0 if inside else -1)
                    want_cs.append(None)
                    ctx.append("F1' %s %d.%d" % ("chunk 2" if chunk2 else "", k, j))
    f4 = [(l, p, lay) for l, pair, lays in zip(g["f4_l"], g["f4_p"], g["f4_layer"]) for p, lay in zip(pair, lays)]
    f4 += [(l, p, lay) for l, p, lay in zip(g["f4_tie_l"], g["f4_tie_p"], g["f4_tie_layer"])]
    f4 += [(l, q, K.ref_layer(orc, q)) for l, pair in zip(g["f4_l"], g["f4_p"])
           for q in _axis_window(pair, int(np.argmax(np.abs(pair[1] - pair[0]))))]
    for k, (l, p, lay) in enumerate(f4):
        s = K.f4_scenario(orc, int(l[0]), int(l[1]), p)
        if s is not None:
            scen.append(s)
            want_co.append(int(lay == l[0]))
            want_cs.append(None)
            ctx.append("F4 %d (layers %d/%d)" % (k, l[0], l[1]))
    # several warp-scan fallback lanes in one disc chunk: B with a far point, and behind it objects C whose last points
    # are the other far points of the fixture (other layers, mostly outside the planning range)
    far = [p for pair, f in zip(g["f4_p"], g["f4_far"]) if f for p in pair] + \
        [p for p, f in zip(g["f4_tie_p"], g["f4_tie_far"]) if f]
    far_l = [l for l, f in zip(g["f4_l"], g["f4_far"]) if f for _ in range(2)] + \
        [l for l, f in zip(g["f4_tie_l"], g["f4_tie_far"]) if f]
    for k, (l, p) in enumerate(zip(far_l, far)):
        s = K.f4_scenario(orc, int(l[0]), int(l[1]), p)
        if s is None:
            continue
        r = orc.lat.refline[int(l[1])]
        s = (s[0], s[1], s[2] + [K.obj(r, pred=[q]) for j, q in enumerate(far) if j != k][:12])
        scen.append(s)
        want_co.append(K.paths_observable(orc, *s)[0])
        want_cs.append(None)
        ctx.append("F4 fallback lanes %d (layers %d/%d)" % (k, l[0], l[1]))
    for k, p in enumerate(g["f7_p"]):
        scen.append(K.f7_scenario(orc, p))
        want_co.append(0)
        want_cs.append(int(g["f7_start"][k]))
        ctx.append("F7 %d (gap %.1e)" % (k, g["f7_gap"][k]))
    return scen, want_co, want_cs, ctx


@pytest.mark.parametrize("tag,windows", [(t, w) for t in SETS for w in (1, 4)])
def test_object_decisions_at_the_boundary(tag, windows):
    """k_plan: in-track test of an object (F1'; it must agree with the ego's F1 on the same points), nearest
    reference-line layer of a disc (F4, incl. exact ties at the closed track's seam and warp-scan fallback lanes),
    neighbour choice on glob_rl for angle gaps of 1e-13 .. 1e-10 rad (F7: angle_cmp_exact)."""
    g = K.golden_set(tag)
    orc = K.oracle_for(tag)
    scen, want_co, want_cs, ctx = _object_scenarios(g, orc)
    reps = max(1, -(-2048 // len(scen))) if windows > 1 else 1   # enough scenarios for 4 windows of >= 512
    pl = D.planner(orc.lat, windows, ax_max_machines=_axm())
    pl.stage_scenarios(_batch(scen * reps))
    pl.upload()
    pl.set_startpos()
    pl.tick()
    f = pl.fetch("closest_obj", "cobj_start", "sc_flags")
    n = len(scen)
    assert np.all(f["sc_flags"] == 0), np.nonzero(f["sc_flags"])[0][:8]
    for r in range(1, reps):
        assert np.array_equal(f["closest_obj"][r * n:(r + 1) * n], f["closest_obj"][:n])
    bad = []
    for b in range(n):
        co = int(f["closest_obj"][b])
        if co != want_co[b]:
            bad.append("%s: closest object %d, want %d" % (ctx[b], co, want_co[b]))
        elif want_cs[b] is not None and int(f["cobj_start"][b]) != want_cs[b]:
            bad.append("%s: glob_rl start %d, want %d" % (ctx[b], int(f["cobj_start"][b]), want_cs[b]))
    assert not bad, "%s, %d windows: %d/%d decisions differ:\n%s" % (tag, windows, len(bad), n, "\n".join(bad[:12]))


@pytest.mark.parametrize("tag", SETS)
def test_collision_decisions_at_the_boundary(tag):
    """k_plan's collision sweep (F5): a v = 0 object whose disc reaches one lattice sample by a hair, misses it by a hair,
    or reaches it EXACTLY (x^2 + y^2 == ref); closest object and node sequences against the fixture, the +-4 ulps
    against the oracle."""
    g = K.golden_set(tag)
    orc = K.oracle_for(tag)
    scen, want, ctx = [], [], []
    for k, pair in enumerate(g["f5_p"]):
        pose = K.ego_pose(orc, int(g["f5_ego"][k]))
        for j, p in enumerate(pair):
            scen.append(pose + ([K.obj(p)],))
            want.append(g["f5_obs"][k, j])
            ctx.append("F5 pair %d.%d" % (k, j))
        for p in _axis_window(pair, int(g["f5_axis"][k])):
            scen.append(pose + ([K.obj(p)],))
            want.append(repr(K.paths_observable(orc, *pose, [K.obj(p)])))
            ctx.append("F5 window %d" % k)
    for k, p in enumerate(g["f5_eq_p"]):
        scen.append(K.ego_pose(orc, int(g["f5_ego"][g["f5_eq_case"][k]])) + ([K.obj(p)],))
        want.append(g["f5_eq_obs"][k])
        ctx.append("F5 equality %d" % k)
    pl = D.planner(orc.lat, 4, ax_max_machines=_axm())
    pl.stage_scenarios(_batch(scen))
    pl.upload()
    pl.set_startpos()
    pl.tick()
    recs = pl.records()
    bad = []
    for b, rec in enumerate(recs):
        got = "out of track" if rec["out_of_track"] else repr(K.observable(rec["closest_obj_index"], rec["nodes"]))
        if got != want[b]:
            bad.append("%s:\n got  %s\n want %s" % (ctx[b], got[:300], want[b][:300]))
    assert not bad, "%s: %d/%d observables differ:\n%s" % (tag, len(bad), len(scen), "\n".join(bad[:6]))


@pytest.mark.parametrize("tag", SETS)
def test_constant_segment_decisions_at_the_boundary(tag):
    """k_plan's check of an object beside / in the constant segment (F6, MOPG:86-122): s_start <= s_obj and
    s_obj <= s_end on the race line, d2 <= oref against the ego position (incl. EXACTLY oref) and against a point inside
    the segment, and race-line near-ties of get_s_coord whose neighbour choice decides s_start <= s_obj.  The segment's
    points come out of float64 sin / cos, so every decision is replayed by the oracle on the device's own segment
    (records()[b]['const_path_seg']); where the inputs are exact (the ego position, the objects) the fixture's
    observable must come out as well."""
    g = K.golden_set(tag)
    orc = K.oracle_for(tag)
    scen, fixed, ctx = [], [], []
    for k, pair in enumerate(g["f6_p"]):
        ego, hd = g["f6_ego"][k], g["f6_hd"][k]
        exact = int(g["f6_kind"][k]) in (0, 2)   # decided by exact inputs only
        for j, p in enumerate(pair):
            scen.append((ego, hd, [K.obj(p)]))
            fixed.append(g["f6_obs"][k, j] if exact else None)
            ctx.append("F6 kind %d pair %d.%d" % (g["f6_kind"][k], k, j))
        for p in _axis_window(pair, int(g["f6_axis"][k])):
            scen.append((ego, hd, [K.obj(p)]))
            fixed.append(None)
            ctx.append("F6 kind %d window %d" % (g["f6_kind"][k], k))
    for k, p in enumerate(g["f6_eq_p"]):
        c = g["f6_eq_case"][k]
        scen.append((g["f6_ego"][c], g["f6_hd"][c], [K.obj(p)]))
        fixed.append(g["f6_eq_obs"][k])
        ctx.append("F6 oref equality %d" % k)
    for k, p in enumerate(g["f6r_p"]):
        scen.append((g["f6r_ego"][k], g["f6r_hd"][k], [K.obj(p)]))
        fixed.append(g["f6r_obs"][k])
        ctx.append("F6 race-line near-tie %d (gap %.1e)" % (k, g["f6r_gap"][k]))
    pl = D.planner(orc.lat, 4, ax_max_machines=_axm())
    pl.stage_scenarios(_batch(scen))
    pl.upload()
    pl.set_startpos()
    pl.tick()
    recs = pl.records()
    bad = []
    for b, rec in enumerate(recs):
        if rec["out_of_track"]:
            bad.append("%s: out of track" % ctx[b])
            continue
        got = repr(K.observable(rec["closest_obj_index"], rec["nodes"]))
        want = repr(K.replay_observable(orc, *scen[b], rec["const_path_seg"]))
        if got != want or (fixed[b] is not None and got != fixed[b]):
            bad.append("%s:\n got    %s\n replay %s\n golden %s" % (ctx[b], got[:200], want[:200], str(fixed[b])[:200]))
    assert not bad, "%s: %d/%d observables differ:\n%s" % (tag, len(bad), len(scen), "\n".join(bad[:6]))
