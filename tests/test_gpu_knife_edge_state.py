"""The stateful tick's float64 decisions at their exact boundaries, on the device (tests/knife_edge_state.py, families
G1-G5; tests/golden/ticks_knife_edge_state.npz for the histories).  Every probe is its own scenario, a copy of its
history (same start pose, no objects, the executed action as sel_action).  The first tick gives each copy the same
memory; the probes are built on that memory as the device downloaded it (its velocity rows are fp32 recurrences stored
in float64, so the reference's ties are no ties here) and one stateful tick takes them with per-scenario t_const /
pos_est.  The replays of tests/knife_edge_state.py, which the fixture pins to the reference, give what k_state and
k_ref must decide: start node, constant-segment length, trim (cut, m, L, pref), vel_plan and vel_course bit for bit,
no fallback flag."""
import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H
from tests import knife_edge_state as KS

pytestmark = pytest.mark.gpu

SETS = ("default", "l216", "open")


def _set(tag):
    g = H.golden("ticks_knife_edge_state.npz")
    return {k.split("__", 1)[1]: g[k] for k in g.files if k.startswith(tag + "__")}


def _batch(g, hist, pos=None):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    hist = np.asarray(hist)
    p = g["h_pos"][hist] if pos is None else np.asarray(pos, dtype=np.float64).reshape(-1, 2)
    return ScenarioBatch.from_object_lists(p.copy(), g["h_heading"][hist].copy(), g["h_vel"][hist].copy(),
                                           [[] for _ in hist])


def _axm():
    return H.golden("ticks_manyobj.npz")["ax_max_machines"]


def _planner(tag, windows, emergency=False):
    return D.planner(H.lattice_for(tag), windows, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=emergency)


def _set_delaycomp(pl, delaycomp, emergency):
    """[DELAY] delaycomp of the planner's online settings"""
    pl.online["delaycomp"] = float(delaycomp)
    pl.set_vel_params(**dict(D.VEL, ax_max_machines=_axm(), incl_emerg_traj=emergency))


def _first(pl, g, hist):
    pl.stage_scenarios(_batch(g, hist))
    pl.upload()
    pl.set_startpos()
    pl.tick()


def _memories(pl, g, hist):
    """the memory of each scenario after a first tick: the executed action's trajectory rows (s, x, y, vx), node
    coordinates, node list and node indices, as raw arrays (byte-comparable)"""
    f = pl.fetch("action_id", "traj_len", "path", "s_vx_ax", "node_idx", "nodes", "n_nodes", "trim", "sc_flags")
    em_vx = pl.t["em_vx"].cpu().numpy() if "em_vx" in pl.t else None
    B = len(hist)
    out = []
    for b, h in enumerate(hist):
        assert int(f["sc_flags"][b]) == 0, "history %d: first tick flags %d" % (h, f["sc_flags"][b])
        em = bool(g["h_em"][h])
        # an executed 'emergency' trajectory: s, x, y of its base (the first trajectory) and the brake profile's vx
        s = int(np.nonzero(f["traj_len"][:, b] > 0)[0][0]) if em else \
            int(np.nonzero(f["action_id"][:, b] == int(g["h_sel"][h]))[0][0])
        q = s * B + b
        n, nn = int(f["traj_len"][s, b]), int(f["n_nodes"][s, b])
        assert (f["trim"][q] == 0).all()
        ni = f["node_idx"][s, b, :nn].copy()
        out.append(dict(traj=np.column_stack((f["s_vx_ax"][0, q, :n], f["path"][0, q, :n], f["path"][1, q, :n],
                                              em_vx[b, :n] if em else f["s_vx_ax"][1, q, :n])),
                        node_xy=f["path"][0:2, q, ni].T.copy(), node_idx=ni, nodes=f["nodes"][s, b, :nn].copy()))
    return out


def _same_memory(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("traj", "node_xy", "node_idx", "nodes"))


def _check_history(g, h, mem):
    """the device plans the reference's node list and row count for the history"""
    nn, n = int(g["h_nn"][h]), int(g["h_n"][h])
    assert mem["nodes"].tolist() == g["h_nodes"][h, :nn].tolist(), "history %d: node list" % h
    assert mem["traj"].shape[0] == n, "history %d: %d rows, reference %d" % (h, mem["traj"].shape[0], n)


def _second(pl, g, hist, pos, t_const, device_batch):
    import torch
    sc = _batch(g, hist, pos)
    sel = g["h_sel"][hist].astype(np.int32)
    if device_batch:
        dev = pl.device
        pl.next_tick(sc.to_device(dev), sel_action=torch.as_tensor(sel, device=dev),
                     t_const=torch.as_tensor(np.asarray(t_const, dtype=np.float64), device=dev))
    else:
        pl.next_tick(sc, sel_action=sel, t_const=np.asarray(t_const, dtype=np.float64))
    f = pl.fetch("sc_flags", "start_node", "const_len", "action_id", "node_idx", "n_nodes", "trim", "t_const")
    f["vel_plan"] = pl._state["vel_plan"].cpu().numpy()
    f["course"] = pl._state["course"].cpu().numpy()
    return f


def _expect_ref(f, b, B, mem, pos, delay, ctx, bad):
    """k_ref of scenario b against ref_idx on the device's memory and the device's second-tick node lists"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    slots = [s for s in range(f["action_id"].shape[0]) if f["action_id"][s, b] != capi.ACT_NONE]
    ni2 = f["node_idx"][slots[0], b, :int(f["n_nodes"][slots[0], b])]
    cut_pos, cut_layer, _, vel_idx, vel_plan, course = KS.ref_idx(mem["traj"], pos, delay, ni2, 0)
    for s in slots:
        m = int(f["node_idx"][s, b, cut_layer])
        got = f["trim"][s * B + b].tolist()
        if got != [m, cut_layer, cut_pos, vel_idx]:
            bad.append("%s slot %d: trim (m, L, cut, pref) %s, want %s" % (ctx, s, got, [m, cut_layer, cut_pos, vel_idx]))
    if f["vel_plan"][b].tobytes() != np.float64(vel_plan).tobytes():
        bad.append("%s: vel_plan %r, want %r" % (ctx, f["vel_plan"][b], vel_plan))
    if f["course"][b, :vel_idx].tobytes() != course.tobytes():
        bad.append("%s: vel_course differs" % ctx)


def _g123(g, mems):
    """[(history, pos, t_const, family, what)] built on the device's memories"""
    rng = np.random.default_rng(77)
    out = []
    for h, mem in enumerate(mems):
        for T, kind, k in KS.g1_probes(mem, all_true=1e3) + KS.g2_probes(mem):
            out.append((h, g["h_pos"][h], T, "G1", kind, "k %d T %r" % (k, T)))
        for p, kind in KS.g3_probes(mem["traj"], rng):
            out.append((h, p, float(g["t0"]), "G3", kind, "pos %r" % p.tolist()))
    return out


def _run_g123(tag, windows, device_batch):
    from graphbasedlocaltrajectoryplanner_b200 import capi
    g = _set(tag)
    nh = g["h_n"].shape[0]
    hist = [h for h in range(nh) if not g["h_em"][h]]
    pl = _planner(tag, windows)
    _first(pl, g, hist)
    mems = _memories(pl, g, hist)
    for h, mem in zip(hist, mems):
        _check_history(g, h, mem)
    probes = [(hist[h],) + p[1:] for p in _g123(g, mems) for h in (p[0],)]
    mems = dict(zip(hist, mems))
    ph = [p[0] for p in probes]
    pl = _planner(tag, windows)
    _first(pl, g, ph)
    got = _memories(pl, g, ph)
    for b, h in enumerate(ph):
        assert _same_memory(got[b], mems[h]), "%s: copy %d of history %d has another memory" % (tag, b, h)
    f = _second(pl, g, ph, [p[1] for p in probes], [p[2] for p in probes], device_batch)
    B = len(probes)
    assert np.array_equal(f["t_const"], np.array([p[2] for p in probes])), "k_stage / staging changed t_const"
    bad = []
    for b, (h, pos, T, fam, kind, what) in enumerate(probes):
        ctx = "%s history %d %s kind %d %s" % (tag, h, fam, kind, what)
        mem = mems[h]
        fl = int(f["sc_flags"][b])
        # a start node far along the memory may leave no room for a whole new plan behind the constant segment: the
        # tick flags SC_CAPACITY after k_state decided (G1 probes of long t_const); the cut probes have none
        if fl not in ((0, capi.SC_CAPACITY) if fam == "G1" else (0,)):
            bad.append("%s: flags %d" % (ctx, fl))
            continue
        sni = KS.memory_start(mem, T)
        want = (mem["nodes"][sni].tolist(), int(mem["node_idx"][sni]) + 1)
        have = (f["start_node"][b].tolist(), int(f["const_len"][b]))
        if have != want:
            bad.append("%s: start node / const_len %s, want %s" % (ctx, have, want))
        if fam == "G3":
            _expect_ref(f, b, B, mem, pos, float(g["delay"]), ctx, bad)
    assert not bad, "%d of %d probes differ:\n%s" % (len(bad), B, "\n".join(bad[:12]))
    c1 = np.bincount([p[4] for p in probes if p[3] == "G1"], minlength=7)
    c3 = np.bincount([p[4] for p in probes if p[3] == "G3"], minlength=7)
    # on the device's memory: start-moving t_const ties, T = 0, all-True, v == 0 (open track's end), every row
    assert c1[KS.G1_TIE] >= 10 and c1[KS.G1_ZERO] >= 2 and c1[KS.G1_ALL] >= 2 and c1[KS.G1_ROW] >= 150, c1
    assert tag != "open" or c1[KS.G1_INF] >= 1, c1
    assert c3[KS.G3_FLIP] >= 20 and c3[KS.G3_TIE] >= 4 and c3[KS.G3_ANGLE] >= 10 and c3[KS.G3_ON_ROW] >= 200, c3
    assert c3[KS.G3_BEYOND] >= 3 and c3[KS.G3_BEFORE] >= 3 and c3[KS.G3_COLLINEAR] >= 2, c3
    return B


@pytest.mark.parametrize("windows", (1, 4))
@pytest.mark.parametrize("tag", SETS)
def test_state_decisions_at_the_boundary(tag, windows):
    """G1 (t_const ties, all-True, T = 0, v == 0), G2 (every row as the predicted position), G3 / G5 (cut index and cut
    layer by pos_est) in one stateful tick"""
    assert _run_g123(tag, windows, device_batch=False) > 300


@pytest.mark.parametrize("tag", SETS)
def test_state_decisions_from_device_inputs(tag):
    """the same probes from a DeviceScenarioBatch with a float64 device t_const: k_stage carries the probe bytes"""
    assert _run_g123(tag, 4, device_batch=True) > 300


@pytest.mark.parametrize("windows", (1, 4))
@pytest.mark.parametrize("tag", SETS)
def test_delaycomp_at_the_boundary(tag, windows):
    """G4 / G5: one second tick per delaycomp D (a planner parameter), on the device's memory: D = the cumsum from the
    cut exactly, its lower neighbour and +-4 ulps, all-True near the end (the nv - 1 clamp), v == 0; also on an
    executed 'emergency' trajectory that reaches standstill (k_ref reads prev_em_vx)"""
    g = _set(tag)
    nh = g["h_n"].shape[0]
    bad, n = [], 0
    kinds = np.zeros((2, 5), dtype=int)
    for em in (False, True):
        hist = [h for h in range(nh) if bool(g["h_em"][h]) == em]
        pl = _planner(tag, windows, emergency=em)
        _first(pl, g, hist)
        mems = _memories(pl, g, hist)
        pd = _planner(tag, windows, emergency=em)
        for h, mem in zip(hist, mems):
            _check_history(g, h, mem)
            for pos, Dc, kind, c in KS.g4_probes(mem["traj"], KS.g4_rows(mem["traj"])):
                _set_delaycomp(pd, Dc, em)
                _first(pd, g, [h])
                assert _same_memory(_memories(pd, g, [h])[0], mem)
                f = _second(pd, g, [h], [pos], [float(g["t0"])], False)
                ctx = "%s history %d G4 kind %d cut %d D %r" % (tag, h, kind, c, Dc)
                if int(f["sc_flags"][0]) != 0:
                    bad.append("%s: flags %d" % (ctx, f["sc_flags"][0]))
                    continue
                _expect_ref(f, 0, 1, mem, pos, Dc, ctx, bad)
                kinds[int(em), kind] += 1
                n += 1
    assert not bad, "%d of %d probes differ:\n%s" % (len(bad), n, "\n".join(bad[:12]))
    assert kinds[0, KS.G4_TIE] >= 12 and kinds[0, KS.G4_ALL] >= 8, kinds
    assert kinds[1, KS.G4_TIE] >= 3 and kinds[1, KS.G4_INF] >= 4, kinds


def _f_points(tag):
    """the F1 - F3 poses of the first tick's fixture (tests/golden/ticks_knife_edge.npz) with the flag bit each one
    decides and its expected value, and for F2 the expected start layer"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from tests import knife_edge as K
    f = K.golden_set(tag)
    orc = K.oracle_for(tag)
    L = orc.lat.num_layers
    out = []   # (pos, heading, bit, want_bit, start_layer or None, what)
    for k, pair in enumerate(f["f1_p"]):
        for j, p in enumerate(pair):
            out.append((p, 0.0, capi.SC_OUT_OF_TRACK, 0 if f["f1_in"][k, j] else capi.SC_OUT_OF_TRACK, None,
                        "F1 pair %d.%d" % (k, j)))
    for k, pair in enumerate(f["f2_p"]):
        for j, p in enumerate(pair):
            out.append((p, 0.0, 0, 0, (int(f["f2_layer"][k, j]) + 2) % (L - 1), "F2 pair %d.%d" % (k, j)))
    for k in range(f["f3_h"].shape[0]):
        pos, _ = K.ego_pose(orc, int(f["f3_layer"][k]))
        for j, hd in enumerate(f["f3_h"][k]):
            out.append((pos, hd, capi.SC_HEADING_MISMATCH, 0 if f["f3_ok"][k, j] else capi.SC_HEADING_MISMATCH, None,
                        "F3 pair %d.%d" % (k, j)))
    return out


@pytest.mark.parametrize("tag", SETS)
def test_restart_at_the_knife_edge(tag):
    """G6: the F1 - F3 flip pairs as restart poses inside a stateful tick (masked k_startpos): each restarted scenario
    gets the in-track / heading decision and the start layer of the first-tick fixture; the unmasked scenario beside
    each of them keeps the bytes of the same tick without restarts"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    g = _set(tag)
    h0 = int(np.nonzero(~g["h_em"])[0][0])
    pts = _f_points(tag)
    B = 2 * len(pts)   # scenario 2 i restarts at point i, 2 i + 1 is its unmasked neighbour
    hist = [h0] * B
    pos = np.repeat(g["h_pos"][h0][None], B, axis=0)
    hd = np.full(B, g["h_heading"][h0])
    for i, (p, h, _, _, _, _) in enumerate(pts):
        pos[2 * i], hd[2 * i] = p, h
    sc = ScenarioBatch.from_object_lists(pos, hd, np.full(B, g["h_vel"][h0]), [[] for _ in range(B)])
    mask = np.arange(B) % 2 == 0
    sel = np.full(B, int(g["h_sel"][h0]), dtype=np.int32)
    tc = np.full(B, float(g["t0"]))
    snaps = []
    for restart in (mask, None):
        pl = _planner(tag, 4)
        _first(pl, g, hist)
        pl.next_tick(sc, sel_action=sel, t_const=tc, restart=restart)
        snaps.append((D.tick_snapshot(pl, emergency=False), pl.fetch("sc_flags", "start_node")))
    (got, f), (ref, _) = snaps
    nb = np.nonzero(~mask)[0]
    for k in ref:
        assert np.array_equal(D.take(got, nb)[k], D.take(ref, nb)[k]), "%s: '%s' of an unmasked neighbour" % (tag, k)
    bad = []
    for i, (_, _, bit, want, layer, what) in enumerate(pts):
        b = 2 * i
        if bit and int(f["sc_flags"][b]) & bit != want:
            bad.append("%s: flag bit %d = %d, want %d" % (what, bit, int(f["sc_flags"][b]) & bit, want))
        if layer is not None and int(f["start_node"][b, 0]) != layer:
            bad.append("%s: start layer %d, want %d" % (what, int(f["start_node"][b, 0]), layer))
    assert not bad, "%s: %d of %d restarted probes differ:\n%s" % (tag, len(bad), len(pts), "\n".join(bad[:12]))
