"""Ticks replayed from CUDA graphs (BatchPlanner.capture_tick / capture_next_tick, TickGraph, k_traj_base): every replay
gives the bytes of the same tick run eagerly from device inputs -- first ticks on three lattices, closed loops over the
multi-tick fixtures and a friction-map loop, eager ticks and replays interleaved from both parities -- with ids that
continue across both.  A replay does no host work, and refused captures, stale graphs and the library's checks of
buffers.traj_base change nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import drivers as D
from tests import gg_map_ref as M
from tests import helpers as H
from tests.test_gpu_device_inputs import MAP, _assert_same, _fixture_inputs, _outputs, _scenarios, _with_pred, \
    _with_zones

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MEMORY = ("st_info", "vel_plan", "course", "zone_s0")


def _axm(tag="default"):
    return H.golden("ticks_%s.npz" % tag)["ax_max_machines"]


def _dev(a, dt=None):
    return None if a is None else torch.as_tensor(np.asarray(a, dtype=dt), device=DEV)


def _results(pl):
    """_outputs with the emergency rows cleared behind their length: a compact export row holds what an earlier tick
    wrote there behind it, and which row a trajectory gets is unspecified"""
    out = _outputs(pl)
    em_rows = out["em_rows"].copy()
    em_rows[0][np.arange(em_rows.shape[2])[None, :] >= out["em_len"][0][:, None]] = 0.0
    out["em_rows"] = em_rows
    return out


def _state(pl):
    """results and, for a stateful planner, the memory records of the last tick, byte-comparable"""
    out = _results(pl)
    if pl._state is not None:
        torch.cuda.synchronize()
        out.update({k: pl._state[k].cpu().numpy() for k in MEMORY})
        out["trim"] = pl.t["trim"].cpu().numpy()
    return out


def _raw(pl):
    """every buffer of the planner as it is (no clearing): for 'changed nothing'"""
    torch.cuda.synchronize()
    out = {k: v.cpu().clone() for k, v in pl.t.items()}
    if pl._state is not None:
        out.update({"st_" + k: pl._state[k].cpu().clone() for k in MEMORY})
    return out


def _assert_raw_same(a, b, ctx):
    assert sorted(a) == sorted(b), ctx
    for k in a:
        assert torch.equal(a[k], b[k]), "%s: '%s' changed" % (ctx, k)


def _ids(pl):
    tid = pl.fetch("traj_id")["traj_id"]
    return np.unique(tid[tid >= 0] // 10)


# ---- first ticks ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag,n,windows", [("default", 384, 4), ("l216", 257, 3), ("open", 200, 1)])
def test_first_tick_replays_equal_eager_ticks(tag, n, windows):
    """capture_tick once, then 4 seeded device batches copied into graph.inputs and replayed: each replay == stage +
    set_startpos + tick of the same device batch on a twin planner, every result incl. traj_id (10, 20, 30, 40) and
    em_info (predictions on the default lattice, zones on l216, the emergency trajectory on)"""
    lat = H.lattice_for(tag)
    vel = dict(ax_max_machines=_axm(tag), incl_emerg_traj=True)
    pg, pe = D.planner(lat, windows, **vel), D.planner(lat, windows, **vel)

    def batch(i):
        sc = _scenarios(tag, n, 9600 + i)
        if tag == "default":
            _with_pred(sc, 12, 9610 + i)
        if tag == "l216":
            z = _with_zones(_scenarios(tag, n, 9600), tag, 9620)   # one zone list for the graph's lifetime
            sc.zones, sc.zone_sel, sc.zone_key = z.zones, np.roll(z.zone_sel, i), np.roll(z.zone_key, i)
        return sc
    sc0 = batch(0)
    graph = pg.capture_tick(sc0.to_device(DEV), vel_est=_dev(sc0.vel))
    assert graph.n_graphs == 1
    for i in range(1, 5):
        sc = batch(i)
        dsc = sc.to_device(DEV)
        graph.inputs.copy_(dsc, vel_est=dsc.vel * 0.97)
        graph.replay()
        D.first_tick(pe, dsc, vel_est=dsc.vel * 0.97)
        got, want = _results(pg), _results(pe)
        _assert_same(got, want, "%s replay %d" % (tag, i))
        assert (want["traj_len"] > 0).sum() > n
        assert list(_ids(pg)) == [i]
        em = pg.fetch("em_info")["em_info"]
        assert (em[:, 0] >= 0).any() and np.all(em[em[:, 0] >= 0, 2] // 10 == i)


# ---- stateful closed loops -----------------------------------------------------------------------------------------
def _union_zones(batches):
    """the zone list of a whole loop (a graph's zone list is fixed): every tick's batch selecting its zones in it"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    keys, zones = {}, []
    for sc in batches:
        for lay, nod in (sc.zones or []):
            if (lay.tobytes(), nod.tobytes()) not in keys:
                keys[(lay.tobytes(), nod.tobytes())] = len(zones)
                zones.append((lay, nod))
    out = []
    for sc in batches:
        sel = np.full(sc.size, -1, dtype=np.int32)
        if sc.zones:
            idx = np.array([keys[(lay.tobytes(), nod.tobytes())] for lay, nod in sc.zones])
            sel = np.where(sc.zone_sel >= 0, idx[np.maximum(sc.zone_sel, 0)], -1).astype(np.int32)
        zkey = np.zeros(sc.size, dtype=np.int64) if sc.zone_key is None else sc.zone_key
        out.append(ScenarioBatch(sc.pos, sc.heading, sc.vel, sc.n_obj, sc.obj, zones or None, sel if zones else None,
                                 zkey if zones else None))
    return out


@pytest.mark.parametrize("fixture,emerg,kind", [
    ("ticks_multitick_ext_default.npz", True, "next_tick"),         # zones + emergency trajectory
    ("ticks_multitick_zswap_default.npz", False, "next_tick"),      # zone id changes (one zone list for both)
    ("ticks_multitick_restart_default.npz", True, "restart"),       # the restart mask as a graph input
    ("ticks_multitick_emsel_default.npz", True, "next_tick"),       # 'emergency' executed
    ("ticks_multitick_ggpp_default.npz", True, "map")])             # friction map, grip drops
def test_closed_loop_replays_equal_eager_loop(fixture, emerg, kind):
    """the fixture's inputs as device tensors on two stateful planners: all-eager next_tick, and one TickGraph
    (captured anew only where gg_scale changes) replayed with the inputs copied in; results and memory (st_info, trim,
    vel_plan, course, zone_s0) byte-equal after every tick"""
    g = H.golden(fixture)
    n_seq, n_ticks = g["dt"].shape
    lat = H.lattice_for("default")
    vel = dict(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emerg)
    pe, pg = (D.planner(lat, 1 + n_seq % 4, stateful=True, **vel) for _ in range(2))
    if kind == "map":
        ax, ay = M.surface_map(MAP[2], x0=MAP[0], y0=MAP[1], width=500.0, height=350.0)
        for pl in (pe, pg):
            pl.set_gg_map(ax, ay, *MAP)
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)]) if kind != "restart" else None
    ticks = [_fixture_inputs(g, kind, k, tc) for k in range(n_ticks)]
    union = _union_zones([t[0] for t in ticks])
    graph, scale, replays = None, None, 0
    for k, (sc, sel, t_c, v_est, restart, gg_scale) in enumerate(ticks):
        if gg_scale != scale:
            for pl in (pe, pg):
                pl.set_vel_params(**dict(D.VEL, gg_scale=gg_scale, **vel))
            scale, graph = gg_scale, None
        args = (_dev(sel, np.int32), _dev(t_c, np.float64))
        kw = dict(vel_est=_dev(v_est, np.float64), restart=_dev(restart, bool))
        if k == 0:
            D.first_tick(pe, sc.to_device(DEV), vel_est=kw["vel_est"])
            D.first_tick(pg, union[k].to_device(DEV), vel_est=kw["vel_est"])
        else:
            pe.next_tick(sc.to_device(DEV), *args, **kw)
            dsc = union[k].to_device(DEV)
            if graph is None:
                graph = pg.capture_next_tick(dsc, *args, **kw)
            graph.inputs.copy_(dsc, *args, **kw)
            graph.replay()
            replays += 1
        _assert_same(_state(pg), _state(pe), "tick %d" % k)
    assert replays == n_ticks - 1 and pg._tick_count == pe._tick_count == n_ticks


def test_friction_map_closed_loop_replays_equal_eager_loop():
    """the closed loop of the friction-map tests (every scenario drives 0.1 s along its first kept trajectory, restarts
    on ticks 2 and 5 through the restart mask, grip drops on ticks 3 and 6, the map off for ticks 4 and 5): one graph
    per stretch of unchanged settings, three states of the buffers where the map was switched (the first tick after a
    switch swaps the gg planes differently from the ticks after it); every tick byte-equal to the eager loop"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    from tests.test_gpu_gg_map import CELL, MAP as GMAP, MAP_OFF_TICKS, X0, Y0
    from tools.workload import closed_loop_step
    lat, sc = H.lattice_for("default"), _scenarios("default", 512, 8300)
    vel = dict(ax_max_machines=_axm(), incl_emerg_traj=True)
    pe, pg = (D.planner(lat, 4, stateful=True, **vel) for _ in range(2))
    for pl in (pe, pg):
        pl.set_gg_map(GMAP[0], GMAP[1], X0, Y0, CELL)
        D.first_tick(pl, sc.to_device(DEV))
    rng = np.random.default_rng(8301)
    pos, v = sc.pos.copy(), sc.vel.copy()
    graph, n_graphs = None, []
    for k in range(1, 8):
        p_new, v_new, sel, ok, head = closed_loop_step(pe.fetch("traj_row", "traj_len", "action_id", "traj"), 0.1)
        pos, v = np.where(ok[:, None], p_new, pos), np.where(ok, v_new, v)
        heading = sc.heading.copy()
        heading[ok] = head[ok]
        restart = (rng.random(sc.size) < 0.1) if k in (2, 5) else np.zeros(sc.size, dtype=bool)
        dsc = ScenarioBatch(pos.copy(), heading, v.copy(), sc.n_obj, sc.obj).to_device(DEV)
        for pl in (pe, pg):
            if k in (3, 6):
                pl.set_vel_params(**dict(D.VEL, gg_scale=0.55 if k == 3 else 0.4, **vel))
            if k == MAP_OFF_TICKS[0]:
                pl.set_gg_map(None)
            elif k == MAP_OFF_TICKS[-1] + 1:
                pl.set_gg_map(GMAP[0], GMAP[1], X0, Y0, CELL)
        args = (_dev(sel, np.int32), 0.2)
        kw = dict(vel_est=_dev(v), restart=_dev(restart))
        pe.next_tick(dsc, *args, **kw)
        if graph is None or k in (3, 4, 6):
            graph = pg.capture_next_tick(dsc, *args, **kw)
            n_graphs.append(graph.n_graphs)
        graph.inputs.copy_(dsc, *args, **kw)
        graph.replay()
        _assert_same(_state(pg), _state(pe), "tick %d" % k)
    assert n_graphs == [2, 2, 3, 3], n_graphs


# ---- parity, interleaving, ids -------------------------------------------------------------------------------------
@pytest.mark.parametrize("shift,host", [(0, False), (1, False), (1, True)], ids=["0", "1", "1-host"])
def test_eager_ticks_and_replays_interleave(shift, host):
    """eager, replay, replay, eager, replay after `shift` eager stateful ticks (the graph captured at either parity) ==
    the all-eager loop, results and memory every tick; the ids count on without a gap or a repeat.  host: the
    capturing planner's eager ticks, the first one included, take the host ScenarioBatch and NumPy arguments (zones
    and zone keys included), so replays and captures follow ticks staged from the host"""
    g = H.golden("ticks_multitick_ext_default.npz")
    n_seq = g["dt"].shape[0]
    lat = H.lattice_for("default")
    vel = dict(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True)
    pe, pg = (D.planner(lat, 3, stateful=True, **vel) for _ in range(2))
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)])
    pattern = ["eager"] * shift + ["eager", "replay", "replay", "eager", "replay"]
    graph = None
    for k, how in enumerate(["first"] + pattern):
        sc, sel, t_c, v_est, _, _ = _fixture_inputs(g, "next_tick", k, tc)
        dsc = sc.to_device(DEV)
        args, kw = (_dev(sel, np.int64), _dev(t_c)), dict(vel_est=_dev(v_est))
        if how == "first":
            D.first_tick(pe, dsc, vel_est=kw["vel_est"])
            D.first_tick(pg, *((sc, v_est) if host else (dsc, kw["vel_est"])))
            continue
        pe.next_tick(dsc, *args, **kw)
        if graph is None and k == 1 + shift:
            graph = pg.capture_next_tick(dsc, *args, **kw)
            assert graph.n_graphs == 2
        if how == "eager" and host:
            pg.next_tick(sc, sel, t_c, vel_est=v_est)
        elif how == "eager":
            pg.next_tick(dsc, *args, **kw)
        else:
            graph.inputs.copy_(dsc, *args, **kw)
            graph.replay()
        _assert_same(_state(pg), _state(pe), "tick %d (%s)" % (k, how))
        assert list(_ids(pg)) == [k + 1], (k, how)


# ---- no host work --------------------------------------------------------------------------------------------------
def test_replay_does_no_host_work():
    """replays under torch.cuda.set_sync_debug_mode('error') without a library call (launch count unchanged); after
    the host arrays the captured batch was made from are overwritten, a replay still gives the eager twin's bytes"""
    sc = _with_zones(_scenarios("default", 256, 9700), "default", 9701)
    lat = H.lattice_for("default")
    pe, pg = (D.planner(lat, 4, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True) for _ in range(2))
    keep = sc.to_device(DEV)
    keep.zones = [(lay.copy(), nod.copy()) for lay, nod in sc.zones]
    for pl in (pe, pg):
        D.first_tick(pl, keep)
    sel = pe.device_results()["action_id"].max(dim=0).values.clamp(min=0)
    restart = torch.zeros(sc.size, dtype=torch.bool, device=DEV)
    restart[::9] = True
    graph = pg.capture_next_tick(sc.to_device(DEV), sel, 0.15, vel_est=keep.vel * 0.9, restart=restart)
    for a in (sc.pos, sc.heading, sc.vel, sc.obj, sc.zone_key):   # the host source arrays, zones included
        a[...] = 7
    sc.n_obj[...] = 99
    sc.zone_sel[...] = 0
    for lay, nod in sc.zones:
        lay[...] = 0
        nod[...] = 0
    n0 = pg.launch_count()
    for k in range(3):
        sel = pe.device_results()["action_id"].max(dim=0).values.clamp(min=0)
        pe.next_tick(keep, sel, 0.15, vel_est=keep.vel * 0.9, restart=restart)
        n_eager = pg.launch_count()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            graph.inputs.copy_(keep, sel, vel_est=keep.vel * 0.9, restart=restart)
            graph.replay()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert pg.launch_count() == n_eager
        _assert_same(_state(pg), _state(pe), "replay %d" % k)
    assert pg.launch_count() > n0   # the eager twin's launches


# ---- refusals, invalidation, the library's checks -------------------------------------------------------------------
def _refused(pl, fn, match):
    before, n0 = _raw(pl), pl.launch_count()
    with pytest.raises(ValueError, match=match):
        fn()
    assert pl.launch_count() == n0, match
    _assert_raw_same(_raw(pl), before, match)


def test_refused_captures_change_nothing():
    sc = _scenarios("default", 96, 9800)
    dsc = sc.to_device(DEV)
    lat = H.lattice_for("default")
    pl = D.planner(lat, 2, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True)
    fresh = D.planner(lat, 2, stateful=True, ax_max_machines=_axm())
    fresh.allocate(sc.size, 3)
    _refused(fresh, lambda: fresh.capture_next_tick(dsc, torch.zeros(96, dtype=torch.int32, device=DEV), 0.1),
             "no previous tick")
    D.first_tick(pl, dsc)
    sel = torch.zeros(sc.size, dtype=torch.int32, device=DEV)
    _refused(pl, lambda: pl.capture_tick(sc), "DeviceScenarioBatch")
    _refused(pl, lambda: pl.capture_next_tick(sc, sel, 0.1), "DeviceScenarioBatch")
    _refused(pl, lambda: pl.capture_tick(dsc, restart=sel > 0), "restart")
    small = _scenarios("default", 95, 9801).to_device(DEV)
    _refused(pl, lambda: pl.capture_next_tick(small, sel[:95], 0.1), "batch")
    pl.set_local_gg_planes(*H.local_gg_planes(pl))
    _refused(pl, lambda: pl.capture_tick(dsc), "local_gg planes")
    _refused(pl, lambda: pl.capture_next_tick(dsc, sel, 0.1), "local_gg planes")
    assert pl._traj_base is None and pl.buf.traj_base is None   # nothing was prepared either


@pytest.mark.parametrize("change", ["allocate", "grow", "set_vel_params", "set_gg_map", "set_local_gg_planes",
                                    "set_subbatches"])
def test_stale_graph_refuses_to_replay(change):
    sc = _scenarios("default", 96, 9900)
    dsc = sc.to_device(DEV)
    pl = D.planner(H.lattice_for("default"), 2, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True)
    D.first_tick(pl, dsc)
    sel = pl.device_results()["action_id"].max(dim=0).values.clamp(min=0)
    graph = pl.capture_next_tick(dsc, sel, 0.1)
    graph.replay()
    if change == "allocate":
        pl.allocate(sc.size + 1, 3)
    elif change == "grow":
        pl.allocate(sc.size, 5)
    elif change == "set_vel_params":
        pl.set_vel_params(**dict(D.VEL, ax_max_machines=_axm(), incl_emerg_traj=True))
    elif change == "set_gg_map":
        pl.set_gg_map(*M.surface_map(MAP[2], x0=MAP[0], y0=MAP[1], width=500.0, height=350.0), *MAP)
    elif change == "set_local_gg_planes":
        pl.set_local_gg_planes(None)
    else:
        pl.set_subbatches(3)
    ticks = pl._tick_count
    _refused(pl, graph.replay, "changed since the capture")
    assert pl._tick_count == ticks
    graph.close()
    with pytest.raises(ValueError, match="closed"):
        graph.replay()


def test_library_refuses_traj_base_misuse_before_launching():
    """buffers.traj_base with params.traj_base_id != 0, and a traj_base that is not 4-byte aligned: every entry point
    with a velocity stage refuses before launching, naming the field"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    sc = _scenarios("default", 64, 9950)
    pl = D.planner(H.lattice_for("default"), 2, stateful=True, ax_max_machines=_axm())
    D.first_tick(pl, sc.to_device(DEV))
    pl.next_tick(sc.to_device(DEV), torch.zeros(64, dtype=torch.int32, device=DEV), 0.1)
    counter = torch.zeros(2, dtype=torch.int32, device=DEV)
    n0 = pl.launch_count()
    for ptr, base, msg in ((counter.data_ptr(), 10, b"traj_base_id"), (counter.data_ptr() + 2, 0, b"aligned")):
        buf, prm = capi.Buffers.from_buffer_copy(pl.buf), capi.Params.from_buffer_copy(pl.params)
        buf.traj_base, prm.traj_base_id = ptr, base
        for name in ("ltpl_tick_batch", "ltpl_calc_vel_profile_batch", "ltpl_next_tick_batch",
                     "ltpl_next_calc_vel_profile_batch"):
            rc = getattr(pl.lib, name)(pl.handle, C.byref(prm), C.byref(pl.dims), C.byref(buf), pl.stream)
            err = pl.lib.ltpl_last_error()
            assert rc < 0 and b"traj_base" in err and msg in err, (name, err)
    assert pl.launch_count() == n0
    assert not counter.any()


def test_null_traj_base_keeps_the_launch_count():
    """with buffers.traj_base NULL a tick issues the launches it always did (4 windows: first tick = k_stage +
    k_startpos + 3 per window; stateful tick = k_stage + 8 per window); once a graph was captured on the planner, its
    eager velocity calls add k_traj_base"""
    sc = _scenarios("default", 128, 9990)
    dsc = sc.to_device(DEV)
    pl = D.planner(H.lattice_for("default"), 4, stateful=True, ax_max_machines=_axm())
    sel = torch.zeros(sc.size, dtype=torch.int32, device=DEV)
    counts = []
    for step in range(2):
        n0 = pl.launch_count()
        D.first_tick(pl, dsc)
        n1 = pl.launch_count()
        pl.next_tick(dsc, sel, 0.1)
        counts.append((n1 - n0, pl.launch_count() - n1))
        if step == 0:
            assert pl.buf.traj_base is None
            pl.capture_next_tick(dsc, sel, 0.1).close()
    assert counts == [(2 + 4 * 3, 1 + 4 * 8), (3 + 4 * 3, 2 + 4 * 8)], counts
