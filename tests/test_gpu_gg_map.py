"""Location dependent friction from a friction map (BatchPlanner.set_gg_map, k_gg_map): the device planes equal the
NumPy evaluation bit for bit, and a tick with the map gives the bytes of the dict form (calc_paths -> planes of the map
along the fetched paths -> set_local_gg_planes -> calc_vel_profile) in first ticks, stateful ticks and every entry point.
The map covers only part of the track, so that points outside it take the border values."""
import numpy as np
import pytest

from tests import drivers as D
from tests import gg_map_ref as M
from tests import helpers as H

pytestmark = pytest.mark.gpu

# a map over the middle of the track only (the race line spans x -531 .. 363 m, y -231 .. 345 m); a cell that is not a
# power of two, so that inv_cell = 1 / cell is rounded
X0, Y0, CELL = -300.0, -150.0, 3.7
MAP = M.surface_map(CELL, x0=X0, y0=Y0, width=500.0, height=350.0)


def _axm(tag="default"):
    return H.golden("ticks_%s.npz" % tag)["ax_max_machines"]


def _scenarios(tag, n, seed):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    track = Track(H.track_csv_for(tag))
    return make_scenarios(track, n, seed=seed, n_obj_min=0, n_obj_max=3,
                          s_max=(track.length - 8.0) if tag == "open" else None)


def _with_map(pl, scale=1.0):
    pl.set_gg_map(MAP[0] * scale, MAP[1] * scale, X0, Y0, CELL)
    return pl


def _dict_form_tick(pl, sc, scale=1.0):
    """set_startpos -> calc_paths -> planes of the map along the fetched paths -> calc_vel_profile"""
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.calc_paths()
    pl.set_local_gg_planes(*M.planes_along(pl, MAP[0] * scale, MAP[1] * scale, X0, Y0, CELL))
    pl.calc_vel_profile()


def _snapshot(pl):
    """every per-path result of the last tick, byte-comparable: tick_snapshot (export rows through traj_row, emergency
    rows) + the path and velocity planes, node indices, trajectory ids and the gg planes, cleared behind path_len and
    n_nodes"""
    snap = D.tick_snapshot(pl, emergency=True)
    f = pl.fetch("path", "path_len", "s_vx_ax", "node_idx", "n_nodes", "traj_id", "gg", "em_info")
    behind = np.arange(f["path"].shape[2])[None, :] >= f["path_len"].reshape(-1)[:, None]
    f["node_idx"][np.arange(f["node_idx"].shape[2])[None, None, :] >= f["n_nodes"][..., None]] = -1
    for k in ("path", "s_vx_ax", "gg"):
        a = f[k].copy()
        a[:, behind] = 0.0
        snap[k] = a
    # em_info: rows and id of the emergency trajectory (its row in the compact export is unspecified)
    snap.update(node_idx=f["node_idx"], traj_id=f["traj_id"], em_info=f["em_info"][None, :, 1:])
    return snap


def _assert_same(a, b, ctx):
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), "%s: '%s' differs" % (ctx, k)


@pytest.mark.parametrize("tag,n,windows", [("default", 256, 1), ("default", 256, 4), ("l216", 203, 3),
                                           ("open", 256, 4), ("open", 131, 1)])
def test_planes_equal_numpy_evaluation(tag, n, windows):
    """t['gg'][:, q, :path_len] of every found path equals the NumPy evaluation of the map at the planned x / y; points
    behind path_len keep what they held"""
    pl = _with_map(D.planner(H.lattice_for(tag), windows, ax_max_machines=_axm(tag)))
    D.first_tick(pl, _scenarios(tag, n, 8100 + n))
    f = pl.fetch("path", "path_len", "gg")
    n_path = f["path_len"].reshape(-1)
    found = np.nonzero(n_path > 0)[0]
    assert found.size > n
    outside = 0
    for q in found:
        k = int(n_path[q])
        x, y = f["path"][0, q, :k], f["path"][1, q, :k]
        gx, gy = M.gg_map_eval(MAP[0], MAP[1], X0, Y0, CELL, x, y)
        assert np.array_equal(f["gg"][0, q, :k], gx) and np.array_equal(f["gg"][1, q, :k], gy), "path %d" % q
        assert np.all(f["gg"][:, q, k:] == 1.0), "path %d: points behind path_len were written" % q
        outside += int(np.any((x < X0) | (x > X0 + 500.0) | (y < Y0) | (y > Y0 + 350.0)))
    assert outside > 0, "no path leaves the map: the clamping is not exercised"
    assert np.all(f["gg"][:, n_path == 0] == 1.0)


@pytest.mark.parametrize("tag,windows", [("default", 4), ("l216", 1)])
def test_tick_with_map_equals_dict_form(tag, windows):
    """tick() with the map == calc_paths -> set_local_gg_planes(map along the fetched paths) -> calc_vel_profile, byte for
    byte, with the emergency trajectory on"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    lat, sc = H.lattice_for(tag), _scenarios(tag, 384, 8200)
    vel = dict(ax_max_machines=_axm(tag), incl_emerg_traj=True)
    pm = _with_map(D.planner(lat, windows, **vel))
    D.first_tick(pm, sc)
    pd = D.planner(lat, windows, **vel)
    _dict_form_tick(pd, sc)
    got, want = _snapshot(pm), _snapshot(pd)
    _assert_same(got, want, tag)
    assert np.sum((got["status"] & capi.ST_TRAJ_VALID) != 0) > sc.size
    assert np.sum(got["em_len"] > 0) > 0
    # the map changes the profiles: the constant tuple gives other velocities
    pc = D.planner(lat, windows, **vel)
    D.first_tick(pc, sc)
    assert not np.array_equal(pc.fetch("s_vx_ax")["s_vx_ax"], pm.fetch("s_vx_ax")["s_vx_ax"])


MAP_OFF_TICKS = (4, 5)   # the map is switched off before tick 4 and on again before tick 6


def test_stateful_closed_loop_equals_split_calls():
    """8 ticks of a closed loop (every scenario drives 0.1 s along its first kept trajectory), grip drops via gg_scale at
    ticks 3 and 6, restarts of some scenarios on ticks 2 and 5, the map switched off between ticks for ticks 4 and 5 and
    on again for tick 6: next_tick with the map == the split calls with the planes evaluated on the host between
    next_calc_paths and next_calc_vel_profile (set_local_gg_planes(None) on ticks 4 and 5), every tick, byte for byte.
    The backup brake of the tick after a switch uses what the last tick's velocity half used: the map's planes on tick 4,
    the constant tuple on tick 6."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    from tools.workload import closed_loop_step
    lat, sc = H.lattice_for("default"), _scenarios("default", 512, 8300)
    vel = dict(ax_max_machines=_axm(), incl_emerg_traj=True)
    pm = _with_map(D.planner(lat, 4, stateful=True, **vel))
    ps = D.planner(lat, 4, stateful=True, **vel)
    D.first_tick(pm, sc)
    _dict_form_tick(ps, sc)
    _assert_same(_snapshot(pm), _snapshot(ps), "first tick")
    rng = np.random.default_rng(8301)
    pos, v = sc.pos.copy(), sc.vel.copy()
    backups = emergencies = restarts = 0
    switch_backups = {}
    for k in range(1, 8):
        p_new, v_new, sel, ok, head = closed_loop_step(pm.fetch("traj_row", "traj_len", "action_id", "traj"), 0.1)
        pos, v = np.where(ok[:, None], p_new, pos), np.where(ok, v_new, v)
        heading = sc.heading.copy()
        heading[ok] = head[ok]
        restart = (rng.random(sc.size) < 0.1) if k in (2, 5) else None
        restarts += 0 if restart is None else int(restart.sum())
        nk = ScenarioBatch(pos.copy(), heading, v.copy(), sc.n_obj, sc.obj)
        if k in (3, 6):
            for pl in (pm, ps):
                pl.set_vel_params(**dict(D.VEL, gg_scale=0.55 if k == 3 else 0.4, **vel))
        if k == MAP_OFF_TICKS[0]:
            pm.set_gg_map(None)
        elif k == MAP_OFF_TICKS[-1] + 1:
            _with_map(pm)
        pm.next_tick(nk, sel, 0.2, vel_est=v, restart=restart)
        ps.next_calc_paths(nk, sel, 0.2, vel_est=v, restart=restart)
        if k in MAP_OFF_TICKS:
            ps.set_local_gg_planes(None)
        else:
            # behind path_len the planes keep what they held in both planners: k_backup's brake on a backup that was
            # itself a backup reads there (the planes follow the path of this tick, not the backup, as uploaded planes
            # do)
            ps.set_local_gg_planes(*M.planes_along(ps, MAP[0], MAP[1], X0, Y0, CELL, keep=True))
        ps.next_calc_vel_profile()
        got = _snapshot(pm)
        _assert_same(got, _snapshot(ps), "tick %d" % k)
        st0, flags = got["status"][0], got["flags"][0]
        both = capi.ST_TRAJ_VALID | capi.ST_VEL_BOUND_VIOL
        n_backup = int(np.sum(((st0 & both) == both) & ((flags & capi.SC_STATE_FALLBACK) == 0)))
        backups += n_backup
        if k in (MAP_OFF_TICKS[0], MAP_OFF_TICKS[-1] + 1):
            switch_backups[k] = n_backup
        emergencies += int(np.sum(got["em_len"] > 0))
    print("closed loop with a friction map: %d backup brakes (%s on the ticks after a switch), %d emergency "
          "trajectories, %d restarts" % (backups, switch_backups, emergencies, restarts))
    assert backups > 0 and emergencies > 0 and restarts > 0
    assert all(n > 0 for n in switch_backups.values()), switch_backups


def test_entry_points():
    """plan_stream with the map gives the bytes of tick() per batch; a map change between calls takes effect;
    set_gg_map(None) gives the bytes of a planner that never had a map; set_local_gg_planes after a map clears it"""
    lat = H.lattice_for("default")
    vel = dict(ax_max_machines=_axm(), incl_emerg_traj=True)
    batches = [_scenarios("default", 200, 8400 + i) for i in range(4)]
    ref = _with_map(D.planner(lat, 4, **vel))
    want = []
    for sc in batches:
        D.first_tick(ref, sc)
        f = ref.fetch("action_id", "status", "traj_len", "traj_id", "traj_row", "traj", "em_info")
        want.append((f, D.export_rows(f, cut=True)))
    pl = _with_map(D.planner(lat, 4, **vel))
    for i, res in enumerate(pl.plan_stream(batches)):
        out = {k: res[k].numpy() for k in ("action_id", "status", "traj_len", "traj_id", "traj_row", "traj")}
        f, rows = want[i]
        for k in ("action_id", "status", "traj_len", "traj_id"):
            assert np.array_equal(out[k], f[k]), "plan_stream batch %d: '%s'" % (i, k)
        got_rows = np.zeros_like(rows)
        ok = out["traj_row"] >= 0
        got_rows[ok] = out["traj"][out["traj_row"][ok]]
        got_rows[np.arange(rows.shape[2])[None, None, :] >= out["traj_len"][..., None]] = 0.0
        assert np.array_equal(got_rows, rows), "plan_stream batch %d: export rows" % i
    sc = batches[0]
    # a map change takes effect on the next call
    _with_map(pl, 0.8)
    D.first_tick(pl, sc)
    fresh = _with_map(D.planner(lat, 4, **vel), 0.8)
    D.first_tick(fresh, sc)
    changed, want_08 = _snapshot(pl), _snapshot(fresh)
    for snap in (changed, want_08):   # trajectory ids count the planner's calls (+10 per call, OTH:669)
        snap["traj_id"] %= 10
        snap["em_info"][..., 1] %= 10
    _assert_same(changed, want_08, "map scaled by 0.8")
    # no map: the bytes of a planner that never had one (no gg planes at all)
    pl.set_gg_map(None)
    D.first_tick(pl, sc)
    never = D.planner(lat, 4, **vel)
    D.first_tick(never, sc)
    assert pl.buf.gg is None and pl.buf.gg_map is None
    a, b = D.tick_snapshot(pl), D.tick_snapshot(never)
    _assert_same(a, b, "set_gg_map(None)")
    # set_local_gg_planes after a map: the uploaded planes are used, the map is gone
    _with_map(pl)
    pl.stage_scenarios(sc)
    pl.upload()
    pl.set_startpos()
    pl.calc_paths()
    const = np.full((3, sc.size, pl.dims.p_max), 4.4), np.full((3, sc.size, pl.dims.p_max), 4.7)
    pl.set_local_gg_planes(*const)
    assert pl.buf.gg_map is None
    pl.calc_vel_profile()
    other = D.planner(lat, 4, **vel)
    other.stage_scenarios(sc)
    other.upload()
    other.set_startpos()
    other.calc_paths()
    other.set_local_gg_planes(*const)
    other.calc_vel_profile()
    _assert_same(D.tick_snapshot(pl), D.tick_snapshot(other), "set_local_gg_planes after a map")


def test_batch_invariance_with_map(monkeypatch):
    """sub-batch, permutation and scenario windows give the same per-scenario bytes with a map"""
    planner = D.planner
    monkeypatch.setattr(D, "planner", lambda *a, **k: _with_map(planner(*a, **k)))
    sc = _scenarios("l216", 300, 8500)
    rng = np.random.default_rng(8501)
    pl = D.assert_batch_invariance(H.lattice_for("l216"), sc, rng.permutation(sc.size),
                                   np.sort(rng.choice(sc.size, 97, replace=False)), ax_max_machines=_axm("l216"))
    assert pl.buf.gg_map is not None


def test_library_refuses_bad_maps_before_launching():
    """a map without gg planes, a map that is not 16-byte aligned and each bad geometry: refused by the C library with the
    field named, nothing launched"""
    pl = _with_map(D.planner(H.lattice_for("default"), 1, ax_max_machines=_axm()))
    sc = _scenarios("default", 64, 8600)
    D.first_tick(pl, sc)
    p, buf = pl.params, pl.buf
    cases = [("gg", None, "buffers.gg"), ("gg_map_nx", 1, "gg_map_nx"), ("gg_map_ny", 0, "gg_map_ny"),
             ("gg_map_nx", 70000, "32-bit"), ("gg_map_inv_cell", 0.0, "gg_map_inv_cell"),
             ("gg_map_inv_cell", -1.0, "gg_map_inv_cell"), ("gg_map_inv_cell", float("inf"), "gg_map_inv_cell"),
             ("gg_map_inv_cell", float("nan"), "gg_map_inv_cell"), ("gg_map_x0", float("nan"), "gg_map_x0"),
             ("gg_map_y0", float("-inf"), "gg_map_y0"), ("gg_map", buf.gg_map + 8, "gg_map must be 16-byte aligned")]
    for field, value, name in cases:
        obj = buf if field in ("gg", "gg_map") else p
        keep = getattr(obj, field)
        setattr(obj, field, value)
        if field == "gg_map_nx" and value == 70000:
            p.gg_map_ny = 70000
        n0 = pl.launch_count()
        for call in (pl.tick, pl.calc_vel_profile):
            with pytest.raises(RuntimeError, match=name):
                call()
        assert pl.launch_count() == n0, field
        setattr(obj, field, keep)
        p.gg_map_ny = MAP[0].shape[0]
    D.first_tick(pl, sc)   # the restored map plans again
