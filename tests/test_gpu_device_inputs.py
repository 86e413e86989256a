"""Scenario inputs that already live on the device (DeviceScenarioBatch, k_stage): staged both ways, the packed device
input buffer holds the same bytes, and every tick entry point gives the bytes of the host path -- first ticks on three
lattices, closed loops over the multi-tick fixtures with sel_action, t_const, vel_est and the restart mask as device
tensors, and a loop that alternates host and device batches.  A device stateful tick does not synchronise with the
host, and malformed inputs are refused before anything launches."""
import numpy as np
import pytest
import torch

from tests import drivers as D
from tests import gg_map_ref as M
from tests import helpers as H

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _axm(tag="default"):
    return H.golden("ticks_%s.npz" % tag)["ax_max_machines"]


def _scenarios(tag, n, seed, omax=3):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    track = Track(H.track_csv_for(tag))
    return make_scenarios(track, n, seed=seed, n_obj_min=0, n_obj_max=omax,
                          s_max=(track.length - 8.0) if tag == "open" else None)


def _with_pred(sc, kp, seed):
    """predictions of kp points on some objects; n_pred -1 (none given) on the others, 0 .. kp points where given"""
    rng = np.random.default_rng(seed)
    B, K = sc.obj.shape[:2]
    sc.n_pred = np.where(rng.random((B, K)) < 0.6, rng.integers(0, kp + 1, size=(B, K)), -1).astype(np.int32)
    t = 0.1 * np.arange(1, kp + 1)
    sc.pred = np.zeros((B, K, kp, 2))
    sc.pred[..., 0] = sc.obj[..., 0:1] - np.sin(sc.obj[..., 2:3]) * sc.obj[..., 3:4] * t
    sc.pred[..., 1] = sc.obj[..., 1:2] + np.cos(sc.obj[..., 2:3]) * sc.obj[..., 3:4] * t
    return sc


def _with_zones(sc, tag, seed):
    from oracle.gen_golden import make_zone
    rng = np.random.default_rng(seed)
    sc.set_zones([{"zone_%d" % b: make_zone(H.lattice_for(tag), rng, sc.pos[b])} if b % 2 == 0 else None
                  for b in range(sc.size)])
    return sc


def _strided(dsc):
    """the same values read through strides: pos as the transpose of a [2][B] tensor, obj inside a wider tensor with
    three extra columns in front and behind"""
    B, K = dsc.obj.shape[:2]
    pos_t = dsc.pos.t().contiguous()
    wide = torch.full((B, K, 11), -7.5, dtype=torch.float64, device=DEV)
    wide[:, :, 3:8] = dsc.obj
    dsc.pos, dsc.obj = pos_t.t(), wide[:, :, 3:]
    assert not dsc.pos.is_contiguous() and dsc.obj.shape[2] == 8
    return dsc


def _outputs(pl):
    """every result of the last tick, byte-comparable: tick_snapshot (export rows gathered through traj_row, whose order
    is unspecified, and emergency rows) + start, constant segment, path and velocity planes cleared behind path_len,
    node indices behind n_nodes, ids and the memory records of a stateful planner"""
    snap = D.tick_snapshot(pl, emergency=True)
    names = ["path", "path_len", "s_vx_ax", "node_idx", "n_nodes", "traj_id", "em_info", "start_node", "const_len",
             "const_seg", "closest_obj", "cobj"]
    if "trim" in pl.t and pl._state is not None:
        names.append("trim")
    f = pl.fetch(*names)
    behind = np.arange(f["path"].shape[2])[None, :] >= f["path_len"].reshape(-1)[:, None]
    f["node_idx"][np.arange(f["node_idx"].shape[2])[None, None, :] >= f["n_nodes"][..., None]] = -1
    for k in ("path", "s_vx_ax"):
        f[k] = f[k].copy()
        f[k][:, behind] = 0.0
    f["em_info"] = f["em_info"][None, :, 1:]
    for k in ("path_len", "n_nodes"):
        f.pop(k)
    snap.update(f)
    return snap


def _assert_same(a, b, ctx):
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), "%s: '%s' differs" % (ctx, k)


def _assert_inputs_equal(ph, pd, ctx, stale_pred=False):
    """the packed device inputs of both planners byte for byte; stale_pred: all but obj_pred, which a host batch without
    predictions leaves as the last batch with predictions staged it and k_stage zero-fills (unread: dims.k_pred = 0)"""
    torch.cuda.synchronize()
    assert ph.d_in_raw.numel() == pd.d_in_raw.numel(), ctx
    if not stale_pred:
        assert torch.equal(ph.d_in_raw, pd.d_in_raw), "%s: the packed device inputs differ" % ctx
        return
    assert pd.dims.k_pred == ph.dims.k_pred == 0
    views_h, views_d = ph.d_in[ph._in_cur][1], pd.d_in[pd._in_cur][1]
    for name in views_h:
        if name != "obj_pred":
            assert torch.equal(views_h[name], views_d[name]), "%s: '%s' differs" % (ctx, name)
    assert not pd.t["obj_pred"].any()


def _stage_both(ph, pd, sc, dsc, ctx, vel_est=None, stale_pred=False):
    ph.stage_scenarios(sc, vel_est=vel_est)
    ph.upload()
    pd.stage_scenarios(dsc, vel_est=None if vel_est is None else torch.as_tensor(vel_est, device=DEV))
    pd.upload()
    _assert_inputs_equal(ph, pd, ctx, stale_pred)


@pytest.mark.parametrize("case", ["fewer_slots", "pred", "zones", "strided", "grow"])
def test_staged_inputs_are_byte_equal(case):
    """d_in_raw after stage_scenarios + upload of the same batch as ScenarioBatch and as DeviceScenarioBatch"""
    lat = H.lattice_for("default")
    ph, pd = (D.planner(lat, 4, ax_max_machines=_axm(), incl_emerg_traj=True) for _ in range(2))
    sc = _scenarios("default", 160, 9100, omax=3)
    vel_est = None
    if case == "fewer_slots":        # 3 of 6 allocated object slots: the slots behind are zero-filled
        for pl in (ph, pd):
            pl.allocate(sc.size, 6)
        vel_est = sc.vel * 0.9
    elif case == "pred":
        _with_pred(sc, 9, 9101)
    elif case == "zones":
        _with_zones(sc, "default", 9102)
    dsc = sc.to_device(DEV)
    if case == "strided":
        dsc = _strided(dsc)
    _stage_both(ph, pd, sc, dsc, case, vel_est)
    if case == "fewer_slots":
        assert pd.dims.k_obj == 6
    if case == "grow":                # more object slots and prediction points than allocated: the inputs grow
        big = _with_pred(_scenarios("default", 160, 9103, omax=5), 4, 9104)
        _stage_both(ph, pd, big, big.to_device(DEV), "grown")
        assert pd.dims.k_obj == 5 and pd._k_pred_cap == 4
        _stage_both(ph, pd, sc, sc.to_device(DEV), "back to 3 objects", stale_pred=True)
    for pl in (ph, pd):
        pl.set_startpos()
        pl.tick()
    _assert_same(_outputs(pd), _outputs(ph), case)


@pytest.mark.parametrize("tag,n,windows", [("default", 384, 4), ("l216", 257, 3), ("open", 200, 1)])
def test_first_tick_equals_host_path(tag, n, windows):
    """set_startpos + tick from a device batch (predictions on the default lattice, zones on l216) == the host path,
    every result buffer"""
    lat = H.lattice_for(tag)
    vel = dict(ax_max_machines=_axm(tag), incl_emerg_traj=True)
    sc = _scenarios(tag, n, 9200 + n)
    if tag == "default":
        _with_pred(sc, 12, 9201)
    if tag == "l216":
        _with_zones(sc, tag, 9202)
    ph, pd = D.planner(lat, windows, **vel), D.planner(lat, windows, **vel)
    D.first_tick(ph, sc)
    D.first_tick(pd, sc.to_device(DEV), vel_est=torch.as_tensor(sc.vel, device=DEV))
    got, want = _outputs(pd), _outputs(ph)
    _assert_same(got, want, tag)
    assert (want["traj_len"] > 0).sum() > n


def test_facade_plan_batch_takes_a_device_batch(tmp_path):
    """Graph_LTPL.set_startpos_batch and plan_batch take a DeviceScenarioBatch and plan what the host batch plans"""
    ltpl = D.facade(tmp_path)
    sc = _scenarios("default", 96, 9250)
    keys = ("action_id", "status", "traj_len", "traj_id", "sc_flags")
    want = {k: v.numpy().copy() for k, v in ltpl.plan_batch(sc).items() if k in keys}
    ltpl.set_startpos_batch(sc.to_device(DEV))
    ltpl.calc_paths_batch()
    got = ltpl.calc_vel_profile_batch()
    for k in keys:   # trajectory ids count the calls (+10 per call, OTH:669)
        w = want[k] + (10 * (want[k] >= 0) if k == "traj_id" else 0)
        assert np.array_equal(got[k].numpy(), w), k
    got = ltpl.plan_batch(sc.to_device(DEV))
    assert np.array_equal(got["traj_len"].numpy(), want["traj_len"])


# ---- closed loops over the multi-tick fixtures ----------------------------------------------------------------------
def _fixture_inputs(g, kind, k, tc):
    """ScenarioBatch, sel_action, t_const, vel_est, restart mask and gg_scale of tick k"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    n_seq = g["dt"].shape[0]
    if kind == "restart":
        sc = ScenarioBatch(g["pos"][:, k].copy(), g["heading"][:, k].copy(), g["vel"][:, k].copy(),
                           g["sc_n_obj"].copy(), g["obj"][:, k].copy())
        return sc, g["sel"][:, k], g["t_const"][:, k], g["vel_est"][:, k], g["restart"][:, k] > 0, \
            float(g["gg_scale"][:, k].min())
    sc = ScenarioBatch(g["pos_est"][:, k].copy(), g["sc_heading"].copy(), g["sc_vel"].copy(), g["sc_n_obj"].copy(),
                       g["obj"][:, k].copy())
    zones = [H.zone_of(g, q, k) for q in range(n_seq)]
    if any(z is not None for z in zones):
        sc.set_zones(zones)
    return sc, g["sel"][:, k], tc[:, k - 1] if k else None, g["vel_est"][:, k], None, float(g["gg_scale"][0, k])


MAP = (-300.0, -150.0, 3.7)


@pytest.mark.parametrize("fixture,tag,emerg,kind", [
    ("ticks_multitick_ext_default.npz", "default", True, "next_tick"),         # zones + emergency trajectory
    ("ticks_multitick_zswap_default.npz", "default", False, "next_tick"),      # zone id changes
    ("ticks_multitick_restart_default.npz", "default", True, "restart"),       # restart masks
    ("ticks_multitick_ggpp_default.npz", "default", True, "ggpp"),             # planes between the two halves
    ("ticks_multitick_ggpp_default.npz", "default", True, "map"),              # friction map, grip drops
    ("ticks_multitick_zswap_default.npz", "default", False, "alternate"),      # host and device batches in turn
    ("ticks_multitick_ext_default.npz", "default", True, "alternate")])
def test_closed_loop_replay_equals_host_path(fixture, tag, emerg, kind):
    """the fixture's inputs replayed on two stateful planners, one fed ScenarioBatch + NumPy arguments, the other
    DeviceScenarioBatch + device tensors (sel_action int64 / int32, t_const, vel_est, restart bool): the packed inputs
    and every result are byte-equal after every tick.  'alternate': the second planner takes host inputs on odd ticks."""
    g = H.golden(fixture)
    n_seq, n_ticks = g["dt"].shape
    lat = H.lattice_for(tag)
    vel = dict(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emerg)
    ph, pd = (D.planner(lat, 1 + n_seq % 4, stateful=True, **vel) for _ in range(2))
    if kind == "map":
        ax, ay = M.surface_map(MAP[2], x0=MAP[0], y0=MAP[1], width=500.0, height=350.0)
        for pl in (ph, pd):
            pl.set_gg_map(ax, ay, *MAP)
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)]) if kind != "restart" else None
    ggpp = kind == "ggpp"
    dev = lambda a, dt=None: None if a is None else torch.as_tensor(np.asarray(a, dtype=dt), device=DEV)  # noqa: E731
    n_traj = 0
    for k in range(n_ticks):
        sc, sel, t_c, v_est, restart, gg_scale = _fixture_inputs(g, kind, k, tc)
        for pl in (ph, pd):
            pl.set_vel_params(**dict(D.VEL, gg_scale=gg_scale, **vel))
        on_device = not (kind == "alternate" and k % 2 == 1)
        dsc = sc.to_device(DEV) if on_device else sc
        d_sel = dev(sel, np.int64 if k % 2 else np.int32) if on_device else sel
        d_tc, d_vel = (dev(t_c, np.float64), dev(v_est, np.float64)) if on_device else (t_c, v_est)
        d_restart = dev(restart, bool) if on_device else restart
        if k == 0:
            D.first_tick(ph, sc, vel_est=v_est, gg=ggpp)
            D.first_tick(pd, dsc, vel_est=d_vel, gg=ggpp)
        elif ggpp:
            ph.next_calc_paths(sc, sel, t_c)
            pd.next_calc_paths(dsc, d_sel, d_tc)
            _assert_inputs_equal(ph, pd, "tick %d" % k)
            for pl in (ph, pd):
                pl.set_local_gg_planes(*H.local_gg_planes(pl))
            ph.next_calc_vel_profile(pos_est=g["pos_est"][:, k], vel_est=v_est)
            pd.next_calc_vel_profile(pos_est=dev(g["pos_est"][:, k]) if on_device else g["pos_est"][:, k],
                                     vel_est=d_vel)
        else:
            ph.next_tick(sc, sel, t_c, vel_est=v_est, restart=restart)
            pd.next_tick(dsc, d_sel, d_tc, vel_est=d_vel, restart=d_restart)
            _assert_inputs_equal(ph, pd, "tick %d" % k)
        got, want = _outputs(pd), _outputs(ph)
        _assert_same(got, want, "tick %d" % k)
        n_traj += int((want["traj_len"] > 0).sum())
    assert n_traj > n_seq * n_ticks


# ---- results on the device, synchronisation, refusals ---------------------------------------------------------------
def _stateful_device_planner(n=128, seed=9300):
    sc = _with_zones(_scenarios("default", n, seed), "default", seed + 1)
    pl = D.planner(H.lattice_for("default"), 4, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True)
    dsc = sc.to_device(DEV)
    D.first_tick(pl, dsc)
    return pl, sc, dsc


def _next_sel(pl):
    """an action every scenario's last tick returned, computed on the device from device_results()"""
    return pl.device_results()["action_id"].max(dim=0).values.clamp(min=0)


def test_device_results_equal_fetch():
    pl, sc, dsc = _stateful_device_planner()
    for step in range(2):
        r = pl.device_results()
        f = pl.fetch(*pl.DEVICE_RESULTS, "traj")
        for k in pl.DEVICE_RESULTS + ("traj",):
            assert r[k].device == torch.device(DEV)
            assert np.array_equal(r[k].cpu().numpy(), f[k]), "tick %d: %s" % (step, k)
        pl.next_tick(dsc, _next_sel(pl), 0.2)


def test_device_stateful_tick_does_not_synchronise():
    """a device next_tick with zones, restarts and every per-scenario argument a device tensor, the next sel_action
    computed from device_results(), under torch.cuda.set_sync_debug_mode('error')"""
    pl, sc, dsc = _stateful_device_planner()
    B = sc.size
    restart = torch.zeros(B, dtype=torch.bool, device=DEV)
    restart[::7] = True
    vel_est = dsc.vel * 0.95
    t_const = torch.full((B,), 0.15, dtype=torch.float64, device=DEV)
    pl.next_tick(dsc, _next_sel(pl), t_const, vel_est=vel_est, restart=restart)   # buffers of the restart mask exist
    n0 = pl.launch_count()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sel = _next_sel(pl)
        pl.next_tick(dsc, sel, t_const, vel_est=vel_est, restart=restart)
        pl.next_calc_paths(dsc, _next_sel(pl), 0.1, vel_est=vel_est)
        pl.next_calc_vel_profile(pos_est=dsc.pos, vel_est=vel_est)
        res = pl.device_results()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert pl.launch_count() > n0
    assert int(res["queue_cnt"][2]) > 0


def test_bad_inputs_are_refused_before_launching():
    """device, dtype, dimensionality, batch size, object slots, obj columns, pred without n_pred and each tick argument:
    ValueError, nothing launched, and the planner plans on afterwards"""
    from dataclasses import replace
    pl, sc, dsc = _stateful_device_planner(64, 9400)
    B = sc.size
    sel = torch.zeros(B, dtype=torch.int32, device=DEV)
    big = pl.max_objects + 1
    batches = [replace(dsc, pos=dsc.pos.cpu()), replace(dsc, pos=dsc.pos.float()),
               replace(dsc, heading=dsc.heading[:, None]), replace(dsc, vel=dsc.vel[:-1]),
               replace(dsc, n_obj=dsc.n_obj.long()), replace(dsc, obj=dsc.obj[:, :, :4]),
               replace(dsc, obj=torch.zeros((B, big, 5), dtype=torch.float64, device=DEV),
                       n_obj=torch.zeros(B, dtype=torch.int32, device=DEV)),
               replace(dsc, pred=torch.zeros((B, dsc.obj.shape[1], 3, 2), dtype=torch.float64, device=DEV)),
               replace(dsc, zone_key=dsc.zone_key.int()), replace(dsc, zone_sel=dsc.zone_sel.cpu())]
    args = [dict(sel_action=sel.float()), dict(sel_action=sel[:-1]), dict(t_const=torch.zeros(B, device=DEV)),
            dict(vel_est=dsc.vel.cpu()), dict(restart=torch.zeros((B, 1), dtype=torch.bool, device=DEV)),
            dict(sel_action=None)]
    n0 = pl.launch_count()
    for bad in batches:
        with pytest.raises(ValueError):
            pl.next_tick(bad, sel, 0.1)
        with pytest.raises(ValueError):
            pl.stage_scenarios(bad)
    for kw in args:
        with pytest.raises(ValueError):
            pl.next_tick(dsc, **dict(dict(sel_action=sel, t_const=0.1), **kw))
    with pytest.raises(ValueError):
        list(pl.plan_stream([dsc]))
    assert pl.launch_count() == n0
    pl.next_tick(dsc, _next_sel(pl), 0.1)
    assert (pl.fetch("traj_len")["traj_len"] > 0).sum() > B


def test_subset_and_round_trip():
    sc = _with_zones(_with_pred(_scenarios("default", 50, 9500), 5, 9501), "default", 9502)
    dsc = sc.to_device(DEV)
    back = dsc.cpu()
    for name in ("pos", "heading", "vel", "n_obj", "obj", "zone_sel", "zone_key", "pred", "n_pred"):
        a, b = getattr(sc, name), getattr(back, name)
        assert a.dtype == b.dtype and np.array_equal(a, b), name
    idx = torch.tensor([3, 1, 40, 7], device=DEV)
    part = dsc.subset(idx).cpu()
    want = sc.subset(idx.cpu().numpy())
    for name in ("pos", "obj", "zone_key", "pred", "n_pred"):
        assert np.array_equal(getattr(part, name), getattr(want, name)), name
    assert part.zones is sc.zones
