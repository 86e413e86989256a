"""Restarts of single scenarios inside a stateful tick (BatchPlanner.next_tick(..., restart=mask), buffers.restart):
the restarted scenarios are planned like the first tick after set_startpos, every other scenario keeps its memory and
gets the bytes of the same tick without restarts (DESIGN.md section 11)."""
import functools

import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H

pytestmark = pytest.mark.gpu

@functools.lru_cache(maxsize=None)
def _track(tag):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    return Track(H.track_csv_for(tag))


def _axm():
    return H.golden("ticks_multitick_default.npz")["ax_max_machines"]


def _stateful(tag, windows, online=None, **vel):
    """a stateful planner on the lattice `tag` (ax_max_machines of the multi-tick fixtures)"""
    return D.planner(H.lattice_for(tag), windows, stateful=True, online=online, ax_max_machines=_axm(), **vel)


def _next_tick(pl, sc, sel, tc, vel_est, restart=None, gg=False):
    if gg:
        pl.next_calc_paths(sc, sel_action=sel, t_const=tc, vel_est=vel_est, restart=restart)
        pl.set_local_gg_planes(*H.local_gg_planes(pl))
        pl.next_calc_vel_profile()
    else:
        pl.next_tick(sc, sel_action=sel, t_const=tc, vel_est=vel_est, restart=restart)


def _state(pl):
    """every output plane and every memory buffer of the last tick, per scenario b (axis 1 of the returned arrays) --
    the export rows gathered through traj_row (their order in the compact buffer is unspecified)"""
    B, NS = pl.dims.batch, 3
    f = pl.fetch("sc_flags", "start_node", "const_len", "action_id", "status", "n_nodes", "nodes", "node_idx",
                 "closest_obj", "cobj", "cobj_start", "path_len", "path", "coeff", "s_vx_ax", "traj", "traj_len",
                 "traj_id", "traj_row", "trim", "em_info", "em_vx")
    st = {k: pl._state[k].cpu().numpy() for k in ("st_info", "vel_plan", "course", "obj_dist", "zone_s0")}
    rows = D.export_rows(f)
    em = np.zeros((1, B) + f["traj"].shape[1:], dtype=np.float32)
    emk = f["em_info"][:, 0] >= 0
    em[0, emk] = f["traj"][f["em_info"][emk, 0]]
    P, Hm = pl.dims.p_max, pl.dims.h_max
    out = dict(sc_flags=f["sc_flags"][None], start_node=f["start_node"][None], const_len=f["const_len"][None],
               closest_obj=f["closest_obj"][None], cobj=f["cobj"][None], cobj_start=f["cobj_start"][None],
               action_id=f["action_id"], status=f["status"], n_nodes=f["n_nodes"], nodes=f["nodes"],
               node_idx=f["node_idx"], path_len=f["path_len"], traj_len=f["traj_len"], traj_id=f["traj_id"],
               path=f["path"].reshape(5, NS, B, P).transpose(1, 0, 2, 3).reshape(NS * 5, B, P),   # [5 s + plane]
               s_vx_ax=f["s_vx_ax"].reshape(3, NS, B, P).transpose(1, 0, 2, 3).reshape(NS * 3, B, P),
               coeff=f["coeff"].reshape(NS, B, Hm, 8), trim=f["trim"].reshape(NS, B, 4), rows=rows,
               em_info=f["em_info"][None, :, 1:],   # (without the unspecified row of the compact export)
               em_rows=em, em_vx=f["em_vx"][None],
               st_info=st["st_info"][None], vel_plan=st["vel_plan"][None], course=st["course"][None],
               obj_dist=st["obj_dist"][None], zone_s0=st["zone_s0"][None])
    return out


class Loop(object):
    """closed loop driven by the device results: the vehicle dummy of oracle/gen_golden.py on the first kept trajectory
    of a rotating action preference, moving opponents, t_const from the moving average of the tick times (as the
    session oracle forms it; a restarted scenario's buffer is kept, OTH:62)"""
    PREFER = ((3, 2, 0, 1), (1, 0, 2, 3), (2, 3, 1, 0), (0, 1, 3, 2))

    def __init__(self, sc0, seed):
        self.sc = sc0
        self.obj = sc0.obj.copy()
        self.pos, self.vel_est = sc0.pos.copy(), sc0.vel.copy()
        self.heading, self.vel = sc0.heading.copy(), sc0.vel.copy()
        self.sel = np.zeros(sc0.size, dtype=np.int32)
        self.rows = None
        self.cbuf = [[] for _ in range(sc0.size)]
        self.tc = np.zeros(sc0.size)
        self.rng = np.random.default_rng(seed)
        self.k = 0
        self.dts = []

    def batch(self):
        from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
        sc = ScenarioBatch(self.pos.copy(), self.heading.copy(), self.vel.copy(), self.sc.n_obj.copy(), self.obj.copy(),
                           pred=None if self.sc.pred is None else self.sc.pred.copy(),
                           n_pred=None if self.sc.n_pred is None else self.sc.n_pred.copy())
        if self.sc.zones is not None:
            sc.zones, sc.zone_sel, sc.zone_key = self.sc.zones, self.sc.zone_sel, self.sc.zone_key
        return sc

    def advance(self):
        """the inputs of the next tick from the last tick's results (self.rows)"""
        from oracle.gen_golden import advance_on_traj
        B = self.sc.size
        dts = self.rng.uniform(0.04, 0.16, size=B)
        self.dts.append(dts)
        self.prev_cbuf = [list(c) for c in self.cbuf]
        for j in range(self.obj.shape[1]):
            live = j < self.sc.n_obj
            self.obj[live, j, 0] -= np.sin(self.obj[live, j, 2]) * self.obj[live, j, 3] * dts[live]
            self.obj[live, j, 1] += np.cos(self.obj[live, j, 2]) * self.obj[live, j, 3] * dts[live]
        aid, tl, rows = self.rows
        for b in range(B):
            for a in self.PREFER[(b + self.k) % 4]:
                s = [i for i in range(3) if aid[i, b] == a and tl[i, b] > 0]
                if s:
                    traj = rows[s[0], b, :tl[s[0], b]].astype(np.float64)
                    self.sel[b] = a
                    if traj.shape[0] >= 2:
                        self.pos[b], self.vel_est[b] = advance_on_traj(traj, float(dts[b]))
                    break
            if len(self.cbuf[b]) >= 5:
                self.cbuf[b].pop(0)
            self.cbuf[b].append(float(dts[b]))
            self.tc[b] = min(float(np.sum(self.cbuf[b]) / len(self.cbuf[b])) * 2.0, 0.5)
        self.k += 1

    def take(self, pl):
        f = pl.fetch("action_id", "traj_len", "traj_row", "traj")
        self.rows = (f["action_id"], f["traj_len"], D.export_rows(f))

    def restart(self, mask, new_pos, new_heading, new_vel):
        self.pos[mask], self.heading[mask], self.vel[mask] = new_pos, new_heading, new_vel
        self.vel_est[mask] = new_vel
        for b in np.nonzero(mask)[0]:   # the restart tick keeps no constant segment: nothing enters the buffer
            self.cbuf[b] = self.prev_cbuf[b]


def _reanchor_heading(rows, b, sel, pos):
    aid, tl, r = rows
    s = [i for i in range(3) if aid[i, b] == sel and tl[i, b] > 0]
    if not s:
        return None
    t = r[s[0], b, :tl[s[0], b]].astype(np.float64)
    return float(t[int(np.argmin(np.hypot(t[:, 1] - pos[0], t[:, 2] - pos[1]))), 3])


def _new_poses(loop, mask, tag, seed, jump_share=0.5):
    """half of the restarted scenarios re-anchored at their position estimate (heading of the driven trajectory there,
    velocity estimate), the others sent to a seeded new start with another start velocity"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_scenarios
    idx = np.nonzero(mask)[0]
    far = make_scenarios(_track(tag), max(idx.size, 1), seed=seed, n_obj_min=0, n_obj_max=0)
    pos, head, vel = far.pos[:idx.size].copy(), far.heading[:idx.size].copy(), far.vel[:idx.size].copy()
    for i, b in enumerate(idx):
        h = _reanchor_heading(loop.rows, b, loop.sel[b], loop.pos[b])
        if i >= int(jump_share * idx.size) and h is not None:
            pos[i], head[i], vel[i] = loop.pos[b], h, loop.vel_est[b]
    return pos, head, vel


def _light(pl):
    """what the session-oracle comparison reads of the last tick (without the large planes)"""
    f = pl.fetch("sc_flags", "action_id", "status", "n_nodes", "nodes", "traj_len", "traj_row", "traj")
    return dict(sc_flags=f["sc_flags"][None], action_id=f["action_id"], status=f["status"], n_nodes=f["n_nodes"],
                nodes=f["nodes"], traj_len=f["traj_len"], rows=D.export_rows(f))


def _assert_scenarios_equal(got, want, idx, ctx, id_shift=0, exact=True):
    """scenarios idx of two _state() results: discrete results exact, path planes bitwise, velocity planes and exported
    rows bitwise (exact=True) or at the parity tolerance"""
    ns = got["action_id"].shape[0]
    for name in ("sc_flags", "start_node", "const_len", "closest_obj", "action_id", "status", "n_nodes", "path_len",
                 "traj_len"):
        assert np.array_equal(got[name][:, idx], want[name][:, idx]), "%s: %s" % (ctx, name)
    tid_g, tid_w = got["traj_id"][:, idx], want["traj_id"][:, idx]
    assert np.array_equal(tid_g >= 0, tid_w >= 0), ctx + ": traj_id presence"
    assert np.array_equal(tid_g[tid_g >= 0] - id_shift, tid_w[tid_w >= 0]), ctx + ": traj_id"
    for i, b in enumerate(idx):
        for s in range(ns):
            nn, n, tl = int(want["n_nodes"][s, b]), int(want["path_len"][s, b]), int(want["traj_len"][s, b])
            c = "%s scenario %d slot %d" % (ctx, b, s)
            assert np.array_equal(got["nodes"][s, b, :nn], want["nodes"][s, b, :nn]), c + " nodes"
            assert np.array_equal(got["node_idx"][s, b, :nn], want["node_idx"][s, b, :nn]), c + " node_idx"
            if nn:
                assert np.array_equal(got["coeff"][s, b, :max(nn - 1, 1)], want["coeff"][s, b, :max(nn - 1, 1)]), \
                    c + " coeff"
            for p in range(5):
                assert np.array_equal(got["path"][5 * s + p, b, :n], want["path"][5 * s + p, b, :n]), c + " path"
            if tl == 0:
                continue
            g_rows, w_rows = got["rows"][s, b, :tl], want["rows"][s, b, :tl]
            g_sv = np.stack([got["s_vx_ax"][3 * s + p, b, :tl] for p in range(3)])
            w_sv = np.stack([want["s_vx_ax"][3 * s + p, b, :tl] for p in range(3)])
            if exact:
                assert np.array_equal(g_sv, w_sv), c + " s_vx_ax"
                assert np.array_equal(g_rows, w_rows), c + " exported rows"
            else:
                H.assert_close("rows", g_rows.astype(np.float64), w_rows.astype(np.float64), D.EXPORT_COLS, c)


def _snap_equal(a, b, idx, ctx):
    for name in a:
        assert np.array_equal(a[name][:, idx], b[name][:, idx]), "%s: %s differs" % (ctx, name)


# ---- 1. the reference's restart sequences -------------------------------------------------------------------------------
@pytest.mark.parametrize("fixture,tag,windows", [("ticks_multitick_restart_default.npz", "default", 1),
                                                 ("ticks_multitick_restart_default.npz", "default", 3),
                                                 ("ticks_multitick_restart_l216.npz", "l216", 2),
                                                 ("ticks_multitick_restart_l216.npz", "l216", 4)])
def test_restart_sequences_match_reference(fixture, tag, windows):
    """the 12 sequences of a fixture as ONE batch: tick 0 = set_startpos + tick, later ticks = next_tick with the
    recorded restart mask, poses and the t_const the reference used; node sequences exact, trajectories at the parity
    tolerance, ids: one counter for the batch (+10 per tick, restarts do not reset it), action part as the reference's"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    g = H.golden(fixture)
    n_seq, n_ticks = g["dt"].shape
    pl = _stateful(tag, windows, incl_emerg_traj=True)
    compared, revived = 0, 0
    rejected_last = g["rejected"][:, 0] > 0
    for k in range(n_ticks):
        sc = ScenarioBatch(g["pos"][:, k].copy(), g["heading"][:, k].copy(), g["vel"][:, k].copy(),
                           g["sc_n_obj"].copy(), g["obj"][:, k].copy())
        pl.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True,
                          **dict(D.VEL, gg_scale=float(g["gg_scale"][:, k].min())))
        if k == 0:
            D.first_tick(pl, sc, g["vel_est"][:, k])
        else:
            _next_tick(pl, sc, g["sel"][:, k], g["t_const"][:, k], g["vel_est"][:, k], restart=g["restart"][:, k] > 0)
        recs = pl.records()
        for q in range(n_seq):
            ctx = "sequence %d tick %d" % (q, k)
            rec = recs[q]
            if g["restart"][q, k]:
                rejected_last[q] = bool(g["rejected"][q, k])
            if not g["planned"][q, k]:
                if rejected_last[q]:
                    assert rec["out_of_track"], ctx + ": a rejected pose stays flagged until a later restart"
                continue
            assert rec["flags"] == 0, "%s: flags %d" % (ctx, rec["flags"])
            revived += int(bool(g["restart"][q, k]) and k > 0 and bool(g["rejected"][q, :k].any()))
            compared += D.compare_multitick_row(rec, g, q, k, ctx, True)
            for a, act in enumerate(H.ACTIONS):   # one id counter for the batch: +10 per tick, restarts do not reset it
                if act in rec["traj"]:
                    assert rec["ids"][act] == 10 * (k + 1) + a, ctx + " id " + act
                    assert rec["ids"][act] % 10 == int(g["traj_id"][q, k, a]) % 10, ctx + " id " + act
    assert compared > 120 and revived >= 2, (compared, revived)


# ---- 2. + 6. a restart is a fresh first tick ---------------------------------------------------------------------------
def _feature_batch(tag, B, feature, seed):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_scenarios
    from oracle.gen_golden import make_zone
    if feature == "manyobj":
        sc = make_scenarios(_track(tag), B, seed=seed, n_obj_min=33, n_obj_max=40, ahead=(20.0, 600.0))
    else:
        sc = make_scenarios(_track(tag), B, seed=seed, n_obj_min=1, n_obj_max=3)
    if feature == "zone":
        rng = np.random.default_rng(seed + 5)
        sc.set_zones([{"zone_%d" % b: make_zone(H.lattice_for(tag), rng, sc.pos[b])} if b % 2 == 0 else None
                      for b in range(B)])
    if feature == "pred":
        rng = np.random.default_rng(seed + 6)
        K, KP = sc.obj.shape[1], 12
        sc.n_pred = np.where(rng.random((B, K)) < 0.6, rng.integers(0, KP + 1, size=(B, K)), -1).astype(np.int32)
        t = 0.1 * np.arange(1, KP + 1)
        sc.pred = np.zeros((B, K, KP, 2))
        sc.pred[..., 0] = sc.obj[..., 0:1] - np.sin(sc.obj[..., 2:3]) * sc.obj[..., 3:4] * t
        sc.pred[..., 1] = sc.obj[..., 1:2] + np.cos(sc.obj[..., 2:3]) * sc.obj[..., 3:4] * t
    return sc


FEATURES = [("default", "plain", 512), ("l216", "plain", 512), ("default", "zone", 256), ("default", "smooth5", 256),
            ("default", "local_gg", 256), ("default", "pred", 256), ("default", "manyobj", 128)]


@pytest.mark.parametrize("tag,feature,B", FEATURES)
def test_restart_equals_fresh_first_tick(tag, feature, B):
    """3 stateful ticks, then a random third of the batch restarts (half re-anchored at the estimate, half sent to a
    new start): every restarted scenario gets what a second planner's set_startpos + tick gives on the same inputs
    (ids up to the call counter).  Features: a zone (unblock window evaluated anew), smoothing window 5, local_gg planes,
    prediction arrays, more than 32 objects."""
    online = dict(filt_window_width=5) if feature == "smooth5" else None
    gg = feature == "local_gg"
    seed = 4100 + 7 * FEATURES.index((tag, feature, B))
    sc0 = _feature_batch(tag, B, feature, seed)
    pl = _stateful(tag, 4, online=online, incl_emerg_traj=True)
    loop = Loop(sc0, seed + 1)
    D.first_tick(pl, loop.batch(), loop.vel_est, gg)
    loop.take(pl)
    for _ in range(3):
        loop.advance()
        _next_tick(pl, loop.batch(), loop.sel, loop.tc, loop.vel_est, gg=gg)
        loop.take(pl)
    loop.advance()
    mask = np.random.default_rng(seed + 2).random(B) < 1.0 / 3.0
    loop.restart(mask, *_new_poses(loop, mask, tag, seed + 3))
    sc = loop.batch()
    _next_tick(pl, sc, loop.sel, loop.tc, loop.vel_est, restart=mask, gg=gg)
    fresh = _stateful(tag, 4, online=online, incl_emerg_traj=True)
    D.first_tick(fresh, sc, loop.vel_est, gg)
    got, want = _state(pl), _state(fresh)
    idx = np.nonzero(mask)[0]
    assert (want["traj_len"][:, idx] > 0).any(axis=0).sum() >= 0.9 * idx.size
    _assert_scenarios_equal(got, want, idx, "%s %s restart" % (tag, feature), id_shift=10 * 4)
    if feature == "zone":   # the zone is processed anew at the restart: zone_s0 = the new start layer
        zs = got["zone_s0"][0, idx]
        assert np.array_equal(zs, want["zone_s0"][0, idx]) and (zs[sc0.zone_sel[idx] >= 0] >= 0).all()


# ---- 3. isolation, 4. edge masks, 7. split calls ---------------------------------------------------------------------
def _twin_loop(tag, B, seed, n_before=3):
    """two planners with identical histories (first tick + n_before stateful ticks)"""
    sc0 = _feature_batch(tag, B, "plain", seed)
    a, c = _stateful(tag, 4, incl_emerg_traj=True), _stateful(tag, 4, incl_emerg_traj=True)
    loop = Loop(sc0, seed + 1)
    for pl in (a, c):
        D.first_tick(pl, loop.batch(), loop.vel_est)
    loop.take(a)
    for _ in range(n_before):
        loop.advance()
        for pl in (a, c):
            _next_tick(pl, loop.batch(), loop.sel, loop.tc, loop.vel_est)
        loop.take(a)
    loop.advance()
    return a, c, loop


def test_restart_leaves_other_scenarios_byte_identical():
    """the same tick with and without restarts from identical states: every scenario that is not restarted has the
    same bytes in every output plane, every memory buffer and its exported rows -- in the restart tick and in the next
    tick.  Some restarts go to poses off the track or facing backwards: those are flagged, the others plan."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    B = 512
    a, c, loop = _twin_loop("default", B, 5300)
    rng = np.random.default_rng(5310)
    mask = rng.random(B) < 0.25
    pos, head, vel = _new_poses(loop, mask, "default", 5320)
    bad = np.nonzero(mask)[0][:16]
    off, back = bad[:8], bad[8:]
    sc = loop.batch()
    inputs_c = (sc, loop.sel.copy(), loop.tc.copy(), loop.vel_est.copy())
    loop.restart(mask, pos, head, vel)
    loop.pos[off] += 40.0 * np.column_stack((np.cos(loop.heading[off]), np.sin(loop.heading[off])))
    loop.heading[back] = np.arctan2(np.sin(loop.heading[back] + np.pi), np.cos(loop.heading[back] + np.pi))
    sc_a = loop.batch()
    _next_tick(a, sc_a, loop.sel, loop.tc, loop.vel_est, restart=mask)
    keep = np.nonzero(~mask)[0]
    sc_c = inputs_c[0]
    sc_c.pos[mask], sc_c.heading[mask], sc_c.vel[mask] = sc_a.pos[mask], sc_a.heading[mask], sc_a.vel[mask]
    _next_tick(c, sc_c, inputs_c[1], inputs_c[2], loop.vel_est)
    sa, sc_state = _state(a), _state(c)
    _snap_equal(sa, sc_state, keep, "restart tick")
    fl = sa["sc_flags"][0]
    assert (fl[off] & capi.SC_OUT_OF_TRACK).all() and (fl[back] & capi.SC_HEADING_MISMATCH).all()
    good = np.setdiff1d(np.nonzero(mask)[0], bad)
    assert (fl[good] == 0).mean() > 0.9
    loop.take(a)
    loop.advance()
    for pl in (a, c):
        _next_tick(pl, loop.batch(), loop.sel, loop.tc, loop.vel_est)
    sa2, sc2 = _state(a), _state(c)
    _snap_equal(sa2, sc2, keep, "tick after the restart")
    assert (sa2["sc_flags"][0, bad] & (capi.SC_OUT_OF_TRACK | capi.SC_HEADING_MISMATCH)).all(), \
        "a rejected pose stays flagged until a later restart"


def test_all_zero_mask_is_no_mask_and_all_ones_is_a_new_session():
    """an all-zero mask equals restart=None byte for byte with the same launches (the pointer is NULL); an all-ones
    mask equals set_startpos + tick of the whole batch"""
    B = 256
    a, c, loop = _twin_loop("l216", B, 5400)
    n0 = a.launch_count()
    _next_tick(a, loop.batch(), loop.sel, loop.tc, loop.vel_est, restart=np.zeros(B, dtype=bool))
    n1 = a.launch_count()
    _next_tick(c, loop.batch(), loop.sel, loop.tc, loop.vel_est)
    assert c.launch_count() - n1 == n1 - n0
    everything = np.arange(B)
    _snap_equal(_state(a), _state(c), everything, "all-zero mask")
    loop.take(a)
    loop.advance()
    ones = np.ones(B, dtype=bool)
    loop.restart(ones, *_new_poses(loop, ones, "l216", 5410))
    sc = loop.batch()
    _next_tick(a, sc, loop.sel, loop.tc, loop.vel_est, restart=ones)
    fresh = _stateful("l216", 4, incl_emerg_traj=True)
    D.first_tick(fresh, sc, loop.vel_est)
    _assert_scenarios_equal(_state(a), _state(fresh), everything, "all-ones mask", id_shift=10 * 5)


def test_split_calls_equal_one_call_with_restarts():
    """next_calc_paths(restart=mask) + next_calc_vel_profile gives the bytes of next_tick(restart=mask): the velocity
    call follows the marker k_state wrote"""
    B = 256
    a, c, loop = _twin_loop("default", B, 5500)
    mask = np.random.default_rng(5510).random(B) < 0.3
    loop.restart(mask, *_new_poses(loop, mask, "default", 5520))
    sc = loop.batch()
    calls, call = [], a._call
    a._call = lambda name: (calls.append(name), call(name))[1]
    a.next_tick(sc, sel_action=loop.sel, t_const=loop.tc, vel_est=loop.vel_est, restart=mask)
    assert calls == ["ltpl_next_tick_batch"]
    c.next_calc_paths(sc, sel_action=loop.sel, t_const=loop.tc, vel_est=loop.vel_est, restart=mask)
    c.next_calc_vel_profile()
    _snap_equal(_state(a), _state(c), np.arange(B), "split calls")


def test_wrong_mask_changes_nothing():
    """a mask of the wrong shape raises before any buffer is swapped: the next tick plans as if it had not been called"""
    B = 128
    a, c, loop = _twin_loop("default", B, 5600, n_before=1)
    with pytest.raises(ValueError):
        a.next_tick(loop.batch(), sel_action=loop.sel, t_const=loop.tc, vel_est=loop.vel_est,
                    restart=np.ones(B + 1, dtype=bool))
    for pl in (a, c):
        _next_tick(pl, loop.batch(), loop.sel, loop.tc, loop.vel_est)
    _snap_equal(_state(a), _state(c), np.arange(B), "after a refused mask")


# ---- 5. recovery --------------------------------------------------------------------------------------------------------
def _oracle_compare(ses, clk, dt, restart, pose, sel, objects, pos, vel_est, snap_b, vel_kw, ctx):
    """one tick of the session oracle against the device results of one scenario (snap_b: action ids, traj lens,
    rows, nodes, n_nodes, status of that scenario); returns the number of compared trajectories"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    clk.t += dt
    if restart:
        assert ses.set_startpos(*pose) is False, ctx
    paths = ses.calc_paths(capi.ACTION_NAMES[int(sel)] if sel != capi.ACT_EMERGENCY else "emergency", objects)
    traj, _ = ses.calc_vel_profile(pos, float(vel_est), **vel_kw)
    aid, tl, rows, nodes, nn, status = snap_b
    got = {capi.ACTION_NAMES[int(aid[s])]: s for s in range(3) if aid[s] >= 0}
    assert sorted(got) == sorted(paths), "%s: paths %s vs %s" % (ctx, sorted(got), sorted(paths))
    n = 0
    for act, s in got.items():
        if not (status[s] & capi.ST_TIE_AMBIGUOUS) and not ses.tie.get(act):
            want = [[-1 if v is None else int(v) for v in p] for p in ses.m_nodes[act][0]] if act in ses.m_nodes else None
            assert want is None or nodes[s, :nn[s]].tolist() == want, "%s: nodes of %s" % (ctx, act)
        assert (tl[s] > 0) == (act in traj), "%s: trajectory %s" % (ctx, act)
        if tl[s] > 0:
            H.assert_close("traj[%s]" % act, rows[s, :tl[s]].astype(np.float64), traj[act][0], D.EXPORT_COLS, ctx)
            n += 1
    return n


def test_flagged_scenarios_plan_again_after_a_restart():
    """scenarios flagged OUT_OF_TRACK, HEADING_MISMATCH (rejected start poses) and STATE_FALLBACK (a first tick that
    broke the brake prefix leaves no usable memory) plan again after a restart, like a fresh first tick, and their next
    four stateful ticks match the session oracle"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from oracle.ltpl_oracle import OracleLTPL
    from tests.restart_session import RestartSession
    B = 96
    sc0 = _feature_batch("default", B, "plain", 5700)
    off, back, fast = np.arange(0, 8), np.arange(8, 16), np.arange(16, 24)
    sc0.pos[off] += 40.0 * np.column_stack((np.cos(sc0.heading[off]), np.sin(sc0.heading[off])))
    sc0.heading[back] = np.arctan2(np.sin(sc0.heading[back] + np.pi), np.cos(sc0.heading[back] + np.pi))
    sc0.vel[fast] = 120.0                                 # > vel_max + 0.1: the first tick reports BRAKE_PREFIX
    pl = _stateful("default", 3)
    loop = Loop(sc0, 5701)
    D.first_tick(pl, loop.batch(), loop.vel_est)
    loop.take(pl)
    loop.advance()
    _next_tick(pl, loop.batch(), loop.sel, loop.tc, loop.vel_est)
    fl = pl.fetch("sc_flags")["sc_flags"]
    assert (fl[off] & capi.SC_OUT_OF_TRACK).all() and (fl[back] & capi.SC_HEADING_MISMATCH).all()
    assert (fl[fast] & capi.SC_STATE_FALLBACK).all(), fl[fast]
    loop.take(pl)
    loop.advance()
    mask = np.zeros(B, dtype=bool)
    mask[:24] = True
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_scenarios
    far = make_scenarios(_track("default"), 24, seed=5702, n_obj_min=0, n_obj_max=0)
    loop.restart(mask, far.pos, far.heading, far.vel)
    for b in range(24):              # never planned with a memory: no calculation time was ever measured
        loop.cbuf[b] = []
    sc = loop.batch()
    _next_tick(pl, sc, loop.sel, loop.tc, loop.vel_est, restart=mask)
    fresh = _stateful("default", 3)
    D.first_tick(fresh, sc, loop.vel_est)
    got = _state(pl)
    ok = np.nonzero(mask & (got["sc_flags"][0] == 0))[0]
    assert ok.size >= 22, got["sc_flags"][0, :24]
    _assert_scenarios_equal(got, _state(fresh), ok, "revived", id_shift=10 * 2)
    # the revived scenarios against the session oracle: the restart tick and four stateful ticks after it
    lat = H.lattice_for("default")
    clks = {b: D.Clock(50.0) for b in ok}
    ses = {b: RestartSession(OracleLTPL(lat), clock=clks[b]) for b in ok}
    vel_kw = dict(D.VEL, ax_max_machines=_axm())
    compared = 0
    for k in range(5):
        if k > 0:
            loop.advance()
            _next_tick(pl, loop.batch(), loop.sel, loop.tc, loop.vel_est)
            sc = loop.batch()
        f = _state(pl)
        for b in ok:
            snap = (f["action_id"][:, b], f["traj_len"][:, b], f["rows"][:, b], f["nodes"][:, b], f["n_nodes"][:, b],
                    f["status"][:, b])
            assert f["sc_flags"][0, b] == 0, "revived scenario %d tick %d flags %d" % (b, k, f["sc_flags"][0, b])
            compared += _oracle_compare(ses[b], clks[b], float(loop.dts[-1][b]), k == 0,
                                        (sc.pos[b], sc.heading[b], sc.vel[b]), loop.sel[b], sc.object_list(b),
                                        sc.pos[b], loop.vel_est[b], snap, vel_kw, "revived %d tick %d" % (b, k))
        loop.take(pl)
    assert compared >= 5 * ok.size


# ---- 8. scale ------------------------------------------------------------------------------------------------------------
def test_restarts_at_scale_window_invariant_and_match_oracle():
    """10 000 scenarios on the ~200 x 11 lattice, 8 ticks, 2 % of the batch restarts per tick (half re-anchored at the
    estimate, half sent to new starts): one and four scenario windows give the same bytes, and 64 sampled sequences
    (most with restarts) match the session oracle tick by tick"""
    from oracle.ltpl_oracle import OracleLTPL
    from tests.restart_session import RestartSession
    B, n_ticks = 10000, 8
    sc0 = _feature_batch("l216", B, "plain", 5800)
    one, four = _stateful("l216", 1), _stateful("l216", 4)
    loop = Loop(sc0, 5801)
    rng = np.random.default_rng(5802)
    masks = [np.zeros(B, dtype=bool)] + [rng.random(B) < 0.02 for _ in range(n_ticks - 1)]
    hit = np.any(masks, axis=0)
    sample = np.concatenate((rng.choice(np.nonzero(hit)[0], 48, replace=False),
                             rng.choice(np.nonzero(~hit)[0], 16, replace=False)))
    lat = H.lattice_for("l216")
    clks = {b: D.Clock(50.0) for b in sample}
    ses = {b: RestartSession(OracleLTPL(lat), clock=clks[b]) for b in sample}
    alive = {b: True for b in sample}
    vel_kw = dict(D.VEL, ax_max_machines=_axm())
    compared, restarts_seen = 0, 0
    for k in range(n_ticks):
        if k == 0:
            sc = loop.batch()
            for pl in (one, four):
                D.first_tick(pl, sc, loop.vel_est)
        else:
            loop.advance()
            if masks[k].any():
                loop.restart(masks[k], *_new_poses(loop, masks[k], "l216", 5810 + k))
            sc = loop.batch()
            for pl in (one, four):
                _next_tick(pl, sc, loop.sel, loop.tc, loop.vel_est, restart=masks[k])
        s1, s4 = D.tick_snapshot(one), D.tick_snapshot(four)
        for name in s1:
            assert np.array_equal(s1[name], s4[name]), "tick %d: %s depends on the scenario windows" % (k, name)
        f = _light(one)
        for b in sample:
            restart = k == 0 or bool(masks[k][b])
            if f["sc_flags"][0, b] != 0:     # (a flagged sequence leaves the comparison for good: the host's moving
                alive[b] = False             # average of the tick times would run on without it)
            if not alive[b]:
                continue
            restarts_seen += int(restart and k > 0)
            dt = 0.0 if k == 0 else float(loop.dts[-1][b])
            snap = (f["action_id"][:, b], f["traj_len"][:, b], f["rows"][:, b], f["nodes"][:, b], f["n_nodes"][:, b],
                    f["status"][:, b])
            compared += _oracle_compare(ses[b], clks[b], dt, restart, (sc.pos[b], sc.heading[b], sc.vel[b]),
                                        loop.sel[b], sc.object_list(b), sc.pos[b], loop.vel_est[b], snap, vel_kw,
                                        "scale sequence %d tick %d" % (b, k))
        loop.take(one)
    assert restarts_seen >= 40 and compared >= 64 * n_ticks // 2, (restarts_seen, compared)
