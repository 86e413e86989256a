"""Stateful tick on the device (csrc/ltpl_state.cuh, BatchPlanner.next_tick) against the closed-loop
sequences of the unmodified reference (tests/golden/ticks_multitick_default.npz, scripted clock): the 16 sequences run
as ONE batch, tick 0 = set_startpos + first tick, ticks 1.. = next_tick with the recorded inputs."""
import ctypes as C

import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H

pytestmark = pytest.mark.gpu


def _raw_call(pl, name):
    """a C-ABI entry point called directly, on the planner's buffers, without the planner's wrapper methods"""
    rc = getattr(pl.lib, name)(pl.handle, C.byref(pl.params), C.byref(pl.dims), C.byref(pl.buf), pl.stream)
    assert rc == 0, pl.lib.ltpl_last_error().decode()


@pytest.mark.parametrize("fixture,emerg,group,tag", [("ticks_multitick_default.npz", False, None, "default"),
                                                     ("ticks_multitick_ext_default.npz", True, None, "default"),
                                                     ("ticks_multitick_ext_default.npz", True, None, "default:raw"),
                                                     ("ticks_multitick_default.npz", False, None, "default:raw"),
                                                     ("ticks_multitick_backup_default.npz", False, 0, "default"),
                                                     ("ticks_multitick_backup_default.npz", False, 1, "default"),
                                                     ("ticks_multitick_emsel_default.npz", True, None, "default"),
                                                     ("ticks_multitick_l216.npz", True, None, "l216"),
                                                     ("ticks_multitick_l430.npz", False, None, "l430"),
                                                     ("ticks_multitick_open.npz", False, None, "open"),
                                                     ("ticks_multitick_zswap_default.npz", False, None, "default"),
                                                     ("ticks_multitick_invalid_default.npz", False, None, "default"),
                                                     ("ticks_multitick_openend.npz", False, None, "open"),
                                                     ("ticks_multitick_pdtan_default.npz", False, None,
                                                      "default:pdtan_exp15"),
                                                     ("ticks_multitick_ggpp_default.npz", True, 0, "default:ggpp"),
                                                     ("ticks_multitick_ggpp_default.npz", True, 1, "default:ggpp")])
def test_next_tick_matches_reference_sequences(fixture, emerg, group, tag):
    """second fixture: a blocked zone on every second sequence + the emergency trajectory in every tick; third fixture:
    the grip (gg_scale) drops on the odd sequences from tick 3 on -> brake on the backup plan (OTH:950-1006); fourth
    fixture: the odd sequences execute the 'emergency' trajectory of ticks 2 .. 4 (sel_action 4; OTH:307-309, 518-601).
    Variant 'raw': a C-ABI caller that calls ltpl_set_startpos_batch, ltpl_tick_batch and ltpl_next_tick_batch itself
    on buffers whose trim, em_info and zone_s0 hold junk.  The first tick has to zero trim (else its trajectories start
    at the junk cut), set_startpos has to reset zone_s0 and, without the emergency trajectory, every tick has to leave
    em_info at -1; the last two are checked on the buffers, because a later kernel may overwrite them."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    g = H.golden(fixture)
    if group is not None:
        g = D.Rows(g, np.arange(group, g["dt"].shape[0], 2))
    n_seq, n_ticks = g["dt"].shape
    n_done = g["n_done"]                                   # open track: sequences end when no trajectory is left
    tag, _, variant = tag.partition(":")
    pl_kw, vel = {}, dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)
    ggpp = variant == "ggpp"   # location dependent local_gg = H.local_gg_field along every path (OTH:649-666), grip drop
    raw = variant == "raw"
    if ggpp or raw:
        variant = ""
    if variant:                                            # other controller / vehicle / velocity parameters (H.VARIANTS)
        online, veh, vel_v, _ = H.VARIANTS[variant]
        pl_kw = dict(online=online, **veh)
        vel.update(vel_v)
    pl = BatchPlanner(H.lattice_for(tag), device="cuda:0", stateful=True, **pl_kw)
    pl.set_subbatches(1 + n_seq % 4)                       # 1 .. 4 scenario windows inside the library
    pl.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emerg, **vel)
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)])       # t_const of ticks 1 ..
    fails, compared = [], 0
    alive = np.ones(n_seq, dtype=bool)
    for k in range(n_ticks):
        sc = ScenarioBatch(g["pos_est"][:, k].copy(), g["sc_heading"].copy(), g["sc_vel"].copy(), g["sc_n_obj"].copy(),
                           g["obj"][:, k].copy())
        zones = [H.zone_of(g, q, k) for q in range(n_seq)]
        if any(z is not None for z in zones):
            sc.set_zones(zones)
        assert len(set(g["gg_scale"][:, k].tolist())) == 1
        pl.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emerg,
                          **dict(vel, gg_scale=float(g["gg_scale"][0, k])))
        if raw:                                            # the planner only allocates the buffers and stages the inputs
            pl.params.traj_base_id = 10 * (k + 1)
            if k == 0:
                pl.stage_scenarios(sc, vel_est=g["vel_est"][:, k])
                pl.upload()
                for name in ("trim", "em_info"):
                    pl.t[name].fill_(1)            # junk, though inside the buffers where a kernel reads it as an index
                pl._state["zone_s0"].fill_(0)
                _raw_call(pl, "ltpl_set_startpos_batch")
                assert (pl._state["zone_s0"].cpu().numpy() == -1).all()
                _raw_call(pl, "ltpl_tick_batch")
            else:
                pl._stage_next(sc, g["sel"][:, k], tc[:, k - 1], g["vel_est"][:, k])
                _raw_call(pl, "ltpl_next_tick_batch")
            if not emerg:
                assert (pl.fetch("em_info")["em_info"] == -1).all(), "tick %d: em_info" % k
        elif k == 0:
            pl.stage_scenarios(sc, vel_est=g["vel_est"][:, k])
            pl.upload()
            pl.set_startpos()
            if ggpp:
                pl.calc_paths()
                pl.set_local_gg_planes(*H.local_gg_planes(pl))
                pl.calc_vel_profile()
            else:
                pl.tick()
        elif ggpp:
            pl.next_calc_paths(sc, sel_action=g["sel"][:, k], t_const=tc[:, k - 1])
            pl.set_local_gg_planes(*H.local_gg_planes(pl))
            pl.next_calc_vel_profile(vel_est=g["vel_est"][:, k])
        else:
            pl.next_tick(sc, sel_action=g["sel"][:, k], t_const=tc[:, k - 1], vel_est=g["vel_est"][:, k])
        recs = pl.records()
        for q in range(n_seq):
            if not alive[q] or k >= int(n_done[q]):
                continue
            ctx = "sequence %d tick %d" % (q, k)
            rec = recs[q]
            try:
                assert not (rec["flags"] & capi.SC_STATE_FALLBACK), ctx + " fell back (flags %d)" % rec["flags"]
                assert not rec["out_of_track"] and "error" not in rec, ctx + " flags %d" % rec["flags"]
                compared += D.compare_multitick_row(rec, g, q, k, ctx, emerg)
            except AssertionError as e:
                fails.append(str(e).split("\n")[0][:400] if "nodes of" not in str(e) else str(e)[:700])
                alive[q] = False            # later ticks of this sequence depend on this one
    assert not fails, "%d sequences diverged (of %d; %d trajectories matched before):\n%s" % (
        len(fails), n_seq, compared, "\n".join(fails[:8]))
    assert compared > (30 if (group is not None or n_seq < 12) else (80 if (emerg or n_seq < 16) else 150))


@pytest.mark.parametrize("fixture,emerg", [("ticks_multitick_invalid_default.npz", False),
                                           ("ticks_multitick_emsel_default.npz", True)])
def test_next_tick_in_one_call_equals_two_calls(fixture, emerg):
    """next_tick is ONE library call (ltpl_next_tick_batch) and gives the bytes of next_calc_paths +
    next_calc_vel_profile in every tick.  First fixture: the restart after an executed action the last tick did not
    return (OTH:393-407), in which k_state takes the start velocity `vel` of the path half; second fixture: the
    executed 'emergency' trajectory."""
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    g = H.golden(fixture)
    n_seq, n_ticks = g["dt"].shape
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)])
    one, two = (BatchPlanner(H.lattice_for("default"), device="cuda:0", stateful=True) for _ in range(2))
    calls, call = [], one._call
    one._call = lambda name: (calls.append(name), call(name))[1]
    for k in range(n_ticks):
        sc = ScenarioBatch(g["pos_est"][:, k].copy(), g["sc_heading"].copy(), g["sc_vel"].copy(), g["sc_n_obj"].copy(),
                           g["obj"][:, k].copy())
        zones = [H.zone_of(g, q, k) for q in range(n_seq)]
        if any(z is not None for z in zones):
            sc.set_zones(zones)
        for pl in (one, two):
            pl.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emerg, vel_max=100.0,
                              gg_scale=float(g["gg_scale"][0, k]), local_gg=(5.0, 5.0), safety_d=30.0)
            if k == 0:
                pl.stage_scenarios(sc, vel_est=g["vel_est"][:, k])
                pl.upload()
                pl.set_startpos()
                pl.tick()
        if k > 0:
            del calls[:]
            one.next_tick(sc, sel_action=g["sel"][:, k], t_const=tc[:, k - 1], vel_est=g["vel_est"][:, k])
            assert calls == ["ltpl_next_tick_batch"]
            two.next_calc_paths(sc, sel_action=g["sel"][:, k], t_const=tc[:, k - 1], vel_est=g["vel_est"][:, k])
            two.next_calc_vel_profile()
        got, want = D.tick_snapshot(one), D.tick_snapshot(two)
        assert (want["traj_len"] > 0).sum() >= n_seq
        for name in want:
            assert np.array_equal(got[name], want[name]), "tick %d: %s" % (k, name)


@pytest.mark.parametrize("tag,n_seq,omin,omax",[("default", 96, 0, 2), ("l216", 64, 1, 3), ("open", 48, 0, 2)])
def test_closed_loop_matches_session_oracle(tag, n_seq, omin, omax):
    """larger closed loop driven by the DEVICE results (vehicle dummy on the selected trajectory, moving opponents,
    changing action preference); the stateful oracle (oracle/ltpl_session.py, pinned against the reference) replays the
    same inputs tick by tick.  Sequences the device flags (memory not usable, capacity) leave the loop -- at most 5 %.
    Second case: BASELINE's ~200 x 11 lattice, whose node lists exceed 32 entries.  Third case: the OPEN track, seeded
    over its whole length -- the vehicles near the end plan reduced horizons, shrinking trajectories and stop."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    g = H.golden("ticks_multitick_default.npz")
    lat = H.lattice_for(tag)
    n_ticks = 8
    vel = dict(D.VEL, ax_max_machines=g["ax_max_machines"])
    trk = Track(H.track_csv_for(tag))
    sc0 = make_scenarios(trk, n_seq, seed=2718, n_obj_min=omin, n_obj_max=omax,
                         s_max=(trk.length - 10.0) if tag == "open" else None)
    prefer = (("right", "left", "straight", "follow"), ("follow", "straight", "left", "right"),
              ("left", "right", "follow", "straight"), ("straight", "follow", "right", "left"))
    pl = D.planner(lat, 5, stateful=True, **vel)           # five scenario windows inside the library (uneven split)
    n = D.closed_loop_vs_session(pl, lat, sc0, np.random.default_rng(2719), vel, prefer,
                                 capi.SC_STATE_FALLBACK | capi.SC_CAPACITY | capi.SC_BRAKE_PREFIX, n_ticks=n_ticks)
    assert n["ticks"] > n_seq * n_ticks // 2 and n["traj"] > n_seq * n_ticks // 2, n
    assert n["flagged"] <= n_seq // 20, "%d of %d sequences were flagged by the device (%d state fallbacks)" % (
        n["flagged"], n_seq, n["fell_back"])


@pytest.mark.parametrize("fixture,seqs,emerg", [("ticks_multitick_default.npz", (0, 5, 11), False),
                                                ("ticks_multitick_emsel_default.npz", (1, 3), True)])
def test_facade_runs_closed_loop_like_the_reference(fixture, seqs, emerg, tmp_path):
    """Graph_LTPL facade with the reference's call sequence over several ticks (main_std_example.py:99-126): an injected
    clock takes the place of time.time(); recorded sequences of the reference are replayed (second case: the caller
    executes the 'emergency' trajectory for three ticks, prev_action_id='emergency')."""
    g = H.golden(fixture)
    assert D.replay_facade(D.facade(tmp_path), g, seqs, emerg) > (20 if emerg else 40)
