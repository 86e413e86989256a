"""Golden vectors of the brake prefix to a lowered vel_max (VpForwardBackward.check_brake_prefix, VPFB:86-139), made by
running the UNMODIFIED reference on the shims of oracle/gen_golden.py and recording the arguments, the instance's memory
and the results of every call.  Writes exactly one file under the repository:

  tests/golden/brake_prefix.npz

Three kinds of call (`kind`):
  0   the reference's own calls inside closed loops (oracle/gen_golden.multitick_fixture) on the default and "216 x 11"
      lattices, with gg_scale dropping between ticks: OTH:747 calls it for every path, with the velocity course of the
      delay compensation as vel_course;
  1   closed loops in which vel_max drops below the planned velocity (and gg_scale with it): the prefix call is recorded,
      then the reference raises at OTH:830 / 919 (the prefix is computed but never joined to the profile) and the loop
      ends there;
  2   direct calls on synthetic inputs, kept so that every label of LABELS occurs, the calls at vel_plan =
      nextafter(vel_max + 0.1, +-inf) and exactly at vel_max + 0.1, and ordered chains of 6 or more calls on one
      instance with vel_max and gg_scale changing between them.
Every call belongs to a chain (`chain`, `step`): the calls of one reference instance in the order it made them, so a
replay can carry the memory (old_gg_scale) from call to call.

Per call: kappa / el / loc_gg rows (loc_gg before the scale, as passed), n_pts, vel_course (n_course), vel_plan, the
instance's parameters (vel_max, gg_scale, dyn_model_exp, drag, mass), its _VpForwardBackward__old_gg_scale before and
after the call, the results vx_prefix (n_prefix), pref_idx, vel_start, a label bitmask and two margins:
  margin        min |vx_decel[k] - vel_max| over the points k <= idx that are not a standstill zero (m/s; inf without
                a brake profile)
  stop_margin   -radicand of the step that ended in standstill at or before idx (m^2/s^2; inf when there is none)
The brake chain on the device is not bit-exact to tph (within 1e-9 relative + 1e-9 m/s): every recorded call keeps
margin > 1e-8 m/s and stop_margin > 1e-6 m^2/s^2, so the cut index and the branch are the same on both sides.  This
generator asserts it for the calls of the closed loops and drops synthetic candidates that miss it.

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_brake_prefix
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

LABELS = ("no_prefix", "prefix_cut", "prefix_unreached", "cut_at_standstill", "empty_course", "per_point_gg",
          "old_ne_current", "exp_1_5", "boundary")
MARGIN_V, MARGIN_W = 1e-8, 1e-6
RECORDS = []
_CUR = {"kind": 0, "boundary": False}
_CHAINS = {}
_KEEP = []   # the instances, so that their ids stay unique


def brake_trace(loc_gg, kappa, el, v_start, exp, drag, mass):
    """tph.calc_vel_profile_brake (the shim's, the reference's own function) and, from its locals at return, the index
    of the first standstill zero (None: none) and -radicand of the step that broke"""
    from oracle import tph_port
    code = tph_port.calc_vel_profile_brake.__code__
    loc = {}

    def tracer(frame, event, arg):
        if frame.f_code is code:
            def local(fr, ev, a):
                if ev == "return":
                    loc.update(fr.f_locals)
                return local
            return local
        return None
    old = sys.gettrace()
    sys.settrace(tracer)
    try:
        vx = tph_port.calc_vel_profile_brake(loc_gg=loc_gg, kappa=kappa, el_lengths=el, v_start=v_start,
                                             dyn_model_exp=exp, drag_coeff=drag, m_veh=mass)
    finally:
        sys.settrace(old)
    r = loc.get("radicand")
    if r is not None and r < 0.0:
        return vx, int(loc["i"]) + 1, -float(r)
    return vx, None, np.inf


def margins(vel_plan, kappa, el, loc_gg, old, vel_max, exp, drag, mass):
    if not vel_plan > vel_max + 0.1:
        return np.inf, np.inf
    vx, stop, stop_w = brake_trace(loc_gg * old, kappa, el, vel_plan, exp, drag, mass)
    idx = int(np.argmax(vx <= vel_max))
    if idx == 0:
        idx = vx.size - 1
    ks = np.arange(idx + 1)
    if stop is not None:
        ks = ks[ks < stop]
    margin = float(np.min(np.abs(vx[ks] - vel_max))) if ks.size else np.inf
    return margin, (stop_w if stop is not None and stop <= idx else np.inf)


def install(graph_ltpl):
    """wrap VpForwardBackward.check_brake_prefix: arguments, memory before / after, results"""
    vpfb = graph_ltpl.online_graph.src.VpForwardBackward.VpForwardBackward
    orig = vpfb.check_brake_prefix

    def method(self, vel_plan, vel_course, kappa, el_lengths, loc_gg):
        g = lambda k: getattr(self, "_VpForwardBackward__" + k)   # noqa: E731
        before = float(g("old_gg_scale"))
        res = orig(self, vel_plan, vel_course, kappa, el_lengths, loc_gg)
        if id(self) not in _CHAINS:
            _CHAINS[id(self)] = [len(_CHAINS), 0]
            _KEEP.append(self)
        chain = _CHAINS[id(self)]
        vel_max, gg_scale, exp = float(g("vel_max")), float(g("gg_scale")), float(g("dyn_model_exp"))
        kappa, el = np.array(kappa, dtype=np.float64), np.array(el_lengths, dtype=np.float64)
        loc_gg, vel_course = np.array(loc_gg, dtype=np.float64), np.array(vel_course, dtype=np.float64).reshape(-1)
        margin, stop_margin = margins(float(vel_plan), kappa, el, loc_gg, before, vel_max, exp, float(g("drag_coeff")),
                                      float(g("m_veh")))
        labels = set()
        if res[1] == 0 and not vel_plan > vel_max + 0.1:
            labels.add("no_prefix")
        else:
            labels.add("prefix_cut" if res[2] <= vel_max else "prefix_unreached")
            if vel_max == 0.0 and res[2] == 0.0:
                labels.add("cut_at_standstill")
            if before != gg_scale:
                labels.add("old_ne_current")
        if vel_course.size == 0:
            labels.add("empty_course")
        if not np.all(loc_gg == loc_gg[0]):
            labels.add("per_point_gg")
        if exp == 1.5:
            labels.add("exp_1_5")
        if _CUR["boundary"]:
            labels.add("boundary")
        RECORDS.append(dict(vel_plan=float(vel_plan), vel_course=vel_course, kappa=kappa, el=el, loc_gg=loc_gg,
                            vel_max=vel_max, gg_scale=gg_scale, dyn_model_exp=exp, drag=float(g("drag_coeff")),
                            mass=float(g("m_veh")), old_before=before, old_after=float(g("old_gg_scale")),
                            vx_prefix=np.array(res[0], dtype=np.float64).reshape(-1), pref_idx=int(res[1]),
                            vel_start=float(res[2]), margin=margin, stop_margin=stop_margin,
                            labels=sum(1 << LABELS.index(b) for b in labels), kind=_CUR["kind"], chain=chain[0],
                            step=chain[1]))
        chain[1] += 1
        return res
    vpfb.check_brake_prefix = method
    return vpfb


def loop_calls(graph_ltpl, ltpl, track, tag, n_seq, n_ticks, seed, gg_fn=None):
    """kind 0: the reference's calls inside closed loops, grip dropping from tick 3 on in every other sequence"""
    vk = dict(vel_max=70.0, gg_scale=0.95, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
              safety_d=25.0, incl_emerg_traj=False)
    n0 = len(RECORDS)
    _CUR["kind"] = 0
    GG.multitick_fixture(graph_ltpl, ltpl, track, n_seq, n_ticks, vk, seed=seed, n_obj=(0, 2), gg_drop=(3, 0.8),
                         gg_fn=gg_fn)
    print("[%s closed loops%s] %d prefix calls" % (tag, " gg" if gg_fn else "", len(RECORDS) - n0))


def drop_calls(graph_ltpl, ltpl, track, tag, n_seq, seed, k_drop=3, n_ticks=6):
    """kind 1: closed loops in which vel_max drops below the planned velocity at tick k_drop (gg_scale with it); the
    reference raises after the prefix call (OTH:830 / 919) and the loop ends there"""
    import graph_ltpl.online_graph.src.OnlineTrajectoryHandler as oth_mod
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_scenarios
    clock = GG.ScriptedClock()
    real_time = oth_mod.time
    oth_mod.time = clock
    n0, raised = len(RECORDS), 0
    _CUR["kind"] = 1
    rng = np.random.default_rng(seed + 1)
    try:
        sc = make_scenarios(track, n_seq, seed=seed, n_obj_min=0, n_obj_max=1)
        for q in range(n_seq):
            if ltpl.set_startpos(pos_est=np.array(sc.pos[q]), heading_est=float(sc.heading[q]), vel_est=float(sc.vel[q])):
                continue
            ltpl._Graph_LTPL__obj_zone = []
            ltpl._Graph_LTPL__obj_list_handler._ObjectListInterface__object_zones = []
            pos_est, vel_est, sel, traj_set = np.array(sc.pos[q]), float(sc.vel[q]), "straight", None
            for k in range(n_ticks):
                dt = float(rng.uniform(0.04, 0.16))
                clock.t += dt
                if traj_set is not None:
                    pos_est, vel_est = advance_on_traj(traj_set[sel][0], dt)
                vk = dict(vel_max=70.0, gg_scale=0.95, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
                          safety_d=25.0, incl_emerg_traj=False)
                if k >= k_drop:
                    vk.update(vel_max=float(max(vel_est - rng.uniform(3.0, 25.0), 0.0)),
                              gg_scale=float(rng.uniform(0.6, 0.9)))
                ltpl.calc_paths(prev_action_id=sel, object_list=[], blocked_zones=None)
                try:
                    traj_set, _, _ = ltpl.calc_vel_profile(pos_est=pos_est, vel_est=vel_est, **vk)
                except ValueError:
                    raised += 1
                    break
                cand = [a for a in ("straight", "left", "right", "follow") if a in traj_set and len(traj_set[a])]
                if not cand:
                    break
                sel = cand[0]
    finally:
        oth_mod.time = real_time
    print("[%s vel_max drops] %d prefix calls, %d loops ended by the reference's exception" % (
        tag, len(RECORDS) - n0, raised))
    return raised


def advance_on_traj(traj, dt):
    return GG.advance_on_traj(traj, dt)


def _path(rng, p, c):
    el = rng.uniform(1.0, 3.5, size=p - 1)
    s = np.concatenate(([0.0], np.cumsum(el)))
    kappa = rng.uniform(0.0, 0.02) * np.sin(s / rng.uniform(20.0, 150.0) + rng.uniform(0, 6.3))
    gg = np.column_stack((4.0 + 1.5 * np.sin(s / 37.0 + c), 4.5 + np.cos(s / 53.0 - c))) if c % 3 == 0 \
        else np.tile([float(rng.uniform(4.0, 6.0)), float(rng.uniform(4.0, 6.0))], (p, 1))
    return kappa, el, gg


def direct_calls(graph_ltpl, axm, n_rand=1500, seed=5151):
    """kind 2: synthetic calls straight into VpForwardBackward; the greedy selection keeps every label several times"""
    vpfb_cls = graph_ltpl.online_graph.src.VpForwardBackward.VpForwardBackward
    rng = np.random.default_rng(seed)
    _CUR["kind"] = 2
    kept = {b: 0 for b in LABELS}

    def one(vp, vel_plan, vel_course, kappa, el, gg, force=False):
        n0 = len(RECORDS)
        vp.check_brake_prefix(vel_plan=vel_plan, vel_course=vel_course, kappa=kappa, el_lengths=el, loc_gg=gg)
        r = RECORDS[-1]
        ok = r["margin"] > MARGIN_V and r["stop_margin"] > MARGIN_W
        bits = [b for b in LABELS if r["labels"] & (1 << LABELS.index(b))]
        if ok and (force or any(kept[b] < 10 for b in bits) or len(RECORDS) % 25 == 0):
            for b in bits:
                kept[b] += 1
            return True
        del RECORDS[n0:]
        return False

    def fresh(exp, gg_scale):
        vp = vpfb_cls(dyn_model_exp=exp, drag_coeff=0.85, m_veh=1000.0, len_veh=4.7, follow_control_type="PD",
                      follow_control_params={"c_p": 1.25, "k_d": 0.025, "k_p": 0.2}, glob_rl=None)
        vp.update_dyn_parameters(vel_max=80.0, gg_scale=gg_scale, ax_max_machines=axm)
        return vp

    # single calls: one instance each; old != current from a first call that needs no brake at another gg_scale
    for c in range(n_rand):
        exp = (1.0, 1.5)[c % 2]
        vp = fresh(exp, float(rng.uniform(0.6, 1.0)))
        if c % 4 == 1:   # the memory: a call that needs no brake at the first scale, then the scale changes
            vp.check_brake_prefix(vel_plan=10.0, vel_course=np.zeros(0), kappa=np.zeros(2), el_lengths=np.ones(1),
                                  loc_gg=np.ones((2, 2)))
            RECORDS.pop()
        p = int(rng.choice([2, 3, 8, 40, 120]))
        cap = int(rng.choice([0, 0, 1, 3, 7]))
        kappa, el, gg = _path(rng, p, c)
        vel_course = rng.uniform(20.0, 60.0, size=cap)
        vel_plan = float(rng.uniform(5.0, 80.0))
        mode = c % 5
        vel_max = float(rng.uniform(0.0, 75.0))
        if mode == 1:
            vel_max = 0.0                                          # brake to standstill
        elif mode == 2:
            vel_max = float(max(vel_plan - rng.uniform(0.5, 4.0), 0.0))   # short paths: the speed is not reached
        vp.update_dyn_parameters(vel_max=vel_max, gg_scale=float(rng.uniform(0.6, 1.0)), ax_max_machines=axm)
        one(vp, vel_plan, vel_course, kappa, el, gg)
    # the float64 boundary of the branch: nextafter(vel_max + 0.1, -inf), exactly vel_max + 0.1, nextafter(.., +inf)
    _CUR["boundary"] = True
    for c, vel_max in enumerate((50.0, 33.3, 12.7, 61.9)):
        for direction in (-np.inf, None, np.inf):
            vp = fresh(1.0, 0.9)
            vp.update_dyn_parameters(vel_max=vel_max, gg_scale=0.8, ax_max_machines=axm)
            b = vel_max + 0.1
            vel_plan = b if direction is None else float(np.nextafter(b, direction))
            kappa, el, gg = _path(rng, 40, c + 1)
            assert one(vp, vel_plan, rng.uniform(20.0, 60.0, size=2), kappa, el, gg, force=True)
    _CUR["boundary"] = False
    # ordered chains on one instance: vel_max and gg_scale change between the calls, the memory carries
    n_chain = 0
    for c in range(40):
        vp = fresh((1.0, 1.5)[c % 2], float(rng.uniform(0.7, 1.0)))
        n0 = len(RECORDS)
        ok = True
        for k in range(8):
            vel_plan = float(rng.uniform(20.0, 70.0))
            vel_max = float(vel_plan + rng.uniform(-15.0, 5.0)) if k % 3 else float(rng.uniform(0.0, vel_plan))
            vp.update_dyn_parameters(vel_max=max(vel_max, 0.0), gg_scale=float(rng.uniform(0.5, 1.0)),
                                     ax_max_machines=axm)
            kappa, el, gg = _path(rng, int(rng.choice([10, 60, 150])), c + k)
            vp.check_brake_prefix(vel_plan=vel_plan, vel_course=rng.uniform(20.0, 60.0, size=int(rng.integers(0, 4))),
                                  kappa=kappa, el_lengths=el, loc_gg=gg)
            r = RECORDS[-1]
            ok = ok and r["margin"] > MARGIN_V and r["stop_margin"] > MARGIN_W
        if not ok or n_chain >= 12:
            del RECORDS[n0:]
        else:
            n_chain += 1
    print("[direct] labels kept %s, %d chains of 8 calls" % (kept, n_chain))


def pack():
    n = len(RECORDS)
    pmax = max(r["kappa"].size for r in RECORDS)
    cmax = max(r["vel_course"].size for r in RECORDS)
    out = dict(kappa=np.zeros((n, pmax)), el=np.zeros((n, pmax - 1)), loc_gg=np.zeros((n, pmax, 2)),
               vel_course=np.zeros((n, cmax)), vx_prefix=np.zeros((n, cmax + pmax - 1)),
               n_pts=np.array([r["kappa"].size for r in RECORDS], dtype=np.int32),
               n_course=np.array([r["vel_course"].size for r in RECORDS], dtype=np.int32),
               n_prefix=np.array([r["vx_prefix"].size for r in RECORDS], dtype=np.int32),
               pref_idx=np.array([r["pref_idx"] for r in RECORDS], dtype=np.int32),
               labels=np.array([r["labels"] for r in RECORDS], dtype=np.int64), label_names=np.array(LABELS),
               kind=np.array([r["kind"] for r in RECORDS], dtype=np.int32),
               chain=np.unique([r["chain"] for r in RECORDS], return_inverse=True)[1].astype(np.int32),
               step=np.array([r["step"] for r in RECORDS], dtype=np.int32),
               has_gg=np.array([not np.all(r["loc_gg"] == r["loc_gg"][0]) for r in RECORDS]))
    for k in ("vel_plan", "vel_max", "gg_scale", "dyn_model_exp", "drag", "mass", "old_before", "old_after",
              "vel_start", "margin", "stop_margin"):
        out[k] = np.array([r[k] for r in RECORDS], dtype=np.float64)
    for i, r in enumerate(RECORDS):
        p, c = r["kappa"].size, r["vel_course"].size
        out["kappa"][i, :p], out["el"][i, :p - 1], out["loc_gg"][i, :p] = r["kappa"], r["el"], r["loc_gg"]
        out["vel_course"][i, :c] = r["vel_course"]
        out["vx_prefix"][i, :r["vx_prefix"].size] = r["vx_prefix"]
    return out


def main():
    graph_ltpl = GG.load_reference()
    install(graph_ltpl)
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    from tests.helpers import local_gg_field
    track = Track(GG.REF + "/inputs/traj_ltpl_cl/traj_ltpl_cl_monteblanco.csv")
    ltpl, _ = GG.make_ltpl(graph_ltpl, "default", {})
    loop_calls(graph_ltpl, ltpl, track, "default", 8, 8, 931)
    loop_calls(graph_ltpl, ltpl, track, "default", 4, 8, 932, gg_fn=local_gg_field)
    l216 = dict(__import__("ast").literal_eval(str(np.load(os.path.join(GG.GOLDEN, "ticks_l216.npz"))["overrides"])))
    l216_ltpl, _ = GG.make_ltpl(graph_ltpl, "l216", l216)
    loop_calls(graph_ltpl, l216_ltpl, track, "l216", 6, 8, 933, gg_fn=local_gg_field)
    for r in RECORDS:
        assert r["margin"] > MARGIN_V and r["stop_margin"] > MARGIN_W, r
    n_loop = len(RECORDS)
    raised = drop_calls(graph_ltpl, ltpl, track, "default", 10, 941)
    raised += drop_calls(graph_ltpl, l216_ltpl, track, "l216", 8, 942)
    assert raised > 0
    for r in RECORDS[n_loop:]:
        assert r["margin"] > MARGIN_V and r["stop_margin"] > MARGIN_W, r
    direct_calls(graph_ltpl, GG.ax_max_machines_table())
    out = pack()
    missing = [b for i, b in enumerate(LABELS) if not np.any(out["labels"] & (1 << i))]
    assert not missing, missing
    assert all(np.any(out["kind"] == k) for k in (0, 1, 2))
    assert np.all(out["margin"] > MARGIN_V) and np.all(out["stop_margin"] > MARGIN_W)
    np.savez_compressed(os.path.join(GG.GOLDEN, "brake_prefix.npz"), **out)
    brake = out["pref_idx"] > 0
    print("brake_prefix.npz: %d calls (%d from closed loops, %d from vel_max drops, %d direct), %d with a brake "
          "prefix, %d chains; smallest margin %.3g m/s, smallest stop margin %.3g m^2/s^2; P <= %d, C <= %d" % (
              out["kind"].size, int((out["kind"] == 0).sum()), int((out["kind"] == 1).sum()),
              int((out["kind"] == 2).sum()), int(brake.sum()), int(out["chain"].max()) + 1, float(out["margin"].min()),
              float(out["stop_margin"].min()), out["kappa"].shape[1], out["vel_course"].shape[1]))


if __name__ == "__main__":
    main()
