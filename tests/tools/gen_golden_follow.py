"""Golden vectors of the follow-mode velocity profile (VpForwardBackward.calc_vel_profile_follow, VPFB:141-192 ->
calc_vel_profile_follow, CVPF:78-313), made by running the UNMODIFIED reference on the shims of oracle/gen_golden.py and
recording the argument and result tuples of the reference's own calls.  Writes exactly one file under the repository:

  tests/golden/vel_follow.npz

Three kinds of call (`kind`):
  0   the calls the reference makes inside first ticks (objects ahead of the ego, so that 'follow' is planned, and a
      velocity estimate beside the planned velocity) on the default and "216 x 11" lattices: PD and PDtan,
      dyn_model_exp 1.0 and 1.5, constant and per-point friction;
  2   the calls inside closed loops (oracle/gen_golden.multitick_fixture: stateful ticks, the start velocity from the
      last trajectory, the estimate from driving along it) on both lattices, constant and per-point friction;
  1   direct VpForwardBackward.calc_vel_profile_follow calls on synthetic inputs, kept so that every branch label of
      tests/vel_follow_ref.BRANCHES is reached (too_close both ways, ego_stop_dist >= s_stop, segment 1 taken and not,
      stop_idx < 2, a control segment of length 0, v_end from the race line, the -1 index wrap of the opponent match).
The branch labels are read off the reference's own locals when its CVPF call returns.

Per call: kappa / el / loc_gg rows (raw loc_gg, padded to the longest call), n_pts, the five scalars, obj_pos, the
planner parameters (vel_max, gg_scale, dyn_model_exp, drag, mass, len_veh, controller), vx, too_close, vel_bound, the
label bitmask and the race-line set (glob_rl_<set>, [M + 1][5] as Lattice.glob_rl stores it).

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_follow
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402
from tests.vel_follow_ref import BRANCHES  # noqa: E402

RECORDS = []
_CUR = {}


def _labels(loc):
    """branch bitmask of one CVPF call from the locals of its frame at return"""
    out = set()
    out.add("too_close" if loc["too_close"] else "not_too_close")
    if not (loc["ego_stop_dist"] < loc["s_stop"]):
        out.add("ego_stop_ge_s_stop")
    else:
        if loc["v_start"] > loc["v_control"] and loc["stop_idx"] >= 2:
            out.add("seg1")
        else:
            out.add("no_seg1")
        if loc["stop_idx"] < 2:
            out.add("stop_idx_lt2")
        if loc["stop_idx"] - loc["idx_c"] == 0:
            out.add("ctrl_len0")
    if loc["s_stop"] > loc["s"][-1]:
        out.add("v_end_rl")
    if loc["idx_s_opp"] == -1:
        out.add("opp_wrap")
    return sum(1 << BRANCHES.index(b) for b in out)


def install(graph_ltpl):
    """wrap VpForwardBackward.calc_vel_profile_follow (arguments, parameters, results) and trace the CVPF frame"""
    vpfb = graph_ltpl.online_graph.src.VpForwardBackward.VpForwardBackward
    mod = graph_ltpl.helper_funcs.src.calc_vel_profile_follow
    fn = mod.calc_vel_profile_follow
    code = fn.__code__

    def traced(**kw):
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
            res = fn(**kw)
        finally:
            sys.settrace(old)
        _CUR["labels"] = _labels(loc)
        return res
    mod.calc_vel_profile_follow = traced
    orig = vpfb.calc_vel_profile_follow

    def method(self, kappa, el_lengths, loc_gg, v_start, v_ego, v_obj, safety_d, obj_dist, obj_pos):
        res = orig(self, kappa, el_lengths, loc_gg, v_start, v_ego, v_obj, safety_d, obj_dist, obj_pos)
        g = lambda k: getattr(self, "_VpForwardBackward__" + k)   # noqa: E731
        RECORDS.append(dict(kappa=np.array(kappa, dtype=np.float64), el=np.array(el_lengths, dtype=np.float64),
                            loc_gg=np.array(loc_gg, dtype=np.float64), v_start=float(v_start), v_ego=float(v_ego),
                            v_obj=float(v_obj), safety_d=float(safety_d), obj_dist=float(obj_dist),
                            obj_pos=np.array(obj_pos, dtype=np.float64), vel_max=float(g("vel_max")),
                            gg_scale=float(g("gg_scale")), ax_max_machines=np.array(g("ax_max_machines")),
                            dyn_model_exp=float(g("dyn_model_exp")), drag=float(g("drag_coeff")),
                            mass=float(g("m_veh")), len_veh=float(g("len_veh")),
                            control_type=g("follow_control_type"), control_params=dict(g("follow_control_params")),
                            glob_rl=g("glob_rl_clsd"), vx=np.array(res[0], dtype=np.float64),
                            too_close=bool(res[1]), vel_bound=bool(res[2]), labels=_CUR["labels"],
                            kind=_CUR.get("kind", 0)))
        return res
    vpfb.calc_vel_profile_follow = method
    return vpfb


def tick_calls(graph_ltpl, track, tag, overrides, controller, exp, n, seed, gg_fn=None):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_scenarios
    ltpl, _ = GG.make_ltpl(graph_ltpl, tag, overrides,   # one stored graph per lattice
                           controller_type=None if controller == "PD" else controller,
                           veh=dict(veh_param_dyn_model_exp=exp))
    vk = dict(vel_max=70.0, gg_scale=0.95, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
              safety_d=25.0, incl_emerg_traj=False)
    sc = make_scenarios(track, n, seed=seed, n_obj_min=1, n_obj_max=3)
    n0 = len(RECORDS)
    _CUR["kind"] = 0
    for b in range(sc.size):
        # the velocity estimate differs from the planned start velocity (the controller's k_d term)
        GG.run_tick(ltpl, sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(b), vk, full=True, gg_fn=gg_fn,
                    vel_est=sc.vel[b] + (1.5 if b % 2 else -2.0))
    print("[%s %s exp %g%s] %d follow calls" % (tag, controller, exp, " gg" if gg_fn else "", len(RECORDS) - n0))
    return ltpl


def loop_calls(graph_ltpl, ltpl, track, tag, n_seq, n_ticks, seed, gg_fn=None):
    """the calls inside closed loops (stateful ticks: the start velocity comes from the last trajectory, the estimate
    from driving along it), 1-3 objects per sequence"""
    vk = dict(vel_max=70.0, gg_scale=0.95, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
              safety_d=25.0, incl_emerg_traj=False)
    n0 = len(RECORDS)
    _CUR["kind"] = 2
    GG.multitick_fixture(graph_ltpl, ltpl, track, n_seq, n_ticks, vk, seed=seed, n_obj=(1, 3), gg_fn=gg_fn)
    print("[%s closed loops%s] %d follow calls" % (tag, " gg" if gg_fn else "", len(RECORDS) - n0))


def direct_calls(graph_ltpl, glob_rl, axm, n_rand=3000, seed=4242):
    """synthetic calls straight into VpForwardBackward; the greedy selection keeps every label several times"""
    vpfb_cls = graph_ltpl.online_graph.src.VpForwardBackward.VpForwardBackward
    rng = np.random.default_rng(seed)
    m = glob_rl.shape[0] - 1
    ctrls = (("PD", {"c_p": 1.25, "k_d": 0.025, "k_p": 0.2}),
             ("PDtan", {"c_p": 1.15, "k_d": 0.025, "k_p": 0.2, "tan_w": 15.0}))
    n0 = len(RECORDS)
    _CUR["kind"] = 1
    for c in range(n_rand):
        ctype, cp = ctrls[c % 2]
        exp = (1.0, 1.5)[(c // 2) % 2]
        vp = vpfb_cls(dyn_model_exp=exp, drag_coeff=0.85, m_veh=1000.0, len_veh=4.7, follow_control_type=ctype,
                      follow_control_params=cp, glob_rl=glob_rl)
        vp.update_dyn_parameters(vel_max=float(rng.choice([40.0, 60.0, 80.0])), gg_scale=float(rng.uniform(0.7, 1.0)),
                                 ax_max_machines=axm)
        p = int(rng.choice([3, 4, 12, 40, 120]))
        el = rng.uniform(1.5, 3.5, size=p)
        s = np.cumsum(el) - el
        kappa = rng.uniform(0.0, 0.012) * np.sin(s / rng.uniform(30.0, 200.0) + rng.uniform(0, 6.3))
        gg = np.column_stack((4.0 + 1.5 * np.sin(s / 37.0 + c), 4.5 + np.cos(s / 53.0 - c))) if c % 3 == 0 \
            else np.tile([5.0, 5.0], (p, 1))
        if c % 17 == 0:   # the opponent just behind race-line point 0: get_s_coord's index -1
            j = 0
            pos = glob_rl[0, 1:3] - 0.3 * (glob_rl[1, 1:3] - glob_rl[0, 1:3])
        else:
            j = int(rng.integers(0, m))
            pos = glob_rl[j, 1:3] + rng.uniform(-2.0, 2.0, size=2)
        v_start = float(rng.uniform(0.0, 70.0))
        v_obj, safety_d, obj_dist = float(rng.uniform(0.0, 60.0)), float(rng.uniform(0.0, 40.0)), \
            float(rng.uniform(-20.0, 300.0))
        if c % 23 == 5:   # the ego at standstill, a stopped opponent s_stop = 1 m ahead: stop_idx 1 < 2
            v_start, v_obj, obj_dist = float(rng.uniform(0.0, 0.1)), 0.0, safety_d + 4.7 + 1.0
        vp.calc_vel_profile_follow(kappa=kappa, el_lengths=el, loc_gg=gg, v_start=v_start,
                                   v_ego=v_start + float(rng.uniform(-2, 2)), v_obj=v_obj, safety_d=safety_d,
                                   obj_dist=obj_dist, obj_pos=list(pos))
    cand = RECORDS[n0:]
    del RECORDS[n0:]
    keep, count = [], {b: 0 for b in BRANCHES}
    for i, r in enumerate(cand):
        bits = [b for b in BRANCHES if r["labels"] & (1 << BRANCHES.index(b))]
        if any(count[b] < 12 for b in bits) or i % 40 == 0:
            keep.append(r)
            for b in bits:
                count[b] += 1
    RECORDS.extend(keep)
    print("[direct] %d of %d calls kept; labels %s" % (len(keep), len(cand), count))


def pack():
    sets = []
    for r in RECORDS:
        key = r["glob_rl"].tobytes()
        if key not in sets:
            sets.append(key)
    glob = {}
    for r in RECORDS:
        glob.setdefault(sets.index(r["glob_rl"].tobytes()), r["glob_rl"])
    n = len(RECORDS)
    pmax = max(r["kappa"].size for r in RECORDS)
    out = dict(kappa=np.zeros((n, pmax)), el=np.zeros((n, pmax)), loc_gg=np.zeros((n, pmax, 2)), vx=np.zeros((n, pmax)),
               n_pts=np.array([r["kappa"].size for r in RECORDS], dtype=np.int32),
               obj_pos=np.array([r["obj_pos"] for r in RECORDS]),
               set=np.array([sets.index(r["glob_rl"].tobytes()) for r in RECORDS], dtype=np.int32),
               labels=np.array([r["labels"] for r in RECORDS], dtype=np.int64), label_names=np.array(BRANCHES),
               control_type=np.array([r["control_type"] for r in RECORDS]),
               control_params=np.array([[r["control_params"].get(k, 0.0) for k in ("c_p", "k_d", "k_p", "tan_w")]
                                        for r in RECORDS]),
               has_gg=np.array([not np.all(r["loc_gg"] == r["loc_gg"][0]) for r in RECORDS]),
               too_close=np.array([r["too_close"] for r in RECORDS]), vel_bound=np.array([r["vel_bound"] for r in RECORDS]),
               kind=np.array([r["kind"] for r in RECORDS], dtype=np.int32))
    for k in ("v_start", "v_ego", "v_obj", "safety_d", "obj_dist", "vel_max", "gg_scale", "dyn_model_exp", "drag",
              "mass", "len_veh"):
        out[k] = np.array([r[k] for r in RECORDS], dtype=np.float64)
    for i, r in enumerate(RECORDS):
        k = r["kappa"].size
        out["kappa"][i, :k], out["el"][i, :k], out["loc_gg"][i, :k], out["vx"][i, :k] = r["kappa"], r["el"], r["loc_gg"], r["vx"]
    axm = RECORDS[0]["ax_max_machines"]
    assert all(np.array_equal(r["ax_max_machines"], axm) for r in RECORDS)
    out["ax_max_machines"] = axm
    for s, g in glob.items():
        out["glob_rl_%d" % s] = g
    return out


def main():
    graph_ltpl = GG.load_reference()
    install(graph_ltpl)
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    from tests.helpers import local_gg_field
    track = Track(GG.REF + "/inputs/traj_ltpl_cl/traj_ltpl_cl_monteblanco.csv")
    ltpl = tick_calls(graph_ltpl, track, "default", {}, "PD", 1.0, 24, 811)
    loop_calls(graph_ltpl, ltpl, track, "default", 8, 8, 821)
    tick_calls(graph_ltpl, track, "default", {}, "PD", 1.0, 16, 812, gg_fn=local_gg_field)
    tick_calls(graph_ltpl, track, "default", {}, "PDtan", 1.5, 24, 813)
    l216 = dict(__import__("ast").literal_eval(str(np.load(os.path.join(GG.GOLDEN, "ticks_l216.npz"))["overrides"])))
    tick_calls(graph_ltpl, track, "l216", l216, "PDtan", 1.0, 16, 814, gg_fn=local_gg_field)
    l216_ltpl = tick_calls(graph_ltpl, track, "l216", l216, "PD", 1.5, 16, 815)
    loop_calls(graph_ltpl, l216_ltpl, track, "l216", 8, 8, 822, gg_fn=local_gg_field)
    glob_rl = ltpl._Graph_LTPL__oth._OnlineTrajectoryHandler__vp_fb._VpForwardBackward__glob_rl_clsd
    direct_calls(graph_ltpl, glob_rl, GG.ax_max_machines_table())
    out = pack()
    missing = [b for i, b in enumerate(BRANCHES) if not np.any(out["labels"] & (1 << i))]
    assert not missing, missing
    np.savez_compressed(os.path.join(GG.GOLDEN, "vel_follow.npz"), **out)
    assert all(np.any(out["kind"] == k) for k in (0, 1, 2))
    print("vel_follow.npz: %d calls (%d from first ticks, %d from closed loops), P <= %d" % (
        out["labels"].size, int((out["kind"] == 0).sum()), int((out["kind"] == 2).sum()), out["kappa"].shape[1]))


if __name__ == "__main__":
    main()
