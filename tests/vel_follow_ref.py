"""Shared pieces of the follow-mode velocity tests (VelocityPlanner.calc_vel_profile_follow): the lattice-free oracle
helper, seeded random inputs on the Monteblanco race line, and the branch labels of tests/golden/vel_follow.npz."""
import types

import numpy as np

from tests import helpers as H

# branch labels of one CVPF call (tests/tools/gen_golden_follow.py reads them off the reference's own locals)
BRANCHES = ("too_close", "not_too_close", "ego_stop_ge_s_stop", "seg1", "no_seg1", "stop_idx_lt2", "ctrl_len0",
            "v_end_rl", "opp_wrap")


def race_line():
    """the closed Monteblanco race line [M + 1][5] as Lattice.glob_rl stores it"""
    return np.asarray(H.lattice_for("default").glob_rl, dtype=np.float64)


def follow_ref(glob_rl, len_veh, control_type, control_params, veh, vk, kappa, el, loc_gg, v_start, v_ego, v_obj,
               safety_d, obj_dist, obj_pos):
    """one path through OracleLTPL.calc_vel_profile_follow (CVPF:78-313) on a namespace that carries only what the
    method reads; returns (vx, ax, too_close, vel_bound) with ax = (v[p+1]^2 - v[p]^2) / (2 el[p]) and 0 at the end.
    veh: dyn_model_exp, drag_coeff, m_veh; vk: vel_max, gg_scale, ax_max_machines; loc_gg a tuple or [P][2]."""
    from oracle.ltpl_oracle import OracleLTPL
    kappa = np.asarray(kappa, dtype=np.float64)
    el = np.asarray(el, dtype=np.float64)
    gg = np.tile(np.asarray(loc_gg, dtype=np.float64), (kappa.size, 1)) if isinstance(loc_gg, tuple) \
        else np.asarray(loc_gg, dtype=np.float64)
    ns = types.SimpleNamespace(lat=types.SimpleNamespace(veh_length=float(len_veh), glob_rl=np.asarray(glob_rl)),
                               p=dict(controller_type=control_type, control_params=dict(control_params)), **veh)
    vk = dict(vk, ax_max_machines=np.atleast_2d(np.asarray(vk["ax_max_machines"], dtype=np.float64)))
    vx, too_close, vel_bound = OracleLTPL.calc_vel_profile_follow(ns, kappa, el, gg, float(v_start), float(v_ego),
                                                                  float(v_obj), float(safety_d), float(obj_dist),
                                                                  list(obj_pos), vk)
    vx = np.asarray(vx, dtype=np.float64)
    ax = np.zeros_like(vx)
    ax[:-1] = (vx[1:] ** 2 - vx[:-1] ** 2) / (2 * el[:vx.size - 1])
    return vx, ax, bool(too_close), bool(vel_bound)


def random_inputs(n, p, seed, glob_rl, lateral=3.0):
    """config-5 curvature rows (make_velocity_microbench) with the path's whole el column, and follow scalars: an
    opponent near a random race-line point, distances, speeds and safety distances that reach every branch"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_velocity_microbench
    mb = make_velocity_microbench(n, p, seed=seed)
    rng = np.random.default_rng(seed + 1)
    m = glob_rl.shape[0] - 1
    j = rng.integers(0, m, size=n)
    obj_pos = glob_rl[j, 1:3] + rng.uniform(-lateral, lateral, size=(n, 2))
    v_start = mb["v_start"] * 1.5
    return dict(kappa=mb["kappa"], el=mb["el"], v_start=v_start, v_ego=v_start + rng.uniform(-2.0, 2.0, size=n),
                v_obj=rng.uniform(0.0, 50.0, size=n), safety_d=rng.uniform(5.0, 40.0, size=n),
                obj_dist=rng.uniform(0.0, 250.0, size=n), obj_pos=obj_pos)


def check_rows(vx, ax, tc, vb, ref, ctx=""):
    """vx / ax at the north-star tolerances (brake-to-standstill tails also in w = v^2, helpers.assert_close), flags
    exact; ref: list of follow_ref results, one per row (rows may be longer: the rest must be 0)"""
    for r, (rvx, rax, rtc, rvb) in enumerate(ref):
        k = rvx.size
        H.assert_close("follow", np.column_stack((vx[r, :k], ax[r, :k])), np.column_stack((rvx, rax)), ["vx", "ax"],
                       ctx="%s row %d" % (ctx, r), w_rel=H.W_REL_BRAKE)
        assert not np.any(vx[r, k:]) and not np.any(ax[r, k:]), "%s row %d: tail not zero" % (ctx, r)
        assert bool(tc[r]) == rtc and bool(vb[r]) == rvb, "%s row %d flags %s %s, want %s %s" % (
            ctx, r, bool(tc[r]), bool(vb[r]), rtc, rvb)
