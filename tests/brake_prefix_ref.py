"""Shared pieces of the brake-prefix tests (VelocityPlanner.check_brake_prefix): the oracle call on one path, the calls
of tests/golden/brake_prefix.npz and their labels."""
import types

import numpy as np

# labels of one recorded call (tests/tools/gen_golden_brake_prefix.py)
LABELS = ("no_prefix", "prefix_cut", "prefix_unreached", "cut_at_standstill", "empty_course", "per_point_gg",
          "old_ne_current", "exp_1_5", "boundary")


def prefix_ref(vel_plan, vel_course, kappa, el, loc_gg, old, vel_max, gg_scale, exp, drag, mass):
    """one path through OracleLTPL.vp_check_brake_prefix (VPFB:86-139) on a namespace that carries only what the method
    reads; returns (vx_prefix, pref_idx, vel_start, old_gg_scale after the call).  loc_gg a tuple or [P][2]."""
    from oracle.ltpl_oracle import OracleLTPL
    kappa = np.asarray(kappa, dtype=np.float64)
    gg = np.tile(np.asarray(loc_gg, dtype=np.float64), (kappa.size, 1)) if isinstance(loc_gg, tuple) \
        else np.asarray(loc_gg, dtype=np.float64)
    ns = types.SimpleNamespace(old_gg_scale=float(old), dyn_model_exp=float(exp), drag_coeff=float(drag),
                               m_veh=float(mass))
    vk = dict(vel_max=float(vel_max), gg_scale=float(gg_scale))
    vx_prefix, pref_idx, vel_start = OracleLTPL.vp_check_brake_prefix(
        ns, float(vel_plan), np.asarray(vel_course, dtype=np.float64), kappa, np.asarray(el, dtype=np.float64), gg, vk)
    return np.asarray(vx_prefix, dtype=np.float64), int(pref_idx), float(vel_start), ns.old_gg_scale


def golden_call(g, c):
    """the arguments of recorded call c: (vel_plan, vel_course, kappa, el, loc_gg, old_before, vel_max, gg_scale, exp,
    drag, mass)"""
    p, k = int(g["n_pts"][c]), int(g["n_course"][c])
    return (float(g["vel_plan"][c]), g["vel_course"][c, :k], g["kappa"][c, :p], g["el"][c, :p - 1], g["loc_gg"][c, :p],
            float(g["old_before"][c]), float(g["vel_max"][c]), float(g["gg_scale"][c]), float(g["dyn_model_exp"][c]),
            float(g["drag"][c]), float(g["mass"][c]))


def has(g, label):
    return (g["labels"] & (1 << LABELS.index(label))) != 0
