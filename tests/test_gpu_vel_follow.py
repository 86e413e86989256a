"""Follow-mode velocity profiles on the device (VelocityPlanner.calc_vel_profile_follow, ltpl_vel_follow_batch): the
reference's own calls (tests/golden/vel_follow.npz), thousands of random paths against the oracle, ragged lengths,
per-point friction, a race line too long for shared memory, strided rows, and calls without a host synchronisation and
from a CUDA graph."""
import numpy as np
import pytest
import torch

from tests import helpers as H
from tests import vel_follow_ref as R
from tests.test_vel_planner_cpu import asym_field

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
PD = ("PD", {"c_p": 1.25, "k_d": 0.025, "k_p": 0.2})
PDTAN = ("PDtan", {"c_p": 1.15, "k_d": 0.025, "k_p": 0.2, "tan_w": 15.0})
LEN_VEH = 4.7


def _axm():
    return H.golden("ticks_default.npz")["ax_max_machines"]


def _planner(ctrl=PD, glob_rl=None, exp=1.0, drag=0.85, mass=1000.0, vel_max=60.0, gg_scale=1.0, len_veh=LEN_VEH,
             axm=None):
    from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner
    vp = VelocityPlanner(veh_param_dyn_model_exp=exp, veh_param_dragcoeff=drag, veh_param_mass=mass, device=DEV,
                         len_veh=len_veh, follow_control_type=ctrl[0], follow_control_params=ctrl[1],
                         glob_rl=R.race_line() if glob_rl is None else glob_rl)
    vp.update_dyn_parameters(vel_max=vel_max, gg_scale=gg_scale, ax_max_machines=_axm() if axm is None else axm)
    return vp


def _refs(d, glob_rl, ctrl, veh, vk, gg=(5.0, 5.0), n_pts=None):
    out = []
    for i in range(d["kappa"].shape[0]):
        k = d["kappa"].shape[1] if n_pts is None else int(n_pts[i])
        g = gg if isinstance(gg, tuple) else gg[i, :k]
        out.append(R.follow_ref(glob_rl, LEN_VEH, ctrl[0], ctrl[1], veh, vk, d["kappa"][i, :k], d["el"][i, :k], g,
                                d["v_start"][i], d["v_ego"][i], d["v_obj"][i], d["safety_d"][i], d["obj_dist"][i],
                                d["obj_pos"][i]))
    return out


def _call(vp, d, gg=(5.0, 5.0), n_pts=None):
    return vp.calc_vel_profile_follow(d["kappa"], d["el"], gg, d["v_start"], d["v_ego"], d["v_obj"], d["safety_d"],
                                      d["obj_dist"], d["obj_pos"], n_pts=n_pts)


def test_reference_calls_from_the_fixture():
    """every recorded call of the reference (first ticks, closed loops and direct calls) on the device: vx / ax at the
    north-star tolerances, both flags exact; every branch label is present"""
    g = H.golden("vel_follow.npz")
    labels = g["labels"]
    names = [str(s) for s in g["label_names"]]
    assert all(np.any(labels & (1 << names.index(b))) for b in R.BRANCHES), "a branch is missing from the fixture"
    groups = {}
    for c in range(labels.size):
        # every parameter a planner holds: one planner per group
        key = (int(g["set"][c]), float(g["dyn_model_exp"][c]), float(g["drag"][c]), float(g["mass"][c]),
               float(g["len_veh"][c]), str(g["control_type"][c]), tuple(float(x) for x in g["control_params"][c]),
               float(g["vel_max"][c]), float(g["gg_scale"][c]), bool(g["has_gg"][c]))
        groups.setdefault(key, []).append(c)
    for (st, exp, drag, mass, len_veh, ctype, cps, vel_max, gg_scale, has_gg), calls in groups.items():
        ctrl = (ctype, {k: v for k, v in zip(("c_p", "k_d", "k_p", "tan_w"), cps) if not (k == "tan_w" and ctype == "PD")})
        vp = _planner(ctrl, glob_rl=g["glob_rl_%d" % st], exp=exp, drag=drag, mass=mass, vel_max=vel_max,
                      gg_scale=gg_scale, len_veh=len_veh, axm=g["ax_max_machines"])
        idx = np.array(calls)
        n_pts = g["n_pts"][idx].astype(np.int32)
        p = int(n_pts.max())
        args = [g["kappa"][idx, :p], g["el"][idx, :p], g["loc_gg"][idx, :p] if has_gg else
                (float(g["loc_gg"][calls[0], 0, 0]), float(g["loc_gg"][calls[0], 0, 1]))]
        args += [g[k][idx] for k in ("v_start", "v_ego", "v_obj", "safety_d", "obj_dist", "obj_pos")]
        vx, ax, tc, vb = vp.calc_vel_profile_follow(*args, n_pts=n_pts)
        ref = [(g["vx"][c, :n_pts[j]], _ax(g["vx"][c, :n_pts[j]], g["el"][c, :n_pts[j]]), bool(g["too_close"][c]),
                bool(g["vel_bound"][c])) for j, c in enumerate(calls)]
        R.check_rows(vx, ax, tc, vb, ref, ctx="fixture set %d %s exp %g" % (st, ctype, exp))


def _ax(vx, el):
    ax = np.zeros_like(vx)
    ax[:-1] = (vx[1:] ** 2 - vx[:-1] ** 2) / (2 * el[:vx.size - 1])
    return ax


@pytest.mark.parametrize("ctrl,exp,seed", [(PD, 1.0, 11), (PDTAN, 1.0, 12), (PD, 1.5, 13), (PDTAN, 1.5, 14)])
def test_random_paths_against_the_oracle(ctrl, exp, seed):
    """1024 paths per case (4096 in all): config-5 curvature, random opponents on the Monteblanco race line"""
    glob_rl = R.race_line()
    d = R.random_inputs(1024, 160, seed, glob_rl)
    vp = _planner(ctrl, exp=exp, gg_scale=0.9)
    vx, ax, tc, vb = _call(vp, d)
    veh = dict(dyn_model_exp=exp, drag_coeff=0.85, m_veh=1000.0)
    vk = dict(vel_max=60.0, gg_scale=0.9, ax_max_machines=_axm())
    ref = _refs(d, glob_rl, ctrl, veh, vk)
    R.check_rows(vx, ax, tc, vb, ref, ctx="random %s %g" % (ctrl[0], exp))
    # the random set reaches both outcomes of both flags
    assert 0 < int(tc.sum()) < tc.size and 0 < int(vb.sum()) < vb.size


def test_ragged_lengths_and_nan_rows():
    """each path against the oracle on its own length, zeros behind it; device lengths out of range give NaN rows and
    both flags False, the other rows keep their bytes"""
    glob_rl = R.race_line()
    d = R.random_inputs(200, 120, 21, glob_rl)
    rng = np.random.default_rng(22)
    n_pts = rng.integers(2, 121, size=200).astype(np.int32)
    vp = _planner()
    vx, ax, tc, vb = _call(vp, d, n_pts=n_pts)
    veh = dict(dyn_model_exp=1.0, drag_coeff=0.85, m_veh=1000.0)
    vk = dict(vel_max=60.0, gg_scale=1.0, ax_max_machines=_axm())
    R.check_rows(vx, ax, tc, vb, _refs(d, glob_rl, PD, veh, vk, n_pts=n_pts), ctx="ragged")
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in d.items()}
    bad = n_pts.copy()
    bad[[3, 50]] = [1, 121]
    dv = vp.calc_vel_profile_follow(t["kappa"], t["el"], (5.0, 5.0), t["v_start"], t["v_ego"], t["v_obj"],
                                    t["safety_d"], t["obj_dist"], t["obj_pos"], n_pts=torch.from_numpy(bad).to(DEV))
    bx, ba, btc, bvb = (x.cpu().numpy() for x in dv)
    assert np.all(np.isnan(bx[[3, 50]])) and np.all(np.isnan(ba[[3, 50]]))
    assert not btc[[3, 50]].any() and not bvb[[3, 50]].any()
    keep = np.setdiff1d(np.arange(200), [3, 50])
    assert np.array_equal(bx[keep], vx[keep]) and np.array_equal(ba[keep], ax[keep])
    assert np.array_equal(btc[keep], tc[keep]) and np.array_equal(bvb[keep], vb[keep])


@pytest.mark.parametrize("exp", [1.0, 1.5])
def test_per_point_friction(exp):
    """loc_gg [N][P][2]: the ego profiles take it times gg_scale, the backward sweeps of both profiles the mirrored point
    of their own slice"""
    glob_rl = R.race_line()
    d = R.random_inputs(256, 150, 31, glob_rl)
    s = np.cumsum(d["el"], axis=1) - d["el"]
    gg = np.stack([asym_field(s[i], phase=0.1 * i) for i in range(256)])
    vp = _planner(PDTAN, exp=exp, gg_scale=0.85)
    vx, ax, tc, vb = _call(vp, d, gg=gg)
    veh = dict(dyn_model_exp=exp, drag_coeff=0.85, m_veh=1000.0)
    vk = dict(vel_max=60.0, gg_scale=0.85, ax_max_machines=_axm())
    R.check_rows(vx, ax, tc, vb, _refs(d, glob_rl, PDTAN, veh, vk, gg=gg), ctx="gg exp %g" % exp)


def test_long_race_line_is_read_through_l2():
    """a race line resampled to >= 10 000 points does not fit into shared memory: same results as the oracle"""
    g = R.race_line()
    m = g.shape[0] - 1
    f = 13
    t = np.arange(m * f) / f
    j, u = t.astype(int), (t - t.astype(int))[:, None]
    nxt = np.append(np.arange(1, m), 0)
    xyk = g[:-1, 1:5][j] * (1 - u) + g[:-1, 1:5][nxt[j]] * u
    seg = np.sqrt(np.sum(np.diff(np.vstack((xyk[:, :2], xyk[:1, :2])), axis=0) ** 2, axis=1))
    s = np.concatenate(([0.0], np.cumsum(seg)))
    long_rl = np.column_stack((s, np.vstack((xyk, xyk[:1]))))
    assert long_rl.shape[0] - 1 >= 10000
    d = R.random_inputs(256, 150, 41, long_rl, lateral=1.0)
    vp = _planner(PD, glob_rl=long_rl)
    vx, ax, tc, vb = _call(vp, d)
    veh = dict(dyn_model_exp=1.0, drag_coeff=0.85, m_veh=1000.0)
    vk = dict(vel_max=60.0, gg_scale=1.0, ax_max_machines=_axm())
    R.check_rows(vx, ax, tc, vb, _refs(d, long_rl, PD, veh, vk), ctx="long race line")


def _device(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in d.items()}


def test_strided_rows_give_the_bytes_of_contiguous_ones():
    glob_rl = R.race_line()
    d = R.random_inputs(100, 90, 51, glob_rl)
    s = np.cumsum(d["el"], axis=1) - d["el"]
    gg = np.stack([asym_field(s[i], phase=0.2 * i) for i in range(100)])
    vp = _planner()
    t = _device(d)
    tg = torch.from_numpy(gg).to(DEV)
    ref = vp.calc_vel_profile_follow(t["kappa"], t["el"], tg, t["v_start"], t["v_ego"], t["v_obj"], t["safety_d"],
                                     t["obj_dist"], t["obj_pos"])
    wide = {k: torch.zeros((100, 97), dtype=torch.float64, device=DEV) for k in ("kappa", "el")}
    for k in wide:
        wide[k][:, :90] = t[k]
    wg = torch.zeros((100, 95, 2), dtype=torch.float64, device=DEV)
    wg[:, :90] = tg
    wp = torch.zeros((100, 3), dtype=torch.float64, device=DEV)
    wp[:, :2] = t["obj_pos"]
    ovx = torch.full((100, 93), -7.0, dtype=torch.float64, device=DEV)
    oax = torch.full((100, 93), -7.0, dtype=torch.float64, device=DEV)
    otc = torch.ones(100, dtype=torch.bool, device=DEV)
    ovb = torch.zeros(100, dtype=torch.bool, device=DEV)
    got = vp.calc_vel_profile_follow(wide["kappa"][:, :90], wide["el"][:, :90], wg[:, :90], t["v_start"], t["v_ego"],
                                     t["v_obj"], t["safety_d"], t["obj_dist"], wp[:, :2],
                                     out=(ovx[:, :90], oax[:, :90], otc, ovb))
    assert got[0].data_ptr() == ovx.data_ptr()
    for a, b in zip(ref, got):
        assert torch.equal(a, b)
    assert torch.all(ovx[:, 90:] == -7.0) and torch.all(oax[:, 90:] == -7.0)


def test_no_host_sync_and_cuda_graph_replay():
    """a device call under sync debug mode "error", and the same call captured once and replayed from a CUDA graph:
    both give the bytes of the eager call"""
    glob_rl = R.race_line()
    d = R.random_inputs(300, 100, 61, glob_rl)
    vp = _planner(PDTAN)
    t = _device(d)
    args = (t["kappa"], t["el"], (5.0, 5.0), t["v_start"], t["v_ego"], t["v_obj"], t["safety_d"], t["obj_dist"],
            t["obj_pos"])
    ref = [x.clone() for x in vp.calc_vel_profile_follow(*args)]
    torch.cuda.synchronize()
    out = (torch.empty((300, 100), dtype=torch.float64, device=DEV),
           torch.empty((300, 100), dtype=torch.float64, device=DEV),
           torch.empty(300, dtype=torch.bool, device=DEV), torch.empty(300, dtype=torch.bool, device=DEV))
    torch.cuda.set_sync_debug_mode("error")
    try:
        vp.calc_vel_profile_follow(*args, out=out)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    for a, b in zip(ref, out):
        assert torch.equal(a, b)
    for x in out:
        x.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            vp.calc_vel_profile_follow(*args, out=out)
    torch.cuda.current_stream().wait_stream(s)
    for x in out:
        x.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(ref, out):
        assert torch.equal(a, b)
