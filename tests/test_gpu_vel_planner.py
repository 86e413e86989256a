"""The stand-alone velocity planner on the device (VelocityPlanner, ltpl_vel_plan_batch): the dense entry's bytes,
per-point friction and ragged lengths against the tph restatement, the brake profile, strided rows, and calls without a
host synchronisation and from a CUDA graph."""
import numpy as np
import pytest
import torch

from tests import helpers as H
from tests.test_vel_planner_cpu import asym_field

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _axm():
    return H.golden("ticks_default.npz")["ax_max_machines"]


def _inputs(n, p, seed):
    from graphbasedlocaltrajectoryplanner_b200.scenarios import make_velocity_microbench
    mb = make_velocity_microbench(n, p, seed=seed)
    s = np.cumsum(mb["el"], axis=1) - mb["el"]
    gg = np.stack([asym_field(s[i], phase=0.1 * i) for i in range(n)])
    return mb, gg


def _planner(exp=1.0, drag=0.85, mass=1000.0, vel_max=60.0, gg_scale=1.0):
    from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner
    vp = VelocityPlanner(veh_param_dyn_model_exp=exp, veh_param_dragcoeff=drag, veh_param_mass=mass, device=DEV)
    vp.update_dyn_parameters(vel_max=vel_max, gg_scale=gg_scale, ax_max_machines=_axm())
    return vp


def _check_tph(vx, ax, ref, el):
    from oracle import tph_port as tph
    ref_ax = tph.calc_ax_profile(ref, el)
    rel = float(np.max(np.abs(vx - ref) / (1e-3 + np.abs(ref))))
    da = float(np.max(np.abs(ax[:-1] - ref_ax)))
    assert rel < 1e-4 and da < 5e-3 and ax[-1] == 0.0, (rel, da, ax[-1])


@pytest.mark.parametrize("n,p,exp,drag,mass,vel_max,gg_scale,gg", [
    (256, 500, 1.0, 0.85, 1000.0, 60.0, 1.0, (5.0, 5.0)), (70, 137, 1.5, 0.9, 1200.0, 55.0, 0.9, (4.5, 5.5))])
def test_constant_friction_gives_the_bytes_of_the_dense_entry(n, p, exp, drag, mass, vel_max, gg_scale, gg):
    """n_pts and gg NULL: the bytes of ltpl_velprofile_batch, with el rows of P (dense solver) and of P - 1 (general
    layout)"""
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    from graphbasedlocaltrajectoryplanner_b200.velprofile import calc_vel_profile_batch
    mb, _ = _inputs(n, p, seed=3)
    pl = BatchPlanner(H.lattice_for("l216"), device=DEV, veh_param_dyn_model_exp=exp, veh_param_dragcoeff=drag,
                      veh_param_mass=mass)
    pl.set_vel_params(vel_max=vel_max, gg_scale=gg_scale, local_gg=gg, ax_max_machines=_axm(), safety_d=30.0)
    vx0, ax0 = calc_vel_profile_batch(pl, mb["kappa"], mb["el"], mb["v_start"], mb["v_end"])
    vp = _planner(exp, drag, mass, vel_max, gg_scale)
    for el in (mb["el"], mb["el"][:, :-1]):
        vx, ax = vp.calc_vel_profile(mb["kappa"], el, gg, mb["v_start"], mb["v_end"])
        assert np.array_equal(vx, vx0) and np.array_equal(ax, ax0)


@pytest.mark.parametrize("exp", [1.0, 1.5])
def test_per_point_friction_matches_tph(exp):
    """loc_gg [N][P][2] from a smooth asymmetric field, times gg_scale, with tph's mirrored friction in the backward
    sweep (test_vel_planner_cpu.py shows the unmirrored solve misses this tolerance)"""
    from oracle import tph_port as tph
    n, p = 48, 160
    mb, gg = _inputs(n, p, seed=5)
    vp = _planner(exp=exp, gg_scale=0.8)
    vx, ax = vp.calc_vel_profile(mb["kappa"], mb["el"][:, :-1], gg, mb["v_start"], mb["v_end"])
    for i in range(n):
        ref = tph.calc_vel_profile(ax_max_machines=_axm(), kappa=mb["kappa"][i], el_lengths=mb["el"][i, :-1],
                                   closed=False, drag_coeff=0.85, m_veh=1000.0, loc_gg=gg[i] * 0.8, v_max=60.0,
                                   v_start=mb["v_start"][i], v_end=mb["v_end"][i], dyn_model_exp=exp)
        _check_tph(vx[i], ax[i], ref, mb["el"][i, :-1])


def _ragged(n, p, seed):
    rng = np.random.default_rng(seed)
    n_pts = rng.integers(2, p + 1, size=n)
    n_pts[:3] = (2, 3, p)
    mb, gg = _inputs(n, p, seed=seed)
    kappa, el = mb["kappa"].copy(), mb["el"].copy()
    for i, m in enumerate(n_pts):   # NaN in every element the planner must not read
        kappa[i, m:] = np.nan
        el[i, m - 1:] = np.nan
        gg[i, m:] = np.nan
    return mb, kappa, el, gg, n_pts


@pytest.mark.parametrize("per_point", [False, True])
def test_ragged_lengths(per_point):
    from oracle import tph_port as tph
    n, p = 64, 150
    mb, kappa, el, gg, n_pts = _ragged(n, p, seed=7)
    loc = gg if per_point else (5.0, 4.5)
    vp = _planner(gg_scale=0.9)
    vx, ax = vp.calc_vel_profile(kappa, el, loc, mb["v_start"], mb["v_end"], n_pts=n_pts)
    for i, m in enumerate(n_pts):
        g = gg[i, :m] if per_point else np.tile(loc, (m, 1))
        ref = tph.calc_vel_profile(ax_max_machines=_axm(), kappa=kappa[i, :m], el_lengths=el[i, :m - 1], closed=False,
                                   drag_coeff=0.85, m_veh=1000.0, loc_gg=g * 0.9, v_max=60.0,
                                   v_start=mb["v_start"][i], v_end=mb["v_end"][i])
        _check_tph(vx[i, :m], ax[i, :m], ref, el[i, :m - 1])
        assert not np.any(vx[i, m:]) and not np.any(ax[i, m:]), i
        # the same path planned alone, with n_points equal to its length
        one = vp.calc_vel_profile(kappa[i:i + 1, :m], el[i:i + 1, :m - 1], gg[i:i + 1, :m] if per_point else loc,
                                  mb["v_start"][i:i + 1], mb["v_end"][i:i + 1])
        assert np.array_equal(one[0][0], vx[i, :m]) and np.array_equal(one[1][0], ax[i, :m]), i
    # a length out of range on the device: a row of NaN, every other row as before
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    bad = n_pts.astype(np.int32)
    bad[5], bad[40] = 1, p + 1
    args = (d(kappa), d(el), d(gg) if per_point else loc, d(mb["v_start"]), d(mb["v_end"]))
    vx2, ax2 = (t.cpu().numpy() for t in vp.calc_vel_profile(*args, n_pts=d(bad)))
    for i in range(n):
        if i in (5, 40):
            assert np.all(np.isnan(vx2[i])) and np.all(np.isnan(ax2[i])), i
        else:
            assert np.array_equal(vx2[i], vx[i]) and np.array_equal(ax2[i], ax[i]), i


@pytest.mark.parametrize("exp", [1.0, 1.5])
@pytest.mark.parametrize("per_point", [False, True])
def test_brake_profile_matches_tph(exp, per_point):
    """tph.calc_vel_profile_brake with the raw friction (no gg_scale), ragged lengths; many paths stop mid-path and
    are zero behind their standstill"""
    from oracle import tph_port as tph
    n, p = 64, 200
    mb, kappa, el, gg, n_pts = _ragged(n, p, seed=9)
    v_start = np.linspace(2.0, 45.0, n)
    v_start[7] = -1.0   # clamped to 0 as tph does
    loc = gg if per_point else (4.0, 5.0)
    vp = _planner(exp=exp, gg_scale=0.5)   # gg_scale is not applied in the brake mode
    vx, ax = vp.calc_vel_brake_em(kappa, el, loc, v_start, n_pts=n_pts)
    worst, stopped = 0.0, 0
    for i, m in enumerate(n_pts):
        g = gg[i, :m] if per_point else np.tile(loc, (m, 1))
        ref = tph.calc_vel_profile_brake(kappa=kappa[i, :m], el_lengths=el[i, :m - 1], v_start=v_start[i],
                                         drag_coeff=0.85, m_veh=1000.0, loc_gg=g, dyn_model_exp=exp)
        err = np.abs(vx[i, :m] - ref)
        assert np.all(err <= 1e-9 * np.abs(ref) + 1e-9), (i, float(err.max()))
        worst = max(worst, float(err.max()))
        ref_ax = tph.calc_ax_profile(ref, el[i, :m - 1], eq_length_output=True)
        assert np.all(np.abs(ax[i, :m] - ref_ax) <= 1e-6), i
        z = np.nonzero(ref[1:] == 0.0)[0]
        if z.size and z[0] + 1 < m - 1:
            stopped += 1
            assert not np.any(vx[i, z[0] + 1:m]), i
        assert not np.any(vx[i, m:]) and not np.any(ax[i, m:]), i
    assert stopped >= 8, stopped
    print("brake exp %.1f per_point %s: worst |vx - tph| = %.3e m/s" % (exp, per_point, worst))


@pytest.mark.parametrize("brake", [False, True])
def test_row_slices_give_the_bytes_of_contiguous_rows(brake):
    n, p = 45, 97
    mb, gg = _inputs(n, p, seed=11)
    vp = _planner()
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)

    def wide(a, extra):
        w = torch.full((a.shape[0], a.shape[1] + extra) + a.shape[2:], float("nan"), dtype=torch.float64, device=DEV)
        w[:, :a.shape[1]] = d(a)
        return w[:, :a.shape[1]]

    def call(k, e, g, vs, ve, out=None):
        if brake:
            return vp.calc_vel_brake_em(k, e, g, vs, out=out)
        return vp.calc_vel_profile(k, e, g, vs, ve, out=out)

    want = call(d(mb["kappa"]), d(mb["el"]), d(gg), d(mb["v_start"]), d(mb["v_end"]))
    ow = [torch.full((n, p + 5), 7.0, dtype=torch.float64, device=DEV) for _ in range(2)]
    got = call(wide(mb["kappa"], 3), wide(mb["el"], 11), wide(gg, 2), d(mb["v_start"]), d(mb["v_end"]),
               out=(ow[0][:, :p], ow[1][:, :p]))
    for g, w, o in zip(got, want, ow):
        assert torch.equal(g, w)
        assert torch.all(o[:, p:] == 7.0)   # nothing written behind the rows
    # element strides that are not 1 (a transposed view): copied once, same bytes
    kt = d(mb["kappa"].T.copy()).T
    got = call(kt, d(mb["el"]), d(gg), d(mb["v_start"]), d(mb["v_end"]))
    assert all(torch.equal(g, w) for g, w in zip(got, want))


def test_device_calls_without_synchronisation_and_from_a_graph():
    n, p = 300, 180
    mb, kappa, el, gg, n_pts = _ragged(n, p, seed=13)
    vp = _planner(gg_scale=0.95)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    args = (d(kappa), d(el), d(gg), d(mb["v_start"]), d(mb["v_end"]))
    dn = d(n_pts.astype(np.int32))
    out = tuple(torch.empty((n, p), dtype=torch.float64, device=DEV) for _ in range(2))
    bout = tuple(torch.empty((n, p), dtype=torch.float64, device=DEV) for _ in range(2))
    vp.calc_vel_profile(*args, n_pts=dn, out=out)
    vp.calc_vel_brake_em(*args[:4], n_pts=dn, out=bout)
    torch.cuda.synchronize()
    want = [t.clone() for t in out + bout]
    torch.cuda.set_sync_debug_mode("error")
    try:
        vp.calc_vel_profile(*args, n_pts=dn, out=out)
        vp.calc_vel_brake_em(*args[:4], n_pts=dn, out=bout)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(out + bout, want))
    for t in out + bout:
        t.zero_()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            vp.calc_vel_profile(*args, n_pts=dn, out=out)
            vp.calc_vel_brake_em(*args[:4], n_pts=dn, out=bout)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        for t in out + bout:
            t.fill_(3.0)
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(out + bout, want))
