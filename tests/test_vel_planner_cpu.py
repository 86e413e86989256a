"""The stand-alone velocity planner without a GPU: the ctypes mirror of LtplVelPlan, the library's refusals (each with
its field named, nothing launched), the Python argument checks, and the friction mirror of tph's backward sweep that the
kernel reproduces."""
import ctypes
import os
import re

import numpy as np
import pytest

from tests import helpers as H

HEADER = os.path.join(H.REPO, "include", "ltpl_b200.h")


def _lib():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    return capi, capi.load_library()


def _valid_plan(capi):
    """every field set (fake device pointers): the checks pass up to the one a test breaks"""
    vp = capi.VelPlan()
    vp.mode, vp.n_paths, vp.n_points = capi.VP_PROFILE, 4, 10
    for name in ("kappa", "el", "v_start", "v_end", "vx", "ax"):
        setattr(vp, name, 256)
    vp.kappa_s, vp.el_s, vp.out_s = 10, 9, 10
    return vp


def _params(capi, vel_max=50.0, axm_top=60.0):
    prm = capi.Params()
    prm.n_axm, prm.vel_max, prm.axm_v[0] = 1, vel_max, axm_top
    return prm


def test_vel_plan_mirror_carries_its_size():
    capi, lib = _lib()
    body = re.search(r"typedef struct LtplVelPlan \{(.*?)\} LtplVelPlan;", open(HEADER).read(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*[;,]", body)
    assert fields == [f for f, _ in capi.VelPlan._fields_], fields
    vp = capi.VelPlan()
    assert vp.struct_bytes == ctypes.sizeof(capi.VelPlan) == 112
    prm = _params(capi, vel_max=70.0)   # refused by the machine-limit check, the last one: nothing can launch

    def error(size):
        vp2 = _valid_plan(capi)
        vp2.struct_bytes = size
        n0 = lib.ltpl_launch_count()
        assert lib.ltpl_vel_plan_batch(ctypes.byref(prm), ctypes.byref(vp2), None) == -1
        assert lib.ltpl_launch_count() == n0
        return lib.ltpl_last_error().decode()

    assert "struct_bytes" not in error(112) and "ax_max_machines" in error(112)
    for size in (0, 104, 120):
        assert "struct_bytes" in error(size)
    # the other structs keep their sizes and the ABI version
    assert lib.ltpl_sizeof(6) == -1 and capi.ABI_VERSION == lib.ltpl_version() == 20
    assert lib.ltpl_sizeof(4) == ctypes.sizeof(capi.VelBatch)


def test_vel_plan_refuses_bad_arguments_before_launching():
    capi, lib = _lib()

    def refused(field, change, prm=None):
        vp = _valid_plan(capi)
        change(vp)
        prm = prm if prm is not None else _params(capi, vel_max=70.0)   # otherwise refused only at the machine limits
        n0 = lib.ltpl_launch_count()
        assert lib.ltpl_vel_plan_batch(ctypes.byref(prm), ctypes.byref(vp), None) == -1
        msg = lib.ltpl_last_error().decode()
        assert field in msg, (field, msg)
        assert lib.ltpl_launch_count() == n0

    refused("vp.mode", lambda v: setattr(v, "mode", 2))
    refused("vp.n_paths", lambda v: setattr(v, "n_paths", 0))
    refused("vp.n_points", lambda v: setattr(v, "n_points", 1))
    for name in ("kappa", "el", "v_start", "v_end", "vx", "ax"):
        refused("vp.%s" % name, lambda v, name=name: setattr(v, name, None))
    refused("vp.kappa_s", lambda v: setattr(v, "kappa_s", 9))
    refused("vp.el_s", lambda v: setattr(v, "el_s", 8))
    refused("vp.out_s", lambda v: setattr(v, "out_s", 9))
    refused("vp.gg_s", lambda v: (setattr(v, "gg", 256), setattr(v, "gg_s", 19)))
    refused("params.n_axm", lambda v: None, prm=_bad_axm(capi))
    refused("ax_max_machines", lambda v: None)
    # the brake mode has no v_end and does not read the machine limits: a plan that passes every check would launch,
    # so it is only broken at its output stride here
    refused("vp.out_s", lambda v: (setattr(v, "mode", capi.VP_BRAKE), setattr(v, "v_end", None),
                                    setattr(v, "out_s", 9)))
    # the old entry goes through the same checks
    vb = capi.VelBatch()
    vb.n_paths, vb.n_points = 4, 1
    assert lib.ltpl_velprofile_batch(ctypes.byref(_params(capi)), ctypes.byref(vb), None) == -1
    assert "n_points" in lib.ltpl_last_error().decode()


def _bad_axm(capi):
    prm = _params(capi)
    prm.n_axm = 0
    return prm


def test_python_argument_checks():
    """shapes, dtypes and host lengths are refused before anything is uploaded or launched (no GPU: a call that passed
    would fail at the upload)"""
    import torch
    from graphbasedlocaltrajectoryplanner_b200 import velprofile
    _lib()
    vp = velprofile.VelocityPlanner(device="cuda:0")
    with pytest.raises(RuntimeError, match="update_dyn_parameters"):
        vp.calc_vel_profile(np.zeros((2, 5)), np.ones((2, 4)), (5.0, 5.0), np.zeros(2), np.zeros(2))
    with pytest.raises(RuntimeError, match="entire velocity range"):
        vp.update_dyn_parameters(vel_max=80.0, gg_scale=1.0, ax_max_machines=[[0.0, 5.0], [60.0, 3.0]])
    vp.update_dyn_parameters(vel_max=50.0, gg_scale=1.0, ax_max_machines=[[0.0, 5.0], [60.0, 3.0]])
    k, e = np.zeros((3, 6)), np.ones((3, 5))
    with pytest.raises(ValueError, match="CUDA tensor"):   # a CPU tensor is not a device tensor
        vp.calc_vel_profile(torch.zeros(3, 6, dtype=torch.float64), e, (5.0, 5.0), np.zeros(3), np.zeros(3))
    upload = velprofile.VelocityPlanner._upload
    with pytest.raises(ValueError, match="n_pts"):
        upload(vp, k, e, (5.0, 5.0), np.zeros(3), np.zeros(3), np.array([2, 7, 6]))
    with pytest.raises(ValueError, match="n_pts"):
        upload(vp, k, e, (5.0, 5.0), np.zeros(3), np.zeros(3), np.array([2, 1, 6]))
    with pytest.raises(ValueError, match="n_pts"):
        upload(vp, k, e, (5.0, 5.0), np.zeros(3), np.zeros(3), np.array([2.0, 3.0, 6.0]))
    with pytest.raises(ValueError, match="kappa"):
        upload(vp, np.zeros(6), e, (5.0, 5.0), np.zeros(3), np.zeros(3), None)
    with pytest.raises(ValueError, match="cannot be mixed"):
        upload(vp, k, torch.ones(3, 5, dtype=torch.float64), (5.0, 5.0), np.zeros(3), np.zeros(3), None)


def _solve_unmirrored(axm, kappa, el, loc_gg, v_max, v_start, v_end):
    """tph_port.calc_vel_profile with the backward sweep reading each point's OWN friction (what tph does not do)"""
    from oracle import tph_port as tph
    orig = tph._solver_fb_acc_profile

    def patched(p_ggv, *args, backwards=False, **kw):
        return orig(np.flipud(p_ggv) if backwards else p_ggv, *args, backwards=backwards, **kw)
    tph._solver_fb_acc_profile = patched
    try:
        return tph.calc_vel_profile(ax_max_machines=axm, kappa=kappa, el_lengths=el, closed=False, drag_coeff=0.85,
                                    m_veh=1000.0, loc_gg=loc_gg, v_max=v_max, v_start=v_start, v_end=v_end)
    finally:
        tph._solver_fb_acc_profile = orig


def asym_field(s, phase=0.0):
    """a smooth friction field that is not symmetric along the path: (ax_max, ay_max) rising and falling unevenly"""
    ax = 3.5 + 2.0 * (s / s[-1]) ** 2 + 0.3 * np.sin(s / 40.0 + phase)
    ay = 4.0 + 2.5 * (s / s[-1]) + 0.4 * np.cos(s / 55.0 + phase)
    return np.column_stack((ax, ay))


def test_backward_sweep_reads_mirrored_friction():
    """the GPU tests bite on the mirror: on one asymmetric friction field, tph's result and the same solve with the
    friction of each point's own position in the backward sweep differ by far more than the GPU tolerance"""
    from oracle import tph_port as tph
    axm = H.golden("ticks_default.npz")["ax_max_machines"]
    n = 300
    el = np.full(n - 1, 2.5)
    s = np.concatenate(([0.0], np.cumsum(el)))
    kappa = 0.012 * np.sin(s / 90.0) + 0.004
    gg = asym_field(s)
    ref = tph.calc_vel_profile(ax_max_machines=axm, kappa=kappa, el_lengths=el, closed=False, drag_coeff=0.85,
                               m_veh=1000.0, loc_gg=gg, v_max=60.0, v_start=20.0, v_end=5.0)
    alt = _solve_unmirrored(axm, kappa, el, gg, 60.0, 20.0, 5.0)
    rel = np.max(np.abs(alt - ref) / (1e-3 + np.abs(ref)))
    assert rel > 100 * 1e-4, rel
