"""Follow-mode velocity profiles without a GPU: the ctypes mirror of LtplVelFollow, the refusals of ltpl_vel_follow_batch
(each with its field named, nothing launched), the Python argument checks, and the lattice-free oracle helper against
every call of the reference recorded in tests/golden/vel_follow.npz."""
import ctypes
import os
import re

import numpy as np
import pytest

from tests import helpers as H
from tests import vel_follow_ref as R

HEADER = os.path.join(H.REPO, "include", "ltpl_b200.h")
SIZE = 192


def _lib():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    return capi, capi.load_library()


def _valid(capi):
    """every field set (fake, aligned device pointers): the checks pass up to the one a test breaks"""
    vf = capi.VelFollow()
    vf.n_paths, vf.n_points, vf.n_glob = 4, 10, 50
    for name in ("kappa", "el", "v_start", "v_ego", "v_obj", "safety_d", "obj_dist", "obj_pos", "glob_rl", "vx", "ax",
                 "too_close", "vel_bound"):
        setattr(vf, name, 256)
    vf.kappa_s, vf.el_s, vf.out_s, vf.obj_pos_s = 10, 10, 10, 2
    return vf


def _params(capi, vel_max=70.0, axm_top=60.0):
    """vel_max above the machine table: refused by the machine-limit check, the last one but one (nothing launches)"""
    prm = capi.Params()
    prm.n_axm, prm.vel_max, prm.axm_v[0] = 1, vel_max, axm_top
    return prm


def test_vel_follow_mirror_matches_the_header_and_carries_its_size():
    capi, lib = _lib()
    body = re.search(r"typedef struct LtplVelFollow \{(.*?)\} LtplVelFollow;", open(HEADER).read(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*[;,]", body)
    assert fields == [f for f, _ in capi.VelFollow._fields_], fields
    vf = capi.VelFollow()
    assert vf.struct_bytes == ctypes.sizeof(capi.VelFollow) == SIZE
    prm = _params(capi)

    def error(size):
        v = _valid(capi)
        v.struct_bytes = size
        n0 = lib.ltpl_launch_count()
        assert lib.ltpl_vel_follow_batch(ctypes.byref(prm), ctypes.byref(v), None) == -1
        assert lib.ltpl_launch_count() == n0
        return lib.ltpl_last_error().decode()

    # the library's sizeof(LtplVelFollow) is the mirror's: only that size gets past the first check
    assert "struct_bytes" not in error(SIZE) and "ax_max_machines" in error(SIZE)
    for size in (0, SIZE - 8, SIZE + 8, 112):
        assert "struct_bytes" in error(size)
    # the struct is not registered in ltpl_sizeof, the ABI version stays
    assert lib.ltpl_sizeof(6) == -1 and capi.ABI_VERSION == lib.ltpl_version() == 20


def test_vel_follow_refuses_bad_arguments_before_launching():
    capi, lib = _lib()

    def refused(field, change, prm=None):
        vf = _valid(capi)
        change(vf)
        prm = prm if prm is not None else _params(capi)
        n0 = lib.ltpl_launch_count()
        assert lib.ltpl_vel_follow_batch(ctypes.byref(prm), ctypes.byref(vf), None) == -1
        msg = lib.ltpl_last_error().decode()
        assert field in msg, (field, msg)
        assert lib.ltpl_launch_count() == n0

    refused("vf.n_paths", lambda v: setattr(v, "n_paths", 0))
    refused("vf.n_points", lambda v: setattr(v, "n_points", 1))
    refused("vf.n_glob", lambda v: setattr(v, "n_glob", 1))
    for name in ("kappa", "el", "v_start", "v_ego", "v_obj", "safety_d", "obj_dist", "obj_pos", "glob_rl", "vx", "ax",
                 "too_close", "vel_bound"):
        refused("vf.%s" % name, lambda v, name=name: setattr(v, name, None))
    for name in ("kappa", "el", "v_start", "v_ego", "v_obj", "safety_d", "obj_dist", "obj_pos", "glob_rl", "vx", "ax"):
        refused("vf.%s" % name, lambda v, name=name: setattr(v, name, 260))   # 4-byte aligned only
    refused("vf.n_pts", lambda v: setattr(v, "n_pts", 258))
    refused("vf.gg", lambda v: setattr(v, "gg", 260))
    refused("vf.kappa_s", lambda v: setattr(v, "kappa_s", 9))
    refused("vf.el_s", lambda v: setattr(v, "el_s", 9))   # el has n_points entries per row here
    refused("vf.gg_s", lambda v: (setattr(v, "gg", 256), setattr(v, "gg_s", 19)))
    refused("vf.obj_pos_s", lambda v: setattr(v, "obj_pos_s", 1))
    refused("vf.out_s", lambda v: setattr(v, "out_s", 9))
    bad = _params(capi, vel_max=50.0)
    bad.n_axm = 0
    refused("params.n_axm", lambda v: None, prm=bad)
    refused("ax_max_machines", lambda v: None)
    ctl = _params(capi, vel_max=50.0)
    ctl.follow_control_type = 2
    refused("params.follow_control_type", lambda v: None, prm=ctl)


def _follow_args():
    return dict(len_veh=4.7, follow_control_type="PDtan",
                follow_control_params={"c_p": 1.15, "k_d": 0.025, "k_p": 0.2, "tan_w": 15.0}, glob_rl=R.race_line())


def test_python_argument_checks():
    """the follow arguments of the constructor, the missing-configuration errors and the host checks of a call, all
    before anything is uploaded or launched (no GPU: a call that passed would fail at the upload)"""
    import torch
    from graphbasedlocaltrajectoryplanner_b200 import velprofile
    _lib()
    vp = velprofile.VelocityPlanner(device="cuda:0")
    assert vp.follow is None and vp.glob_rl is None
    with pytest.raises(RuntimeError, match="len_veh, follow_control_type"):
        vp.calc_vel_profile_follow(np.zeros((2, 5)), np.ones((2, 5)), (5.0, 5.0), *([np.zeros(2)] * 5),
                                   np.zeros((2, 2)))
    check = velprofile.check_follow_args
    a = _follow_args()
    g6 = check(a["len_veh"], a["follow_control_type"], a["follow_control_params"], a["glob_rl"])
    rl = a["glob_rl"]
    assert g6["glob_rl"].shape == (rl.shape[0] - 1, 6)
    assert np.array_equal(g6["glob_rl"][:, :5], rl[:-1]) and np.array_equal(g6["glob_rl"][:, 5], np.diff(rl[:, 0]))
    assert check(None, None, None, None) is None
    with pytest.raises(ValueError, match="missing glob_rl"):
        check(4.7, "PD", {"c_p": 1.0, "k_d": 0.0, "k_p": 0.1}, None)
    with pytest.raises(ValueError, match="PD"):
        check(4.7, "PID", {"c_p": 1.0, "k_d": 0.0, "k_p": 0.1}, rl)
    with pytest.raises(ValueError, match="tan_w"):
        check(4.7, "PDtan", {"c_p": 1.0, "k_d": 0.0, "k_p": 0.1}, rl)
    with pytest.raises(ValueError, match="glob_rl"):
        check(4.7, "PD", {"c_p": 1.0, "k_d": 0.0, "k_p": 0.1}, rl[:, :4])
    with pytest.raises(ValueError, match="repeated at the end"):
        check(4.7, "PD", {"c_p": 1.0, "k_d": 0.0, "k_p": 0.1}, rl[:-1])
    with pytest.raises(ValueError, match="glob_rl"):
        velprofile.VelocityPlanner(device="cuda:0", **dict(a, glob_rl=rl[:-1]))
    # a planner with follow arguments (built without its upload: no GPU here)
    vp.follow = dict(len_veh=4.7, control_type="PD", control_params={"c_p": 1.0, "k_d": 0.0, "k_p": 0.1})
    with pytest.raises(RuntimeError, match="update_dyn_parameters"):
        vp.calc_vel_profile_follow(np.zeros((2, 5)), np.ones((2, 5)), (5.0, 5.0), *([np.zeros(2)] * 5),
                                   np.zeros((2, 2)))
    vp.update_dyn_parameters(vel_max=50.0, gg_scale=1.0, ax_max_machines=[[0.0, 5.0], [60.0, 3.0]])
    assert vp.params.follow_control_type == 0 and vp.params.follow_c_p == 1.0 and vp.params.follow_k_p == 0.1
    up = vp._upload_follow
    sc = {k: np.zeros(3) for k in ("v_start", "v_ego", "v_obj", "safety_d", "obj_dist")}
    with pytest.raises(ValueError, match=r"whole el column \[N\]\[P\]"):
        vp.calc_vel_profile_follow(np.zeros((3, 6)), np.ones((3, 5)), (5.0, 5.0), *([np.zeros(3)] * 5),
                                   np.zeros((3, 2)))
    with pytest.raises(ValueError, match="CUDA tensor"):
        vp.calc_vel_profile_follow(torch.zeros(3, 6, dtype=torch.float64), torch.ones(3, 6, dtype=torch.float64),
                                   (5.0, 5.0), *([torch.zeros(3, dtype=torch.float64)] * 5),
                                   torch.zeros(3, 2, dtype=torch.float64))
    with pytest.raises(ValueError, match="n_pts"):
        up(np.zeros((3, 6)), np.ones((3, 6)), (5.0, 5.0), sc, np.zeros((3, 2)), np.array([2, 7, 6]))
    with pytest.raises(ValueError, match="cannot be mixed"):
        up(np.zeros((3, 6)), np.ones((3, 6)), (5.0, 5.0), dict(sc, v_obj=torch.zeros(3)), np.zeros((3, 2)), None)
    with pytest.raises(ValueError, match="obj_pos: a numeric array"):
        up(np.zeros((3, 6)), np.ones((3, 6)), (5.0, 5.0), sc, np.array([["a", "b"]] * 3), None)


def _fixture_call(g, c):
    k = int(g["n_pts"][c])
    ctype = str(g["control_type"][c])
    cp = dict(zip(("c_p", "k_d", "k_p", "tan_w"), (float(x) for x in g["control_params"][c])))
    if ctype == "PD":
        cp.pop("tan_w")
    veh = dict(dyn_model_exp=float(g["dyn_model_exp"][c]), drag_coeff=float(g["drag"][c]), m_veh=float(g["mass"][c]))
    vk = dict(vel_max=float(g["vel_max"][c]), gg_scale=float(g["gg_scale"][c]), ax_max_machines=g["ax_max_machines"])
    return R.follow_ref(g["glob_rl_%d" % int(g["set"][c])], float(g["len_veh"][c]), ctype, cp, veh, vk,
                        g["kappa"][c, :k], g["el"][c, :k], g["loc_gg"][c, :k], g["v_start"][c], g["v_ego"][c],
                        g["v_obj"][c], g["safety_d"][c], g["obj_dist"][c], g["obj_pos"][c])


def test_oracle_helper_reproduces_every_fixture_call():
    """the lattice-free helper (OracleLTPL.calc_vel_profile_follow on a namespace) against the reference's own calls:
    vx within float64 rounding, both flags exact; the fixture holds calls from ticks and every branch label"""
    g = H.golden("vel_follow.npz")
    names = [str(s) for s in g["label_names"]]
    assert names == list(R.BRANCHES)
    for i, b in enumerate(names):
        assert np.any(g["labels"] & (1 << i)), b
    # calls from first ticks (0), direct calls (1) and calls inside closed loops (2), on both lattices' race lines; the
    # calls from ticks carry a velocity estimate other than the planned velocity (the controller's k_d term)
    assert all(np.any(g["kind"] == k) for k in (0, 1, 2))
    for k in (0, 2):
        assert np.any(g["v_ego"][g["kind"] == k] != g["v_start"][g["kind"] == k])
    assert set(str(s) for s in g["control_type"]) == {"PD", "PDtan"}
    assert set(float(e) for e in g["dyn_model_exp"]) == {1.0, 1.5} and g["has_gg"].any()
    for c in range(g["labels"].size):
        k = int(g["n_pts"][c])
        vx, _, tc, vb = _fixture_call(g, c)
        want = g["vx"][c, :k]
        assert vx.shape == want.shape
        assert np.allclose(vx, want, rtol=1e-12, atol=1e-9), (c, float(np.max(np.abs(vx - want))))
        assert tc == bool(g["too_close"][c]) and vb == bool(g["vel_bound"][c]), c
