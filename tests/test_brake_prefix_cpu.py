"""Brake prefixes without a GPU: the ctypes mirror of LtplBrakePrefix, the refusals of ltpl_brake_prefix_batch (each
with its field named, nothing launched), the Python argument checks, and the oracle against every call of the reference
recorded in tests/golden/brake_prefix.npz, bit for bit."""
import ctypes
import os
import re

import numpy as np
import pytest

from tests import brake_prefix_ref as R
from tests import helpers as H

HEADER = os.path.join(H.REPO, "include", "ltpl_b200.h")
SIZE = 160


def _lib():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    return capi, capi.load_library()


def _valid(capi, cap=3):
    """every field set (fake, aligned device pointers): the checks pass up to the one a test breaks"""
    bp = capi.BrakePrefix()
    bp.n_paths, bp.n_points, bp.n_course_cap = 4, 10, cap
    for name in ("kappa", "el", "vel_plan", "vel_course", "old_gg_scale", "vx_prefix", "n_prefix", "pref_idx",
                 "vel_start"):
        setattr(bp, name, 256)
    bp.kappa_s, bp.el_s, bp.vel_course_s, bp.vx_prefix_s = 10, 9, cap, cap + 9
    return bp


def _refused(capi, lib, bp, field):
    prm = capi.Params()
    n0 = lib.ltpl_launch_count()
    assert lib.ltpl_brake_prefix_batch(ctypes.byref(prm), ctypes.byref(bp), None) == -1
    msg = lib.ltpl_last_error().decode()
    assert field in msg, (field, msg)
    assert lib.ltpl_launch_count() == n0
    return msg


def test_brake_prefix_mirror_matches_the_header_and_carries_its_size():
    capi, lib = _lib()
    body = re.search(r"typedef struct LtplBrakePrefix \{(.*?)\} LtplBrakePrefix;", open(HEADER).read(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*[;,]", body)
    assert fields == [f for f, _ in capi.BrakePrefix._fields_], fields
    bp = capi.BrakePrefix()
    assert bp.struct_bytes == ctypes.sizeof(capi.BrakePrefix) == SIZE
    # the library's sizeof(LtplBrakePrefix) is the mirror's: only that size gets past the first check (to n_paths)
    v = _valid(capi)
    v.n_paths = 0
    assert "struct_bytes" not in _refused(capi, lib, v, "bp.n_paths")
    for size in (0, SIZE - 8, SIZE + 8, 192):
        v = _valid(capi)
        v.struct_bytes = size
        _refused(capi, lib, v, "struct_bytes")
    # the struct is not registered in ltpl_sizeof, the ABI version stays
    assert lib.ltpl_sizeof(6) == -1 and capi.ABI_VERSION == lib.ltpl_version() == 20


def test_brake_prefix_refuses_bad_arguments_before_launching():
    capi, lib = _lib()

    def refused(field, change, cap=3):
        bp = _valid(capi, cap)
        change(bp)
        _refused(capi, lib, bp, field)

    refused("bp.n_paths", lambda v: setattr(v, "n_paths", 0))
    refused("bp.n_points", lambda v: setattr(v, "n_points", 1))
    refused("bp.n_course_cap", lambda v: setattr(v, "n_course_cap", -1))
    for name in ("kappa", "el", "vel_plan", "old_gg_scale", "vx_prefix", "n_prefix", "pref_idx", "vel_start",
                 "vel_course"):
        refused("bp.%s" % name, lambda v, name=name: setattr(v, name, None))
    for name in ("kappa", "el", "vel_plan", "old_gg_scale", "vx_prefix", "vel_start", "vel_course"):
        refused("bp.%s" % name, lambda v, name=name: setattr(v, name, 260))   # 4-byte aligned only
    for name in ("n_prefix", "pref_idx", "n_pts", "n_course"):
        refused("bp.%s" % name, lambda v, name=name: setattr(v, name, 258))
    refused("bp.gg", lambda v: setattr(v, "gg", 260))
    refused("bp.kappa_s", lambda v: setattr(v, "kappa_s", 9))
    refused("bp.el_s", lambda v: setattr(v, "el_s", 8))
    refused("bp.gg_s", lambda v: (setattr(v, "gg", 256), setattr(v, "gg_s", 19)))
    refused("bp.vel_course_s", lambda v: setattr(v, "vel_course_s", 2))
    refused("bp.vx_prefix_s", lambda v: setattr(v, "vx_prefix_s", 11))
    # without a course capacity the course pointer may be NULL; the prefix stride is still C + P - 1
    refused("bp.vx_prefix_s", lambda v: (setattr(v, "vel_course", None), setattr(v, "vx_prefix_s", 8)), cap=0)


def test_python_argument_checks():
    """the missing-parameter error and the host checks of a call, all before anything is uploaded or launched (no GPU:
    a call that passed would fail at the upload)"""
    import torch
    from graphbasedlocaltrajectoryplanner_b200 import velprofile
    _lib()
    vp = velprofile.VelocityPlanner(device="cuda:0")
    k, el, vc = np.zeros((3, 6)), np.ones((3, 5)), np.zeros((3, 2))
    mem = np.ones(3)
    with pytest.raises(RuntimeError, match="update_dyn_parameters"):
        vp.check_brake_prefix(np.zeros(3), vc, k, el, (5.0, 5.0), mem)
    vp.update_dyn_parameters(vel_max=50.0, gg_scale=0.9, ax_max_machines=[[0.0, 5.0], [60.0, 3.0]])
    with pytest.raises(ValueError, match="old_gg_scale: a writeable float64"):
        vp.check_brake_prefix(np.zeros(3), vc, k, el, (5.0, 5.0), np.ones(3, dtype=np.float32))
    with pytest.raises(ValueError, match="old_gg_scale: a writeable float64"):
        vp.check_brake_prefix(np.zeros(3), vc, k, el, (5.0, 5.0), np.ones(4))
    with pytest.raises(ValueError, match="old_gg_scale: a writeable float64"):
        vp.check_brake_prefix(np.zeros(3), vc, k, el, (5.0, 5.0), [1.0, 1.0, 1.0])
    with pytest.raises(ValueError, match=r"n_course: every length must be in \[0, 2\]"):
        vp.check_brake_prefix(np.zeros(3), vc, k, el, (5.0, 5.0), mem, n_course=[0, 3, 1])
    with pytest.raises(ValueError, match="n_course: an integer array"):
        vp.check_brake_prefix(np.zeros(3), vc, k, el, (5.0, 5.0), mem, n_course=[0.0, 1.0, 1.0])
    with pytest.raises(ValueError, match="n_pts"):
        vp.check_brake_prefix(np.zeros(3), vc, k, el, (5.0, 5.0), mem, n_pts=[2, 7, 6])
    with pytest.raises(ValueError, match=r"vel_course: an array \[3\]\[C\]"):
        vp.check_brake_prefix(np.zeros(3), np.zeros(3), k, el, (5.0, 5.0), mem)
    with pytest.raises(ValueError, match="cannot be mixed"):
        vp.check_brake_prefix(torch.zeros(3), vc, k, el, (5.0, 5.0), mem)
    with pytest.raises(ValueError, match="vel_plan: a numeric array"):
        vp.check_brake_prefix(np.array(["a"] * 3), vc, k, el, (5.0, 5.0), mem)
    with pytest.raises(ValueError, match="CUDA tensor"):
        t = lambda *s: torch.zeros(*s, dtype=torch.float64)   # noqa: E731
        vp.check_brake_prefix(t(3), t(3, 2), t(3, 6), t(3, 5), (5.0, 5.0), t(3))
    assert np.array_equal(mem, np.ones(3))   # nothing was written


def _oracle(g, c):
    vel_plan, vc, kappa, el, gg, old, vel_max, gg_scale, exp, drag, mass = R.golden_call(g, c)
    return R.prefix_ref(vel_plan, vc, kappa, el, gg, old, vel_max, gg_scale, exp, drag, mass)


def test_oracle_reproduces_every_fixture_call_bit_for_bit():
    """OracleLTPL.vp_check_brake_prefix against the reference's own calls: the prefix, pref_idx, vel_start and the
    memory after the call, bit for bit; every label, every kind, chains whose memory carries from call to call"""
    g = H.golden("brake_prefix.npz")
    assert [str(s) for s in g["label_names"]] == list(R.LABELS)
    for b in R.LABELS:
        assert R.has(g, b).any(), b
    assert all(np.any(g["kind"] == k) for k in (0, 1, 2))
    assert g["has_gg"].any() and set(float(e) for e in g["dyn_model_exp"]) == {1.0, 1.5}
    assert np.any((g["kind"] == 0) & (g["n_course"] > 0))   # the tick passes its delay-compensation course
    assert np.any((g["kind"] == 1) & (g["pref_idx"] > 0))   # a lowered vel_max inside a closed loop
    for c in range(g["kind"].size):
        vx_prefix, pref_idx, vel_start, old = _oracle(g, c)
        n = int(g["n_prefix"][c])
        assert vx_prefix.size == n and pref_idx == int(g["pref_idx"][c]), c
        assert vx_prefix.tobytes() == g["vx_prefix"][c, :n].tobytes(), c
        assert np.float64(vel_start).tobytes() == g["vel_start"][c].tobytes(), c
        assert old == float(g["old_after"][c]), c
        assert not np.any(g["vx_prefix"][c, n:])
    # a chain is one instance's calls in order: each call starts from the memory the previous one left
    for ch in np.unique(g["chain"]):
        idx = np.flatnonzero(g["chain"] == ch)
        idx = idx[np.argsort(g["step"][idx])]
        assert np.array_equal(g["old_before"][idx[1:]], g["old_after"][idx[:-1]]), ch
    steps = np.bincount(g["chain"][g["kind"] == 2])
    assert np.sum(steps >= 6) >= 6
    # the margins that keep the device's cut and branch on the reference's side
    assert np.all(g["margin"] > 1e-8) and np.all(g["stop_margin"] > 1e-6)


def test_boundary_calls_take_the_float64_branch():
    """vel_plan = nextafter(vel_max + 0.1, -inf), vel_max + 0.1 (no brake) and nextafter(.., +inf) (brake)"""
    g = H.golden("brake_prefix.npz")
    sel = np.flatnonzero(R.has(g, "boundary"))
    seen = set()
    for c in sel:
        b = float(g["vel_max"][c]) + 0.1
        v = float(g["vel_plan"][c])
        side = -1 if v == np.nextafter(b, -np.inf) else 0 if v == b else 1 if v == np.nextafter(b, np.inf) else None
        assert side is not None, c
        seen.add(side)
        assert (int(g["pref_idx"][c]) > 0) == (side == 1), c
        assert (float(g["old_after"][c]) == float(g["gg_scale"][c])) == (side != 1), c
        assert _oracle(g, c)[1] == int(g["pref_idx"][c])
    assert seen == {-1, 0, 1}
