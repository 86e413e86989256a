"""The trajectory each scenario takes, without a GPU: the NumPy rule (tests/select_ref.py) against the selections the
reference's closed loops recorded, its corner cases, k_select's stack frame, the ctypes mirror of LtplSelect and the
argument checks of BatchPlanner.select / plan_batch(prefer=...)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from tests import helpers as H
from tests.select_ref import select_ref

# the three rotating orders of oracle/gen_golden.py:multitick_fixture (sequence q uses order q % 3)
ORDERS = (("right", "left", "straight", "follow"), ("follow", "straight", "left", "right"),
          ("left", "straight", "follow", "right"))
HEADER = os.path.join(H.REPO, "include", "ltpl_b200.h")
IDS = dict(straight=0, follow=1, left=2, right=3, emergency=4)


def _tick_arrays(g, k):
    """the device layout of tick k of a multi-tick fixture, one scenario per sequence: slot 0 straight | follow, 1 left,
    2 right; an action without a kept trajectory keeps its slot with traj_row -1; rows numbered apart"""
    n_seq = g["traj_len"].shape[0]
    action_id = np.full((3, n_seq), -1, dtype=np.int32)
    traj_row = np.full((3, n_seq), -1, dtype=np.int32)
    traj_len = np.zeros((3, n_seq), dtype=np.int32)
    traj_id = np.full((3, n_seq), -1, dtype=np.int32)
    em_info = np.full((n_seq, 3), -1, dtype=np.int32)
    for q in range(n_seq):
        assert not (g["path_len"][q, k, 0] and g["path_len"][q, k, 1]), "straight and follow share slot 0"
        for a, act in enumerate(H.ACTIONS):
            s = max(a - 1, 0)
            if g["path_len"][q, k, a]:
                action_id[s, q] = a
            if g["traj_len"][q, k, a]:
                traj_row[s, q], traj_len[s, q], traj_id[s, q] = 3 * q + s, g["traj_len"][q, k, a], g["traj_id"][q, k, a]
        if g["em_len"][q, k]:
            em_info[q] = (3 * n_seq + q, g["em_len"][q, k], 7)
    return action_id, traj_row, traj_len, traj_id, em_info


@pytest.mark.parametrize("fixture,emergency", [("ticks_multitick_default.npz", False),
                                               ("ticks_multitick_ext_default.npz", True)])
def test_rule_reproduces_the_recorded_selections(fixture, emergency):
    """the rule applied to the action set of tick k gives the action the reference's loop passed to calc_paths of tick
    k + 1; with 'emergency' listed first, the emergency trajectory wherever the reference returned one"""
    g = H.golden(fixture)
    n_seq, n_ticks = g["sel"].shape
    prefer = np.array([[IDS[a] for a in ORDERS[q % 3]] for q in range(n_seq)])
    checked = 0
    for k in range(n_ticks - 1):
        live = g["n_done"] > k + 1
        arrays = _tick_arrays(g, k)
        sel, info = select_ref(*arrays, emergency, prefer)
        assert np.array_equal(sel[live], g["sel"][live, k + 1]), "tick %d: %s vs %s" % (k, sel, g["sel"][:, k + 1])
        action_id, traj_row, traj_len, traj_id, em_info = arrays
        for q in np.flatnonzero(live):
            s = max(int(sel[q]) - 1, 0)
            assert tuple(info[q]) == (sel[q], traj_row[s, q], traj_len[s, q], traj_id[s, q])
        checked += int(live.sum())
        sel_em, info_em = select_ref(*arrays, emergency, np.concatenate((np.full((n_seq, 1), 4), prefer), axis=1))
        want = np.where(emergency & (g["em_len"][:, k] > 0), 4, sel)
        assert np.array_equal(sel_em, want), "tick %d with 'emergency' first" % k
        em = sel_em == 4
        assert np.array_equal(info_em[em, 1:], em_info[em])
    assert checked >= 80
    assert len(set(g["sel"][:, 1:].ravel().tolist())) >= 3   # the orders pick different actions


def _one(action_id, traj_row, em_row=-1, n=1):
    a = np.array(action_id, dtype=np.int32).reshape(3, n)
    r = np.array(traj_row, dtype=np.int32).reshape(3, n)
    em = np.tile(np.array([em_row, 40, 17], dtype=np.int32), (n, 1))
    return a, r, np.where(r >= 0, 115, 0).astype(np.int32), np.where(r >= 0, 10 + a, -1).astype(np.int32), em


def test_rule_corner_cases():
    kept_follow_left = _one([1, 2, -1], [5, 6, -1], em_row=9)
    # an empty list selects nothing
    sel, info = select_ref(*kept_follow_left, True, np.zeros((1, 0), dtype=np.int64))
    assert sel.tolist() == [-1] and info.tolist() == [[-1, -1, 0, -1]]
    # ids that are not one of the five are skipped, whatever their width
    sel, _ = select_ref(*kept_follow_left, True, np.array([[7, -1, 2 ** 32 + 2, 2]]))
    assert sel.tolist() == [2]
    # 'straight' and 'follow' share slot 0: the id decides, not the slot
    sel, _ = select_ref(*kept_follow_left, True, np.array([[0, 3]]))
    assert sel.tolist() == [-1]
    sel, info = select_ref(*kept_follow_left, True, np.array([[0, 1, 2]]))
    assert sel.tolist() == [1] and info.tolist() == [[1, 5, 115, 11]]
    # an action whose path exists but whose trajectory was not kept is not returned
    sel, _ = select_ref(*_one([0, 2, 3], [-1, 6, -1]), True, np.array([[0, 3, 2]]))
    assert sel.tolist() == [2]
    # 'emergency' needs a kept trajectory beside it ...
    nothing_kept = _one([0, 2, -1], [-1, -1, -1], em_row=9)
    sel, _ = select_ref(*nothing_kept, True, np.array([[4, 0, 2]]))
    assert sel.tolist() == [-1]
    # ... and a velocity call with incl_emerg_traj: em_info of a buffer set without memory may be stale
    sel, _ = select_ref(*kept_follow_left, False, np.array([[4, 2]]))
    assert sel.tolist() == [2]
    sel, info = select_ref(*kept_follow_left, True, np.array([[4, 2]]))
    assert sel.tolist() == [4] and info.tolist() == [[4, 9, 40, 17]]


def test_select_kernel_has_no_stack_frame():
    from tests.test_kernel_frames import _stack_frames
    frames = _stack_frames()
    sel = [s for f, s in frames.items() if f.startswith("_Z8k_select")]
    assert len(sel) == 1, sorted(frames)
    assert sel[0] == 0, sel


def test_select_mirror_carries_its_size():
    """LtplSelect is checked by its own size at every call (ltpl_sizeof and the ABI version of the other structs stay
    as they were): the mirror has the header's field order, fills struct_bytes itself, and the library accepts that
    size -- a refusal then names another field -- while any other size is refused by name"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    lib = capi.load_library()
    body = re.search(r"typedef struct LtplSelect \{(.*?)\} LtplSelect;", open(HEADER).read(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)(?:\[\d\])?\s*;", body)
    assert fields == [f for f, _ in capi.Select._fields_], fields
    assert "#define LTPL_SELECT_MAX %d" % capi.SELECT_MAX in open(HEADER).read() and capi.SELECT_MAX == 8
    sel = capi.Select()
    assert sel.struct_bytes == ctypes.sizeof(capi.Select) == 72
    prm, dims, buf = capi.Params(), capi.Dims(), capi.Buffers()
    dims.batch, dims.n_export = 4, 115
    sel.sel_traj = 256   # without buffers.traj: refused, never launched

    def error(size):
        sel.struct_bytes = size
        rc = lib.ltpl_select_batch(ctypes.byref(prm), ctypes.byref(dims), ctypes.byref(buf), ctypes.byref(sel), None)
        assert rc == -1
        return lib.ltpl_last_error().decode()

    assert "struct_bytes" not in error(72)
    for size in (0, 64, 80):
        assert "struct_bytes" in error(size)
    assert lib.ltpl_sizeof(6) == -1 and capi.ABI_VERSION == lib.ltpl_version() == 20


def test_select_batch_refuses_bad_arguments_before_launching():
    """the library's checks, each with its field named (the struct's size: test_select_mirror_carries_its_size).  No argument set here passes them all: sel_traj without
    buffers.traj, the last check, stays refused throughout, so nothing can be launched"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    lib = capi.load_library()
    prm, dims, buf, sel = capi.Params(), capi.Dims(), capi.Buffers(), capi.Select()
    dims.batch, dims.n_export = 4, 115
    fake = 256
    for name in ("action_id", "traj_row", "traj_len", "traj_id"):
        setattr(buf, name, fake)
    sel.sel_action, sel.sel_info, sel.sel_traj, sel.prefer, sel.prefer_len, sel.prefer_bytes = fake, fake, fake, fake, 2, 4

    def refused(field):
        n0 = lib.ltpl_launch_count()
        rc = lib.ltpl_select_batch(ctypes.byref(prm), ctypes.byref(dims), ctypes.byref(buf), ctypes.byref(sel), None)
        assert rc == -1 and field in lib.ltpl_last_error().decode(), (field, lib.ltpl_last_error())
        assert lib.ltpl_launch_count() == n0

    refused("buffers.traj")
    sel.prefer_len = 9
    refused("prefer_len")
    sel.prefer_len, sel.prefer_bytes = 2, 2
    refused("prefer_bytes")
    sel.prefer_bytes, sel.prefer = 8, None
    refused("sel.prefer")
    sel.prefer, sel.sel_info = fake, None
    refused("sel_info")
    sel.sel_info, sel.sel_action = fake, None
    refused("sel_action")
    sel.sel_action, prm.incl_emerg_traj = fake, 1
    refused("em_info")
    prm.incl_emerg_traj, buf.traj_id = 0, None
    refused("traj_id")


def test_prefer_checks():
    from graphbasedlocaltrajectoryplanner_b200.planner import check_prefer
    ids = check_prefer(["follow", "emergency", "left"], 5, "cpu")
    assert ids.tolist() == [[1, 4, 2]] and ids.dtype == np.int64
    assert check_prefer([], 5, "cpu").shape == (1, 0)
    assert check_prefer(np.zeros((5, 8), dtype=np.uint8), 5, "cpu").shape == (5, 8)
    t = torch.zeros((8, 5), dtype=torch.int8).t()   # any strides
    assert check_prefer(t, 5, "cpu") is t
    bad = [(["straight", "overtake"], "unknown action"), (["left"] * 9, "shape"), ([2, 3], "unknown action"),
           (np.zeros((4, 2), dtype=np.int32), "shape"), (np.zeros((5,), dtype=np.int32), "shape"),
           (np.zeros((5, 2)), "integers"), (torch.zeros((5, 2)), "int8"), (torch.zeros((5, 2), dtype=torch.int16), "int8"),
           (torch.zeros((5, 9), dtype=torch.int32), "shape"), ("straight", "list of action names")]
    for prefer, msg in bad:
        with pytest.raises(ValueError, match=msg):
            check_prefer(prefer, 5, "cpu")
    with pytest.raises(ValueError, match="on cuda"):
        check_prefer(torch.zeros((5, 2), dtype=torch.int32), 5, "cuda:0")
