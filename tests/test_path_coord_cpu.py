"""Positions on polylines without a GPU: the ctypes mirror of LtplPathCoord, the refusals of ltpl_path_coord_batch (each
with its field named, nothing launched), the Python argument checks, and the oracle against every call of the reference
recorded in tests/golden/path_coord.npz, bit for bit."""
import ctypes
import os
import re

import numpy as np
import pytest

from tests import helpers as H
from tests import path_coord_ref as R

HEADER = os.path.join(H.REPO, "include", "ltpl_b200.h")
SIZE = 176


def _lib():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    return capi, capi.load_library()


def _valid(capi, mode=0):
    """every field set (fake, aligned device pointers): the checks pass up to the one a test breaks"""
    pc = capi.PathCoord()
    pc.mode, pc.n_queries, pc.m_points = mode, 4, 10
    for name in ("x", "y", "x2", "y2", "pos", "s", "closest", "idx", "inside"):
        setattr(pc, name, 256)
    pc.line_s, pc.pt_s, pc.line2_s, pc.pt2_s = 20, 2, 20, 2
    pc.pos_s[0], pc.pos_s[1] = 2, 1
    return pc


def _refused(capi, lib, pc, field):
    n0 = lib.ltpl_launch_count()
    assert lib.ltpl_path_coord_batch(ctypes.byref(pc), None) == -1
    msg = lib.ltpl_last_error().decode()
    assert field in msg, (field, msg)
    assert lib.ltpl_launch_count() == n0
    return msg


def test_path_coord_mirror_matches_the_header_and_carries_its_size():
    capi, lib = _lib()
    body = re.search(r"typedef struct LtplPathCoord \{(.*?)\} LtplPathCoord;", open(HEADER).read(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)(?:\[\d+\])?\s*[;,]", body)
    assert fields == [f for f, _ in capi.PathCoord._fields_], fields
    assert ctypes.sizeof(capi.PathCoord) == capi.PathCoord().struct_bytes == SIZE
    modes = dict(re.findall(r"#define (LTPL_PC_\w+)\s+(\d+)", open(HEADER).read()))
    assert modes == {"LTPL_PC_S_COORD": "0", "LTPL_PC_S_INDEX": "1", "LTPL_PC_CLOSEST": "2",
                     "LTPL_PC_INSIDE_BOUNDS": "3"}
    assert (capi.PC_S_COORD, capi.PC_S_INDEX, capi.PC_CLOSEST, capi.PC_INSIDE_BOUNDS) == (0, 1, 2, 3)
    v = _valid(capi)
    v.m_points = 1
    assert "struct_bytes" not in _refused(capi, lib, v, "pc.m_points")
    for size in (0, SIZE - 8, SIZE + 8):
        v = _valid(capi)
        v.struct_bytes = size
        _refused(capi, lib, v, "struct_bytes")
    assert lib.ltpl_sizeof(6) == -1 and capi.ABI_VERSION == lib.ltpl_version() == 20


def test_path_coord_refuses_bad_arguments_before_launching():
    capi, lib = _lib()

    def refused(field, change, mode=0):
        pc = _valid(capi, mode)
        change(pc)
        _refused(capi, lib, pc, field)

    refused("pc.mode", lambda v: setattr(v, "mode", 4))
    refused("pc.mode", lambda v: setattr(v, "mode", -1))
    refused("pc.n_queries", lambda v: setattr(v, "n_queries", -1))
    refused("pc.m_points", lambda v: setattr(v, "m_points", 1))
    for name in ("x", "y", "pos", "s", "closest"):
        refused("pc.%s" % name, lambda v, name=name: setattr(v, name, None))
        refused("pc.%s" % name, lambda v, name=name: setattr(v, name, 258 if name == "closest" else 260))
    refused("pc.closest", lambda v: setattr(v, "closest", None), mode=1)
    refused("pc.s", lambda v: setattr(v, "s", 260), mode=1)
    refused("pc.idx", lambda v: setattr(v, "idx", None), mode=2)
    refused("pc.idx", lambda v: setattr(v, "idx", 258), mode=2)
    for name in ("x2", "y2", "inside"):
        refused("pc.%s" % name, lambda v, name=name: setattr(v, name, None), mode=3)
    refused("pc.x2", lambda v: setattr(v, "x2", 260), mode=3)
    refused("pc.s_array", lambda v: setattr(v, "s_array", 260))
    refused("pc.n_pts", lambda v: setattr(v, "n_pts", 258))
    refused("pc.pt_s", lambda v: setattr(v, "pt_s", 0))
    refused("pc.line_s", lambda v: setattr(v, "line_s", 18))
    refused("pc.pt2_s", lambda v: setattr(v, "pt2_s", 0), mode=3)
    refused("pc.line2_s", lambda v: setattr(v, "line2_s", 5), mode=3)
    refused("pc.s_array_es", lambda v: (setattr(v, "s_array", 256), setattr(v, "s_array_s", 10)))
    refused("pc.s_array_s", lambda v: (setattr(v, "s_array", 256), setattr(v, "s_array_es", 1),
                                       setattr(v, "s_array_s", 9)))
    refused("pc.s_array_s", lambda v: (setattr(v, "s_array", 256), setattr(v, "s_array_es", 1),
                                       setattr(v, "s_array_s", 0)))
    # a column of the [B][115][7] selection: element stride 7, rows of 7 * 115 -- only the last element has to fit
    refused("pc.s_array_s", lambda v: (setattr(v, "s_array", 256), setattr(v, "s_array_es", 7),
                                       setattr(v, "s_array_s", 63)))
    refused("pc.pos_s", lambda v: v.pos_s.__setitem__(1, 0))
    refused("pc.pos_s", lambda v: v.pos_s.__setitem__(0, -1))
    # accepted without a launch: no queries, with or without pointers (empty tensors have none)
    def empty(v):
        v.n_queries = 0
        for name in ("x", "y", "x2", "y2", "pos", "s", "closest", "idx", "inside"):
            setattr(v, name, None)
    for change in (lambda v: setattr(v, "n_queries", 0), empty):
        pc = _valid(capi)
        change(pc)
        n0 = lib.ltpl_launch_count()
        assert lib.ltpl_path_coord_batch(ctypes.byref(pc), None) == 0
        assert lib.ltpl_launch_count() == n0


def test_python_argument_checks():
    """the host checks of every function, before anything is uploaded or launched (no GPU: a call that passed would
    fail at the upload)"""
    import torch
    from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P
    _lib()
    line, pos = np.zeros((3, 6, 2)), np.zeros((3, 2))
    with pytest.raises(ValueError, match="cannot be mixed"):
        P.get_s_coord(line, torch.zeros(3, 2, dtype=torch.float64))
    with pytest.raises(ValueError, match="pos: an array"):
        P.get_s_coord(line, np.zeros((3, 3)))
    with pytest.raises(ValueError, match=r"ref_line: an array \[3\]\[M >= 2\]\[2\]"):
        P.get_s_coord(np.zeros((4, 6, 2)), pos)
    with pytest.raises(ValueError, match="ref_line: an array"):
        P.get_s_coord(np.zeros((1, 2)), pos)
    with pytest.raises(ValueError, match="path: a numeric array"):
        P.closest_path_index(np.array([["a", "b"]] * 3), pos)
    with pytest.raises(ValueError, match=r"n_pts: every length must be in \[2, 6\]"):
        P.closest_path_index(line, pos, n_pts=[2, 7, 6])
    with pytest.raises(ValueError, match="n_pts: an integer array"):
        P.check_inside_bounds(line, line, pos, n_pts=[2.0, 3.0, 4.0])
    with pytest.raises(ValueError, match="bound2: an array"):
        P.check_inside_bounds(line, np.zeros((3, 6, 3)), pos)
    t = lambda *s: torch.zeros(*s, dtype=torch.float64)   # noqa: E731
    with pytest.raises(ValueError, match="CUDA tensor"):
        P.get_s_coord(t(3, 6, 2), t(3, 2))


def test_oracle_reproduces_every_fixture_call_bit_for_bit():
    """oracle/ltpl_oracle.py's get_s_coord, closest_path_index and check_inside_bounds against the reference's own
    calls: s bit for bit (NaN where the reference returned None or raised), the index pairs, idx and inside"""
    g = H.golden("path_coord.npz")
    for b in (str(s) for s in g["label_names"]):
        assert R.has(g, b).any(), b
    assert all(np.any(g["fn"] == f) for f in (0, 1, 2)) and all(np.any(g["kind"] == k) for k in (0, 1))
    assert np.any((g["kind"] == 0) & (g["fn"] == R.FN_S) & (g["sarr_id"] >= 0) & g["closed"])   # MOPG's race line
    assert np.any((g["kind"] == 0) & (g["fn"] == R.FN_S) & (g["sarr_id"] >= 0) & ~g["closed"])  # OTH:774-782
    assert np.any((g["kind"] == 0) & (g["fn"] == R.FN_INSIDE))
    for c in range(g["fn"].size):
        s, ci, idx, inside = R.oracle(g, c)
        assert R.same_s(s, float(g["s"][c])), c
        fn = int(g["fn"][c])
        if fn == R.FN_S:
            assert ci == tuple(int(v) for v in g["closest"][c]), c
            assert np.isnan(g["s"][c]) == (bool(g["only_index"][c]) or bool(g["raised"][c]) or np.isnan(s)), c
        elif fn == R.FN_CLOSEST:
            assert idx == int(g["idx"][c]), c
        else:
            assert inside == int(g["inside"][c]), c
    # exact angle ties: the segment for s (ang1 > ang2) and the index pair (ang1 >= ang2) differ, on both ends
    tie = np.flatnonzero(R.has(g, "angle_tie"))
    assert np.all(g["ang_margin"][tie] == 0.0) and np.all(g["fn"][tie] == R.FN_S)
    ci = g["closest"][tie]
    end = np.isnan(g["s"][tie]) & (ci[:, 1] == ci[:, 0] + 1) & ~g["only_index"][tie]
    start = (ci[:, 0] == 0) & (ci[:, 1] == 0) & np.isfinite(g["s"][tie])
    assert end.sum() >= 8 and start.sum() >= 8 and np.any(start & (g["sarr_id"][tie] >= 0))
    # the margins that keep the device's float64 atan2 on the reference's side
    fin = g["fn"] != R.FN_CLOSEST
    assert np.all((g["ang_margin"][fin] > 1e-12) | (g["ang_margin"][fin] == 0.0))
