"""
Positions on the caller's polylines on the device (``ltpl_path_coord_batch`` of the C-ABI), N queries per call:

- ``get_s_coord``          -> helper_funcs/src/get_s_coord.py (get_s_coord, angle3pt)
- ``closest_path_index``   -> helper_funcs/src/closest_path_index.py (n_closest=1)
- ``check_inside_bounds``  -> online_graph/src/check_inside_bounds.py

Lines: ``[N][M][2]`` (one polyline per query) or ``[M][2]`` (one polyline shared by every query: a race line, the track
bounds), float64 with any strides -- e.g. ``sel_traj.double()[:, :, 1:3]``, the x / y columns of BatchPlanner.select's
``[B][n_export][7]`` rows, is read in place.  ``pos`` ``[N][2]`` float64, any strides.  ``n_pts`` ``[N]`` int32
(host or device, optional): points of each row, 2 <= n <= M; nothing at or behind a row's end is read.

Device tensors in give device tensors out, enqueued on the current stream without a host synchronisation; with ``out=``
(and ``n_pts`` on the device or None) nothing is allocated, so a call can be captured in a CUDA graph.  NumPy arrays in give NumPy arrays out.  Bad shapes,
dtypes, devices and host lengths raise ValueError before anything is launched.  A query is invalid when its device
length is out of range, its position is not finite, or no point of its row is at a finite distance: it gets s = NaN,
closest_indexes = (-2, -2), idx = -1 and inside = -1.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import capi
from .velprofile import _describe, _host, _host_lengths


def get_s_coord(ref_line, pos, s_array=None, only_index=False, closed=False, n_pts=None, out=None):
    """get_s_coord.py:8-99 per query: the nearest point (first minimum), the neighbour on the side of the larger angle,
    s = s_array[index] + the distance to the foot of the perpendicular.  Returns ``(s, closest_indexes)``: s float64
    [N], closest_indexes int32 [N][2].  The reference's quirks are kept:

    - closed, nearest point 0: the index pair holds NumPy's -1, and s reads s_array[-1] (the last element);
    - s_array[0] > 0.05: a leading 0 is inserted, which shifts the index into s_array by one;
    - ang1 > ang2 chooses the segment for s, ang1 >= ang2 the index pair;
    - s_array None: the chord lengths are summed in index order (np.cumsum's bytes); without the insertion that array
      is one element short, and where the reference raises its IndexError s is NaN;
    - only_index: s is NaN (the reference returns None).

    s_array (optional): [N][M] with per-query lines, [M] with a shared line, float64 with any strides (e.g. the s column
    ``sel_traj.double()[:, :, 0]`` of the selection, read in place); the line's values for the first n points of each
    row.  out=(s, closest_indexes) allocates nothing."""
    mode = capi.PC_S_INDEX if only_index else capi.PC_S_COORD
    res = _run(mode, (("ref_line", ref_line),), pos, n_pts, out, s_array=s_array, closed=closed)
    return res[0], res[1]


def closest_path_index(path, pos, n_pts=None, out=None):
    """closest_path_index.py:4-32 with n_closest=1, as every caller in graph_ltpl uses it: idx int32 [N], the index of
    the nearest point.  Ties go to the first minimum, as in the tick (argpartition's tie order is undefined).  The
    reference's second result, the [N][M] array of squared distances, is not returned.  out=idx allocates nothing."""
    return _run(capi.PC_CLOSEST, (("path", path),), pos, n_pts, out)[0]


def check_inside_bounds(bound1, bound2, pos, n_pts=None, out=None):
    """check_inside_bounds.py:26-59: centre line (bound1 + bound2) / 2, the closed index pair of get_s_coord on it, the
    three 50-point linspaces, the nearest interpolated centre point and the two squared-distance comparisons.  bound1 and
    bound2 have the same shape.  Returns inside int8 [N]: 1 inside, 0 outside (-1 invalid).  out=inside allocates
    nothing."""
    return _run(capi.PC_INSIDE_BOUNDS, (("bound1", bound1), ("bound2", bound2)), pos, n_pts, out)[0]


# -- arguments -----------------------------------------------------------------------------------------------------
_OUTS = {capi.PC_S_COORD: (("s", torch.float64, 1), ("closest_indexes", torch.int32, 2)),
         capi.PC_S_INDEX: (("s", torch.float64, 1), ("closest_indexes", torch.int32, 2)),
         capi.PC_CLOSEST: (("idx", torch.int32, 1),),
         capi.PC_INSIDE_BOUNDS: (("inside", torch.int8, 1),)}


def _run(mode, lines, pos, n_pts, out, s_array=None, closed=False):
    on_device = isinstance(lines[0][1], torch.Tensor)
    if not on_device:
        lines, pos, s_array, n_pts = _upload(lines, pos, s_array, n_pts)
    dev = lines[0][1].device
    if dev.type != "cuda":
        raise ValueError("%s: a CUDA tensor or a NumPy array, got a tensor on %s" % (lines[0][0], dev))
    if not isinstance(pos, torch.Tensor) or pos.device != dev or pos.dtype != torch.float64 or pos.dim() != 2 \
            or pos.shape[1] != 2:
        raise ValueError("pos: a float64 tensor [N][2] on %s, got %s" % (dev, _describe(pos)))
    n = pos.shape[0]
    shape = tuple(lines[0][1].shape)
    for name, t in lines:
        if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.float64 or t.dim() not in (2, 3) \
                or t.shape[-1] != 2 or t.shape[-2] < 2 or (t.dim() == 3 and t.shape[0] != n):
            raise ValueError("%s: a float64 tensor [%d][M >= 2][2] or [M >= 2][2] on %s, got %s"
                             % (name, n, dev, _describe(t)))
        if tuple(t.shape) != shape:
            raise ValueError("%s: the shape of %s %s, got %s" % (name, lines[0][0], list(shape), _describe(t)))
    m, shared = shape[-2], len(shape) == 2
    if n_pts is not None:
        if isinstance(n_pts, torch.Tensor) and n_pts.device.type == "cuda":
            if n_pts.device != dev or n_pts.dtype != torch.int32 or tuple(n_pts.shape) != (n,):
                raise ValueError("n_pts: an int32 tensor [%d] on %s, got %s" % (n, dev, _describe(n_pts)))
            n_pts = n_pts.contiguous()
        else:
            h = n_pts.numpy() if isinstance(n_pts, torch.Tensor) else n_pts
            n_pts = torch.from_numpy(_host_lengths(h, n, m)).to(dev)
    if s_array is not None:
        want = (m,) if shared else (n, m)
        if not isinstance(s_array, torch.Tensor) or s_array.device != dev or s_array.dtype != torch.float64 \
                or tuple(s_array.shape) != want:
            raise ValueError("s_array: a float64 tensor %s on %s (the line's row length), got %s"
                             % (list(want), dev, _describe(s_array)))
        es = s_array.stride(-1)
        if es < 1 or (not shared and 0 < s_array.stride(0) < (m - 1) * es + 1):   # repeated elements, overlapping rows
            s_array = s_array.contiguous()
    outs = _OUTS[mode]
    if out is None:
        res = [torch.empty((n,) if w == 1 else (n, w), dtype=dt, device=dev) for _, dt, w in outs]
    else:
        res = list(out) if isinstance(out, (tuple, list)) else [out]
        if len(res) != len(outs):
            raise ValueError("out: (%s)" % ", ".join(name for name, _, _ in outs))
        for (name, dt, w), t in zip(outs, res):
            want = (n,) if w == 1 else (n, w)
            if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != dt or tuple(t.shape) != want \
                    or not t.is_contiguous():
                raise ValueError("out %s: a contiguous %s tensor %s on %s, got %s" % (name, dt, list(want), dev,
                                                                                     _describe(t)))
    if pos.stride(1) < 1:
        pos = pos.contiguous()
    pc = capi.PathCoord()
    pc.mode, pc.closed, pc.n_queries, pc.m_points = mode, int(bool(closed)), n, m
    for k, (_, t) in enumerate(lines):
        t, line_s, pt_s = _line(t, m, shared)
        x, y = t.data_ptr(), t.data_ptr() + 8 * t.stride(-1)
        if k == 0:
            pc.x, pc.y, pc.line_s, pc.pt_s = x, y, line_s, pt_s
        else:
            pc.x2, pc.y2, pc.line2_s, pc.pt2_s = x, y, line_s, pt_s
    if s_array is not None:
        pc.s_array, pc.s_array_es = s_array.data_ptr(), s_array.stride(-1)
        pc.s_array_s = 0 if shared else s_array.stride(0)
    pc.pos, pc.pos_s[0], pc.pos_s[1] = pos.data_ptr(), pos.stride(0), pos.stride(1)
    pc.n_pts = n_pts.data_ptr() if n_pts is not None else None
    if mode in (capi.PC_S_COORD, capi.PC_S_INDEX):
        pc.s, pc.closest = res[0].data_ptr(), res[1].data_ptr()
    elif mode == capi.PC_CLOSEST:
        pc.idx = res[0].data_ptr()
    else:
        pc.inside = res[0].data_ptr()
    lib = capi.load_library()
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    capi.check(lib, lib.ltpl_path_coord_batch(C.byref(pc), stream), "ltpl_path_coord_batch")
    if on_device:
        return res
    torch.cuda.current_stream(dev).synchronize()
    return [t.cpu().numpy() for t in res]


def _line(t, m, shared):
    """(tensor, row stride, point stride) of a line: points with stride 0, or rows that overlap, are copied once"""
    pt_s = t.stride(-2)
    line_s = 0 if shared else t.stride(0)
    if pt_s < 1 or (line_s != 0 and line_s < (m - 1) * pt_s + 1):
        t = t.contiguous()
        pt_s, line_s = t.stride(-2), 0 if shared else t.stride(0)
    return t, line_s, pt_s


def _upload(lines, pos, s_array, n_pts):
    """NumPy arguments to device tensors on the current CUDA device, checked on the host first"""
    h = [(name, _host(t, name)) for name, t in lines]
    pos = _host(pos, "pos")
    if pos.ndim != 2 or pos.shape[1] != 2:
        raise ValueError("pos: an array [N][2], got %s" % _describe(pos))
    for name, a in h:
        if a.ndim not in (2, 3) or a.shape[-1] != 2 or a.shape[-2] < 2 or (a.ndim == 3 and a.shape[0] != pos.shape[0]):
            raise ValueError("%s: an array [%d][M >= 2][2] or [M >= 2][2], got %s" % (name, pos.shape[0], _describe(a)))
    n_pts = _host_lengths(n_pts, pos.shape[0], h[0][1].shape[-2])
    if s_array is not None:
        s_array = _host(s_array, "s_array")
    dev = torch.device("cuda", torch.cuda.current_device())
    if s_array is not None:
        s_array = torch.from_numpy(s_array).to(dev)
    up = lambda a: torch.from_numpy(a).to(dev) if a is not None else None   # noqa: E731
    return [(name, up(a)) for name, a in h], up(pos), s_array, up(n_pts)
