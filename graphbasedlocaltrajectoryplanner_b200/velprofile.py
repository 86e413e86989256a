"""
Stand-alone batched velocity planner on the caller's paths (``ltpl_vel_plan_batch`` of the C-ABI).

``VelocityPlanner`` replaces ``VpForwardBackward`` (graph_ltpl/online_graph/src/VpForwardBackward.py)
without a lattice: ``calc_vel_profile`` -> ``tph.calc_vel_profile(closed=False)`` (VPFB:194-227) and
``calc_vel_brake_em`` -> ``tph.calc_vel_profile_brake`` (VPFB:229-255), for N paths at once, each with its own length
and, optionally, its own friction per point.  ``velprofile_batch_device`` / ``calc_vel_profile_batch`` are the dense
constant-friction form of BASELINE.json config 5, with the vehicle parameters of a BatchPlanner.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import capi


def _rows(t: torch.Tensor, width: int) -> tuple:
    """(tensor, row stride): rows whose elements are not contiguous, or that overlap, are copied once"""
    if t.stride(-1) != 1 or (t.dim() == 3 and t.stride(1) != 2) or t.stride(0) < width:
        t = t.contiguous()
    return t, t.stride(0)


def plan_velocity(lib, params, stream, mode: int, kappa: torch.Tensor, el: torch.Tensor, gg, v_start: torch.Tensor,
                  v_end, n_pts, vx: torch.Tensor, ax: torch.Tensor) -> None:
    """one ltpl_vel_plan_batch call on checked device tensors: kappa, vx, ax [N][P], el [N][>= P - 1], gg [N][P][2] or
    None, v_start / v_end [N] (v_end None in brake mode), n_pts [N] int32 or None; every array with unit element
    stride within a row (gg: pairs)."""
    n, p = kappa.shape
    vp = capi.VelPlan()
    vp.mode, vp.n_paths, vp.n_points = mode, n, p
    vp.n_pts = n_pts.data_ptr() if n_pts is not None else None
    vp.kappa, vp.kappa_s = kappa.data_ptr(), kappa.stride(0)
    vp.el, vp.el_s = el.data_ptr(), el.stride(0)
    if gg is not None:
        vp.gg, vp.gg_s = gg.data_ptr(), gg.stride(0)
    vp.v_start = v_start.data_ptr()
    vp.v_end = v_end.data_ptr() if v_end is not None else None
    vp.vx, vp.ax, vp.out_s = vx.data_ptr(), ax.data_ptr(), vx.stride(0)
    capi.check(lib, lib.ltpl_vel_plan_batch(C.byref(params), C.byref(vp), stream), "ltpl_vel_plan_batch")


def velprofile_batch_device(planner, kappa: torch.Tensor, el: torch.Tensor, v_start: torch.Tensor, v_end: torch.Tensor,
                            vx: torch.Tensor, ax: torch.Tensor) -> None:
    """device tensors in / out (float64, [n_paths][n_points], contiguous); vehicle / gg parameters from
    ``planner.params`` (set_vel_params)."""
    for t in (kappa, el, vx, ax):
        if t.dtype != torch.float64 or not t.is_contiguous() or t.shape != kappa.shape:
            raise ValueError("kappa, el, vx, ax must be contiguous float64 tensors of identical shape")
    plan_velocity(planner.lib, planner.params, planner.stream, capi.VP_PROFILE, kappa, el, None, v_start, v_end, None,
                  vx, ax)


def calc_vel_profile_batch(planner, kappa: np.ndarray, el_lengths: np.ndarray, v_start: np.ndarray,
                           v_end: np.ndarray) -> tuple:
    """host arrays in, host arrays out: kappa [N][P], el_lengths [N][P-1] or [N][P]; returns (vx [N][P], ax [N][P])."""
    kappa = np.ascontiguousarray(kappa, dtype=np.float64)
    n, p = kappa.shape
    el = np.zeros((n, p))
    el[:, :el_lengths.shape[1]] = el_lengths
    dev = planner.device
    d_k = torch.from_numpy(kappa).to(dev)
    d_e = torch.from_numpy(el).to(dev)
    d_s = torch.from_numpy(np.ascontiguousarray(v_start, dtype=np.float64)).to(dev)
    d_t = torch.from_numpy(np.ascontiguousarray(v_end, dtype=np.float64)).to(dev)
    vx = torch.empty_like(d_k)
    ax = torch.empty_like(d_k)
    velprofile_batch_device(planner, d_k, d_e, d_s, d_t, vx, ax)
    torch.cuda.synchronize(dev)
    return vx.cpu().numpy(), ax.cpu().numpy()


class VelocityPlanner(object):
    """VpForwardBackward's calc_vel_profile and calc_vel_brake_em on the device, for N paths per call, without a
    lattice.  One parameter set per instance, as a VpForwardBackward instance holds it (update_dyn_parameters).

    Arrays: ``kappa`` [N][P]; ``el_lengths`` [N][P - 1] (tph's shape) or [N][P]; ``loc_gg`` a tuple (ax_max, ay_max)
    for every point or an array [N][P][2]; ``v_start`` / ``v_end`` [N]; ``n_pts`` [N] points per path (2 <= n <= P,
    None: P each; elements at or behind a path's end are not read).  Results ``(vx, ax)`` [N][P], ax = (v[p+1]^2 -
    v[p]^2) / (2 el[p]) and 0 at each path's last point, both 0 behind it.

    Device tensors in give device tensors out, enqueued on the current stream without a host synchronisation, and with
    ``out=(vx, ax)`` without an allocation: such a call can be captured in a CUDA graph.  Rows whose elements are not
    contiguous are copied once; row strides are passed through.  A length in a device ``n_pts`` cannot be checked
    without a synchronisation: a path whose length is out of range gets a row of NaN.  NumPy arrays in give NumPy
    arrays out (after one synchronisation).  Bad shapes, dtypes or devices, and host lengths out of range, raise
    ValueError before anything is launched."""

    def __init__(self, veh_param_dyn_model_exp: float = 1.0, veh_param_dragcoeff: float = 0.85,
                 veh_param_mass: float = 1000.0, device=None):
        self.lib = capi.load_library()
        self.device = torch.device(device if device is not None else "cuda:0")
        self.veh = dict(dyn_model_exp=float(veh_param_dyn_model_exp), drag_coeff=float(veh_param_dragcoeff),
                        m_veh=float(veh_param_mass))
        self.params = None       # set by update_dyn_parameters
        self._brake_params = self._fill(0.0, 1.0, [[0.0, 0.0]])   # the brake mode reads the vehicle parameters only

    def _fill(self, vel_max, gg_scale, ax_max_machines):
        from .planner import DEFAULT_ONLINE, fill_vel_params
        params = capi.Params()
        fill_vel_params(params, DEFAULT_ONLINE, self.veh, vel_max=float(vel_max), gg_scale=float(gg_scale),
                        local_gg=(1.0, 1.0), ax_max_machines=ax_max_machines, safety_d=0.0, incl_emerg_traj=False)
        return params

    def update_dyn_parameters(self, vel_max: float, gg_scale: float, ax_max_machines) -> None:
        """VPFB.update_dyn_parameters: maximum velocity, gg scale applied to loc_gg in calc_vel_profile, and the
        machine limits [[vx, ax_max], ...] (ascending vx, covering vel_max)."""
        self.params = self._fill(vel_max, gg_scale, ax_max_machines)

    def calc_vel_profile(self, kappa, el_lengths, loc_gg, v_start, v_end, n_pts=None, out=None):
        """tph.calc_vel_profile(closed=False) with loc_gg * gg_scale, v_max, ax_max_machines (VPFB:194-227)"""
        if self.params is None:
            raise RuntimeError("calc_vel_profile: call update_dyn_parameters first")
        return self._plan(capi.VP_PROFILE, self.params, kappa, el_lengths, loc_gg, v_start, v_end, n_pts, out)

    def calc_vel_brake_em(self, kappa, el_lengths, loc_gg, v_start, n_pts=None, out=None):
        """tph.calc_vel_profile_brake with the raw loc_gg, no gg_scale (VPFB:229-255): zeros after standstill"""
        return self._plan(capi.VP_BRAKE, self._brake_params, kappa, el_lengths, loc_gg, v_start, None, n_pts, out)

    # -- arguments ---------------------------------------------------------------------------------------------------
    def _plan(self, mode, params, kappa, el, loc_gg, v_start, v_end, n_pts, out):
        on_device = isinstance(kappa, torch.Tensor)
        if not on_device:
            kappa, el, loc_gg, v_start, v_end, n_pts = self._upload(kappa, el, loc_gg, v_start, v_end, n_pts)
        dev = kappa.device
        if dev.type != "cuda":
            raise ValueError("kappa: a CUDA tensor or a NumPy array, got a tensor on %s" % dev)
        if kappa.dim() != 2 or kappa.shape[0] < 1 or kappa.shape[1] < 2:
            raise ValueError("kappa must be [N >= 1][P >= 2], got %s" % (tuple(kappa.shape),))
        n, p = kappa.shape
        gg = None if isinstance(loc_gg, tuple) else loc_gg
        if gg is None and (len(loc_gg) != 2 or not all(np.isscalar(g) for g in loc_gg)):
            raise ValueError("loc_gg: a tuple (ax_max, ay_max) or an array [N][P][2]")
        el_cols = el.shape[-1] if isinstance(el, torch.Tensor) and el.dim() == 2 and el.shape[-1] in (p - 1, p) else p
        arrays = dict(kappa=(kappa, (n, p)), el_lengths=(el, (n, el_cols)), v_start=(v_start, (n,)))
        if gg is not None:
            arrays["loc_gg"] = (gg, (n, p, 2))
        if v_end is not None:
            arrays["v_end"] = (v_end, (n,))
        for name, (t, shape) in arrays.items():
            if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.float64 or tuple(t.shape) != shape:
                raise ValueError("%s: a float64 tensor %s on %s, got %s" % (name, list(shape), dev, _describe(t)))
        if n_pts is not None:
            if not isinstance(n_pts, torch.Tensor) or n_pts.device != dev or n_pts.dtype != torch.int32 \
                    or tuple(n_pts.shape) != (n,):
                raise ValueError("n_pts: an int32 tensor [%d] on %s, got %s" % (n, dev, _describe(n_pts)))
            n_pts = n_pts.contiguous()
        if out is None:
            vx = torch.empty((n, p), dtype=torch.float64, device=dev)
            ax = torch.empty((n, p), dtype=torch.float64, device=dev)
        else:
            vx, ax = out
            for name, t in (("vx", vx), ("ax", ax)):
                if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.float64 \
                        or tuple(t.shape) != (n, p) or t.stride(1) != 1 or t.stride(0) < p:
                    raise ValueError("out %s: a float64 tensor [%d][%d] on %s with contiguous rows, got %s"
                                     % (name, n, p, dev, _describe(t)))
            if vx.stride(0) != ax.stride(0):
                raise ValueError("out: vx and ax must have the same row stride, got %d and %d"
                                 % (vx.stride(0), ax.stride(0)))
        kappa, _ = _rows(kappa, p)
        el, _ = _rows(el, el.shape[1])
        if gg is not None:
            gg, _ = _rows(gg, 2 * p)
        v_start = v_start.contiguous()
        v_end = v_end.contiguous() if v_end is not None else None
        if gg is None:
            params = capi.Params.from_buffer_copy(params)
            params.gg_ax, params.gg_ay = float(loc_gg[0]), float(loc_gg[1])
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        plan_velocity(self.lib, params, stream, mode, kappa, el, gg, v_start, v_end, n_pts, vx, ax)
        if on_device:
            return vx, ax
        torch.cuda.current_stream(dev).synchronize()
        return vx.cpu().numpy(), ax.cpu().numpy()

    def _upload(self, kappa, el, loc_gg, v_start, v_end, n_pts):
        """NumPy arguments to device tensors; host lengths are checked here, before anything is uploaded"""
        def host(a, name, dtype=np.float64):
            if isinstance(a, torch.Tensor):
                raise ValueError("%s: NumPy arrays and tensors cannot be mixed in one call" % name)
            a = np.asarray(a)
            if a.dtype.kind not in "iuf":
                raise ValueError("%s: a numeric array, got %s" % (name, a.dtype))
            return np.ascontiguousarray(a, dtype=dtype)

        kappa = host(kappa, "kappa")
        if kappa.ndim != 2 or kappa.shape[0] < 1 or kappa.shape[1] < 2:
            raise ValueError("kappa must be [N >= 1][P >= 2], got %s" % (kappa.shape,))
        if n_pts is not None:
            h = np.asarray(n_pts)
            if h.dtype.kind not in "iu" or h.shape != (kappa.shape[0],):
                raise ValueError("n_pts: an integer array [%d], got %s" % (kappa.shape[0], _describe(n_pts)))
            if np.any(h < 2) or np.any(h > kappa.shape[1]):
                raise ValueError("n_pts: every length must be in [2, %d], got %d .. %d"
                                 % (kappa.shape[1], h.min(), h.max()))
            n_pts = host(h, "n_pts", np.int32)
        arrays = [kappa, host(el, "el_lengths"), loc_gg if isinstance(loc_gg, tuple) else host(loc_gg, "loc_gg"),
                  host(v_start, "v_start"), host(v_end, "v_end") if v_end is not None else None, n_pts]
        return [torch.from_numpy(a).to(self.device) if isinstance(a, np.ndarray) else a for a in arrays]


def _describe(t) -> str:
    if isinstance(t, torch.Tensor):
        return "%s %s on %s" % (t.dtype, list(t.shape), t.device)
    if isinstance(t, np.ndarray):
        return "%s %s (NumPy)" % (t.dtype, list(t.shape))
    return type(t).__name__
