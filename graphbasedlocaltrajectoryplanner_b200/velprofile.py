"""
Stand-alone batched velocity planner on the caller's paths (``ltpl_vel_plan_batch`` of the C-ABI).

``VelocityPlanner`` replaces ``VpForwardBackward`` (graph_ltpl/online_graph/src/VpForwardBackward.py)
without a lattice: ``calc_vel_profile`` -> ``tph.calc_vel_profile(closed=False)`` (VPFB:194-227),
``calc_vel_brake_em`` -> ``tph.calc_vel_profile_brake`` (VPFB:229-255), ``calc_vel_profile_follow`` ->
``calc_vel_profile_follow`` (VPFB:141-192, ``ltpl_vel_follow_batch``) and ``check_brake_prefix`` (VPFB:86-139,
``ltpl_brake_prefix_batch``), for N paths at once, each with its own length and, optionally, its own friction per point.
``velprofile_batch_device`` / ``calc_vel_profile_batch`` are the dense constant-friction form of BASELINE.json config 5,
with the vehicle parameters of a BatchPlanner.
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
    """VpForwardBackward's calc_vel_profile, calc_vel_brake_em, calc_vel_profile_follow and check_brake_prefix on the
    device, for N paths per call, without a lattice.  One parameter set per instance, as a VpForwardBackward instance
    holds it (update_dyn_parameters); the instance's old_gg_scale of check_brake_prefix is a per-path array the caller
    keeps.

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
                 veh_param_mass: float = 1000.0, device=None, len_veh=None, follow_control_type=None,
                 follow_control_params=None, glob_rl=None):
        """len_veh, follow_control_type ('PD' or 'PDtan'), follow_control_params (k_p, k_d, c_p and, for PDtan, tan_w:
        the online ini's [FOLLOW] form) and glob_rl (the closed race line [M + 1][5] s, x, y, kappa, vx with its first
        point repeated at the end, as Lattice.glob_rl stores it) enable calc_vel_profile_follow (VPFB:22-60); all four
        or none.  The race line is checked and uploaded here, once."""
        self.lib = capi.load_library()
        self.device = torch.device(device if device is not None else "cuda:0")
        self.veh = dict(dyn_model_exp=float(veh_param_dyn_model_exp), drag_coeff=float(veh_param_dragcoeff),
                        m_veh=float(veh_param_mass))
        self.follow = check_follow_args(len_veh, follow_control_type, follow_control_params, glob_rl)
        self.glob_rl = None      # device [M][6] s, x, y, kappa, vx, el (CVPF:166)
        if self.follow is not None:
            self.glob_rl = torch.from_numpy(self.follow.pop("glob_rl")).to(self.device)
        self.params = None       # set by update_dyn_parameters
        self._brake_params = self._fill(0.0, 1.0, [[0.0, 0.0]])   # the brake mode reads the vehicle parameters only

    def _fill(self, vel_max, gg_scale, ax_max_machines):
        from .planner import DEFAULT_ONLINE, fill_vel_params
        params = capi.Params()
        online = DEFAULT_ONLINE
        if self.follow is not None:
            online = dict(DEFAULT_ONLINE, controller_type=self.follow["control_type"],
                          control_params=self.follow["control_params"])
        fill_vel_params(params, online, self.veh, vel_max=float(vel_max), gg_scale=float(gg_scale),
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

    def calc_vel_profile_follow(self, kappa, el_lengths, loc_gg, v_start, v_ego, v_obj, safety_d, obj_dist, obj_pos,
                                n_pts=None, out=None):
        """calc_vel_profile_follow (VPFB:141-192, CVPF:78-313) with loc_gg * gg_scale, vel_max and ax_max_machines of
        update_dyn_parameters.  kappa [N][P]; el_lengths [N][P], the path's whole el column as the reference passes it
        (its last element enters the ego stop distance); loc_gg a tuple or [N][P][2]; v_start, v_ego, v_obj, safety_d,
        obj_dist [N]; obj_pos [N][2].  Returns (vx, ax, too_close, vel_bound): vx, ax [N][P] as in calc_vel_profile,
        too_close and vel_bound (vel_bound_fulfilled) bool [N].  out=(vx, ax, too_close, vel_bound) allocates nothing.
        A path whose device length is out of range gets a row of NaN and both flags False."""
        if self.follow is None:
            raise RuntimeError("calc_vel_profile_follow: construct the VelocityPlanner with len_veh, follow_control_type, "
                               "follow_control_params and glob_rl")
        if self.params is None:
            raise RuntimeError("calc_vel_profile_follow: call update_dyn_parameters first")
        scal = dict(v_start=v_start, v_ego=v_ego, v_obj=v_obj, safety_d=safety_d, obj_dist=obj_dist)
        on_device = isinstance(kappa, torch.Tensor)
        if not on_device:
            kappa, el_lengths, loc_gg, scal, obj_pos, n_pts = self._upload_follow(kappa, el_lengths, loc_gg, scal,
                                                                                  obj_pos, n_pts)
        dev = kappa.device
        if dev.type != "cuda":
            raise ValueError("kappa: a CUDA tensor or a NumPy array, got a tensor on %s" % dev)
        if kappa.dim() != 2 or kappa.shape[0] < 1 or kappa.shape[1] < 2:
            raise ValueError("kappa must be [N >= 1][P >= 2], got %s" % (tuple(kappa.shape),))
        n, p = kappa.shape
        gg = None if isinstance(loc_gg, tuple) else loc_gg
        if gg is None and (len(loc_gg) != 2 or not all(np.isscalar(g) for g in loc_gg)):
            raise ValueError("loc_gg: a tuple (ax_max, ay_max) or an array [N][P][2]")
        if isinstance(el_lengths, torch.Tensor) and el_lengths.dim() == 2 and tuple(el_lengths.shape) == (n, p - 1):
            raise ValueError("el_lengths: calc_vel_profile_follow takes the path's whole el column [N][P] = [%d][%d] "
                             "(the last element enters the ego stop distance), got [N][P - 1]" % (n, p))
        arrays = dict(kappa=(kappa, (n, p)), el_lengths=(el_lengths, (n, p)), obj_pos=(obj_pos, (n, 2)))
        arrays.update({k: (v, (n,)) for k, v in scal.items()})
        if gg is not None:
            arrays["loc_gg"] = (gg, (n, p, 2))
        for name, (t, shape) in arrays.items():
            if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.float64 or tuple(t.shape) != shape:
                raise ValueError("%s: a float64 tensor %s on %s, got %s" % (name, list(shape), dev, _describe(t)))
        if dev != self.glob_rl.device:
            raise ValueError("kappa: tensors on %s, the planner's race line is on %s" % (dev, self.glob_rl.device))
        if n_pts is not None:
            if not isinstance(n_pts, torch.Tensor) or n_pts.device != dev or n_pts.dtype != torch.int32 \
                    or tuple(n_pts.shape) != (n,):
                raise ValueError("n_pts: an int32 tensor [%d] on %s, got %s" % (n, dev, _describe(n_pts)))
            n_pts = n_pts.contiguous()
        if out is None:
            vx = torch.empty((n, p), dtype=torch.float64, device=dev)
            ax = torch.empty((n, p), dtype=torch.float64, device=dev)
            too_close = torch.empty(n, dtype=torch.bool, device=dev)
            vel_bound = torch.empty(n, dtype=torch.bool, device=dev)
        else:
            if len(out) != 4:
                raise ValueError("out: (vx, ax, too_close, vel_bound)")
            vx, ax, too_close, vel_bound = out
            for name, t in (("vx", vx), ("ax", ax)):
                if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.float64 \
                        or tuple(t.shape) != (n, p) or t.stride(1) != 1 or t.stride(0) < p:
                    raise ValueError("out %s: a float64 tensor [%d][%d] on %s with contiguous rows, got %s"
                                     % (name, n, p, dev, _describe(t)))
            if vx.stride(0) != ax.stride(0):
                raise ValueError("out: vx and ax must have the same row stride, got %d and %d"
                                 % (vx.stride(0), ax.stride(0)))
            for name, t in (("too_close", too_close), ("vel_bound", vel_bound)):
                if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.bool \
                        or tuple(t.shape) != (n,) or not t.is_contiguous():
                    raise ValueError("out %s: a contiguous bool tensor [%d] on %s, got %s" % (name, n, dev, _describe(t)))
        kappa, _ = _rows(kappa, p)
        el_lengths, _ = _rows(el_lengths, p)
        if gg is not None:
            gg, _ = _rows(gg, 2 * p)
        if obj_pos.stride(-1) != 1 or obj_pos.stride(0) < 2:
            obj_pos = obj_pos.contiguous()
        scal = {k: v.contiguous() for k, v in scal.items()}
        params = self.params
        if gg is None:
            params = capi.Params.from_buffer_copy(params)
            params.gg_ax, params.gg_ay = float(loc_gg[0]), float(loc_gg[1])
        vf = capi.VelFollow()
        vf.n_paths, vf.n_points = n, p
        vf.n_pts = n_pts.data_ptr() if n_pts is not None else None
        vf.kappa, vf.kappa_s = kappa.data_ptr(), kappa.stride(0)
        vf.el, vf.el_s = el_lengths.data_ptr(), el_lengths.stride(0)
        if gg is not None:
            vf.gg, vf.gg_s = gg.data_ptr(), gg.stride(0)
        for k, v in scal.items():
            setattr(vf, k, v.data_ptr())
        vf.obj_pos, vf.obj_pos_s = obj_pos.data_ptr(), obj_pos.stride(0)
        vf.glob_rl, vf.n_glob = self.glob_rl.data_ptr(), self.glob_rl.shape[0]
        vf.veh_length = self.follow["len_veh"]
        vf.vx, vf.ax, vf.out_s = vx.data_ptr(), ax.data_ptr(), vx.stride(0)
        vf.too_close, vf.vel_bound = too_close.data_ptr(), vel_bound.data_ptr()
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        capi.check(self.lib, self.lib.ltpl_vel_follow_batch(C.byref(params), C.byref(vf), stream),
                   "ltpl_vel_follow_batch")
        if on_device:
            return vx, ax, too_close, vel_bound
        torch.cuda.current_stream(dev).synchronize()
        return vx.cpu().numpy(), ax.cpu().numpy(), too_close.cpu().numpy(), vel_bound.cpu().numpy()

    def check_brake_prefix(self, vel_plan, vel_course, kappa, el_lengths, loc_gg, old_gg_scale, n_course=None,
                           n_pts=None, out=None):
        """VPFB.check_brake_prefix (VPFB:86-139) for N paths, the instance's old_gg_scale kept per path in the caller's
        ``old_gg_scale`` [N] (float64, updated in place).  Create it filled with the gg_scale of the first
        update_dyn_parameters call, as the reference's instance sets old_gg_scale on its first update_dyn_parameters
        (VPFB:78-80); then pass the same array to every later call.

        Per path i, c = n_course[i] (None: C each), n = n_pts[i]: when vel_plan[i] > vel_max + 0.1 (float64), the brake
        profile tph.calc_vel_profile_brake(loc_gg * old_gg_scale[i], v_start=vel_plan[i]) is cut at idx = the first
        point at or below vel_max (n - 1 when there is none or it is point 0): vx_prefix = vel_course[:c] followed by
        the profile's points [0, idx), pref_idx = idx, vel_start = the profile at idx, and old_gg_scale[i] stays.
        Otherwise vx_prefix = vel_course[:c], pref_idx = 0, vel_start = vel_plan[i] and old_gg_scale[i] = gg_scale.

        vel_plan [N]; vel_course [N][C] (C = 0 allowed); kappa [N][P]; el_lengths [N][P - 1] or [N][P]; loc_gg a tuple
        or [N][P][2] (before the scale).  Returns (vx_prefix, n_prefix, pref_idx, vel_start): vx_prefix float64
        [N][C + P - 1], 0 behind n_prefix[i] = c + pref_idx[i]; n_prefix, pref_idx int32 [N]; vel_start float64 [N].
        out=(vx_prefix, n_prefix, pref_idx, vel_start) allocates nothing.  A device length out of range (n_pts outside
        [2, P], n_course outside [0, C]) gives a row of NaN, n_prefix = pref_idx = -1, vel_start NaN and leaves the
        path's old_gg_scale as it was."""
        if self.params is None:
            raise RuntimeError("check_brake_prefix: call update_dyn_parameters first")
        on_device = isinstance(kappa, torch.Tensor)
        host_memory = None
        if not on_device:
            host_memory = old_gg_scale
            vel_plan, vel_course, kappa, el_lengths, loc_gg, old_gg_scale, n_course, n_pts = self._upload_prefix(
                vel_plan, vel_course, kappa, el_lengths, loc_gg, old_gg_scale, n_course, n_pts)
        dev = kappa.device
        if dev.type != "cuda":
            raise ValueError("kappa: a CUDA tensor or a NumPy array, got a tensor on %s" % dev)
        if kappa.dim() != 2 or kappa.shape[0] < 1 or kappa.shape[1] < 2:
            raise ValueError("kappa must be [N >= 1][P >= 2], got %s" % (tuple(kappa.shape),))
        n, p = kappa.shape
        gg = None if isinstance(loc_gg, tuple) else loc_gg
        if gg is None and (len(loc_gg) != 2 or not all(np.isscalar(g) for g in loc_gg)):
            raise ValueError("loc_gg: a tuple (ax_max, ay_max) or an array [N][P][2]")
        if not isinstance(vel_course, torch.Tensor) or vel_course.dim() != 2:
            raise ValueError("vel_course: a float64 tensor [%d][C] on %s, got %s" % (n, dev, _describe(vel_course)))
        cap = vel_course.shape[1]
        el_cols = el_lengths.shape[-1] if isinstance(el_lengths, torch.Tensor) and el_lengths.dim() == 2 \
            and el_lengths.shape[-1] in (p - 1, p) else p
        arrays = dict(kappa=(kappa, (n, p)), el_lengths=(el_lengths, (n, el_cols)), vel_plan=(vel_plan, (n,)),
                      vel_course=(vel_course, (n, cap)), old_gg_scale=(old_gg_scale, (n,)))
        if gg is not None:
            arrays["loc_gg"] = (gg, (n, p, 2))
        for name, (t, shape) in arrays.items():
            if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.float64 or tuple(t.shape) != shape:
                raise ValueError("%s: a float64 tensor %s on %s, got %s" % (name, list(shape), dev, _describe(t)))
        if not old_gg_scale.is_contiguous():
            raise ValueError("old_gg_scale: updated in place, so it must be contiguous")
        lengths = dict(n_pts=n_pts, n_course=n_course)
        for name, t in lengths.items():
            if t is not None:
                if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.int32 or tuple(t.shape) != (n,):
                    raise ValueError("%s: an int32 tensor [%d] on %s, got %s" % (name, n, dev, _describe(t)))
                lengths[name] = t.contiguous()
        width = cap + p - 1
        if out is None:
            vx_prefix = torch.empty((n, width), dtype=torch.float64, device=dev)
            n_prefix = torch.empty(n, dtype=torch.int32, device=dev)
            pref_idx = torch.empty(n, dtype=torch.int32, device=dev)
            vel_start = torch.empty(n, dtype=torch.float64, device=dev)
        else:
            if len(out) != 4:
                raise ValueError("out: (vx_prefix, n_prefix, pref_idx, vel_start)")
            vx_prefix, n_prefix, pref_idx, vel_start = out
            if not isinstance(vx_prefix, torch.Tensor) or vx_prefix.device != dev or vx_prefix.dtype != torch.float64 \
                    or tuple(vx_prefix.shape) != (n, width) or vx_prefix.stride(1) != 1 or vx_prefix.stride(0) < width:
                raise ValueError("out vx_prefix: a float64 tensor [%d][%d] on %s with contiguous rows, got %s"
                                 % (n, width, dev, _describe(vx_prefix)))
            for name, t, dt in (("n_prefix", n_prefix, torch.int32), ("pref_idx", pref_idx, torch.int32),
                                ("vel_start", vel_start, torch.float64)):
                if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != dt or tuple(t.shape) != (n,) \
                        or not t.is_contiguous():
                    raise ValueError("out %s: a contiguous %s tensor [%d] on %s, got %s" % (name, dt, n, dev, _describe(t)))
        kappa, _ = _rows(kappa, p)
        el_lengths, _ = _rows(el_lengths, el_lengths.shape[1])
        if gg is not None:
            gg, _ = _rows(gg, 2 * p)
        vel_plan = vel_plan.contiguous()
        params = self.params
        if gg is None:
            params = capi.Params.from_buffer_copy(params)
            params.gg_ax, params.gg_ay = float(loc_gg[0]), float(loc_gg[1])
        bp = capi.BrakePrefix()
        bp.n_paths, bp.n_points = n, p
        bp.n_pts = lengths["n_pts"].data_ptr() if lengths["n_pts"] is not None else None
        bp.kappa, bp.kappa_s = kappa.data_ptr(), kappa.stride(0)
        bp.el, bp.el_s = el_lengths.data_ptr(), el_lengths.stride(0)
        if gg is not None:
            bp.gg, bp.gg_s = gg.data_ptr(), gg.stride(0)
        bp.vel_plan = vel_plan.data_ptr()
        if cap > 0:
            vel_course, _ = _rows(vel_course, cap)
            bp.vel_course, bp.vel_course_s = vel_course.data_ptr(), vel_course.stride(0)
        bp.n_course_cap = cap
        bp.n_course = lengths["n_course"].data_ptr() if lengths["n_course"] is not None else None
        bp.old_gg_scale = old_gg_scale.data_ptr()
        bp.vx_prefix, bp.vx_prefix_s = vx_prefix.data_ptr(), vx_prefix.stride(0)
        bp.n_prefix, bp.pref_idx, bp.vel_start = n_prefix.data_ptr(), pref_idx.data_ptr(), vel_start.data_ptr()
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        capi.check(self.lib, self.lib.ltpl_brake_prefix_batch(C.byref(params), C.byref(bp), stream),
                   "ltpl_brake_prefix_batch")
        if on_device:
            return vx_prefix, n_prefix, pref_idx, vel_start
        torch.cuda.current_stream(dev).synchronize()
        host_memory[...] = old_gg_scale.cpu().numpy()
        return vx_prefix.cpu().numpy(), n_prefix.cpu().numpy(), pref_idx.cpu().numpy(), vel_start.cpu().numpy()

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
        h = _host_arrays(kappa, n_pts, el_lengths=el, loc_gg=loc_gg, v_start=v_start, v_end=v_end)
        return [self._to_device(h[k]) for k in ("kappa", "el_lengths", "loc_gg", "v_start", "v_end", "n_pts")]

    def _upload_follow(self, kappa, el, loc_gg, scal, obj_pos, n_pts):
        """NumPy arguments of calc_vel_profile_follow to device tensors, all checked on the host first"""
        h = _host_arrays(kappa, n_pts, el_lengths=el, loc_gg=loc_gg, obj_pos=obj_pos, **scal)
        k = h["kappa"]
        if h["el_lengths"].shape == (k.shape[0], k.shape[1] - 1):
            raise ValueError("el_lengths: calc_vel_profile_follow takes the path's whole el column [N][P] = [%d][%d] "
                             "(the last element enters the ego stop distance), got [N][P - 1]" % k.shape)
        d = {name: self._to_device(a) for name, a in h.items()}
        return d["kappa"], d["el_lengths"], d["loc_gg"], {name: d[name] for name in scal}, d["obj_pos"], d["n_pts"]

    def _upload_prefix(self, vel_plan, vel_course, kappa, el, loc_gg, old_gg_scale, n_course, n_pts):
        """NumPy arguments of check_brake_prefix to device tensors, all checked on the host first; old_gg_scale must be
        a float64 NumPy array [N] (it is written back after the call)"""
        h = _host_arrays(kappa, n_pts, el_lengths=el, loc_gg=loc_gg, vel_plan=vel_plan, vel_course=vel_course)
        n = h["kappa"].shape[0]
        if h["vel_course"].ndim != 2 or h["vel_course"].shape[0] != n:
            raise ValueError("vel_course: an array [%d][C], got %s" % (n, _describe(h["vel_course"])))
        if not isinstance(old_gg_scale, np.ndarray) or old_gg_scale.dtype != np.float64 or old_gg_scale.shape != (n,) \
                or not old_gg_scale.flags.writeable:
            raise ValueError("old_gg_scale: a writeable float64 NumPy array [%d] (updated in place), got %s"
                             % (n, _describe(old_gg_scale)))
        if n_course is not None:
            cap = h["vel_course"].shape[1]
            c = np.asarray(n_course)
            if c.dtype.kind not in "iu" or c.shape != (n,):
                raise ValueError("n_course: an integer array [%d], got %s" % (n, _describe(n_course)))
            if np.any(c < 0) or np.any(c > cap):
                raise ValueError("n_course: every length must be in [0, %d], got %d .. %d" % (cap, c.min(), c.max()))
            n_course = np.ascontiguousarray(c, dtype=np.int32)
        d = {name: self._to_device(a) for name, a in h.items()}
        return (d["vel_plan"], d["vel_course"], d["kappa"], d["el_lengths"], d["loc_gg"],
                self._to_device(np.ascontiguousarray(old_gg_scale)), self._to_device(n_course), d["n_pts"])

    def _to_device(self, a):
        return torch.from_numpy(a).to(self.device) if isinstance(a, np.ndarray) else a


def _host_arrays(kappa, n_pts, **arrays) -> dict:
    """host checks shared by the NumPy paths: kappa [N >= 1][P >= 2], n_pts (integers in [2, P]) and every other array
    numeric and not a tensor; returns contiguous float64 arrays (n_pts int32; a loc_gg tuple and None pass through)"""
    kappa = _host(kappa, "kappa")
    if kappa.ndim != 2 or kappa.shape[0] < 1 or kappa.shape[1] < 2:
        raise ValueError("kappa must be [N >= 1][P >= 2], got %s" % (kappa.shape,))
    out = dict(kappa=kappa, n_pts=_host_lengths(n_pts, kappa.shape[0], kappa.shape[1]))
    for name, a in arrays.items():
        out[name] = a if a is None or (name == "loc_gg" and isinstance(a, tuple)) else _host(a, name)
    return out


def _host(a, name, dtype=np.float64):
    """a numeric host array (not a tensor) as a contiguous array of dtype"""
    if isinstance(a, torch.Tensor):
        raise ValueError("%s: NumPy arrays and tensors cannot be mixed in one call" % name)
    a = np.asarray(a)
    if a.dtype.kind not in "iuf":
        raise ValueError("%s: a numeric array, got %s" % (name, a.dtype))
    return np.ascontiguousarray(a, dtype=dtype)


def _host_lengths(n_pts, n, p):
    """host lengths n_pts: None, or integers [n] in [2, p] as contiguous int32"""
    if n_pts is None:
        return None
    h = np.asarray(n_pts)
    if h.dtype.kind not in "iu" or h.shape != (n,):
        raise ValueError("n_pts: an integer array [%d], got %s" % (n, _describe(n_pts)))
    if np.any(h < 2) or np.any(h > p):
        raise ValueError("n_pts: every length must be in [2, %d], got %d .. %d" % (p, h.min(), h.max()))
    return _host(h, "n_pts", np.int32)


def check_follow_args(len_veh, control_type, control_params, glob_rl):
    """the follow arguments of VelocityPlanner: None when none is given, else a dict with the race line in CVPF:166's
    form [M][6] (s, x, y, kappa, vx, el) as float64 NumPy; ValueError for anything incomplete or malformed"""
    given = dict(len_veh=len_veh, follow_control_type=control_type, follow_control_params=control_params,
                 glob_rl=glob_rl)
    if all(v is None for v in given.values()):
        return None
    missing = [k for k, v in given.items() if v is None]
    if missing:
        raise ValueError("follow mode needs len_veh, follow_control_type, follow_control_params and glob_rl; missing %s"
                         % ", ".join(missing))
    if control_type not in ("PD", "PDtan"):
        raise ValueError('follow_control_type: "PD" or "PDtan", got %r' % (control_type,))
    keys = ("k_p", "k_d", "c_p") + (("tan_w",) if control_type == "PDtan" else ())
    if not isinstance(control_params, dict) or any(k not in control_params for k in keys):
        raise ValueError("follow_control_params: a dict with %s for %s, got %r" % (", ".join(keys), control_type,
                                                                                 control_params))
    cp = {k: float(control_params[k]) for k in keys}
    g = np.asarray(glob_rl, dtype=np.float64) if not isinstance(glob_rl, torch.Tensor) else None
    if g is None or g.ndim != 2 or g.shape[0] < 3 or g.shape[1] != 5:
        raise ValueError("glob_rl: the closed race line [M + 1 >= 3][5] (s, x, y, kappa, vx), got %s"
                         % _describe(glob_rl))
    if not np.all(np.isfinite(g)):
        raise ValueError("glob_rl: every value must be finite")
    if not np.array_equal(g[-1, 1:3], g[0, 1:3]):
        raise ValueError("glob_rl: the first point must be repeated at the end (a closed race line, as "
                         "Lattice.glob_rl stores it)")
    g6 = np.ascontiguousarray(np.column_stack((g[:-1], np.diff(g[:, 0]))))   # CVPF:166
    return dict(len_veh=float(len_veh), control_type=control_type, control_params=cp, glob_rl=g6)


def _describe(t) -> str:
    if isinstance(t, torch.Tensor):
        return "%s %s on %s" % (t.dtype, list(t.shape), t.device)
    if isinstance(t, np.ndarray):
        return "%s %s (NumPy)" % (t.dtype, list(t.shape))
    return type(t).__name__
