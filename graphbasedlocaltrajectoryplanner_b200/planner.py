"""
BatchPlanner -- host side of the batched planning tick.  PyTorch is used ONLY as the owner of device buffers and
streams (``tensor.data_ptr()`` / ``torch.cuda.current_stream().cuda_stream``); all compute happens in the hand-written
sm_90a kernels behind the C-ABI (capi.py -> libltpl_b200.so).

Mirrors, batched over B independent scenarios, the reference call sequence of one planning tick
(main_min_example.py:69-104):

    set_startpos (LTPL:262-296)  ->  calc_paths (LTPL:300-340)  ->  calc_vel_profile (LTPL:344-408)
"""

from __future__ import annotations

import configparser
import ctypes as C
import json
from dataclasses import dataclass, replace

import numpy as np
import torch

from . import capi
from .lattice import Lattice
from .lattice_blob import pack_lattice
from .scenarios import DeviceScenarioBatch, ScenarioBatch

NSLOT = capi.NSLOT


def check_filt_window(w) -> int:
    """[SMOOTHING] filt_window_width: width of the moving-average window over every velocity profile (tph.conv_filt;
    1 = no smoothing).  The reference raises on its first calc_vel_profile; here the value is refused up front."""
    if int(w) != w or w < 1:
        raise ValueError("filt_window_width must be a positive odd integer, got %r" % (w,))
    if w % 2 != 1:
        raise RuntimeError("Window width of moving average filter must be odd!")   # tph.conv_filt
    return int(w)


def max_objects(header, cap: dict) -> int:
    """largest object list per scenario a planner over this lattice header and these capacities can plan: k_plan keeps
    one record per on-track object in shared memory (ltpl_max_objects; several hundred on every lattice)."""
    return int(capi.load_library().ltpl_max_objects(C.byref(header), int(cap["h_max"])))


def check_object_count(k_obj: int, bound: int) -> int:
    """object slots per scenario: at least 1, at most ``bound`` (max_objects); refused before anything is launched."""
    k_obj = max(1, int(k_obj))
    if k_obj > bound:
        raise ValueError("%d objects per scenario exceed k_plan's shared memory on this lattice: at most %d"
                         % (k_obj, bound))
    return k_obj


def read_online_config(path: str) -> dict:
    """online ini keys the batched path needs (reference: OTH:99-122, LTPL:168-173)."""
    cfg = configparser.ConfigParser()
    if not cfg.read(path):
        raise ValueError('Specified cost config file does not exist or is empty!')
    ctype = cfg.get('FOLLOW', 'controller_type')
    vp_type = cfg.get('VP', 'vp_type')
    if vp_type != "fb":
        raise ValueError('Only the forward-backward velocity planner (vp_type=fb) is available in the batched path!')
    return dict(max_heading_offset=json.loads(cfg.get('GENERAL', 'max_heading_offset')),
                nmbr_export_points=json.loads(cfg.get('EXPORT', 'nmbr_export_points')),
                v_max_offset=cfg.getfloat('ACTIONSET', 'v_max_offset'),
                max_solutions=cfg.getint('ACTIONSET', 'max_solutions'),
                filt_window_width=check_filt_window(cfg.getint('SMOOTHING', 'filt_window_width')),
                w_last_edges=json.loads(cfg.get('COST', 'w_last_edges')),
                controller_type=ctype,
                control_params=json.loads(cfg.get('FOLLOW', 'control_params_' + ctype)),
                delaycomp=cfg.getfloat('DELAY', 'delaycomp'))


def check_gg_map(ax, ay, x0, y0, cell):
    """input checks of a friction map (BatchPlanner.set_gg_map): ``ax``, ``ay`` 2-D [ny][nx] arrays (NumPy or torch) of
    equal shape with ny, nx >= 2 and finite values > 0; ``x0``, ``y0`` finite; ``cell`` finite and > 0.  Raises
    ValueError; returns (nx, ny, inv_cell) with inv_cell = 1 / cell in float64."""
    shape_x, shape_y = tuple(ax.shape), tuple(ay.shape)
    if shape_x != shape_y or len(shape_x) != 2:
        raise ValueError("gg map: ax and ay must be 2-D arrays [ny][nx] of equal shape, got %s and %s"
                         % (shape_x, shape_y))
    ny, nx = shape_x
    if nx < 2 or ny < 2:
        raise ValueError("gg map: at least 2 x 2 vertices, got %d x %d" % (nx, ny))
    if nx * ny > 2 ** 31 - 1:
        raise ValueError("gg map: %d x %d vertices exceed 32-bit indexing" % (nx, ny))
    for name, a in (("ax", ax), ("ay", ay)):
        ok = bool(torch.all(torch.isfinite(a) & (a > 0))) if isinstance(a, torch.Tensor) \
            else bool(np.all(np.isfinite(a) & (a > 0)))
        if not ok:
            raise ValueError("gg map: every %s value must be finite and > 0" % name)
    x0, y0, cell = float(x0), float(y0), float(cell)
    if not (np.isfinite(x0) and np.isfinite(y0)):
        raise ValueError("gg map: the origin (x0, y0) must be finite")
    if not (np.isfinite(cell) and cell > 0.0):
        raise ValueError("gg map: cell must be finite and > 0, got %r" % cell)
    return nx, ny, 1.0 / cell


def check_gg_planes(ax, ay, batch: int, p_max: int, device) -> None:
    """input checks of friction planes given as device tensors (BatchPlanner.set_local_gg_planes, the local_gg of a
    split capture): ``ax``, ``ay`` float64 tensors on ``device`` of equal shape [NSLOT][batch][P <= p_max], any strides.
    Shapes, dtypes and devices only (no values, no synchronisation); raises ValueError."""
    for name, a in (("ax", ax), ("ay", ay)):
        if not isinstance(a, torch.Tensor) or a.device != device or a.dtype != torch.float64:
            raise ValueError("local_gg planes: %s must be a float64 tensor on %s, got %s" % (
                name, device, "%s on %s" % (a.dtype, a.device) if isinstance(a, torch.Tensor) else type(a).__name__))
    if ax.shape != ay.shape or ax.dim() != 3 or tuple(ax.shape[:2]) != (NSLOT, batch) or ax.shape[2] > p_max:
        raise ValueError("local_gg planes must have the shape [NSLOT][B][P <= p_max] = [%d][%d][<= %d], got %s and %s"
                         % (NSLOT, batch, p_max, tuple(ax.shape), tuple(ay.shape)))


def fill_vel_params(p, online: dict, veh: dict, vel_max: float, gg_scale: float, local_gg, ax_max_machines,
                    safety_d: float, incl_emerg_traj: bool) -> None:
    """fills LtplParams ``p`` from the online ini keys (``online``, see read_online_config), the vehicle parameters of
    graph_init (``veh``: dyn_model_exp, drag_coeff, m_veh) and the per-call arguments of Graph_LTPL.calc_vel_profile
    (LTPL:344-352).  Every check runs before the first field is written: a refused call leaves ``p`` as it was."""
    if type(local_gg) is not tuple or len(local_gg) != 2:   # OTH:651-653 (dict form: Graph_LTPL / set_local_gg_planes)
        raise ValueError("Provided local_gg does not satisfy requested format! Read parameter documentation.")
    axm = np.atleast_2d(np.asarray(ax_max_machines, dtype=np.float64))
    if axm.shape[1] != 2:
        raise RuntimeError("ax_max_machines must consist of the two columns [vx, ax_max_machines]!")
    if axm.shape[0] > capi.MAX_AXM:
        raise ValueError("ax_max_machines has more than %d rows" % capi.MAX_AXM)
    if axm[-1, 0] < vel_max:                               # tph.calc_vel_profile input check
        raise RuntimeError("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!")
    o = online
    if o["controller_type"] not in ("PD", "PDtan"):
        raise ValueError('Unsupported control type "' + o["controller_type"] + '"!')
    p.max_heading_offset = o["max_heading_offset"]
    p.v_max_offset = o["v_max_offset"]
    cp = o["control_params"]
    p.follow_c_p, p.follow_k_d, p.follow_k_p = cp["c_p"], cp["k_d"], cp["k_p"]
    p.follow_tan_w = cp.get("tan_w", 1.0)
    p.follow_control_type = 0 if o["controller_type"] == "PD" else 1
    p.nmbr_export_points = int(o["nmbr_export_points"])
    p.dyn_model_exp, p.drag_coeff, p.m_veh = veh["dyn_model_exp"], veh["drag_coeff"], veh["m_veh"]
    p.vel_max, p.gg_scale, p.gg_ax, p.gg_ay, p.safety_d = vel_max, gg_scale, local_gg[0], local_gg[1], safety_d
    p.n_axm = axm.shape[0]
    p.delaycomp = float(o.get("delaycomp", 0.1))
    for i in range(3):
        p.w_last_edges[i] = float(o["w_last_edges"][i]) if i < len(o["w_last_edges"]) else 1.0
    p.incl_emerg_traj = 1 if incl_emerg_traj else 0
    p.filt_window = int(o["filt_window_width"])
    for i in range(axm.shape[0]):
        p.axm_v[i] = axm[i, 0]
        p.axm_a[i] = axm[i, 1]
    for i in range(axm.shape[0] - 1):   # slopes exactly as np.interp forms them
        p.axm_s[i] = (axm[i + 1, 1] - axm[i, 1]) / (axm[i + 1, 0] - axm[i, 0])


PREFER_IDS = {"straight": capi.ACT_STRAIGHT, "follow": capi.ACT_FOLLOW, "left": capi.ACT_LEFT, "right": capi.ACT_RIGHT,
              "emergency": capi.ACT_EMERGENCY}
_PREFER_DTYPES = (torch.int8, torch.uint8, torch.int32, torch.int64)


def check_prefer(prefer, batch: int, device):
    """input checks of an action preference (BatchPlanner.select): a list of action names (PREFER_IDS; one list for the
    whole batch), a host integer array [batch][L] or an integer tensor [batch][L] on ``device`` (int8, uint8, int32 or
    int64, any strides), L <= capi.SELECT_MAX.  Names, shapes, dtypes and devices only (no tensor values, no
    synchronisation); raises ValueError.  Returns the tensor as it is, or the ids as an int64 NumPy array [1][L] (a
    list) or [batch][L] (an array)."""
    if isinstance(prefer, torch.Tensor):
        if prefer.device != torch.device(device) or prefer.dtype not in _PREFER_DTYPES:
            raise ValueError("prefer: a tensor must be int8 / uint8 / int32 / int64 on %s, got %s on %s"
                             % (device, prefer.dtype, prefer.device))
        ids = prefer
    elif isinstance(prefer, (list, tuple)):
        bad = [a for a in prefer if not isinstance(a, str) or a not in PREFER_IDS]
        if bad:
            raise ValueError("prefer: unknown action name(s) %s; the names are %s" % (bad, sorted(PREFER_IDS)))
        ids = np.array([[PREFER_IDS[a] for a in prefer]], dtype=np.int64).reshape(1, len(prefer))
    elif isinstance(prefer, np.ndarray):
        if prefer.dtype.kind not in "iu":
            raise ValueError("prefer: a host array must hold integers, got %s" % prefer.dtype)
        ids = prefer.astype(np.int64)
    else:
        raise ValueError("prefer: a list of action names, an integer array or a device tensor [B][L], got %s"
                         % type(prefer).__name__)
    rows = 1 if isinstance(prefer, (list, tuple)) else batch
    if ids.ndim != 2 or ids.shape[0] != rows or ids.shape[1] > capi.SELECT_MAX:
        raise ValueError("prefer: shape [%d][L <= %d], got %s" % (batch, capi.SELECT_MAX, tuple(ids.shape)))
    return ids


DEFAULT_ONLINE = dict(max_heading_offset=0.8, nmbr_export_points=115, v_max_offset=0.1, max_solutions=1,
                      filt_window_width=1, w_last_edges=[0.0, 0.5, 0.8], controller_type="PD",
                      control_params={"c_p": 1.25, "k_d": 0.025, "k_p": 0.2}, delaycomp=0.1)


@dataclass
class TickState:
    """what a tick changes on the planner's host side besides dims and the buffer dicts, with the flags that choose the
    optional bindings of buffer_sources.  A TickGraph keeps a copy per captured state and installs it after a replay."""
    in_cur: int = 0                  # the device input copy in use (stateful ticks alternate the two)
    pos_last: torch.Tensor = None    # `pos` of the input copy the last tick used; set from the first stateful staging on
    gg_planes_used: bool = False     # the last velocity call ran with gg planes (decides the next tick's prev_gg)
    gg: bool = False                 # this tick's gg planes are bound (set_local_gg_planes; a friction map binds them too)
    prev_gg: bool = False            # the last stateful staging kept planes as memory: buffers.prev_gg
    restart: bool = False            # the last stateful staging had a restart mask: buffers.restart
    export: int = 0                  # the traj_bufs set the tick exports into (plan_stream's set)
    gg_uploaded: bool = False        # the planes set_local_gg_planes bound last came from host arrays
    zone_key_kept: bool = False      # a staging since allocate(): the next stateful tick applies the zone rule
    zone_key_zero: bool = True       # the device zone keys (_zone_key) are all zero
    zones: tuple = None              # the zone list whose bitmasks are on the device (None: none yet)
    staged_on_device: bool = False   # the last staged batch was a DeviceScenarioBatch: upload() has nothing to copy
    ticked: bool = False             # the buffers hold a tick (a velocity call ran since they were allocated)
    emerg: bool = False              # the last velocity call ran with incl_emerg_traj ('emergency' for select)
    selected: bool = False           # select() ran since the last velocity call: sel_action="selected" may be staged


SWAPPED = ("path", "node_idx", "nodes", "coeff", "s_vx_ax", "em_vx")            # stateful memory swapped by pointer
CARRIED = ("action_id", "traj_len", "em_info", "path_len", "n_nodes", "trim")  # stateful memory carried by ONE copy
_PER_BATCH = tuple(n for n in capi.BUFFER_FIELDS if n not in capi.STATE_FIELDS and n != "traj")


def buffer_sources(t: dict, state: dict, traj_bufs: list, tick: TickState, gg_map=None, traj_base=None,
                   export_rows=None) -> dict:
    """the tensor behind every field of capi.BUFFER_FIELDS (None: NULL), the one rule for what BatchPlanner passes, from
    its tables -- ``t`` (the batch's buffers and input copy in use), the memory ``state`` (None without), the export
    sets, map, id counter and export override when set -- and the flags of ``tick`` that choose optional bindings."""
    src = dict.fromkeys(capi.BUFFER_FIELDS)
    src.update((n, t[n]) for n in _PER_BATCH)   # inputs, outputs, scratch; obj_pred and zone_bits may be placeholders
    src["traj"] = traj_bufs[tick.export] if export_rows is None else export_rows
    if tick.gg or gg_map is not None:   # the library evaluates a map into this tick's planes
        src["gg"] = t["gg"]
    src["gg_map"], src["traj_base"] = gg_map, traj_base
    if state is not None:
        src["trim"], src["em_vx"], src["zone_s0"] = t["trim"], t["em_vx"], state["zone_s0"]
    if state is not None and tick.pos_last is not None:   # from the first stateful staging on
        src.update(("prev_" + k, state["other"][k]) for k in SWAPPED)
        src.update(("prev_" + k, state["prev_small"][k]) for k in CARRIED)
        src.update((k, state[k]) for k in ("st_info", "vel_plan", "course", "obj_dist"))
        src["sel_action"], src["t_const"], src["pos_last"] = t["sel_action"], t["t_const"], tick.pos_last
        src["prev_gg"] = state["other"]["gg"] if tick.prev_gg else None
        src["restart"] = state["restart"] if tick.restart else None
    return src


class BatchPlanner(object):
    N_SETS = 3   # host staging / export buffer sets of the pipelined path (plan_stream)

    def __init__(self, lattice: Lattice = None, online: dict = None, device=None, veh_param_dyn_model_exp: float = 1.0,
                 veh_param_dragcoeff: float = 0.85, veh_param_mass: float = 1000.0, packed: tuple = None,
                 blob_tensor: torch.Tensor = None, stateful: bool = False):
        """``packed`` = (LatticeHeader, capacities) + ``blob_tensor`` (device uint8) when the blob arrived through a
        collective instead of being uploaded from ``lattice`` (parallel.broadcast_lattice)."""
        self.handle = None
        self.online = dict(DEFAULT_ONLINE)
        if online:
            self.online.update(online)
        self.online["filt_window_width"] = check_filt_window(self.online["filt_window_width"])
        self.lib = capi.load_library()
        if not torch.cuda.is_available():
            raise RuntimeError("BatchPlanner needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.device = torch.device(device if device is not None else "cuda:0")
        torch.cuda.set_device(self.device)
        self.veh = dict(dyn_model_exp=float(veh_param_dyn_model_exp), drag_coeff=float(veh_param_dragcoeff),
                        m_veh=float(veh_param_mass))
        if packed is None:
            self.header, blob, self.cap = pack_lattice(lattice)
            self.blob = torch.from_numpy(blob).to(self.device)
        else:
            self.header, self.cap = packed
            self.blob = blob_tensor
            if self.blob.device != self.device or self.blob.dtype != torch.uint8 \
                    or self.blob.numel() != self.header.blob_bytes:
                raise ValueError("blob tensor does not match the lattice header")
        self._stateful = bool(stateful)
        if stateful:   # stateful ticks carry constant nodes / points of earlier ticks in front of the new plan
            self.cap = dict(self.cap, h_max=self.cap["h_max"] + 8, p_max=self.cap["p_max"] + 96)
        self.max_objects = max_objects(self.header, self.cap)
        handle = C.c_void_p()
        capi.check(self.lib, self.lib.ltpl_lattice_create(C.byref(self.header), C.c_void_p(self.blob.data_ptr()),
                                                          C.byref(handle)), "ltpl_lattice_create")
        self.handle = handle
        # node offsets per layer (zone bitmasks address nodes as node_off[layer] + node), read back from the blob
        off = int(self.header.off_node_off)
        self.node_off = self.blob[off: off + 4 * (int(self.header.num_layers) + 1)].cpu().numpy().view(np.int32) \
            .astype(np.int64)
        self.lattice_nodes = int(self.header.num_nodes)
        self.dims = None
        self._k_pred_cap = 0
        self.buf = capi.Buffers()     # the one struct every call passes, for the planner's life (bound by _bind)
        self._src = None              # the tensors _bind wrote into buf (buffer_sources)
        self._export_rows = None      # rows that replace the export set (set_export_rows), or None
        self.t = {}
        self.params = capi.Params()
        self._tick_count = 0
        self._gg_map = None           # device [ny][nx][2] friction map of set_gg_map, or None
        self.on_device_start = None   # optional callable, called where a stateful tick's host staging ends (timing)
        self._tick = TickState()
        self._generation = 0          # bumped by every change a captured TickGraph cannot follow (tick_graph.py)
        self._plane_bumps = 0         # the part of _generation set_local_gg_planes bumped (split graphs with planes)
        self._split_pending = None    # (SplitTickGraph, velocity half) after its replay_paths(), until the next call
        self._traj_base = None        # [1] int32 device id counter of buffers.traj_base, from the first capture on
        self._copy_stream = None      # second stream of plan_stream (trajectory downloads), created on first use
        self._sel = self._sel_host = None   # per set: selection buffers of select(), device / pinned (created on use)
        self.set_vel_params()

    def __del__(self):
        try:
            if self.handle:
                self.lib.ltpl_lattice_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def set_subbatches(self, n: int) -> None:
        """number of scenario windows a tick is split into inside the library (1 .. capi.MAX_SUB; default 4 for windows
        of >= 512 scenarios): window s runs on an internal stream, so kernels of different stages overlap.  The results
        do not depend on it (only the unspecified order of the compact export rows)."""
        capi.check(self.lib, self.lib.ltpl_set_subbatches(self.handle, int(n)), "ltpl_set_subbatches")
        self._generation += 1

    # -- parameters ------------------------------------------------------------------------------------------------------
    def set_vel_params(self, vel_max: float = 100.0, gg_scale: float = 1.0, local_gg=(5.0, 5.0),
                       ax_max_machines=np.atleast_2d([100.0, 5.0]), safety_d: float = 30.0,
                       incl_emerg_traj: bool = False) -> None:
        """per-call arguments of Graph_LTPL.calc_vel_profile (LTPL:344-352)."""
        if local_gg is None:        # location dependent friction: the planes of set_local_gg_planes() are used
            local_gg = (1.0, 1.0)
        fill_vel_params(self.params, self.online, self.veh, vel_max=vel_max, gg_scale=gg_scale, local_gg=local_gg,
                        ax_max_machines=ax_max_machines, safety_d=safety_d, incl_emerg_traj=incl_emerg_traj)
        self._generation += 1   # after the checks: a refused call leaves captured graphs valid

    # -- buffers -----------------------------------------------------------------------------------------------------------
    @staticmethod
    def _packed(spec, make):
        """one raw byte buffer + named views into it (sections 256-byte aligned)"""
        offs, total = {}, 0
        for name, shape, dt in spec:
            nbytes = int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
            offs[name] = (total, nbytes, shape, dt)
            total += (nbytes + 255) // 256 * 256
        raw = make(total)
        views = {name: raw[o:o + nb].view(dt).view(shape) for name, (o, nb, shape, dt) in offs.items()}
        return raw, views

    def _bind(self, *names) -> None:
        """writes buffer_sources into self.buf in place: every field, or only ``names`` where nothing else changed"""
        src = buffer_sources(self.t, self._state, self.traj_bufs, self._tick, self._gg_map, self._traj_base,
                             self._export_rows)
        for name in names or capi.BUFFER_FIELDS:
            setattr(self.buf, name, None if src[name] is None else src[name].data_ptr())
        self._src = src

    def set_export_rows(self, rows=None) -> None:
        """the compact export rows (buffers.traj) go to ``rows``, a device tensor [(NSLOT + 1) * B][n_export][7] float32
        that may be peer memory (parallel.PeerGather), instead of the planner's own export sets; None: back to them"""
        self._export_rows = rows
        self._bind("traj")

    def _alloc_inputs(self, batch: int, k_obj: int, k_pred: int) -> None:
        """The scenario inputs live in ONE packed device buffer (one H2D copy per tick) with N_SETS pinned host staging
        sets.  Only these buffers depend on the object / prediction capacities, so a batch with more objects or with
        its first 'prediction' array re-creates them and nothing else: the memory of a stateful session stays intact.
        Two device copies are kept and used alternately by stateful ticks: the position estimate of the previous
        calc_vel_profile (pos_last, OTH:537, MOPG:80-84) is then simply the other copy's ``pos``."""
        B, K, dev = int(batch), int(k_obj), self.device
        f64, i32 = torch.float64, torch.int32
        in_spec = [("pos", (B, 2), f64), ("heading", (B,), f64), ("vel", (B,), f64), ("vel_est", (B,), f64),
                   ("n_obj", (B,), i32), ("obj", (B, K, 5), f64), ("zone_sel", (B,), i32), ("n_pred", (B, K), i32),
                   ("sel_action", (B,), i32), ("t_const", (B,), f64)]
        if k_pred > 0:
            in_spec.append(("obj_pred", (B, K, int(k_pred), 2), f64))
        self._k_pred_cap = int(k_pred)
        self.d_in = []
        for _ in range(2):
            raw, views = self._packed(in_spec, lambda n: torch.zeros(n, dtype=torch.uint8, device=dev))
            if k_pred == 0:
                views["obj_pred"] = torch.zeros((1,), dtype=f64, device=dev)
            self.d_in.append((raw, views))
        self.h_in_raw, self.h_in_sets = [], []
        for _ in range(self.N_SETS):
            raw, views = self._packed(in_spec, lambda n: torch.zeros(n, dtype=torch.uint8).pin_memory())
            self.h_in_raw.append(raw)
            self.h_in_sets.append(views)
        self.h_in = self.h_in_sets[0]
        self._h2d_ev = [None] * self.N_SETS
        self.dims.k_obj = K
        self._use_inputs(0)

    def _use_inputs(self, which: int) -> None:
        self._tick.in_cur = which
        self.t.update(self.d_in[which][1])

    @property
    def _in_cur(self) -> int:
        return self._tick.in_cur

    @property
    def d_in_raw(self) -> torch.Tensor:
        """the packed device input copy in use (upload() copies a pinned staging set into it)"""
        return self.d_in[self._tick.in_cur][0]

    def allocate(self, batch: int, k_obj: int = 3, k_pred: int = 0) -> None:
        k_obj = check_object_count(k_obj, self.max_objects)
        if self.dims is not None and self.dims.batch == batch:
            if self.dims.k_obj >= k_obj and self._k_pred_cap >= k_pred:
                return
            # more object slots / prediction points than before: only the input buffers grow (see _alloc_inputs)
            torch.cuda.current_stream(self.device).synchronize()
            self._alloc_inputs(batch, max(k_obj, self.dims.k_obj), max(int(k_pred), self._k_pred_cap))
            self._bind()
            self._generation += 1
            return
        d = capi.Dims()
        d.batch, d.k_obj = int(batch), k_obj
        d.p0_max, d.p_max, d.h_max = self.cap["p0_max"], self.cap["p_max"], self.cap["h_max"]
        d.n_export = int(self.online["nmbr_export_points"])
        B, P0, P, H, NE = d.batch, d.p0_max, d.p_max, d.h_max, d.n_export
        dev = self.device
        f64, i32, f32 = torch.float64, torch.int32, torch.float32
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)   # noqa: E731
        # the small per-path result arrays live in one packed buffer (one D2H copy per tick)
        # (the first six are what a stateful tick keeps of the previous one: one contiguous block, carried by one copy)
        meta_spec = [("action_id", (NSLOT, B), i32), ("traj_len", (NSLOT, B), i32), ("em_info", (B, 3), i32),
                     ("path_len", (NSLOT, B), i32), ("n_nodes", (NSLOT, B), i32), ("trim", (NSLOT * B, 4), i32),
                     ("exp_q", (NSLOT * B,), i32), ("traj_row", (NSLOT, B), i32), ("traj_id", (NSLOT, B), i32),
                     ("status", (NSLOT, B), i32), ("sc_flags", (B,), i32), ("queue_cnt", (4 + 4 * capi.MAX_SUB,), i32)]
        self._carry_spec = meta_spec[:6]
        self._meta_spec = meta_spec
        self.d_meta_raw, t_meta = self._packed(meta_spec, lambda n: torch.zeros(n, dtype=torch.uint8, device=dev))
        t = dict(
            start_node=z((B, 2), i32), const_len=z((B,), i32), const_seg=z((5, B, P0), f64),
            const_coeff=z((B, 8), f64),
            nodes=z((NSLOT, B, H, 2), i32), node_idx=z((NSLOT, B, H), i32),
            edge_seq=z((NSLOT, B, H), i32), closest_obj=z((B,), i32), cobj=z((B, 4), f64), cobj_start=z((B,), i32),
            path=z((5, NSLOT * B, P), f64), coeff=z((NSLOT * B, H, 8), f64), queue=z((2, NSLOT * B), i32),
            s_vx_ax=z((3, NSLOT * B, P), f64),
            traj=z(((NSLOT + 1) * B, NE, 7), f32))
        t.update(t_meta)
        t["zone_bits"] = torch.zeros((1, 1), dtype=torch.int32, device=dev)   # replaced by _stage_zones()
        d.k_pred = 0
        d.n_zones, d.n_zone_words = 0, (self.lattice_nodes + 31) // 32
        self.t, self.dims = t, d
        self._export_rows = None   # sized for the old batch
        self._generation += 1
        self._tick = TickState()
        # zone keys of the last staged batch, which the next stateful tick compares with (k_stage reads and writes them);
        # one buffer per allocation, so that captured graphs keep its address
        self._zone_key = z((B,), torch.int64)
        self._alloc_inputs(B, k_obj, k_pred)
        self._state = None   # buffers of the stateful tick, allocated by next_tick()
        # further compact export buffers: the pipelined stream planner lets the D2H of step i overlap step i + 1
        self.traj_bufs = [t["traj"]] + [z(((NSLOT + 1) * B, NE, 7), f32) for _ in range(self.N_SETS - 1)]
        self._sel, self._sel_host = [None] * self.N_SETS, [None] * self.N_SETS
        # pinned host staging of the per-tick results (N_SETS sets for the pipelined path)
        pin = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory()   # noqa: E731
        self.h_meta_raw, self.h_out_sets = [], []
        for _ in range(self.N_SETS):
            raw, views = self._packed(meta_spec, lambda n: torch.zeros(n, dtype=torch.uint8).pin_memory())
            views["traj"] = pin(((NSLOT + 1) * B, NE, 7), f32)
            self.h_meta_raw.append(raw)
            self.h_out_sets.append(views)
        self.h_out = self.h_out_sets[0]
        self._meta_names = tuple(n for n, _, _ in meta_spec)
        self._row_bytes = NE * 7 * 4
        if self._stateful:
            self._alloc_state()   # incl. zone_s0, which the FIRST tick has to fill
        if self._gg_map is not None:
            self._gg_planes(t)
        self._bind()

    def set_local_gg_planes(self, ax=None, ay=None) -> None:
        """location dependent friction (calc_vel_profile(local_gg={action: [ndarray(P, 2)]}), OTH:649-666) for the batch:
        ``ax``, ``ay`` [NSLOT][B][P] (P <= p_max) = longitudinal / lateral limit at every point of every path (slot 0:
        straight | follow, 1: left, 2: right), aligned with the paths of the last calc_paths; None: back to the constant
        tuple of set_vel_params().  The values are taken without gg_scale (VPFB:213-214 applies it).  Clears the friction
        map of set_gg_map().
        ``ax``, ``ay`` may also be float64 tensors on the planner's device (any strides, e.g. a friction model evaluated
        on the device along device_results()["path"]): they are copied into this tick's planes on the current stream,
        without a host synchronisation, and give the bytes of the same values as NumPy arrays.  Such tensors are
        checked (device, dtype, shape) before anything changes; a refusal raises ValueError."""
        B, P = self.dims.batch, self.dims.p_max
        on_device = isinstance(ax, torch.Tensor) or isinstance(ay, torch.Tensor)
        if on_device:
            check_gg_planes(ax, ay, B, P, self.device)
        elif ax is not None:
            ax = np.asarray(ax, dtype=np.float64)
            ay = np.asarray(ay, dtype=np.float64)
            if ax.shape != ay.shape or ax.ndim != 3 or ax.shape[:2] != (NSLOT, B) or ax.shape[2] > P:
                raise ValueError("local_gg planes must have the shape [NSLOT][B][P <= p_max]")
        self._generation += 1 if self._gg_map is None else 2   # captured graphs evaluate a map: they go stale with it
        self._gg_map = None
        self._plane_bumps += 1
        self._split_pending = None
        self._tick.gg, self._tick.gg_uploaded = ax is not None, ax is not None and not on_device
        if on_device:   # the given values, then 1.0 behind them: what the host path writes
            n = ax.shape[2]
            rows = self._gg_planes(self.t).view(2, NSLOT, B, P)
            rows[0, :, :, :n].copy_(ax)
            rows[1, :, :, :n].copy_(ay)
            if n < P:
                rows[:, :, :, n:].fill_(1.0)
        elif ax is not None:
            host = np.ones((2, NSLOT * B, P))
            host[0, :, :ax.shape[2]] = ax.reshape(NSLOT * B, -1)
            host[1, :, :ay.shape[2]] = ay.reshape(NSLOT * B, -1)
            self._gg_planes(self.t).copy_(torch.from_numpy(host))
        self._bind("gg", "gg_map")

    def set_gg_map(self, ax=None, ay=None, x0: float = 0.0, y0: float = 0.0, cell: float = 1.0) -> None:
        """location dependent friction from a map of the track surface, for the whole batch: ``ax``, ``ay`` [ny][nx] =
        longitudinal / lateral limit (without gg_scale, like the local_gg rows) at the vertices of a regular grid with
        vertex [0][0] at (x0, y0) and spacing ``cell`` metres.  NumPy arrays or torch tensors on this planner's device.
        From now on the velocity half of every tick (tick, calc_vel_profile, next_tick, next_calc_vel_profile,
        plan_stream) evaluates the map on the device along every planned path (bilinear, clamped to the grid; DESIGN.md
        section 7), as calc_vel_profile(local_gg={action: [map(path[:, 0:2])]}) would take it.  The map is uploaded once
        and stays until it is changed.  None: back to the constant tuple of set_vel_params().  Clears the planes of
        set_local_gg_planes().  Bad input raises ValueError and changes nothing."""
        if ax is not None:
            for a in (ax, ay):
                if isinstance(a, torch.Tensor) and a.device != self.device:
                    raise ValueError("gg map: a torch tensor must be on the planner's device %s, got %s"
                                     % (self.device, a.device))
            if not isinstance(ax, torch.Tensor):
                ax = np.asarray(ax, dtype=np.float64)
            if not isinstance(ay, torch.Tensor):
                ay = np.asarray(ay, dtype=np.float64)
            nx, ny, inv_cell = check_gg_map(ax, ay, x0, y0, cell)
            dev = lambda a: torch.as_tensor(a, dtype=torch.float64).to(self.device)   # noqa: E731
            ax = torch.stack((dev(ax), dev(ay)), dim=-1).contiguous()   # [ny][nx][2]: one 16-byte load per vertex
            p = self.params
            p.gg_map_x0, p.gg_map_y0, p.gg_map_inv_cell = float(x0), float(y0), inv_cell
            p.gg_map_nx, p.gg_map_ny = nx, ny
        self._gg_map, self._tick.gg = ax, False
        self._generation += 1
        if self.dims is not None:   # (allocate binds them otherwise)
            if ax is not None:   # the planes the library evaluates the map into
                self._gg_planes(self.t)
            self._bind("gg", "gg_map")

    def _gg_planes(self, planes: dict) -> torch.Tensor:
        """``planes["gg"]``: the gg planes [2][NSLOT * B][p_max] of this batch (this tick's in ``t``, the last tick's in
        the stateful memory), created as ones on first use"""
        if "gg" not in planes:
            planes["gg"] = torch.ones((2, NSLOT * self.dims.batch, self.dims.p_max), dtype=torch.float64,
                                      device=self.device)
        return planes["gg"]

    def device_bytes(self) -> int:
        return int(sum(v.numel() * v.element_size() for v in self.t.values()) + self.blob.numel())

    @property
    def stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # -- scenario upload (host -> device) -------------------------------------------------------------------------------------
    def h2d_bytes(self) -> int:
        return int(sum(v.numel() * v.element_size() for v in self.h_in.values()))

    def d2h_bytes(self, n_rows: int = None) -> int:
        """bytes of one result download: the small per-path arrays + n_rows compact trajectory rows."""
        meta = sum(self.h_out[n].numel() * self.h_out[n].element_size() for n in self._meta_names)
        rows = self.h_out["traj"].shape[0] if n_rows is None else n_rows
        return int(meta + rows * self._row_bytes)

    def stage_scenarios(self, sc, vel_est=None, which: int = 0) -> None:
        """copy a scenario batch into the pinned staging buffers (host memcpy).  A DeviceScenarioBatch is written into
        the device inputs instead, by one kernel on the current stream (k_stage, no host synchronisation unless the
        batch brings more object slots or prediction points than allocated); upload() then has nothing to copy.
        ``vel_est`` may then be a device tensor [B]."""
        if isinstance(sc, DeviceScenarioBatch):
            vel_est = self._device_args(sc, vel_est)[0]
        self._stage(sc, vel_est, which)

    def _stage(self, sc, vel_est, which: int, tick_args: tuple = None) -> None:
        """staging of both batch kinds: the buffers grown for the batch and the zone bitmasks, then ONE kind-specific
        step -- a ScenarioBatch is copied into pinned staging set ``which`` (upload() copies it to the device), a
        DeviceScenarioBatch is written into the device inputs by k_stage -- then the zone keys of the batch.
        ``tick_args`` = (sel_action, t_const, restart) of a stateful tick: they are staged along, and the tick's zone
        rule applies (a zone under a NEW id is a new zone object: its unblock window is evaluated at this tick,
        OLI:155-237, GLNT:43-77)."""
        self._split_pending = None
        self._grow_for(sc)
        self._stage_zones(sc.zones)
        ts = self._tick
        on_device = isinstance(sc, DeviceScenarioBatch)
        sel_action, t_const, restart = tick_args or (None, None, None)
        zone_rule = tick_args is not None and ts.zone_key_kept
        if not on_device:
            self._fill_staging(sc, vel_est, which, sel_action, t_const)
        if tick_args is not None and self.on_device_start is not None:   # the host staging ends here (timing)
            self.on_device_start()
        if on_device:
            self._launch_stage(sc, vel_est, sel_action, t_const, restart, zone_rule)
        else:
            self._put_zone_key(sc.zone_key, zone_rule)
            if restart is not None:   # one small H2D copy of the mask (the packed upload stays as it is)
                self._state["restart"].copy_(torch.from_numpy(restart.astype(np.int32)).pin_memory(),
                                             non_blocking=True)
        self.dims.k_pred = 0 if sc.n_pred is None else self._k_pred_cap
        ts.staged_on_device = on_device
        ts.zone_key_kept, ts.zone_key_zero = True, sc.zone_key is None

    def _grow_for(self, sc) -> None:
        """buffers for the batch size, object slots and prediction points of a batch (see allocate: growing them
        synchronises)"""
        kp = 0 if sc.pred is None else int(sc.pred.shape[2])
        if self.dims is None or sc.size != self.dims.batch or sc.obj.shape[1] > self.dims.k_obj or kp > self._k_pred_cap:
            self.allocate(sc.size, sc.obj.shape[1], kp)

    def _fill_staging(self, sc: ScenarioBatch, vel_est, which: int, sel_action=None, t_const=None) -> None:
        """a host batch (and the sel_action / t_const of a stateful tick) into pinned staging set ``which``"""
        if self._h2d_ev[which] is not None:   # an asynchronous upload may still read this pinned set
            self._h2d_ev[which].synchronize()
            self._h2d_ev[which] = None
        h = self.h_in_sets[which]
        k = sc.obj.shape[1]
        h["pos"].numpy()[...] = sc.pos
        h["heading"].numpy()[...] = sc.heading
        h["vel"].numpy()[...] = sc.vel
        h["vel_est"].numpy()[...] = sc.vel if vel_est is None else vel_est
        h["n_obj"].numpy()[...] = sc.n_obj
        if k < h["obj"].shape[1]:
            h["obj"].numpy()[:, k:, :] = 0.0
        h["obj"].numpy()[:, :k, :] = sc.obj
        h["zone_sel"].numpy()[...] = -1 if sc.zone_sel is None else sc.zone_sel
        h["n_pred"].numpy()[...] = -1
        if sc.n_pred is not None:     # with pred, so _grow_for provided the obj_pred staging
            h["n_pred"].numpy()[:, :k] = sc.n_pred
            h["obj_pred"].numpy()[...] = 0.0
            h["obj_pred"].numpy()[:, :k, :sc.pred.shape[2], :] = sc.pred
        if sel_action is not None:
            h["sel_action"].numpy()[...] = np.asarray(sel_action, dtype=np.int32).reshape(-1)
            h["t_const"].numpy()[...] = np.broadcast_to(np.asarray(t_const, dtype=np.float64), (self.dims.batch,))

    def _put_zone_key(self, zone_key, zone_rule: bool) -> None:
        """the zone keys of a host batch into _zone_key, where k_stage puts those of a device batch: a copy from pinned
        memory on the stream, none while _zone_key is all zero and the batch has no keys.  zone_rule: first zone_s0[b]
        = -1 where the new key is non-zero and differs from the last one (k_stage's rule), as a masked fill"""
        if zone_key is None:
            if not self._tick.zone_key_zero:
                self._zone_key.zero_()
            return
        key = torch.from_numpy(np.ascontiguousarray(zone_key, dtype=np.int64)).pin_memory()
        key = key.to(self.device, non_blocking=True)
        if zone_rule:
            self._state["zone_s0"].masked_fill_((key != self._zone_key) & (key != 0), -1)
        self._zone_key.copy_(key)

    def _stage_zones(self, zones) -> None:
        """zone bitmasks: bit (node_off[layer] + node) of mask z = that node is blocked by zone z (GLNT:46, 96-99);
        uploaded (pinned, asynchronously) only when the zone list changed"""
        if not zones:
            self.dims.n_zones = 0
            return
        key = tuple((np.asarray(lay).tobytes(), np.asarray(nod).tobytes()) for lay, nod in zones)
        if key != self._tick.zones:
            bits = torch.from_numpy(self._zone_bits(zones)).pin_memory()
            self.t["zone_bits"] = bits.to(self.device, non_blocking=True)
            self._bind("zone_bits")
            self._tick.zones = key
        self.dims.n_zones = len(zones)

    def _zone_bits(self, zones) -> np.ndarray:
        """the int32 [n_zones][n_zone_words] bitmasks of a zone list; ValueError for ids outside the lattice"""
        w = int(self.dims.n_zone_words)
        bits = np.zeros((len(zones), w), dtype=np.uint32)
        for z, (lay, nod) in enumerate(zones):
            if lay.size and (lay.min() < 0 or lay.max() >= self.node_off.size - 1):
                raise ValueError("zone layer id outside the lattice")
            g = self.node_off[lay] + nod
            if lay.size and (np.any(nod < 0) or np.any(g >= self.node_off[lay + 1])):
                raise ValueError("zone node id outside its layer")
            np.bitwise_or.at(bits[z], g >> 5, (np.uint32(1) << (g & 31).astype(np.uint32)))
        return bits.view(np.int32)

    # -- scenario inputs from device tensors (DeviceScenarioBatch -> k_stage) ----------------------------------------------
    def _device_args(self, sc: DeviceScenarioBatch, vel_est=None, sel_action=None, t_const=None, restart=None):
        """checks of a device batch and of the per-scenario arguments of its tick, from shapes, dtypes and devices only
        (no values, no synchronisation): ValueError before anything launches.  Returns vel_est, sel_action, t_const,
        restart as device tensors [B] or None; t_const may also come back as a float (broadcast by k_stage).  Host
        arrays are accepted and uploaded here (a synchronous copy)."""
        sc.check(self.device)
        check_object_count(sc.obj.shape[1], self.max_objects)
        B, dev = sc.size, sc.pos.device

        def arg(name, a, dtypes, np_dt):
            if a is None:
                return None
            if not isinstance(a, torch.Tensor):
                try:
                    a = np.broadcast_to(np.asarray(a, dtype=np_dt), (B,))
                except ValueError:
                    raise ValueError("%s must broadcast to shape [%d]" % (name, B)) from None
                return torch.as_tensor(np.ascontiguousarray(a)).to(dev)
            if a.device != dev or a.dtype not in dtypes or tuple(a.shape) != (B,):
                raise ValueError("%s must be a tensor [%d] of %s on %s, got %s %s on %s" % (
                    name, B, " / ".join(str(d) for d in dtypes), dev, a.dtype, tuple(a.shape), a.device))
            return a
        if t_const is not None and not isinstance(t_const, torch.Tensor) and np.ndim(t_const) == 0:
            t_const = float(t_const)
        else:
            t_const = arg("t_const", t_const, (torch.float64,), np.float64)
        return (arg("vel_est", vel_est, (torch.float64,), np.float64),
                arg("sel_action", sel_action, (torch.int32, torch.int64), np.int32), t_const,
                arg("restart", restart, (torch.bool, torch.uint8, torch.int8, torch.int32, torch.int64), np.int32))

    def _launch_stage(self, sc: DeviceScenarioBatch, vel_est, sel_action, t_const, restart, zone_rule: bool) -> None:
        """k_stage: the inputs of a device batch into the input copy in use, the bytes _fill_staging + upload() write
        (with sel_action also those of a stateful tick), and its zone keys into _zone_key; zone_rule: the zone rule of
        a stateful tick"""
        src = capi.StageSrc()

        def put(name, a):
            if a is not None:
                setattr(src, name, a.data_ptr())
                stride = a.stride()
                if isinstance(getattr(src, name + "_s"), int):
                    setattr(src, name + "_s", stride[0])
                else:
                    getattr(src, name + "_s")[:] = stride[:len(getattr(src, name + "_s"))]
        for name in ("pos", "heading", "vel", "n_obj", "obj", "zone_sel", "zone_key", "pred", "n_pred"):
            put(name, getattr(sc, name))
        put("vel_est", vel_est)
        src.k_src = int(sc.obj.shape[1])
        src.kp_src = 0 if sc.pred is None else int(sc.pred.shape[2])
        src.kp_dst = self._k_pred_cap
        if sel_action is not None:
            put("sel_action", sel_action)
            src.sel_action_bytes = sel_action.element_size()
            if isinstance(t_const, torch.Tensor):
                put("t_const", t_const)
            else:
                src.t_const_value = float(t_const)
        if restart is not None:
            put("restart", restart)
            src.restart_bytes = restart.element_size()
        src.zone_key_rule = int(zone_rule)
        src.zone_key_last = self._zone_key.data_ptr()
        capi.check(self.lib, self.lib.ltpl_stage_inputs_batch(C.byref(self.dims), C.byref(self.buf), C.byref(src),
                                                              self.stream), "ltpl_stage_inputs_batch")

    def upload(self, which: int = 0) -> None:
        if self._tick.staged_on_device:   # k_stage has already written the device inputs
            return
        self.d_in_raw.copy_(self.h_in_raw[which], non_blocking=True)      # one packed H2D copy
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._h2d_ev[which] = ev

    def set_estimates(self, pos_est=None, vel_est=None) -> None:
        """position / velocity estimates of calc_vel_profile (LTPL:344-346) for the staged batch: written into the pinned
        staging set 0 and copied to the device on the current stream.  Device tensors (float64 on the planner's device,
        [B][2] / [B]) are copied on the stream without the host."""
        for name, a in (("pos", pos_est), ("vel_est", vel_est)):
            if isinstance(a, torch.Tensor):
                if a.device != self.t[name].device or a.dtype != torch.float64 or a.numel() != self.t[name].numel():
                    raise ValueError("%s: a float64 tensor of %d values on %s, got %s %s on %s" % (
                        name, self.t[name].numel(), self.t[name].device, a.dtype, tuple(a.shape), a.device))
        self._split_pending = None
        for name, a in (("pos", pos_est), ("vel_est", vel_est)):
            if isinstance(a, torch.Tensor):
                self.t[name].copy_(a.reshape(self.t[name].shape))
        pos_est = None if isinstance(pos_est, torch.Tensor) else pos_est
        vel_est = None if isinstance(vel_est, torch.Tensor) else vel_est
        if pos_est is None and vel_est is None:
            return
        if self._h2d_ev[0] is not None:
            self._h2d_ev[0].synchronize()
            self._h2d_ev[0] = None
        t = self.t
        if pos_est is not None:
            self.h_in["pos"].numpy()[...] = np.asarray(pos_est, dtype=np.float64).reshape(-1, 2)
            t["pos"].copy_(self.h_in["pos"], non_blocking=True)
        if vel_est is not None:
            self.h_in["vel_est"].numpy()[...] = np.asarray(vel_est, dtype=np.float64).reshape(-1)
            t["vel_est"].copy_(self.h_in["vel_est"], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._h2d_ev[0] = ev

    def _download_meta(self, which: int) -> None:
        self.h_meta_raw[which].copy_(self.d_meta_raw, non_blocking=True)  # one packed D2H copy

    def download(self, which: int = 0) -> dict:
        """synchronous-style download on the current stream: per-path arrays + the filled rows of the compact
        trajectory list (the row count is read back first)."""
        out = self.h_out_sets[which]
        stream = torch.cuda.current_stream(self.device)
        self._download_meta(which)
        stream.synchronize()
        n = int(out["queue_cnt"][2])
        if n:
            out["traj"][:n].copy_(self._src["traj"][:n], non_blocking=True)
            stream.synchronize()   # the caller reads pinned host memory: the copy has to be complete
        out["n_rows"] = n
        out["incl_emerg_traj"] = bool(self.params.incl_emerg_traj)
        return out

    def plan_stream(self, batches, vel_est=None, device_hook=None, prefer=None):
        """Pipelined end-to-end planning of a sequence of ScenarioBatch objects (generator of result dicts, in order).

        Per step: host staging (pinned) -> H2D -> k_startpos -> tick kernels -> D2H of the per-path arrays on the compute
        stream; the large D2H of the compact trajectory rows runs on a second stream and overlaps the kernels of the
        next step (CUDA events for the hand-over).  With N_SETS = 3 staging / export buffer sets the host stages step
        i + 1 while the GPU runs step i and the copy engine drains step i - 1, so the GPU never waits for the host.
        Results are views of pinned host memory; a result stays valid until N_SETS - 1 further results were taken.
        With ``prefer`` (see select) every step selects one trajectory per scenario on the device and its result is
        download_selected()'s dict instead: the fixed-size copy of the selected rows is issued on the second stream
        without waiting for the row count."""
        ns = self.N_SETS
        compute = torch.cuda.current_stream(self.device)
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        copy_stream = self._copy_stream
        ev_meta = [torch.cuda.Event() for _ in range(ns)]
        ev_d2h = [None] * ns
        pending = []          # sets submitted, trajectory copy not yet issued
        inflight = []         # sets whose trajectory copy is issued, oldest first

        def issue_copy(k):
            if prefer is not None:   # fixed size: the copy stream waits for the step on the device, not the host
                copy_stream.wait_event(ev_meta[k])
                with torch.cuda.stream(copy_stream):
                    results[k] = self._copy_selected(k)
                    ev = torch.cuda.Event()
                    ev.record(copy_stream)
                ev_d2h[k] = ev
                inflight.append(k)
                return
            ev_meta[k].synchronize()
            out = self.h_out_sets[k]
            n = int(out["queue_cnt"][2])
            with torch.cuda.stream(copy_stream):
                if n:
                    out["traj"][:n].copy_(self.traj_bufs[k][:n], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(copy_stream)
            ev_d2h[k] = ev
            out["n_rows"] = n
            out["incl_emerg_traj"] = bool(self.params.incl_emerg_traj)
            results[k] = out
            inflight.append(k)

        results = [None] * ns   # per set: the dict a step yields
        try:
            for i, sc in enumerate(batches):
                k = i % ns
                if self.dims is not None and sc.size != self.dims.batch and (pending or inflight):
                    raise ValueError("plan_stream: the batch size changed while results are in flight")
                while inflight and (inflight[0] == k or ev_d2h[inflight[0]].query()):
                    # hand out finished results in order; the set about to be reused must have left the device first
                    j = inflight.pop(0)
                    ev_d2h[j].synchronize()
                    yield results[j]
                if isinstance(sc, DeviceScenarioBatch):
                    raise ValueError("plan_stream overlaps the host staging of ScenarioBatch objects; plan a "
                                     "DeviceScenarioBatch with plan_batch or tick()")
                if prefer is not None and i == 0:
                    prefer = self._prefer_tensor(check_prefer(prefer, sc.size, self.device))
                if device_hook is not None and hasattr(device_hook, "before"):
                    device_hook.before(k)   # e.g. wait until a collective that still reads buffer set k has finished
                self.stage_scenarios(sc, vel_est=vel_est, which=k)
                self._tick.export = k
                self._bind("traj")
                self.upload(which=k)
                self.set_startpos()
                self.tick()
                if prefer is not None:
                    self._select(prefer, None, k)
                if device_hook is not None:     # e.g. an all-gather of the device-side action sets (multi-GPU)
                    device_hook(k)
                self._download_meta(k)
                ev_meta[k].record(compute)
                pending.append(k)
                if len(pending) > 1:            # issue the trajectory copy of the previous step; it overlaps this step
                    issue_copy(pending.pop(0))
            while pending:
                issue_copy(pending.pop(0))
            for j in inflight:
                ev_d2h[j].synchronize()
                yield results[j]
        finally:
            if self.dims is not None:   # (a refusal may come before the first batch allocated anything)
                self._tick.export = 0
                self._bind("traj")

    # -- kernels ---------------------------------------------------------------------------------------------------------------
    def _call(self, name):
        self._split_pending = None   # a split replay's velocity half follows only its own paths half
        capi.check(self.lib, getattr(self.lib, name)(self.handle, C.byref(self.params), C.byref(self.dims),
                                                     C.byref(self.buf), self.stream), name)

    # -- the trajectory each scenario takes (ltpl_select_batch, csrc/ltpl_select.cuh) ---------------------------------------
    def select(self, prefer, sel_action=None) -> dict:
        """the reference loop's step after every tick, on the device: per scenario the first action of ``prefer`` that
        the last velocity call returned (main_min_example.py:83-85) -- a slot action whose trajectory was kept, or
        'emergency' when that call had incl_emerg_traj and kept anything (OTH:1027-1034).
        ``prefer``: a list of action names (PREFER_IDS) for the whole batch, a host integer array [B][L] or an integer
        tensor [B][L] on the planner's device (any strides) of action ids (capi.ACT_*; other values are skipped),
        L <= capi.SELECT_MAX.  Enqueues one kernel on the current stream, without a host synchronisation, and returns
        device views the planner owns, valid until the next select(): ``sel_action`` [B] int32 (capi.ACT_NONE where
        nothing in the list was returned), ``sel_info`` [B][4] int32 (action, row in device_results()["traj"] or -1,
        rows, trajectory id) and ``sel_traj`` [B][n_export][7] float32 (a copy of the selected row, zeros without a
        selection).  ``sel_action``: an int32 tensor [B] on the device (any stride) that receives the actions instead.
        The next stateful tick takes these actions with sel_action="selected".  Bad arguments raise ValueError before
        anything is launched."""
        self._check_select("select")
        prefer = check_prefer(prefer, self.dims.batch, self.device)
        if sel_action is not None and (not isinstance(sel_action, torch.Tensor) or sel_action.device != self.device
                                       or sel_action.dtype != torch.int32 or tuple(sel_action.shape) != (self.dims.batch,)):
            raise ValueError("select: sel_action must be an int32 tensor [%d] on %s" % (self.dims.batch, self.device))
        return self._select(self._prefer_tensor(prefer), sel_action, 0)

    def _check_select(self, what: str) -> None:
        if not self._tick.ticked:
            raise ValueError("%s: no velocity call ran on this planner's buffers" % what)
        if all(tb.data_ptr() != self.buf.traj for tb in self.traj_bufs):
            raise ValueError("%s: buffers.traj points at peer memory (a PeerGather is attached)" % what)

    def _sel_buffers(self, which: int) -> dict:
        """the device selection buffers of set ``which``, created on first use for the allocated batch: ``info`` [B][4]
        int32, ``traj`` [B][n_export][7] float32"""
        if self._sel[which] is None:
            B, NE = self.dims.batch, self.dims.n_export
            self._sel[which] = dict(info=torch.full((B, 4), -1, dtype=torch.int32, device=self.device),
                                    traj=torch.zeros((B, NE, 7), dtype=torch.float32, device=self.device))
        return self._sel[which]

    def _prefer_tensor(self, prefer) -> torch.Tensor:
        """a preference checked by check_prefer as a device tensor: host ids are copied from pinned memory on the current
        stream, without a host synchronisation"""
        if isinstance(prefer, torch.Tensor):
            return prefer
        return torch.from_numpy(prefer).pin_memory().to(self.device, non_blocking=True)

    def _select(self, prefer: torch.Tensor, sel_action, which: int) -> dict:
        """k_select into selection set ``which`` (sel_action None: column 0 of its info)"""
        sel = self._sel_buffers(which)
        out = sel["info"][:, 0] if sel_action is None else sel_action
        s = capi.Select()
        s.prefer_len = int(prefer.shape[1])
        s.prefer_bytes = prefer.element_size()
        if s.prefer_len:
            s.prefer = prefer.data_ptr()
            s.prefer_s[0] = 0 if prefer.shape[0] == 1 else prefer.stride(0)   # one list for the batch
            s.prefer_s[1] = prefer.stride(1)
        s.sel_action, s.sel_action_s = out.data_ptr(), out.stride(0)
        s.sel_info, s.sel_traj = sel["info"].data_ptr(), sel["traj"].data_ptr()
        prm = capi.Params.from_buffer_copy(self.params)
        prm.incl_emerg_traj = int(self._tick.emerg)
        capi.check(self.lib, self.lib.ltpl_select_batch(C.byref(prm), C.byref(self.dims), C.byref(self.buf), C.byref(s),
                                                        self.stream), "ltpl_select_batch")
        self._tick.selected = True
        return dict(sel_action=out, sel_info=sel["info"], sel_traj=sel["traj"])

    def download_selected(self, which: int = 0) -> dict:
        """the last tick's small per-path arrays (as download()) and the selection of the last select(): ``sel_info``
        [B][4], ``sel_action`` (its column 0) and ``sel_traj`` [B][n_export][7], copied into pinned host memory on the
        current stream, both copies back to back, then one synchronisation.  The rows have a fixed size (scenario b in
        row b), so nothing is read back first.  Views of pinned buffers, valid until the next download_selected()."""
        if self._sel is None or self._sel[0] is None:
            raise ValueError("download_selected: no select() ran on this planner's buffers")
        self._download_meta(which)
        out = self._copy_selected(which, 0)
        torch.cuda.current_stream(self.device).synchronize()
        return out

    def _copy_selected(self, which: int, sel_set: int = None) -> dict:
        """the D2H copy of selection set ``sel_set`` (default: ``which``) into its pinned buffers on the current stream,
        and the result dict with the per-path arrays of host set ``which`` (_download_meta)"""
        sel_set = which if sel_set is None else sel_set
        if self._sel_host[sel_set] is None:
            self._sel_host[sel_set] = {k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True)
                                       for k, v in self._sel[sel_set].items()}
        h = self._sel_host[sel_set]
        for k in ("info", "traj"):
            h[k].copy_(self._sel[sel_set][k], non_blocking=True)
        out = {n: self.h_out_sets[which][n] for n in self._meta_names}
        out.update(sel_info=h["info"], sel_action=h["info"][:, 0], sel_traj=h["traj"],
                   incl_emerg_traj=bool(self._tick.emerg))
        return out

    def _call_vel(self, name):
        """a call that includes calc_vel_profile: its trajectories get the next ids (+10 per call, OTH:669).  Once a
        TickGraph was captured on this planner the ids come from the device counter buffers.traj_base (k_traj_base),
        so that eager calls and replays number alike."""
        self._tick_count += 1
        self.params.traj_base_id = 10 * self._tick_count if self._traj_base is None else 0
        self._call(name)
        self._tick.gg_planes_used = self._src["gg"] is not None
        self._tick.ticked = True
        self._tick.emerg, self._tick.selected = bool(self.params.incl_emerg_traj), False

    def set_startpos(self) -> None:
        self._call("ltpl_set_startpos_batch")

    def calc_paths(self) -> None:
        self._call("ltpl_calc_paths_batch")

    def calc_vel_profile(self) -> None:
        self._call_vel("ltpl_calc_vel_profile_batch")

    def tick(self) -> None:
        """calc_paths + calc_vel_profile back to back."""
        self._call_vel("ltpl_tick_batch")

    # -- stateful tick (DESIGN.md section 11, csrc/ltpl_state.cuh) ----------------------------------------------
    def _alloc_state(self) -> None:
        dev, B = self.device, self.dims.batch
        f64, i32 = torch.float64, torch.int32
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)   # noqa: E731
        t = self.t
        t["em_vx"] = z((B, self.dims.n_export), f64)   # f64 velocity of the emergency trajectory (executed 'emergency')
        t["em_info"].fill_(-1)
        prev_raw, prev_small = self._packed(self._carry_spec, lambda n: torch.zeros(n, dtype=torch.uint8, device=dev))
        prev_small["em_info"].fill_(-1)
        st = dict(other={k: torch.zeros_like(t[k]) for k in SWAPPED}, prev_raw=prev_raw, prev_small=prev_small,
                  st_info=z((B, 8), i32), vel_plan=z((B,), f64), course=z((B, self.dims.n_export), f64),
                  obj_dist=z((B,), f64))
        st["zone_s0"] = torch.full((B,), -1, dtype=i32, device=dev)
        st["restart"] = z((B,), i32)   # buffers.restart of the ticks with a restart mask
        self._state = st

    def _restart_mask(self, restart):
        """the restart mask of a stateful tick as a bool array [B], or None when no scenario restarts"""
        if restart is None:
            return None
        mask = np.asarray(restart)
        if mask.shape != (self.dims.batch,):
            raise ValueError("restart must be a boolean array of shape [%d], got shape %s" % (self.dims.batch,
                                                                                          mask.shape))
        mask = mask.astype(bool)
        return mask if mask.any() else None

    def _stage_next(self, sc, sel_action, t_const, vel_est, restart=None) -> None:
        """host side of a stateful tick: pointer swaps, ONE device copy (the small per-path arrays of the last tick),
        then the staging of stage_scenarios into the other input copy with sel_action / t_const and the restart mask.
        A ScenarioBatch: host memcpy into the pinned staging set and ONE packed H2D copy, with restarts one more small
        H2D copy (the mask).  A DeviceScenarioBatch: one k_stage launch."""
        if sc.size != self.dims.batch:
            raise ValueError("stateful tick: the batch size must not change within a session (re-anchor with "
                             "set_startpos on a new batch, or restart single scenarios with `restart`)")
        # before the swaps below: refused inputs change nothing
        if sel_action is None or t_const is None:
            raise ValueError("stateful tick: sel_action and t_const are required")
        selected = self._selected(sel_action) if isinstance(sel_action, str) else None
        if selected is not None:   # a device batch stages the selection through k_stage, a host batch copies it below
            sel_action = selected if isinstance(sc, DeviceScenarioBatch) else 0
        if isinstance(sc, DeviceScenarioBatch):
            vel_est, sel_action, t_const, restart = self._device_args(sc, vel_est, sel_action, t_const, restart)
        else:
            check_object_count(sc.obj.shape[1], self.max_objects)
            restart = self._restart_mask(restart)
        if self._state is None:
            self._alloc_state()
        st, t, ts = self._state, self.t, self._tick
        n_carry = st["prev_raw"].numel()
        st["prev_raw"].copy_(self.d_meta_raw[:n_carry])       # the last tick's small per-path arrays
        for k in SWAPPED:                                     # this tick writes the other set, the last one is memory
            t[k], st["other"][k] = st["other"][k], t[k]
        # location dependent local_gg of the last tick = backup for a brake on the old plan (__backup_path_gg, OTH:970)
        if ts.gg_planes_used:
            t["gg"], st["other"]["gg"] = self._gg_planes(st["other"]), t["gg"]
        ts.prev_gg = ts.gg_planes_used
        ts.gg = False   # this tick's local_gg arrives with its calc_vel_profile, or from the friction map
        ts.restart = restart is not None
        # pos_est of the previous calc_vel_profile (OTH:537) = `pos` of the input copy the last tick used; this tick
        # stages into the other copy (a batch with more objects than before re-creates only the input buffers)
        ts.pos_last = t["pos"]
        self._grow_for(sc)
        self._use_inputs(1 - ts.in_cur)
        self._bind()
        self._stage(sc, vel_est, 0, (sel_action, t_const, restart))
        self.upload()   # a ScenarioBatch: ONE packed H2D copy (k_stage has written a DeviceScenarioBatch)
        if selected is not None and not isinstance(sc, DeviceScenarioBatch):
            t["sel_action"].copy_(selected)

    def _selected(self, name: str) -> torch.Tensor:
        """sel_action="selected": the actions of the last select() (column 0 of its sel_info, a device view), which must
        have run after the last velocity call"""
        if name != "selected":
            raise ValueError('sel_action: action ids or "selected", got %r' % name)
        if not self._tick.selected:
            raise ValueError('sel_action="selected": no select() ran after the last velocity call')
        return self._sel[0]["info"][:, 0]

    def next_calc_paths(self, sc: ScenarioBatch, sel_action, t_const, vel_est=None, restart=None) -> None:
        """calc_paths of a stateful tick (OTH:289-516 with the iterative memory): ``sc`` carries the object
        lists (its poses are only used by ``next_calc_vel_profile``), ``sel_action`` = action id (capi.ACT_*) every
        scenario executed since the last tick, ``t_const`` = min(average calculation time * calc_time_safety, 0.5) per
        scenario (OTH:353-375; the caller keeps the moving average).  The previous tick (tick() / calc_paths() +
        calc_vel_profile() after set_startpos(), or a stateful tick) must have run on this planner.
        ``sel_action="selected"`` takes the actions of the last select() on the device, without a copy through the host.
        ``restart``: boolean array [B]; a true entry restarts that scenario inside this tick, as set_startpos(sc.pos[b],
        sc.heading[b], sc.vel[b]) on a live planner followed by a first tick (its memory is dropped, its sel_action and
        t_const are ignored); the other scenarios keep theirs.  A wrong shape raises ValueError and changes nothing.
        With a DeviceScenarioBatch, ``sel_action`` (int32 / int64), ``t_const`` (float64 or a scalar), ``vel_est``
        (float64) and ``restart`` (bool or integer) may be device tensors [B]; the tick then runs without a host
        synchronisation (a mask tensor is passed to the library as it is, whether or not an entry is set)."""
        self._stage_next(sc, sel_action, t_const, vel_est, restart)
        self._call("ltpl_next_calc_paths_batch")

    def next_calc_vel_profile(self, pos_est=None, vel_est=None) -> None:
        """calc_vel_profile of a stateful tick (OTH:518-601 + 603-1040): position / velocity estimates per
        scenario (None: the poses / velocities staged by ``next_calc_paths``)."""
        if pos_est is not None or vel_est is not None:
            self.set_estimates(pos_est, vel_est)
        self._call_vel("ltpl_next_calc_vel_profile_batch")

    def next_tick(self, sc: ScenarioBatch, sel_action, t_const, vel_est=None, restart=None) -> None:
        """One stateful tick for the whole batch in one library call: ``sc.pos`` = position estimates (and the new start
        poses of the scenarios ``restart`` marks, see next_calc_paths)."""
        self._stage_next(sc, sel_action, t_const, vel_est, restart)   # vel_est travels in the packed upload
        self._call_vel("ltpl_next_tick_batch")

    # -- ticks replayed from CUDA graphs (tick_graph.py, DESIGN.md section 11) -------------------------------------------
    def capture_tick(self, sc, vel_est=None, restart=None, prefer=None):
        """capture a first tick -- k_stage + set_startpos + tick of ``sc`` (a DeviceScenarioBatch) -- into a CUDA graph
        and return a TickGraph: write each tick's inputs into ``graph.inputs`` (TickInputs.copy_) and call
        ``graph.replay()``, which enqueues the tick with no host work.  The arguments are those of the eager device
        calls.  Everything that could allocate or copy from the host happens here, before the capture (a batch of
        another size starts a new session, as in stage_scenarios); the zone list ``sc.zones`` is fixed for the graph's
        lifetime.  Nothing is launched and the planner's state is left as it was.
        ``prefer`` (see select): the graph ends with select(prefer) from a device copy it owns (``graph.prefer``, which
        may be rewritten in place), so a replay leaves the selection for a stateful tick with sel_action="selected"."""
        from .tick_graph import capture
        if restart is not None:
            raise ValueError("capture_tick: a first tick takes no restart mask (capture_next_tick does)")
        return capture(self, False, sc, vel_est=vel_est, prefer=prefer)

    def capture_next_tick(self, sc, sel_action, t_const, vel_est=None, restart=None, prefer=None):
        """capture a stateful tick (next_tick with the same arguments) into CUDA graphs, one per ping-pong parity of
        the planner's buffers, and return a TickGraph (see capture_tick).  A replay runs the graph of the planner's
        current parity and then does the host side of the tick (pointer swaps, tick count), so eager ticks and replays
        may be interleaved freely.  Needs a previous tick in this session and the session's batch size.
        ``sel_action="selected"`` stages the last selection on the device (see next_calc_paths); with ``prefer`` every
        per-parity graph ends with select(prefer): replays then run a closed loop with no host work for the pick."""
        from .tick_graph import capture
        return capture(self, True, sc, vel_est=vel_est, sel_action=sel_action, t_const=t_const, restart=restart,
                       prefer=prefer)

    def capture_split_tick(self, sc, vel_est=None, pos_est=None, local_gg=None, prefer=None):
        """capture a first tick as two halves and return a SplitTickGraph: ``replay_paths()`` = k_stage + set_startpos +
        calc_paths of ``sc`` (a DeviceScenarioBatch), ``replay_vel_profile()`` = calc_vel_profile with the estimates
        ``pos_est`` [B][2] / ``vel_est`` [B] (set_estimates) and, with ``local_gg=(ax, ay)``, the friction planes
        [NSLOT][B][P] (set_local_gg_planes), all float64 device tensors.  Between the two replays the caller may read
        device_results()["path"] and write the velocity half's inputs (``graph.vel_inputs``) on the device: the
        reference's loop (calc_paths, then local_gg along the new paths, then calc_vel_profile) with no host work.
        Everything else as capture_tick; ``local_gg`` excludes a friction map (set_gg_map).  With ``prefer`` the velocity
        half ends with select(prefer), as in capture_tick."""
        from .tick_graph import capture_split
        return capture_split(self, False, sc, vel_est=vel_est, pos_est=pos_est, local_gg=local_gg, prefer=prefer)

    def capture_next_split_tick(self, sc, sel_action, t_const, vel_est=None, restart=None, pos_est=None,
                                local_gg=None, prefer=None):
        """capture a stateful tick as its two halves, next_calc_paths(sc, sel_action, t_const, restart=restart) and
        next_calc_vel_profile(pos_est, vel_est) with the friction planes ``local_gg`` set between them, and return a
        SplitTickGraph (see capture_split_tick and capture_next_tick)"""
        from .tick_graph import capture_split
        return capture_split(self, True, sc, vel_est=vel_est, pos_est=pos_est, local_gg=local_gg,
                             sel_action=sel_action, t_const=t_const, restart=restart, prefer=prefer)

    def _prepare_capture(self, inputs, stateful: bool, planes: bool = False, select: bool = False) -> None:
        """everything a tick of these inputs could allocate, grow or copy from the host, done before a capture: the
        buffers for the batch, the memory buffers a stateful tick creates on first use, the zone bitmasks, the id
        counter and the kernels' attributes (ltpl_prepare_batch).  planes: the tick's velocity half sets gg planes;
        select: the tick ends with select() (its buffers)"""
        sc = inputs.sc
        pos = self.t["pos"] if stateful else None
        self._grow_for(sc)
        if pos is not None and self.t["pos"] is not pos:
            # more object slots or prediction points: the input copies were re-created (the current one is copy 0).  A
            # stateful tick reads the last tick's positions as pos_last from the current copy; the eager tick keeps the
            # old copy for it instead, so the current copy takes its values here
            self.t["pos"].copy_(pos)
        if planes:
            self._gg_planes(self.t)
        if select:
            self._sel_buffers(0)
        if stateful:
            if self._state is None:
                self._alloc_state()
            if "gg" in self.t:   # what the first gg swap would create
                self._gg_planes(self._state["other"])
        self._stage_zones(sc.zones)
        if self._traj_base is None:   # the ids an all-eager session would give next
            self._traj_base = torch.full((1,), 10 * self._tick_count, dtype=torch.int32, device=self.device)
        self.params.traj_base_id = 0
        ts = self._tick
        self._tick = replace(ts, gg=ts.gg or planes)   # bound as the velocity half will bind them
        self._bind()
        rc = self.lib.ltpl_prepare_batch(self.handle, C.byref(self.params), C.byref(self.dims), C.byref(self.buf))
        self._tick = ts
        self._bind("gg")
        capi.check(self.lib, rc, "ltpl_prepare_batch")

    def _host_state(self) -> dict:
        """what a tick changes on the host: dims, the buffer dicts (by reference) and the TickState record, from which
        _bind derives the pointer fields"""
        return dict(dims=capi.Dims.from_buffer_copy(self.dims), t=dict(self.t),
                    other=None if self._state is None else dict(self._state["other"]), tick=replace(self._tick))

    def _set_host_state(self, hs: dict) -> None:
        C.memmove(C.addressof(self.dims), C.addressof(hs["dims"]), C.sizeof(capi.Dims))
        self.t.clear()
        self.t.update(hs["t"])
        if hs["other"] is not None:
            self._state["other"].clear()
            self._state["other"].update(hs["other"])
        self._tick = replace(hs["tick"])   # a copy: the record in hs serves every replay of its graph
        self._bind()

    def _tick_key(self, stateful: bool) -> tuple:
        """the buffers the next tick would use: the input copy, the ping-pong planes, the gg planes and, for a stateful
        tick, whether the last velocity call ran with planes (it decides the gg swap and prev_gg)"""
        key = (self._tick.in_cur,) + tuple(self.t[k].data_ptr() if k in self.t else 0 for k in SWAPPED + ("gg",))
        return key + (self._tick.gg_planes_used,) if stateful else key

    def launch_count(self) -> int:
        return int(self.lib.ltpl_launch_count())

    DEVICE_RESULTS = ("action_id", "traj_len", "traj_row", "traj_id", "status", "sc_flags", "path_len", "queue_cnt")

    def device_results(self) -> dict:
        """the last tick's results as torch views of the device buffers, without a copy or a synchronisation:
        ``action_id``, ``traj_len``, ``traj_row``, ``traj_id``, ``status``, ``path_len`` [NSLOT][B], ``sc_flags`` [B],
        ``queue_cnt`` (entry 2 = filled rows of ``traj``) and ``traj``, the compact export rows [(NSLOT + 1) * B]
        [n_export][7] float32 (path (s, b) in row traj_row[s, b]).  For a caller that computes the next tick's
        sel_action / pos_est on the device.  Work queued on the planner's stream after the tick sees them complete.
        The views are valid until the next tick: it rewrites these buffers, and a stateful tick swaps planes by pointer,
        so read or clone what is needed before staging the next tick.
        ``path`` [5][NSLOT * B][p_max] float64 holds the planned paths (x, y, psi, kappa, el; row q = slot * B + b,
        points [0, path_len[slot, b])), valid right after calc_paths / next_calc_paths: a friction model on the device
        evaluates them for set_local_gg_planes.  A stateful tick swaps this plane by pointer, so the view belongs to
        the tick that produced it; take device_results() anew after every calc_paths."""
        out = {n: self.t[n] for n in self.DEVICE_RESULTS}
        out["traj"] = self._src["traj"]
        out["path"] = self.t["path"]
        return out

    # -- result access (device -> host, test / facade use) ----------------------------------------------------------------------
    def fetch(self, *names) -> dict:
        torch.cuda.synchronize(self.device)
        return {n: self.t[n].cpu().numpy() for n in names}

    def records(self, indices=None) -> list:
        """per-scenario result dicts in the reference's vocabulary ({action: [ndarray]}), for parity tests and the
        single-scenario facade.  Copies every result buffer to the host."""
        f = self.fetch("sc_flags", "start_node", "action_id", "status", "n_nodes", "nodes", "node_idx", "closest_obj",
                       "path_len", "path", "coeff", "s_vx_ax", "traj", "traj_row", "traj_len", "traj_id", "const_seg",
                       "const_len", "em_info")
        trim = self.t["trim"].cpu().numpy() if "trim" in self.t else None   # stateful ticks: trajectories start at the cut
        B = self.dims.batch
        out = []
        for b in (range(B) if indices is None else indices):
            rec = dict(flags=int(f["sc_flags"][b]))
            rec["out_of_track"] = bool(rec["flags"] & (capi.SC_OUT_OF_TRACK | capi.SC_HEADING_MISMATCH))
            if rec["flags"] & (capi.SC_CAPACITY | capi.SC_BRAKE_PREFIX):
                rec["error"] = rec["flags"]
            if rec["out_of_track"]:
                out.append(rec)
                continue
            rec["start_node"] = f["start_node"][b].tolist()
            co = int(f["closest_obj"][b])
            rec["closest_obj_index"] = None if co < 0 else co
            n0 = int(f["const_len"][b])
            rec["const_path_seg"] = f["const_seg"][:, b, :n0].T.copy()
            for key in ("paths", "nodes", "node_idx", "coeff", "red_len", "tie", "traj_full", "traj", "ids", "status"):
                rec[key] = {}
            for s in range(NSLOT):
                a = int(f["action_id"][s, b])
                if a == capi.ACT_NONE:
                    continue
                name = capi.ACTION_NAMES[a]
                q = s * B + b
                st = int(f["status"][s, b])
                n = int(f["path_len"][s, b])
                nn = int(f["n_nodes"][s, b])
                rec["status"][name] = st
                rec["paths"][name] = [f["path"][:, q, :n].T.copy()]
                nodes = f["nodes"][s, b, :nn].tolist()
                rec["nodes"][name] = [[[None, None] if p[0] < 0 else p for p in nodes]]
                rec["node_idx"][name] = [f["node_idx"][s, b, :nn].copy()]
                rec["coeff"][name] = [f["coeff"][q, :max(nn - 1, 1)].copy()]
                rec["red_len"][name] = [bool(st & capi.ST_REDUCED_HORIZON)]
                rec["tie"][name] = bool(st & capi.ST_TIE_AMBIGUOUS)
                if st & capi.ST_TRAJ_VALID:
                    cut = 0 if trim is None else int(trim[q, 2])
                    m = n - cut
                    full = np.column_stack((f["s_vx_ax"][0, q, :m], f["path"][0:4, q, cut:n].T, f["s_vx_ax"][1, q, :m],
                                            f["s_vx_ax"][2, q, :m]))
                    rec["traj_full"][name] = [full]
                    tl = int(f["traj_len"][s, b])
                    rec["traj"][name] = [f["traj"][int(f["traj_row"][s, b]), :tl].astype(np.float64)]
                    rec["ids"][name] = int(f["traj_id"][s, b])
            if self.params.incl_emerg_traj and rec["traj"] and int(f["em_info"][b, 0]) >= 0:   # OTH:1027-1034
                row, n_em, em_id = (int(v) for v in f["em_info"][b])
                rec["traj"]["emergency"] = [f["traj"][row, :n_em].astype(np.float64)]
                rec["ids"]["emergency"] = em_id
            out.append(rec)
        return out
