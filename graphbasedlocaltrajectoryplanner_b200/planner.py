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

import numpy as np
import torch

from . import capi
from .lattice import Lattice
from .lattice_blob import pack_lattice
from .scenarios import ScenarioBatch

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


DEFAULT_ONLINE = dict(max_heading_offset=0.8, nmbr_export_points=115, v_max_offset=0.1, max_solutions=1,
                      filt_window_width=1, w_last_edges=[0.0, 0.5, 0.8], controller_type="PD",
                      control_params={"c_p": 1.25, "k_d": 0.025, "k_p": 0.2}, delaycomp=0.1)


class BatchPlanner(object):
    N_SETS = 3   # host staging / export buffer sets of the pipelined path (plan_stream)

    def __init__(self, lattice: Lattice = None, online: dict = None, device=None, veh_param_dyn_model_exp: float = 1.0,
                 veh_param_dragcoeff: float = 0.85, veh_param_mass: float = 1000.0, packed: tuple = None,
                 blob_tensor: torch.Tensor = None, stateful: bool = False):
        """``packed`` = (LatticeHeader, capacities) + ``blob_tensor`` (device uint8) when the blob arrived through a
        collective instead of being uploaded from ``lattice`` (parallel.broadcast_lattice)."""
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
        self.buf = None
        self.t = {}
        self.params = capi.Params()
        self._tick_count = 0
        self.on_device_start = None   # optional callable, called where a stateful tick's host staging ends (timing)
        self.set_vel_params()

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.ltpl_lattice_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def set_subbatches(self, n: int) -> None:
        """number of scenario windows a tick is split into inside the library (1 .. capi.MAX_SUB; default 4 for windows
        of >= 512 scenarios): window s runs on an internal stream, so kernels of different stages overlap.  The results
        do not depend on it (only the unspecified order of the compact export rows)."""
        capi.check(self.lib, self.lib.ltpl_set_subbatches(self.handle, int(n)), "ltpl_set_subbatches")

    # -- parameters ------------------------------------------------------------------------------------------------------
    def set_vel_params(self, vel_max: float = 100.0, gg_scale: float = 1.0, local_gg=(5.0, 5.0),
                       ax_max_machines=np.atleast_2d([100.0, 5.0]), safety_d: float = 30.0,
                       incl_emerg_traj: bool = False) -> None:
        """per-call arguments of Graph_LTPL.calc_vel_profile (LTPL:344-352)."""
        if local_gg is None:        # location dependent friction: the planes of set_local_gg_planes() are used
            local_gg = (1.0, 1.0)
        if type(local_gg) is not tuple or len(local_gg) != 2:   # OTH:651-653 (dict form: Graph_LTPL / set_local_gg_planes)
            raise ValueError("Provided local_gg does not satisfy requested format! Read parameter documentation.")
        axm = np.atleast_2d(np.asarray(ax_max_machines, dtype=np.float64))
        if axm.shape[1] != 2:
            raise RuntimeError("ax_max_machines must consist of the two columns [vx, ax_max_machines]!")
        if axm.shape[0] > capi.MAX_AXM:
            raise ValueError("ax_max_machines has more than %d rows" % capi.MAX_AXM)
        if axm[-1, 0] < vel_max:                               # tph.calc_vel_profile input check
            raise RuntimeError("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!")
        p = self.params
        o = self.online
        p.max_heading_offset = o["max_heading_offset"]
        p.v_max_offset = o["v_max_offset"]
        cp = o["control_params"]
        p.follow_c_p, p.follow_k_d, p.follow_k_p = cp["c_p"], cp["k_d"], cp["k_p"]
        p.follow_tan_w = cp.get("tan_w", 1.0)
        if o["controller_type"] not in ("PD", "PDtan"):
            raise ValueError('Unsupported control type "' + o["controller_type"] + '"!')
        p.follow_control_type = 0 if o["controller_type"] == "PD" else 1
        p.nmbr_export_points = int(o["nmbr_export_points"])
        p.dyn_model_exp, p.drag_coeff, p.m_veh = self.veh["dyn_model_exp"], self.veh["drag_coeff"], self.veh["m_veh"]
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

    _IN_NAMES = ("pos", "heading", "vel", "vel_est", "n_obj", "obj", "zone_sel", "n_pred", "sel_action", "t_const",
                 "obj_pred")

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
        self._in_cur = which
        self.d_in_raw, views = self.d_in[which]
        self.t.update(views)
        for name in self._IN_NAMES:
            if name in views and name not in ("sel_action", "t_const"):
                setattr(self.buf, name, views[name].data_ptr())

    def allocate(self, batch: int, k_obj: int = 3, k_pred: int = 0) -> None:
        k_obj = check_object_count(k_obj, self.max_objects)
        if self.dims is not None and self.dims.batch == batch:
            if self.dims.k_obj >= k_obj and self._k_pred_cap >= k_pred:
                return
            # more object slots / prediction points than before: only the input buffers grow (see _alloc_inputs)
            torch.cuda.current_stream(self.device).synchronize()
            self._alloc_inputs(batch, max(k_obj, self.dims.k_obj), max(int(k_pred), self._k_pred_cap))
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
        buf = capi.Buffers()
        t["zone_bits"] = torch.zeros((1, 1), dtype=torch.int32, device=dev)   # replaced by _upload_zones()
        d.k_pred = 0
        d.n_zones, d.n_zone_words = 0, (self.lattice_nodes + 31) // 32
        for name in capi.BUFFER_FIELDS:
            if name not in capi.STATE_FIELDS and name in t:   # `trim` is a state field: NULL unless the planner is stateful
                setattr(buf, name, t[name].data_ptr())
        self.t, self.buf, self.dims = t, buf, d
        self._alloc_inputs(B, k_obj, k_pred)
        self._state = None   # buffers of the stateful tick, allocated by next_tick()
        # further compact export buffers: the pipelined stream planner lets the D2H of step i overlap step i + 1
        self.traj_bufs = [t["traj"]] + [z(((NSLOT + 1) * B, NE, 7), f32) for _ in range(self.N_SETS - 1)]
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

    def set_local_gg_planes(self, ax=None, ay=None) -> None:
        """location dependent friction (calc_vel_profile(local_gg={action: [ndarray(P, 2)]}), OTH:649-666) for the batch:
        ``ax``, ``ay`` [NSLOT][B][P] (P <= p_max) = longitudinal / lateral limit at every point of every path (slot 0:
        straight | follow, 1: left, 2: right), aligned with the paths of the last calc_paths; None: back to the constant
        tuple of set_vel_params().  The values are taken without gg_scale (VPFB:213-214 applies it)."""
        if ax is None:
            self.buf.gg = None
            self._gg_active = False
            return
        ax = np.asarray(ax, dtype=np.float64)
        ay = np.asarray(ay, dtype=np.float64)
        B, P = self.dims.batch, self.dims.p_max
        if ax.shape != ay.shape or ax.ndim != 3 or ax.shape[:2] != (NSLOT, B) or ax.shape[2] > P:
            raise ValueError("local_gg planes must have the shape [NSLOT][B][P <= p_max]")
        if "gg" not in self.t:
            self.t["gg"] = torch.ones((2, NSLOT * B, P), dtype=torch.float64, device=self.device)
        host = np.ones((2, NSLOT * B, P))
        host[0, :, :ax.shape[2]] = ax.reshape(NSLOT * B, -1)
        host[1, :, :ay.shape[2]] = ay.reshape(NSLOT * B, -1)
        self.t["gg"].copy_(torch.from_numpy(host))
        self.buf.gg = self.t["gg"].data_ptr()
        self._gg_active = True

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

    def stage_scenarios(self, sc: ScenarioBatch, vel_est=None, which: int = 0) -> None:
        """copy a scenario batch into the pinned staging buffers (host memcpy)."""
        kp = 0 if sc.pred is None else int(sc.pred.shape[2])
        if self.dims is None or sc.size != self.dims.batch or sc.obj.shape[1] > self.dims.k_obj or kp > self._k_pred_cap:
            self.allocate(sc.size, sc.obj.shape[1], kp)
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
        self.dims.k_pred = 0
        if sc.n_pred is not None:     # kp >= 1 here, so allocate() above provided the obj_pred staging
            h["n_pred"].numpy()[:, :k] = sc.n_pred
            h["obj_pred"].numpy()[...] = 0.0
            h["obj_pred"].numpy()[:, :k, :kp, :] = sc.pred
            self.dims.k_pred = self._k_pred_cap
        self._upload_zones(sc.zones)
        self._zone_key = sc.zone_key.copy() if sc.zone_key is not None else np.zeros(sc.size, dtype=np.int64)

    def _upload_zones(self, zones) -> None:
        """zone bitmasks: bit (node_off[layer] + node) of mask z = that node is blocked by zone z (GLNT:46, 96-99)."""
        if not zones:
            self.dims.n_zones = 0
            return
        w = int(self.dims.n_zone_words)
        bits = np.zeros((len(zones), w), dtype=np.uint32)
        for z, (lay, nod) in enumerate(zones):
            if lay.size and (lay.min() < 0 or lay.max() >= self.node_off.size - 1):
                raise ValueError("zone layer id outside the lattice")
            g = self.node_off[lay] + nod
            if lay.size and (np.any(nod < 0) or np.any(g >= self.node_off[lay + 1])):
                raise ValueError("zone node id outside its layer")
            np.bitwise_or.at(bits[z], g >> 5, (np.uint32(1) << (g & 31).astype(np.uint32)))
        self.t["zone_bits"] = torch.from_numpy(bits.view(np.int32)).to(self.device)
        self.buf.zone_bits = self.t["zone_bits"].data_ptr()
        self.dims.n_zones = len(zones)

    def upload(self, which: int = 0) -> None:
        self.d_in_raw.copy_(self.h_in_raw[which], non_blocking=True)      # one packed H2D copy
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._h2d_ev[which] = ev

    def set_estimates(self, pos_est=None, vel_est=None) -> None:
        """position / velocity estimates of calc_vel_profile (LTPL:344-346) for the staged batch: written into the pinned
        staging set 0 and copied to the device on the current stream."""
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
            src = next(tb for tb in self.traj_bufs if tb.data_ptr() == self.buf.traj)   # the set the kernels wrote
            out["traj"][:n].copy_(src[:n], non_blocking=True)
            stream.synchronize()   # the caller reads pinned host memory: the copy has to be complete
        out["n_rows"] = n
        out["incl_emerg_traj"] = bool(self.params.incl_emerg_traj)
        return out

    def plan_stream(self, batches, vel_est=None, device_hook=None):
        """Pipelined end-to-end planning of a sequence of ScenarioBatch objects (generator of result dicts, in order).

        Per step: host staging (pinned) -> H2D -> k_startpos -> tick kernels -> D2H of the per-path arrays on the compute
        stream; the large D2H of the compact trajectory rows runs on a second stream and overlaps the kernels of the
        next step (CUDA events for the hand-over).  With N_SETS = 3 staging / export buffer sets the host stages step
        i + 1 while the GPU runs step i and the copy engine drains step i - 1, so the GPU never waits for the host.
        Results are views of pinned host memory; a result stays valid until N_SETS - 1 further results were taken."""
        dev = self.device
        ns = self.N_SETS
        compute = torch.cuda.current_stream(dev)
        copy_stream = getattr(self, "_copy_stream", None)
        if copy_stream is None:
            copy_stream = self._copy_stream = torch.cuda.Stream(device=dev)
        ev_meta = [torch.cuda.Event() for _ in range(ns)]
        ev_d2h = [None] * ns
        pending = []          # sets submitted, trajectory copy not yet issued
        inflight = []         # sets whose trajectory copy is issued, oldest first

        def issue_copy(k):
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
            inflight.append(k)

        try:
            yield from self._plan_stream_loop(batches, vel_est, device_hook, ns, compute, ev_meta, ev_d2h, pending,
                                              inflight, issue_copy)
        finally:
            self.buf.traj = self.traj_bufs[0].data_ptr()

    def _plan_stream_loop(self, batches, vel_est, device_hook, ns, compute, ev_meta, ev_d2h, pending, inflight,
                          issue_copy):
        i = 0
        for sc in batches:
            k = i % ns
            if self.dims is not None and sc.size != self.dims.batch and (pending or inflight):
                raise ValueError("plan_stream: the batch size changed while results are in flight")
            while inflight and (inflight[0] == k or ev_d2h[inflight[0]].query()):
                # hand out finished results in order; the set about to be reused must have left the device first
                j = inflight.pop(0)
                ev_d2h[j].synchronize()
                yield self.h_out_sets[j]
            if device_hook is not None and hasattr(device_hook, "before"):
                device_hook.before(k)   # e.g. wait until a collective that still reads buffer set k has finished
            self.stage_scenarios(sc, vel_est=vel_est, which=k)
            self.buf.traj = self.traj_bufs[k].data_ptr()
            self.upload(which=k)
            self.set_startpos()
            self.tick()
            if device_hook is not None:     # e.g. an all-gather of the device-side action sets (multi-GPU)
                device_hook(k)
            self._download_meta(k)
            ev_meta[k].record(compute)
            pending.append(k)
            if len(pending) > 1:            # issue the trajectory copy of the previous step; it overlaps this step
                issue_copy(pending.pop(0))
            i += 1
        while pending:
            issue_copy(pending.pop(0))
        for j in inflight:
            ev_d2h[j].synchronize()
            yield self.h_out_sets[j]

    # -- kernels ---------------------------------------------------------------------------------------------------------------
    def _call(self, name):
        capi.check(self.lib, getattr(self.lib, name)(self.handle, C.byref(self.params), C.byref(self.dims),
                                                     C.byref(self.buf), self.stream), name)

    def _call_vel(self, name):
        """a call that includes calc_vel_profile: its trajectories get the next ids (+10 per call, OTH:669)"""
        self._tick_count += 1
        self.params.traj_base_id = 10 * self._tick_count
        self._call(name)

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
    _BIG = ("path", "node_idx", "nodes", "coeff", "s_vx_ax", "em_vx")            # swapped by pointer
    _SMALL = ("action_id", "traj_len", "em_info", "path_len", "n_nodes", "trim")  # carried by ONE device copy

    def _alloc_state(self) -> None:
        dev, B = self.device, self.dims.batch
        f64, i32 = torch.float64, torch.int32
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)   # noqa: E731
        t = self.t
        t["em_vx"] = z((B, self.dims.n_export), f64)   # f64 velocity of the emergency trajectory (executed 'emergency')
        self.buf.em_vx = t["em_vx"].data_ptr()
        t["em_info"].fill_(-1)
        prev_raw, prev_small = self._packed(self._carry_spec, lambda n: torch.zeros(n, dtype=torch.uint8, device=dev))
        prev_small["em_info"].fill_(-1)
        st = dict(other={k: torch.zeros_like(t[k]) for k in self._BIG}, prev_raw=prev_raw, prev_small=prev_small,
                  st_info=z((B, 8), i32), vel_plan=z((B,), f64), course=z((B, self.dims.n_export), f64),
                  obj_dist=z((B,), f64))
        st["zone_s0"] = torch.full((B,), -1, dtype=i32, device=dev)
        self.buf.zone_s0 = st["zone_s0"].data_ptr()
        self.buf.trim = t["trim"].data_ptr()
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

    def _stage_restart(self, mask) -> None:
        """buffers.restart: NULL without restarts; else its own small H2D copy (the packed input upload stays as it is)"""
        if mask is None:
            self.buf.restart = None
            return
        st = self._state
        if "restart" not in st:
            st["restart"] = torch.zeros((self.dims.batch,), dtype=torch.int32, device=self.device)
            st["h_restart"] = torch.zeros((self.dims.batch,), dtype=torch.int32).pin_memory()
            st["restart_ev"] = None
        if st["restart_ev"] is not None:      # the last copy may still read the pinned staging
            st["restart_ev"].synchronize()
        st["h_restart"].numpy()[...] = mask
        st["restart"].copy_(st["h_restart"], non_blocking=True)
        st["restart_ev"] = torch.cuda.Event()
        st["restart_ev"].record(torch.cuda.current_stream(self.device))
        self.buf.restart = st["restart"].data_ptr()

    def _stage_next(self, sc: ScenarioBatch, sel_action, t_const, vel_est, restart=None) -> None:
        """host side of a stateful tick: pointer swaps, the host memcpy into the pinned staging set, ONE packed H2D copy
        (scenario arrays incl. sel_action / t_const) and ONE device copy (the small per-path arrays of the last tick);
        with restarts one more small H2D copy (the mask)."""
        if sc.size != self.dims.batch:
            raise ValueError("stateful tick: the batch size must not change within a session (re-anchor with "
                             "set_startpos on a new batch, or restart single scenarios with `restart`)")
        check_object_count(sc.obj.shape[1], self.max_objects)   # before the swaps below: a refused list changes nothing
        mask = self._restart_mask(restart)                       # (likewise)
        if self._state is None:
            self._alloc_state()
        st, t, buf = self._state, self.t, self.buf
        n_carry = st["prev_raw"].numel()
        st["prev_raw"].copy_(self.d_meta_raw[:n_carry])       # the last tick's small per-path arrays
        for k in self._BIG:                                   # this tick writes the other set, the last one is memory
            t[k], st["other"][k] = st["other"][k], t[k]
            setattr(buf, k, t[k].data_ptr())
            setattr(buf, "prev_" + k, st["other"][k].data_ptr())
        for k in self._SMALL:
            setattr(buf, "prev_" + k, st["prev_small"][k].data_ptr())
        # location dependent local_gg of the last tick = backup for a brake on the old plan (__backup_path_gg, OTH:970)
        if getattr(self, "_gg_active", False):
            if "gg" not in st["other"]:
                st["other"]["gg"] = torch.ones_like(t["gg"])
            t["gg"], st["other"]["gg"] = st["other"]["gg"], t["gg"]
            buf.prev_gg = st["other"]["gg"].data_ptr()
        else:
            buf.prev_gg = None
        buf.gg = None            # this tick's local_gg arrives with its calc_vel_profile
        self._gg_active = False
        # a zone under a NEW id is a new zone object: its unblock window is evaluated at this tick (OLI:155-237, GLNT:43-77)
        zkey = sc.zone_key if sc.zone_key is not None else np.zeros(sc.size, dtype=np.int64)
        last = getattr(self, "_zone_key", None)               # of the batch staged for the previous tick
        if last is not None and last.shape == zkey.shape:
            changed = np.nonzero((zkey != last) & (zkey != 0))[0]
            if changed.size:
                st["zone_s0"][torch.as_tensor(changed, device=self.device)] = -1
        # pos_est of the previous calc_vel_profile (OTH:537) = `pos` of the input copy the last tick used; this tick
        # uploads into the other copy (a batch with more objects than before re-creates only the input buffers)
        self._pos_last = t["pos"]
        self.stage_scenarios(sc, vel_est=vel_est)
        self._use_inputs(1 - self._in_cur)
        buf.pos_last = self._pos_last.data_ptr()
        for k in ("st_info", "vel_plan", "course", "obj_dist"):
            setattr(buf, k, st[k].data_ptr())
        buf.sel_action = t["sel_action"].data_ptr()
        buf.t_const = t["t_const"].data_ptr()
        self.h_in["sel_action"].numpy()[...] = np.asarray(sel_action, dtype=np.int32).reshape(-1)
        self.h_in["t_const"].numpy()[...] = np.broadcast_to(np.asarray(t_const, dtype=np.float64), (self.dims.batch,))
        if self.on_device_start is not None:   # measurement hook: the host staging ends here, the device work begins
            self.on_device_start()
        self.upload()
        self._stage_restart(mask)

    def next_calc_paths(self, sc: ScenarioBatch, sel_action, t_const, vel_est=None, restart=None) -> None:
        """calc_paths of a stateful tick (OTH:289-516 with the iterative memory): ``sc`` carries the object
        lists (its poses are only used by ``next_calc_vel_profile``), ``sel_action`` = action id (capi.ACT_*) every
        scenario executed since the last tick, ``t_const`` = min(average calculation time * calc_time_safety, 0.5) per
        scenario (OTH:353-375; the caller keeps the moving average).  The previous tick (tick() / calc_paths() +
        calc_vel_profile() after set_startpos(), or a stateful tick) must have run on this planner.
        ``restart``: boolean array [B]; a true entry restarts that scenario inside this tick, as set_startpos(sc.pos[b],
        sc.heading[b], sc.vel[b]) on a live planner followed by a first tick (its memory is dropped, its sel_action and
        t_const are ignored); the other scenarios keep theirs.  A wrong shape raises ValueError and changes nothing."""
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

    def launch_count(self) -> int:
        return int(self.lib.ltpl_launch_count())

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
