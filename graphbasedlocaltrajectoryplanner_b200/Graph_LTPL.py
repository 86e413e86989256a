"""
``Graph_LTPL`` -- drop-in facade with the call surface of the reference class
(graph_ltpl/Graph_LTPL.py:26-532) for the online planning path, executed by the sm_90a kernels.

Kept signatures (same names, argument meaning, return structure and error behaviour):

    Graph_LTPL(path_dict, visual_mode=False, log_to_file=True)                                   LTPL:41-181
    graph_init(veh_param_dyn_model_exp=1.0, veh_param_dragcoeff=0.85, veh_param_mass=1000.0)     LTPL:189-258
    set_startpos(pos_est, heading_est, vel_est=0.0) -> out_of_track                              LTPL:262-296
    calc_paths(prev_action_id, prev_traj_idx=0, object_list=None, blocked_zones=None) -> dict    LTPL:300-340
    calc_vel_profile(pos_est, vel_est, vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0),
                     ax_max_machines=[[100.0, 5.0]], safety_d=30.0, incl_emerg_traj=False)
                     -> (action_set, action_set_id, traj_time)                                   LTPL:344-408

plus the batched variants ``set_startpos_batch`` / ``calc_paths_batch`` / ``calc_vel_profile_batch`` / ``plan_batch``
over a ``ScenarioBatch`` (thousands of independent ego-start x obstacle scenarios per call).

    log() / visual()   documented no-ops (LTPL:412-463, 465-532): the reference's loops call them every tick
                       (main_min_example.py:107, main_std_example.py:132-135); file logging and live plots themselves
                       are out of scope (SURVEY 2)

Scope (SURVEY 8): the first ``calc_paths`` / ``calc_vel_profile`` pair after ``set_startpos`` is the stateless first
tick; every later pair is a STATEFUL tick whose iterative memory (OTH:64-87) lives on the device (DESIGN.md section 11,
csrc/ltpl_state.cuh) -- the wall clock the reference reads (OTH:353-378) is ``self.clock`` here (injectable).
``blocked_zones`` takes one zone per scenario ('nodes' type, GLNT:43-99); ``incl_emerg_traj=True`` adds the 'emergency'
entry (OTH:1027-1034); ``local_gg`` is the tuple of the reference or its location dependent dict form
``{action: [ndarray(P, 2)]}`` (OTH:649-666).  Offline graph generation is replaced by the flat lattice blob (lattice.py).
"""

from __future__ import annotations

import logging
import time

import numpy as np

from . import capi
from .lattice import load_or_build_lattice
from .planner import BatchPlanner, read_online_config
from .scenarios import ScenarioBatch

# required path dict entries (LTPL:22-23)
REQ_PATH_DICT_ENTRIES = ['globtraj_input_path', 'graph_store_path', 'ltpl_offline_param_path', 'ltpl_online_param_path',
                         'graph_log_id', 'log_path']


def physical_objects(object_list) -> list:
    """the entries the object filter sees (OLI:104-112): 'physical' ones, in list order, on the track or not (the track
    test runs on the device); their number is bounded by BatchPlanner.max_objects, not by the on-track count."""
    return [o for o in (object_list or []) if o.get('type') == 'physical']


class ActionSetView(object):
    """Lazy sequence over the scenarios of a batched result (Graph_LTPL.unpack_batch): ``view[b]`` ->
    ({action: [ndarray(rows, 7)]}, {action: trajectory id}) exactly as the reference's calc_vel_profile returns them
    (LTPL:344-408), incl. the 'emergency' entry when it was requested."""

    def __init__(self, out: dict):
        self._rows, self._lens, self._ids, self._acts = (out[k].numpy() for k in ("traj_row", "traj_len", "traj_id",
                                                                                  "action_id"))
        self._traj = out["traj"].numpy()
        self._em = out["em_info"].numpy() if out.get("incl_emerg_traj") else None

    def __len__(self) -> int:
        return int(self._rows.shape[1])

    def __getitem__(self, b: int) -> tuple:
        if b < 0:
            b += len(self)
        if not 0 <= b < len(self):
            raise IndexError(b)
        t, i = {}, {}
        for s in range(self._rows.shape[0]):
            r = self._rows[s, b]
            if r >= 0:
                name = capi.ACTION_NAMES[int(self._acts[s, b])]
                t[name] = [self._traj[r, :self._lens[s, b]]]
                i[name] = int(self._ids[s, b])
        if self._em is not None and t and self._em[b, 0] >= 0:
            t["emergency"] = [self._traj[self._em[b, 0], :self._em[b, 1]]]
            i["emergency"] = int(self._em[b, 2])
        return t, i

    def __iter__(self):
        return (self[b] for b in range(len(self)))

    def kept(self) -> np.ndarray:
        """[NSLOT][B] bool: which (slot, scenario) holds a trajectory -- vectorised access without building dicts"""
        return self._rows >= 0


class Graph_LTPL(object):
    def __init__(self, path_dict: dict, visual_mode: bool = False, log_to_file: bool = True, device=None) -> None:
        for entry in REQ_PATH_DICT_ENTRIES:   # LTPL:62-68
            if entry not in path_dict:
                if log_to_file or 'log' not in entry:
                    raise ValueError('Missing path specification in path_dict (Missing entry: "' + entry + '")!')
        self.__log = logging.getLogger("local_trajectory_logger")
        # live plots / file logs of the reference (LTPL:96-104, 146-166) are out of scope: the flags are accepted so that
        # the reference's own loops run unchanged, visual() / log() are no-ops
        self.__visual_mode = bool(visual_mode)
        self.__log_to_file = bool(log_to_file)
        if visual_mode:
            self.__log.warning("visual_mode=True: live visualisation is not part of the batched GPU planning path; visual() "
                               "is a no-op")
        self.__path_dict = path_dict
        self.__device = device
        self.__online = read_online_config(path_dict['ltpl_online_param_path'])
        self.__planner = None
        self.__lattice = None
        self.__state = None          # None | "start" | "paths"
        self.__records = None
        self.__zones = None          # the last blocked_zones dict: the reference keeps its zone objects when none is passed
        self.__start_vel = 0.0
        self.__pos = None
        self.__heading = None
        self.__objects = None
        # iterative memory across ticks (DESIGN.md section 11): the clock is injectable for tests
        self.clock = time.time
        self.__tick_no = 0
        self.__last_path_timestamp = None
        self.__calc_buffer = []

    # ------------------------------------------------------------------------------------------------------------------
    def graph_init(self, veh_param_dyn_model_exp: float = 1.0, veh_param_dragcoeff: float = 0.85,
                   veh_param_mass: float = 1000.0, lattice_overrides: dict = None) -> None:
        """load (md5-keyed cache) or build the lattice, upload it, create the planner (LTPL:189-258)."""
        self.__lattice, _ = load_or_build_lattice(self.__path_dict['globtraj_input_path'],
                                                  self.__path_dict['ltpl_offline_param_path'],
                                                  store_path=self.__path_dict.get('graph_store_path'),
                                                  overrides=lattice_overrides)
        self.__planner = BatchPlanner(self.__lattice, online=self.__online, device=self.__device,
                                      veh_param_dyn_model_exp=veh_param_dyn_model_exp,
                                      veh_param_dragcoeff=veh_param_dragcoeff, veh_param_mass=veh_param_mass,
                                      stateful=True)

    @property
    def lattice(self):
        return self.__lattice

    @property
    def planner(self) -> BatchPlanner:
        if self.__planner is None:
            raise ValueError("Graph is not initialized yet. Call graph_init() first!")
        return self.__planner

    # ------------------------------------------------------------------------------------------------------------------
    # single-scenario API (reference signatures)
    # ------------------------------------------------------------------------------------------------------------------
    def set_startpos(self, pos_est: np.ndarray, heading_est: float, vel_est: float = 0.0) -> bool:
        if self.__planner is None:   # LTPL:277-280
            raise ValueError("Could not set start position, since graph is not initialized yet. "
                             "Call graph_init() first!")
        self.__pos = np.asarray(pos_est, dtype=np.float64).reshape(2)
        self.__heading = float(np.asarray(heading_est).reshape(-1)[0])
        self.__start_vel = float(vel_est)
        sc = ScenarioBatch.from_object_lists([self.__pos], [self.__heading], [self.__start_vel], [[]])
        pl = self.__planner
        pl.stage_scenarios(sc)
        pl.upload()
        pl.set_startpos()
        flags = int(pl.fetch("sc_flags")["sc_flags"][0])
        if flags & capi.SC_OUT_OF_TRACK:
            self.__log.warning("Vehicle is out of track, check if correct reference line is provided!")
        if flags & capi.SC_HEADING_MISMATCH:
            self.__log.warning("Heading mismatch between vehicle and track grid, check if vehicle oriented correctly!")
        if flags & capi.SC_CAPACITY:
            raise RuntimeError("start pose too far from the lattice for the constant-segment capacity")
        out_of_track = bool(flags & (capi.SC_OUT_OF_TRACK | capi.SC_HEADING_MISMATCH))
        self.__state = None if out_of_track else "start"
        self.__tick_no = 0
        self.__last_path_timestamp = None
        self.__calc_buffer = []
        return out_of_track

    def calc_paths(self, prev_action_id: str, prev_traj_idx: int = 0, object_list: list = None,
                   blocked_zones: dict = None) -> dict:
        if self.__state is None:
            raise ValueError("calc_paths() needs a start pose: call set_startpos() first (after an out-of-track result or "
                             "a memory fallback again)")
        if blocked_zones:                # LTPL:324-329: update_zone only runs for a passed dict, the zone objects persist
            self.__zones = blocked_zones
        blocked_zones = self.__zones
        if self.__state == "next":   # stateful tick: the memory of the last tick lives on the device
            return self.__calc_paths_next(prev_action_id, object_list, blocked_zones)
        self.__last_path_timestamp = self.clock()   # OTH:395
        sc = ScenarioBatch.from_object_lists([self.__pos], [self.__heading], [self.__start_vel],
                                             [physical_objects(object_list)],
                                             blocked_zones=[blocked_zones] if blocked_zones else None)
        for o in (object_list or []):
            if o.get('type') != 'physical':   # OLI:140-141
                self.__log.warning("Found non-supported object of type '%s' in object list!" % o.get('type'))
        pl = self.__planner
        pl.stage_scenarios(sc)
        pl.upload()
        pl.set_startpos()
        pl.calc_paths()
        self.__records = pl.records()[0]
        self.__state = "paths"
        if not self.__records["paths"]:
            self.__log.critical("Could not find a path solution for any of the points in the given destination layer! "
                                "Track useems to be blocked.")
        return {k: [a.copy() for a in v] for k, v in self.__records["paths"].items()}

    def __calc_paths_next(self, prev_action_id, object_list, blocked_zones):
        """OTH:346-392 on the device: the calculation time since the last calc_paths (moving average over 5 ticks, safety
        factor 2, at most 0.5 s -- ltpl_config_online.ini:84-94) decides how much of the last trajectory stays constant."""
        if prev_action_id not in ("straight", "follow", "left", "right", "emergency"):
            raise ValueError("unknown prev_action_id '%s'" % prev_action_id)
        now = self.clock()
        calc_time = now - self.__last_path_timestamp
        self.__last_path_timestamp = self.clock()
        if len(self.__calc_buffer) >= 5:
            self.__calc_buffer.pop(0)
        self.__calc_buffer.append(calc_time)
        t_const = min(float(np.sum(self.__calc_buffer) / len(self.__calc_buffer)) * 2.0, 0.5)
        sc = ScenarioBatch.from_object_lists([self.__pos], [self.__heading], [self.__start_vel],
                                             [physical_objects(object_list)],
                                             blocked_zones=[blocked_zones] if blocked_zones else None)
        # 'emergency': the device translates it to the action its profile was based on (OTH:307-309)
        sel = dict({v: k for k, v in capi.ACTION_NAMES.items()}, emergency=capi.ACT_EMERGENCY)[prev_action_id]
        pl = self.__planner
        pl.next_calc_paths(sc, [sel], t_const)
        rec = pl.records()[0]
        if rec["flags"] & capi.SC_STATE_FALLBACK:
            self.__state = None
            raise RuntimeError("the last trajectory of action '%s' cannot serve as memory (flags 0x%x, see "
                               "LTPL_SC_REASON_SHIFT): call set_startpos() again" % (prev_action_id, rec["flags"]))
        self.__records = rec
        self.__state = "paths_next"
        return {k: [a.copy() for a in v] for k, v in rec["paths"].items()}

    def calc_vel_profile(self, pos_est: np.ndarray, vel_est: float, vel_max: float = 100.0, gg_scale: float = 1.0,
                         local_gg: dict = (5.0, 5.0), ax_max_machines: np.ndarray = np.atleast_2d([100.0, 5.0]),
                         safety_d: float = 30.0, incl_emerg_traj: bool = False) -> tuple:
        if self.__state not in ("paths", "paths_next"):
            raise ValueError("calc_paths() must be called before calc_vel_profile()")
        pl = self.__planner
        gg_planes = None
        if type(local_gg) is dict:   # location dependent friction: one (P, 2) array per path of this tick (OTH:649-666)
            n_pts = pl.dims.p_max
            gg_planes = np.ones((2, capi.NSLOT, 1, n_pts))
            slot_of = {"straight": 0, "follow": 0, "left": 1, "right": 2}
            for action, paths in self.__records["paths"].items():
                if action not in local_gg:   # the reference indexes local_gg[action_id] for every action (OTH:708)
                    raise KeyError(action)
                arr = np.asarray(local_gg[action][0], dtype=np.float64)
                if arr.ndim != 2 or arr.shape != (paths[0].shape[0], 2):
                    raise ValueError("local_gg['%s'][0] must have the shape (%d, 2) of the action's path" % (
                        action, paths[0].shape[0]))
                gg_planes[:, slot_of[action], 0, :arr.shape[0]] = arr.T
            local_gg = None
        pl.set_vel_params(vel_max=vel_max, gg_scale=gg_scale, local_gg=local_gg, ax_max_machines=ax_max_machines,
                          safety_d=safety_d, incl_emerg_traj=incl_emerg_traj)
        if gg_planes is not None:
            pl.set_local_gg_planes(gg_planes[0], gg_planes[1])
        else:
            pl.set_local_gg_planes(None)
        pos = np.asarray(pos_est, dtype=np.float64).reshape(2)
        if self.__state == "paths_next":
            pl.next_calc_vel_profile(pos_est=[pos], vel_est=[float(vel_est)])
        else:
            # first tick: the position estimate only enters the follow-mode distance (OTH:779-784)
            pl.set_estimates(pos_est=[pos], vel_est=[float(vel_est)])
            pl.calc_vel_profile()
        rec = pl.records()[0]
        if rec.get("error", 0) & capi.SC_BRAKE_PREFIX:
            raise ValueError("vel_plan exceeds vel_max: the reference's brake-prefix branch (OTH:747-754) yields arrays "
                             "of mismatching length and raises; not planned")
        if (rec["flags"] & capi.SC_STATE_FALLBACK) and ((rec["flags"] >> capi.SC_REASON_SHIFT) & 7) == 7:
            self.__state = None   # the reference raises here as well (np.argmin of an empty array, OTH:570)
            raise ValueError("pos_est lies at the last row of the last trajectory: no velocity course left "
                             "(OTH:558-574); call set_startpos() again")
        if rec.get("error", 0) & capi.SC_CAPACITY:
            raise RuntimeError("a capacity of the batched path was exceeded (LTPL_SC_CAPACITY, flags 0x%x)" % rec["flags"])
        self.__records = rec
        for name, st in rec["status"].items():
            if st & capi.ST_TOO_CLOSE:
                self.__log.warning("Too close to object! Entering safety distance... [Follow-Mode]")
            if (st & capi.ST_VEL_BOUND_VIOL) and not (st & capi.ST_TRAJ_VALID):
                self.__log.warning("Removed action set, since vel constraints were broken! (Action Set: " + name + ")")
        self.__pos = pos
        # later ticks continue from the device-resident memory; when the velocity planner removed every trajectory the
        # memory is empty and the next calc_paths() takes the "no valid last solution" branch (OTH:393-407) on the device
        self.__state = "next"
        return ({k: [a.copy() for a in v] for k, v in rec["traj"].items()}, dict(rec["ids"]), time.time())

    def log(self) -> None:
        """LTPL:412-463 writes the tick to the graph log file; file logging is out of scope (SURVEY 2) -- no-op, kept so
        that the reference's loops (main_std_example.py:132) run unchanged."""
        return None

    def visual(self) -> None:
        """LTPL:465-532 updates the live plot; visualisation is out of scope (SURVEY 2) -- no-op, kept so that the
        reference's loops (main_min_example.py:107, main_std_example.py:135) run unchanged."""
        return None

    def last_node_sequences(self) -> dict:
        """node sequences of the last calc_paths() call ({action: [[[layer, node], ...]]}, cf. OTH:509)."""
        return {} if self.__records is None else dict(self.__records["nodes"])

    # ------------------------------------------------------------------------------------------------------------------
    # batched API
    # ------------------------------------------------------------------------------------------------------------------
    def set_startpos_batch(self, scenarios: ScenarioBatch, vel_est=None) -> None:
        pl = self.planner
        pl.stage_scenarios(scenarios, vel_est=vel_est)
        pl.upload()
        pl.set_startpos()

    def calc_paths_batch(self) -> None:
        self.planner.calc_paths()

    def calc_vel_profile_batch(self, **vel_kwargs) -> dict:
        pl = self.planner
        if vel_kwargs:
            pl.set_vel_params(**vel_kwargs)
        pl.calc_vel_profile()
        return pl.download()

    def plan_batch(self, scenarios: ScenarioBatch = None, synchronize: bool = True) -> dict:
        """One end-to-end batched tick: host scenario arrays -> (H2D) -> set_startpos -> calc_paths -> calc_vel_profile
        -> (D2H) -> pinned host action sets: ``traj`` [n_rows][n_export][7] fp32 (compact: one row per kept
        trajectory), ``exp_q`` (row -> path id q = slot * B + b), ``traj_row`` [NSLOT][B] (path -> row or -1),
        ``traj_len``, ``traj_id``, ``action_id``, ``status``, ``sc_flags``, ``n_rows``.
        With ``scenarios=None`` the previously staged batch is planned again."""
        pl = self.planner
        if scenarios is not None:
            pl.stage_scenarios(scenarios)
        pl.upload()
        pl.set_startpos()
        pl.tick()
        out = pl.download()
        if synchronize:
            import torch
            torch.cuda.current_stream(pl.device).synchronize()
        return out

    @staticmethod
    def unpack_batch(out: dict) -> "ActionSetView":
        """per-scenario view of a plan_batch / plan_stream result in the reference's return structure of
        calc_vel_profile (LTPL:344-408): a sequence of ({action: [ndarray(rows, 7)]}, {action: id}), one entry per
        scenario.  The sequence is LAZY: it keeps the packed index arrays and builds a scenario's two dicts when it is
        indexed or iterated; the arrays are views of the pinned host buffer (fp32), nothing is copied."""
        return ActionSetView(out)

    def plan_stream(self, batches, vel_est=None, device_hook=None):
        """Pipelined variant of ``plan_batch`` over an iterable of ScenarioBatch objects: yields one result dict per
        batch, in order; the device-to-host copy of step i overlaps the kernels of step i + 1
        (``BatchPlanner.plan_stream``)."""
        return self.planner.plan_stream(batches, vel_est=vel_est, device_hook=device_hook)
