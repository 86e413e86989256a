"""
ctypes binding of ``libltpl_b200.so`` (C-ABI declared in include/ltpl_b200.h).

The product path has NO CPU fallback: if the shared library is missing or a call fails, a ``RuntimeError`` is raised
(the oracle under oracle/ is test infrastructure and is never imported from here).
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

ABI_VERSION = 20
MAX_SUB = 8
NSLOT = 3
MAX_AXM = 32

ACT_NONE, ACT_STRAIGHT, ACT_FOLLOW, ACT_LEFT, ACT_RIGHT = -1, 0, 1, 2, 3
ACT_EMERGENCY = 4   # only as the executed action of a stateful tick (OTH:307-309) and in preference lists (select)
ACTION_NAMES = {ACT_STRAIGHT: "straight", ACT_FOLLOW: "follow", ACT_LEFT: "left", ACT_RIGHT: "right"}
SELECT_MAX = 8      # entries of a preference list (LtplSelect.prefer_len)

ST_FOUND, ST_REDUCED_HORIZON, ST_TIE_AMBIGUOUS, ST_START_BLOCKED = 1, 2, 4, 8
ST_TRAJ_VALID, ST_VEL_BOUND_VIOL, ST_TOO_CLOSE, ST_CONST_ONLY, ST_RENAMED_STRAIGHT = 16, 32, 64, 128, 256
SC_OUT_OF_TRACK, SC_HEADING_MISMATCH, SC_CAPACITY, SC_BRAKE_PREFIX, SC_STATE_FALLBACK = 1, 2, 4, 8, 16
SC_REASON_SHIFT = 8   # bits 8..10 of sc_flags: why SC_STATE_FALLBACK was raised (include/ltpl_b200.h)
SC_REASON_MASK = 7 << SC_REASON_SHIFT
SC_REASON_NOT_IN_MEMORY, SC_REASON_SHORT_TRAJ, SC_REASON_FEW_NODES, SC_REASON_PLACEHOLDER = 1, 2, 3, 4
SC_REASON_CONST_LONG, SC_REASON_NO_BACKUP, SC_REASON_LAST_ROW = 5, 6, 7

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC_DIR = os.path.join(PKG_DIR, "csrc")
INCLUDE_DIR = os.path.join(os.path.dirname(PKG_DIR), "include")
LIB_PATH = os.path.join(PKG_DIR, "libltpl_b200.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-fmad=false", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


class LatticeHeader(C.Structure):
    _fields_ = ([("abi_version", C.c_int32)]
                + [(n, C.c_int32) for n in ("num_layers", "num_nodes", "num_edges", "num_samples", "n_glob_rl", "closed",
                                            "plan_horizon_mode", "max_nodes_per_layer", "max_window_edges",
                                            "max_pair_edges", "tab_stride", "grid_nx", "grid_ny")]
                + [(n, C.c_double) for n in ("lat_offset", "lat_resolution", "sampled_resolution", "vel_decrease_lat",
                                             "veh_width", "veh_length", "virt_goal_node_cost", "min_plan_horizon",
                                             "grid_x0", "grid_y0", "grid_inv_cell")]
                + [(n, C.c_uint64) for n in (
                    "off_node_off", "off_raceline_index", "off_s_raceline", "off_vel_raceline", "off_refline",
                    "off_raceline", "off_bound1", "off_bound2", "off_centerline", "off_node_xy", "off_node_psi",
                    "off_node_layer", "off_in_off", "off_edge_layer_off", "off_edge_src", "off_edge_dst",
                    "off_edge_cost", "off_edge_len", "off_edge_psi1", "off_edge_psi0", "off_samp_off", "off_samp_xy", "off_samp_el",
                    "off_samp_edge", "off_glob_rl", "off_glob_xy", "off_edge_rec", "off_tab_reach", "off_tab_node",
                    "off_tab_edge", "off_grid_center", "off_grid_refline", "off_grid_raceline", "off_grid_glob",
                    "blob_bytes")])


class Params(C.Structure):
    _fields_ = [("max_heading_offset", C.c_double), ("v_max_offset", C.c_double), ("follow_c_p", C.c_double),
                ("follow_k_d", C.c_double), ("follow_k_p", C.c_double), ("follow_tan_w", C.c_double),
                ("follow_control_type", C.c_int32), ("nmbr_export_points", C.c_int32),
                ("dyn_model_exp", C.c_double), ("drag_coeff", C.c_double), ("m_veh", C.c_double),
                ("vel_max", C.c_double), ("gg_scale", C.c_double), ("gg_ax", C.c_double), ("gg_ay", C.c_double),
                ("safety_d", C.c_double), ("n_axm", C.c_int32), ("traj_base_id", C.c_int32),
                ("incl_emerg_traj", C.c_int32), ("filt_window", C.c_int32), ("delaycomp", C.c_double),
                ("w_last_edges", C.c_double * 4),
                ("axm_v", C.c_double * MAX_AXM), ("axm_a", C.c_double * MAX_AXM), ("axm_s", C.c_double * MAX_AXM),
                ("gg_map_x0", C.c_double), ("gg_map_y0", C.c_double), ("gg_map_inv_cell", C.c_double),
                ("gg_map_nx", C.c_int32), ("gg_map_ny", C.c_int32)]


class Dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "k_obj", "p0_max", "p_max", "h_max", "n_export", "n_zone_words",
                                            "n_zones", "k_pred", "sub_id", "sub_off", "sub_cnt")]


BUFFER_FIELDS = ("pos", "heading", "vel", "vel_est", "n_obj", "obj", "sc_flags", "start_node", "const_len", "const_seg",
                 "const_coeff", "action_id", "status", "n_nodes", "nodes", "node_idx", "edge_seq", "closest_obj", "cobj", "cobj_start",
                 "path_len", "path", "coeff", "queue", "queue_cnt", "exp_q", "traj_row", "s_vx_ax",
                 "traj", "traj_len", "traj_id", "zone_bits", "zone_sel", "em_info", "obj_pred",
                 "n_pred", "prev_path", "prev_path_len", "prev_node_idx", "prev_nodes", "prev_n_nodes", "prev_coeff",
                 "prev_s_vx_ax", "prev_action_id", "prev_traj_len", "prev_trim", "sel_action", "pos_last", "t_const",
                 "st_info", "trim", "vel_plan", "course", "obj_dist", "zone_s0", "em_vx", "prev_em_vx", "prev_em_info",
                 "gg", "prev_gg", "restart", "gg_map", "traj_base")
STATE_FIELDS = BUFFER_FIELDS[BUFFER_FIELDS.index("prev_path"):]   # NULL unless a stateful tick is planned


class Buffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in BUFFER_FIELDS]


class VelBatch(C.Structure):
    _fields_ = [("n_paths", C.c_int32), ("n_points", C.c_int32), ("kappa", C.c_void_p), ("el", C.c_void_p),
                ("v_start", C.c_void_p), ("v_end", C.c_void_p), ("vx", C.c_void_p), ("ax", C.c_void_p)]


VP_PROFILE, VP_BRAKE = 0, 1   # LtplVelPlan.mode: tph.calc_vel_profile | tph.calc_vel_profile_brake


class VelPlan(C.Structure):
    """LtplVelPlan; it carries its size (struct_bytes), which ltpl_vel_plan_batch checks at every call"""
    _fields_ = [("struct_bytes", C.c_int32), ("mode", C.c_int32), ("n_paths", C.c_int32), ("n_points", C.c_int32),
                ("n_pts", C.c_void_p), ("kappa", C.c_void_p), ("kappa_s", C.c_int64), ("el", C.c_void_p),
                ("el_s", C.c_int64), ("gg", C.c_void_p), ("gg_s", C.c_int64), ("v_start", C.c_void_p),
                ("v_end", C.c_void_p), ("vx", C.c_void_p), ("ax", C.c_void_p), ("out_s", C.c_int64)]

    def __init__(self):
        super().__init__()
        self.struct_bytes = C.sizeof(VelPlan)


class VelFollow(C.Structure):
    """LtplVelFollow; it carries its size (struct_bytes), which ltpl_vel_follow_batch checks at every call"""
    _fields_ = [("struct_bytes", C.c_int32), ("n_paths", C.c_int32), ("n_points", C.c_int32), ("n_pts", C.c_void_p),
                ("kappa", C.c_void_p), ("kappa_s", C.c_int64), ("el", C.c_void_p), ("el_s", C.c_int64),
                ("gg", C.c_void_p), ("gg_s", C.c_int64), ("v_start", C.c_void_p), ("v_ego", C.c_void_p),
                ("v_obj", C.c_void_p), ("safety_d", C.c_void_p), ("obj_dist", C.c_void_p), ("obj_pos", C.c_void_p),
                ("obj_pos_s", C.c_int64), ("glob_rl", C.c_void_p), ("n_glob", C.c_int32), ("veh_length", C.c_double),
                ("vx", C.c_void_p), ("ax", C.c_void_p), ("out_s", C.c_int64), ("too_close", C.c_void_p),
                ("vel_bound", C.c_void_p)]

    def __init__(self):
        super().__init__()
        self.struct_bytes = C.sizeof(VelFollow)


class BrakePrefix(C.Structure):
    """LtplBrakePrefix; it carries its size (struct_bytes), which ltpl_brake_prefix_batch checks at every call"""
    _fields_ = [("struct_bytes", C.c_int32), ("n_paths", C.c_int32), ("n_points", C.c_int32), ("n_pts", C.c_void_p),
                ("kappa", C.c_void_p), ("kappa_s", C.c_int64), ("el", C.c_void_p), ("el_s", C.c_int64),
                ("gg", C.c_void_p), ("gg_s", C.c_int64), ("vel_plan", C.c_void_p), ("vel_course", C.c_void_p),
                ("vel_course_s", C.c_int64), ("n_course_cap", C.c_int32), ("n_course", C.c_void_p),
                ("old_gg_scale", C.c_void_p), ("vx_prefix", C.c_void_p), ("vx_prefix_s", C.c_int64),
                ("n_prefix", C.c_void_p), ("pref_idx", C.c_void_p), ("vel_start", C.c_void_p)]

    def __init__(self):
        super().__init__()
        self.struct_bytes = C.sizeof(BrakePrefix)


PC_S_COORD, PC_S_INDEX, PC_CLOSEST, PC_INSIDE_BOUNDS = 0, 1, 2, 3   # LtplPathCoord.mode


class PathCoord(C.Structure):
    """LtplPathCoord; it carries its size (struct_bytes), which ltpl_path_coord_batch checks at every call"""
    _fields_ = [("struct_bytes", C.c_int32), ("mode", C.c_int32), ("closed", C.c_int32), ("n_queries", C.c_int32),
                ("m_points", C.c_int32), ("x", C.c_void_p), ("y", C.c_void_p), ("line_s", C.c_int64),
                ("pt_s", C.c_int64), ("x2", C.c_void_p), ("y2", C.c_void_p), ("line2_s", C.c_int64),
                ("pt2_s", C.c_int64), ("s_array", C.c_void_p), ("s_array_s", C.c_int64), ("s_array_es", C.c_int64),
                ("pos", C.c_void_p),
                ("pos_s", C.c_int64 * 2), ("n_pts", C.c_void_p), ("s", C.c_void_p), ("closest", C.c_void_p),
                ("idx", C.c_void_p), ("inside", C.c_void_p)]

    def __init__(self):
        super().__init__()
        self.struct_bytes = C.sizeof(PathCoord)


class StageSrc(C.Structure):
    _fields_ = [("pos", C.c_void_p), ("pos_s", C.c_int64 * 2), ("heading", C.c_void_p), ("heading_s", C.c_int64),
                ("vel", C.c_void_p), ("vel_s", C.c_int64), ("vel_est", C.c_void_p), ("vel_est_s", C.c_int64),
                ("n_obj", C.c_void_p), ("n_obj_s", C.c_int64), ("obj", C.c_void_p), ("obj_s", C.c_int64 * 3),
                ("pred", C.c_void_p), ("pred_s", C.c_int64 * 4), ("n_pred", C.c_void_p), ("n_pred_s", C.c_int64 * 2),
                ("zone_sel", C.c_void_p), ("zone_sel_s", C.c_int64), ("zone_key", C.c_void_p), ("zone_key_s", C.c_int64),
                ("zone_key_last", C.c_void_p), ("sel_action", C.c_void_p), ("sel_action_s", C.c_int64),
                ("t_const", C.c_void_p), ("t_const_s", C.c_int64), ("restart", C.c_void_p), ("restart_s", C.c_int64),
                ("t_const_value", C.c_double), ("k_src", C.c_int32), ("kp_src", C.c_int32), ("kp_dst", C.c_int32),
                ("sel_action_bytes", C.c_int32), ("restart_bytes", C.c_int32), ("zone_key_rule", C.c_int32)]


class Select(C.Structure):
    """LtplSelect; it carries its size (struct_bytes), which ltpl_select_batch checks at every call"""
    _fields_ = [("struct_bytes", C.c_int32), ("prefer_len", C.c_int32), ("prefer", C.c_void_p),
                ("prefer_s", C.c_int64 * 2), ("prefer_bytes", C.c_int32), ("sel_action", C.c_void_p),
                ("sel_action_s", C.c_int64), ("sel_info", C.c_void_p), ("sel_traj", C.c_void_p)]

    def __init__(self):
        super().__init__()
        self.struct_bytes = C.sizeof(Select)


EXPORTS = ("ltpl_version", "ltpl_last_error", "ltpl_sizeof", "ltpl_max_objects", "ltpl_lattice_create",
           "ltpl_lattice_destroy", "ltpl_set_startpos_batch", "ltpl_calc_paths_batch", "ltpl_calc_vel_profile_batch",
           "ltpl_tick_batch", "ltpl_velprofile_batch", "ltpl_launch_count", "ltpl_launch_stage", "ltpl_next_tick_batch",
           "ltpl_next_calc_paths_batch", "ltpl_next_calc_vel_profile_batch", "ltpl_set_subbatches",
           "ltpl_stage_inputs_batch", "ltpl_prepare_batch", "ltpl_select_batch", "ltpl_vel_plan_batch",
           "ltpl_vel_follow_batch", "ltpl_brake_prefix_batch", "ltpl_path_coord_batch")


def build_library(verbose: bool = False) -> str:
    """nvcc cross-compile for sm_90a (works without a GPU); the .so is written next to this module."""
    src = os.path.join(CSRC_DIR, "ltpl_api.cu")
    deps = [src] + [os.path.join(CSRC_DIR, f) for f in os.listdir(CSRC_DIR) if f.endswith(".cuh")] \
        + [os.path.join(INCLUDE_DIR, "ltpl_b200.h"), os.path.abspath(__file__)]   # this file holds NVCC_FLAGS
    if os.path.isfile(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-I" + INCLUDE_DIR, "-o", LIB_PATH, src]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout)
    return LIB_PATH


_lib = None


def load_library():
    """dlopen libltpl_b200.so; raises RuntimeError (never falls back) when it is missing or its ABI does not match."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError("libltpl_b200.so not found at %s -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a). There is no CPU fallback for the planning path." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise RuntimeError("libltpl_b200.so does not export %s" % name)
    lib.ltpl_version.restype = C.c_int
    lib.ltpl_last_error.restype = C.c_char_p
    lib.ltpl_sizeof.argtypes = [C.c_int]
    lib.ltpl_sizeof.restype = C.c_int
    lib.ltpl_launch_count.restype = C.c_uint64
    lib.ltpl_lattice_create.argtypes = [C.POINTER(LatticeHeader), C.c_void_p, C.POINTER(C.c_void_p)]
    lib.ltpl_lattice_destroy.argtypes = [C.c_void_p]
    lib.ltpl_max_objects.argtypes = [C.POINTER(LatticeHeader), C.c_int]
    lib.ltpl_max_objects.restype = C.c_int
    lib.ltpl_set_subbatches.argtypes = [C.c_void_p, C.c_int]
    lib.ltpl_set_subbatches.restype = C.c_int
    for fn in (lib.ltpl_set_startpos_batch, lib.ltpl_calc_paths_batch, lib.ltpl_calc_vel_profile_batch,
               lib.ltpl_tick_batch, lib.ltpl_next_tick_batch, lib.ltpl_next_calc_paths_batch,
               lib.ltpl_next_calc_vel_profile_batch):
        fn.argtypes = [C.c_void_p, C.POINTER(Params), C.POINTER(Dims), C.POINTER(Buffers), C.c_void_p]
        fn.restype = C.c_int
    lib.ltpl_launch_stage.argtypes = [C.c_int, C.c_void_p, C.POINTER(Params), C.POINTER(Dims), C.POINTER(Buffers),
                                      C.c_void_p]
    lib.ltpl_launch_stage.restype = C.c_int
    lib.ltpl_velprofile_batch.argtypes = [C.POINTER(Params), C.POINTER(VelBatch), C.c_void_p]
    lib.ltpl_velprofile_batch.restype = C.c_int
    lib.ltpl_vel_plan_batch.argtypes = [C.POINTER(Params), C.POINTER(VelPlan), C.c_void_p]
    lib.ltpl_vel_plan_batch.restype = C.c_int
    lib.ltpl_vel_follow_batch.argtypes = [C.POINTER(Params), C.POINTER(VelFollow), C.c_void_p]
    lib.ltpl_vel_follow_batch.restype = C.c_int
    lib.ltpl_brake_prefix_batch.argtypes = [C.POINTER(Params), C.POINTER(BrakePrefix), C.c_void_p]
    lib.ltpl_brake_prefix_batch.restype = C.c_int
    lib.ltpl_path_coord_batch.argtypes = [C.POINTER(PathCoord), C.c_void_p]
    lib.ltpl_path_coord_batch.restype = C.c_int
    lib.ltpl_stage_inputs_batch.argtypes = [C.POINTER(Dims), C.POINTER(Buffers), C.POINTER(StageSrc), C.c_void_p]
    lib.ltpl_stage_inputs_batch.restype = C.c_int
    lib.ltpl_prepare_batch.argtypes = [C.c_void_p, C.POINTER(Params), C.POINTER(Dims), C.POINTER(Buffers)]
    lib.ltpl_prepare_batch.restype = C.c_int
    lib.ltpl_select_batch.argtypes = [C.POINTER(Params), C.POINTER(Dims), C.POINTER(Buffers), C.POINTER(Select),
                                      C.c_void_p]
    lib.ltpl_select_batch.restype = C.c_int
    if lib.ltpl_version() != ABI_VERSION:
        raise RuntimeError("libltpl_b200.so ABI version %d != binding %d" % (lib.ltpl_version(), ABI_VERSION))
    for which, st in enumerate((LatticeHeader, Params, Dims, Buffers, VelBatch, StageSrc)):
        if lib.ltpl_sizeof(which) != C.sizeof(st):
            raise RuntimeError("ctypes mirror of %s has %d bytes, library says %d" % (st.__name__, C.sizeof(st),
                                                                                      lib.ltpl_sizeof(which)))
    _lib = lib
    return lib


def check(lib, rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, lib.ltpl_last_error().decode()))
