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

ABI_VERSION = 17
MAX_SUB = 8
NSLOT = 3
MAX_AXM = 32

ACT_NONE, ACT_STRAIGHT, ACT_FOLLOW, ACT_LEFT, ACT_RIGHT = -1, 0, 1, 2, 3
ACT_EMERGENCY = 4   # only as the executed action of a stateful tick (OTH:307-309)
ACTION_NAMES = {ACT_STRAIGHT: "straight", ACT_FOLLOW: "follow", ACT_LEFT: "left", ACT_RIGHT: "right"}

ST_FOUND, ST_REDUCED_HORIZON, ST_TIE_AMBIGUOUS, ST_START_BLOCKED = 1, 2, 4, 8
ST_TRAJ_VALID, ST_VEL_BOUND_VIOL, ST_TOO_CLOSE, ST_CONST_ONLY, ST_RENAMED_STRAIGHT = 16, 32, 64, 128, 256
SC_OUT_OF_TRACK, SC_HEADING_MISMATCH, SC_CAPACITY, SC_BRAKE_PREFIX, SC_STATE_FALLBACK = 1, 2, 4, 8, 16
SC_REASON_SHIFT = 8   # bits 8..10 of sc_flags: why SC_STATE_FALLBACK was raised (include/ltpl_b200.h)

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
                ("axm_v", C.c_double * MAX_AXM), ("axm_a", C.c_double * MAX_AXM), ("axm_s", C.c_double * MAX_AXM)]


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
                 "gg", "prev_gg", "restart")
STATE_FIELDS = BUFFER_FIELDS[BUFFER_FIELDS.index("prev_path"):]   # NULL unless a stateful tick is planned


class Buffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in BUFFER_FIELDS]


class VelBatch(C.Structure):
    _fields_ = [("n_paths", C.c_int32), ("n_points", C.c_int32), ("kappa", C.c_void_p), ("el", C.c_void_p),
                ("v_start", C.c_void_p), ("v_end", C.c_void_p), ("vx", C.c_void_p), ("ax", C.c_void_p)]


EXPORTS = ("ltpl_version", "ltpl_last_error", "ltpl_sizeof", "ltpl_max_objects", "ltpl_lattice_create",
           "ltpl_lattice_destroy", "ltpl_set_startpos_batch", "ltpl_calc_paths_batch", "ltpl_calc_vel_profile_batch",
           "ltpl_tick_batch", "ltpl_velprofile_batch", "ltpl_launch_count", "ltpl_launch_stage", "ltpl_next_tick_batch",
           "ltpl_next_calc_paths_batch", "ltpl_next_calc_vel_profile_batch", "ltpl_set_subbatches")


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
    if lib.ltpl_version() != ABI_VERSION:
        raise RuntimeError("libltpl_b200.so ABI version %d != binding %d" % (lib.ltpl_version(), ABI_VERSION))
    for which, st in enumerate((LatticeHeader, Params, Dims, Buffers, VelBatch)):
        if lib.ltpl_sizeof(which) != C.sizeof(st):
            raise RuntimeError("ctypes mirror of %s has %d bytes, library says %d" % (st.__name__, C.sizeof(st),
                                                                                      lib.ltpl_sizeof(which)))
    _lib = lib
    return lib


def check(lib, rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, lib.ltpl_last_error().decode()))
