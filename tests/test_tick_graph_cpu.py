"""Ticks replayed from CUDA graphs, without a GPU: k_traj_base's stack frame in the built library, the ctypes mirror of
LtplBuffers with the appended traj_base against the header and the library, and the ABI version."""
import ctypes
import os
import re

from tests.test_kernel_frames import _stack_frames

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "ltpl_b200.h")


def _header_buffer_fields():
    """the field names of LtplBuffers in the header, in order (every field is one pointer)"""
    text = open(HEADER).read()
    body = re.search(r"typedef struct LtplBuffers \{(.*?)\} LtplBuffers;", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [m.group(1) for m in re.finditer(r"\*\s*(\w+)\s*;", body)]


def test_traj_base_kernel_has_no_stack_frame():
    frames = _stack_frames()
    k = [s for f, s in frames.items() if f.startswith("_Z11k_traj_base")]
    assert len(k) == 1, sorted(frames)
    assert k[0] == 0, k


def test_buffers_mirror_matches_header_and_library():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    lib = capi.load_library()
    names = _header_buffer_fields()
    assert tuple(names) == capi.BUFFER_FIELDS
    assert names[-1] == "traj_base" and names[-2] == "gg_map"
    assert lib.ltpl_sizeof(3) == ctypes.sizeof(capi.Buffers) == 8 * len(names)
    assert capi.Buffers.traj_base.offset == 8 * (len(names) - 1) == capi.Buffers.gg_map.offset + 8


def test_abi_version_is_20():
    from graphbasedlocaltrajectoryplanner_b200 import capi
    capi.build_library()
    assert re.search(r"#define LTPL_ABI_VERSION (\d+)", open(HEADER).read()).group(1) == "20"
    assert capi.ABI_VERSION == 20 and capi.load_library().ltpl_version() == 20
    assert hasattr(capi.load_library(), "ltpl_prepare_batch")
