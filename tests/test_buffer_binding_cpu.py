"""The binding rule of BatchPlanner without a GPU: planner.buffer_sources on CPU tensors standing in for the planner's
device tables, for first ticks, planners with memory before and after their first stateful staging, every kind of
friction, export sets, a peer export and the id counter.  Every case names the table entry behind every bound field."""
from dataclasses import replace

import pytest
import torch

from graphbasedlocaltrajectoryplanner_b200 import capi
from graphbasedlocaltrajectoryplanner_b200.planner import CARRIED, SWAPPED, TickState, buffer_sources

FIELDS = capi.BUFFER_FIELDS
REQUIRED = FIELDS[:FIELDS.index("zone_bits")]   # ltpl validate(): never NULL
# the memory of a stateful tick; gg, gg_map and traj_base serve first ticks as well
MEMORY = tuple(n for n in capi.STATE_FIELDS if n not in ("gg", "gg_map", "traj_base"))
PER_BATCH = tuple(n for n in FIELDS if n not in capi.STATE_FIELDS and n != "traj")


def _tables(memory: bool):
    """stand-ins for BatchPlanner.t, _state, traj_bufs, the map, the id counter, peer rows and the last `pos`, and the
    name of every tensor in them"""
    t = {n: torch.zeros(1) for n in PER_BATCH + ("trim", "sel_action", "t_const", "gg")}
    state = None
    if memory:
        t["em_vx"] = torch.zeros(1)
        state = dict(other={k: torch.zeros(1) for k in SWAPPED + ("gg",)},
                     prev_small={k: torch.zeros(1) for k in CARRIED},
                     **{k: torch.zeros(1) for k in ("st_info", "vel_plan", "course", "obj_dist", "zone_s0", "restart")})
    extra = dict(traj_bufs=[torch.zeros(1) for _ in range(3)], gg_map=torch.zeros(1), traj_base=torch.zeros(1),
                 peer=torch.zeros(1), pos_last=torch.zeros(1))
    names = {id(v): "t." + k for k, v in t.items()}
    names.update({id(v): "traj_bufs[%d]" % i for i, v in enumerate(extra["traj_bufs"])})
    names.update({id(extra[k]): k for k in ("gg_map", "traj_base", "peer", "pos_last")})
    if state is not None:
        for group in ("other", "prev_small"):
            names.update({id(v): group + "." + k for k, v in state[group].items()})
        names.update({id(v): "state." + k for k, v in state.items() if isinstance(v, torch.Tensor)})
    return t, state, extra, names


FIRST = {**{n: "t." + n for n in PER_BATCH}, "traj": "traj_bufs[0]"}
WITH_MEMORY = {**FIRST, "trim": "t.trim", "em_vx": "t.em_vx", "zone_s0": "state.zone_s0"}
STAGED = {**WITH_MEMORY, **{"prev_" + k: "other." + k for k in SWAPPED},
          **{"prev_" + k: "prev_small." + k for k in CARRIED},
          **{k: "state." + k for k in ("st_info", "vel_plan", "course", "obj_dist")},
          "sel_action": "t.sel_action", "t_const": "t.t_const", "pos_last": "pos_last"}

# case: (memory, TickState fields, map, id counter, peer rows, expected field -> source; every other field NULL)
CASES = {
    "first_tick": (False, {}, False, False, False, FIRST),
    "memory_before_staging": (True, {}, False, False, False, WITH_MEMORY),
    "memory_staged": (True, dict(staged=True), False, False, False, STAGED),
    "memory_staged_restart": (True, dict(staged=True, restart=True), False, False, False,
                              {**STAGED, "restart": "state.restart"}),
    "host_planes": (False, dict(gg=True, gg_uploaded=True), False, False, False, {**FIRST, "gg": "t.gg"}),
    "device_planes": (False, dict(gg=True), False, False, False, {**FIRST, "gg": "t.gg"}),
    "map": (False, {}, True, False, False, {**FIRST, "gg": "t.gg", "gg_map": "gg_map"}),
    "planes_after_swap": (True, dict(staged=True, prev_gg=True), False, False, False,
                          {**STAGED, "prev_gg": "other.gg"}),
    "map_after_swap": (True, dict(staged=True, prev_gg=True, gg_planes_used=True), True, False, False,
                       {**STAGED, "prev_gg": "other.gg", "gg": "t.gg", "gg_map": "gg_map"}),
    "export_set": (False, dict(export=2), False, False, False, {**FIRST, "traj": "traj_bufs[2]"}),
    "peer_export": (True, dict(staged=True, export=1), False, False, True, {**STAGED, "traj": "peer"}),
    "id_counter": (False, {}, False, True, False, {**FIRST, "traj_base": "traj_base"}),
    "id_counter_staged": (True, dict(staged=True, restart=True), True, True, False,
                          {**STAGED, "restart": "state.restart", "gg": "t.gg", "gg_map": "gg_map",
                           "traj_base": "traj_base"}),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_binding_rule(case):
    memory, flags, with_map, with_counter, with_peer, expected = CASES[case]
    t, state, extra, names = _tables(memory)
    flags = dict(flags)
    tick = replace(TickState(), pos_last=extra["pos_last"] if flags.pop("staged", False) else None, **flags)
    src = buffer_sources(t, state, extra["traj_bufs"], tick, extra["gg_map"] if with_map else None,
                         extra["traj_base"] if with_counter else None, extra["peer"] if with_peer else None)
    assert tuple(src) == FIELDS   # every field decided
    assert all(v is None or isinstance(v, torch.Tensor) for v in src.values())
    assert all(src[n] is not None for n in REQUIRED)
    if not memory:
        assert all(src[n] is None for n in MEMORY)
    assert src["gg_map"] is None or src["gg"] is not None
    assert {n: names[id(v)] for n, v in src.items() if v is not None} == expected
