"""Long object lists without a GPU: the oracle reproduces the reference's golden vectors of 17-64 objects per scenario
(tests/golden/ticks_manyobj.npz), the fixture covers what k_plan's chunked object stage has to get right, and the planner
accepts any object list up to the shared-memory bound of k_plan and refuses a longer one up front."""
import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H

SETS = ("default", "l216", "open")


def subset(name):
    return H._Sub(H.golden("ticks_manyobj.npz"), name, upcast=True)


def vel_kwargs():
    return dict(D.VEL, ax_max_machines=H.golden("ticks_manyobj.npz")["ax_max_machines"])


@pytest.mark.parametrize("name", SETS)
def test_oracle_matches_reference_many_objects(name):
    from oracle.ltpl_oracle import OracleLTPL
    sub = subset(name)
    orc = OracleLTPL(H.lattice_for(str(sub["lattice"])))
    vk = vel_kwargs()
    for b in range(sub["sc_pos"].shape[0]):
        rec = orc.tick(sub["sc_pos"][b], sub["sc_heading"][b], sub["sc_vel"][b], H.object_list(sub, b), vk)
        H.compare_first_tick(rec, sub, b, ctx="manyobj " + name)


def _vehicles(orc, objs):
    """object slots of the on-track objects (the vehicle list, OLI:104-112), in list order"""
    from oracle.ltpl_oracle import check_inside_bounds
    return [k for k, o in enumerate(objs) if check_inside_bounds(orc.bound1, orc.bound2, [o['X'], o['Y']])]


def test_fixture_covers_chunks_and_rounds():
    """more than 32 slots with more than 30 on-track vehicles; a closest object with vehicle index >= 16 and one in slot
    >= 32; an object beside the constant path segment with vehicle index >= 30 (past the first s-coordinate round);
    prediction discs of a vehicle in slot >= 32."""
    from oracle.ltpl_oracle import OracleLTPL, get_s_coord
    big = coi16 = coi_slot32 = beside30 = pred32 = 0
    for s in SETS:
        sub = subset(s)
        orc = OracleLTPL(H.lattice_for(str(sub["lattice"])))
        lt = orc.lat
        vk = vel_kwargs()
        for b in range(sub["sc_pos"].shape[0]):
            objs = H.object_list(sub, b)
            veh = _vehicles(orc, objs)
            big += int(len(objs) > 32 and len(veh) > 30)
            pred32 += int(any(k >= 32 and int(sub["sc_n_pred"][b, k]) > 0 for k in veh))
            coi = int(sub["closest_obj_index"][b])
            if coi >= 0:
                coi16 += int(coi >= 16)
                coi_slot32 += int(veh[coi] >= 32)
            if bool(sub["out_of_track"][b]) or len(veh) <= 30:
                continue
            seg = orc.tick(sub["sc_pos"][b], sub["sc_heading"][b], sub["sc_vel"][b], objs, vk)["const_path_seg"]
            s0 = get_s_coord(lt.raceline, seg[0, 0:2], lt.s_raceline, closed=True)[0]
            s1 = get_s_coord(lt.raceline, seg[-1, 0:2], lt.s_raceline, closed=True)[0]
            for v in range(30, len(veh)):
                so = get_s_coord(lt.raceline, [objs[veh[v]]['X'], objs[veh[v]]['Y']], lt.s_raceline, closed=True)[0]
                beside30 += int(s0 <= so <= s1 or (s0 > s1 and (so > s0 or so < s1)))
    assert big >= 10, big
    assert coi16 >= 5 and coi_slot32 >= 5, (coi16, coi_slot32)
    assert beside30 >= 2, beside30
    assert pred32 >= 10, pred32


def test_planner_object_bound_without_gpu():
    """the planner accepts 17+ objects per scenario (the facade passes every 'physical' entry, on the track or not) and
    refuses a list beyond k_plan's shared-memory bound with a ValueError that names the bound."""
    from graphbasedlocaltrajectoryplanner_b200.Graph_LTPL import physical_objects
    from graphbasedlocaltrajectoryplanner_b200.lattice_blob import pack_lattice
    from graphbasedlocaltrajectoryplanner_b200.planner import check_object_count, max_objects
    for tag in ("default", "l216", "l430", "open"):
        header, _, cap = pack_lattice(H.lattice_for(tag))
        bound = max_objects(header, cap)
        assert 500 <= bound <= 1000, (tag, bound)
        assert max_objects(header, dict(cap, h_max=cap["h_max"] + 8)) <= bound   # a stateful planner's h_max
        for k in (17, 33, 64, 200, bound):
            assert check_object_count(k, bound) == k
        with pytest.raises(ValueError, match="at most %d" % bound):
            check_object_count(bound + 1, bound)
    ol = [{'id': k, 'type': 'physical' if k % 4 else 'static', 'X': float(k), 'Y': 0.0, 'theta': 0.0, 'v': 1.0,
           'length': 5.0} for k in range(40)]
    phys = physical_objects(ol)
    assert len(phys) == 30 and [o['id'] for o in phys] == [k for k in range(40) if k % 4]
    assert check_object_count(len(phys), bound) == 30
    assert np.all([o['type'] == 'physical' for o in phys])
