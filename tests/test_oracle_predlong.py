"""Pins the oracle against golden vectors of objects with long 'prediction' arrays (tests/golden/ticks_predlong.npz, made
by tests/tools/gen_golden_predlong.py from the unmodified reference): up to 80 points per object, scenarios with far
more than 32 obstacle discs, and objects whose last point leaves the planning range (quirk q14: such an object is not
the closest object, although its earlier discs still block edges)."""
import numpy as np
import pytest

from tests import helpers as H

SETS = ("default", "l216", "open")


def subset(name):
    return H._Sub(H.golden("ticks_predlong.npz"), name, upcast=True)


@pytest.mark.parametrize("name", SETS)
def test_oracle_matches_reference_long_predictions(name):
    from oracle.ltpl_oracle import OracleLTPL
    sub = subset(name)
    n = sub["sc_pos"].shape[0]
    assert int((sub["n_disc"] > 32).sum()) > n // 2
    orc = OracleLTPL(H.lattice_for(str(sub["lattice"])))
    vk = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=sub.g["ax_max_machines"], safety_d=30.0)
    for b in range(n):
        rec = orc.tick(sub["sc_pos"][b], sub["sc_heading"][b], sub["sc_vel"][b], H.object_list(sub, b), vk)
        H.compare_first_tick(rec, sub, b, ctx="predlong " + name)


def test_fixture_covers_chunks_and_q14():
    """the fixture holds what the chunked disc stage has to get right: vehicles whose discs straddle a 32-disc chunk
    boundary, and objects that are on the track now but whose last prediction point is outside the planning range."""
    from oracle.ltpl_oracle import OracleLTPL
    n_all = sum(subset(s)["sc_pos"].shape[0] for s in SETS)
    n_long = sum(int((subset(s)["n_disc"] > 32).sum()) for s in SETS)
    assert 3 * n_long >= 2 * n_all
    assert any(int(subset(s)["n_disc"].max()) > 128 for s in SETS)
    straddle = 0
    for s in SETS:
        sub = subset(s)
        for b in range(sub["sc_pos"].shape[0]):
            d0 = 0
            for k in range(int(sub["sc_n_obj"][b])):
                m = int(sub["sc_n_pred"][b, k])
                d1 = d0 + 1 + (1 if m < 0 else m)
                straddle += int(d0 // 32 != (d1 - 1) // 32)
                d0 = d1
    assert straddle > 10
    # q14: the LAST point decides the object's layer -- with every array cut to its first point, the closest object
    # (or whether there is one) changes in some scenarios
    sub = subset("default")
    orc = OracleLTPL(H.lattice_for("default"))
    vk = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=sub.g["ax_max_machines"], safety_d=30.0)
    changed = 0
    for b in range(sub["sc_pos"].shape[0]):
        objs = H.object_list(sub, b)
        if bool(sub["out_of_track"][b]):
            continue
        short = [dict(o, prediction=o["prediction"][:1]) if len(o.get("prediction", ())) else o for o in objs]
        r_short = orc.tick(sub["sc_pos"][b], sub["sc_heading"][b], sub["sc_vel"][b], short, vk)
        c_short = -1 if r_short["closest_obj_index"] is None else int(r_short["closest_obj_index"])
        changed += int(c_short != int(sub["closest_obj_index"][b]))
    assert changed >= 1
    assert np.all(sub["sc_n_pred"] <= 80)
