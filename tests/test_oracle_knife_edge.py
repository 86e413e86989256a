"""The planner's float64 decisions at their exact boundaries, without a GPU (tests/golden/ticks_knife_edge.npz, made by
tests/tools/gen_golden_knife_edge.py; constructions in tests/knife_edge.py): the oracle takes the reference's decision on
both sides of every flip pair, on every exact tie and equality; the fixture covers what the device tests need; and every
flip pair changes the observable through which the device tests see it -- otherwise they could not notice a wrong
decision."""
import numpy as np
import pytest

from tests import knife_edge as K

SETS = ("default", "l216", "open")


@pytest.mark.parametrize("tag", SETS)
def test_oracle_reproduces_knife_edge_decisions(tag):
    g = K.golden_set(tag)
    orc = K.oracle_for(tag)
    for k, pair in enumerate(g["f1_p"]):
        assert [K.in_track(orc, p) for p in pair] == g["f1_in"][k].tolist(), ("F1", k)
    for k, pair in enumerate(g["f2_p"]):
        assert [K.start_layer_of(orc, p) for p in pair] == g["f2_layer"][k].tolist(), ("F2", k)
    assert [K.start_layer_of(orc, p) for p in g["f2_tie_p"]] == g["f2_tie_layer"].tolist()
    for k in range(g["f3_h"].shape[0]):
        assert [K.heading_ok(orc, h, g["f3_psi"][k]) for h in g["f3_h"][k]] == g["f3_ok"][k].tolist(), ("F3", k)
        assert K.ego_pose(orc, int(g["f3_layer"][k]))[1] == g["f3_psi"][k]
    for k, pair in enumerate(g["f4_p"]):
        assert [K.ref_layer(orc, p) for p in pair] == g["f4_layer"][k].tolist(), ("F4", k)
    assert [K.ref_layer(orc, p) for p in g["f4_tie_p"]] == g["f4_tie_layer"].tolist()
    for k, pair in enumerate(g["f5_p"]):
        pose = K.ego_pose(orc, int(g["f5_ego"][k]))
        assert [repr(K.paths_observable(orc, *pose, [K.obj(p)])) for p in pair] == g["f5_obs"][k].tolist(), ("F5", k)
    for k, p in enumerate(g["f5_eq_p"]):
        pose = K.ego_pose(orc, int(g["f5_ego"][g["f5_eq_case"][k]]))
        assert repr(K.paths_observable(orc, *pose, [K.obj(p)])) == g["f5_eq_obs"][k], ("F5 equality", k)
    assert [K.glob_start(orc, p) for p in g["f7_p"]] == g["f7_start"].tolist()
    for k, pair in enumerate(g["f6_p"]):
        ego, hd = g["f6_ego"][k], g["f6_hd"][k]
        assert [K.rl_s(orc, p) for p in pair] == g["f6_s"][k].tolist(), ("F6 s", k)
        assert [repr(K.paths_observable(orc, ego, hd, [K.obj(p)])) for p in pair] == g["f6_obs"][k].tolist(), ("F6", k)
    for k, p in enumerate(g["f6_eq_p"]):
        c = g["f6_eq_case"][k]
        assert repr(K.paths_observable(orc, g["f6_ego"][c], g["f6_hd"][c], [K.obj(p)])) == g["f6_eq_obs"][k], k
    for k, p in enumerate(g["f6r_p"]):
        assert K.rl_s(orc, p) == g["f6r_s"][k] and K.rl_s(orc, g["f6r_ego"][k]) == g["f6r_s0"][k], ("F6 race line", k)
        assert repr(K.paths_observable(orc, g["f6r_ego"][k], g["f6r_hd"][k], [K.obj(p)])) == g["f6r_obs"][k], k


@pytest.mark.parametrize("tag", SETS)
def test_every_flip_pair_changes_its_observable(tag):
    g = K.golden_set(tag)
    orc = K.oracle_for(tag)
    lt = orc.lat
    L = lt.num_layers
    # F1: the ego's in-track flag is the observable (SC_OUT_OF_TRACK); F1': the closest object, 0 on the track, else none
    assert np.all(g["f1_in"][:, 0] != g["f1_in"][:, 1])
    n_obj = 0
    for k, pair in enumerate(g["f1_p"]):
        for chunk2 in (False, True):
            sc = [K.f1_scenario(orc, p, chunk2) for p in pair]
            if sc[0] is None:
                continue
            obs = [K.paths_observable(orc, *s)[0] for s in sc]
            want = [0 if i else -1 for i in g["f1_in"][k]]
            assert obs == want, ("F1'", k, chunk2, obs, want)
            n_obj += 1
    assert n_obj >= g["f1_p"].shape[0]
    # F2: start node = (closest layer + 2) % (L - 1); ties: the two tied nodes lie in different layers
    st = (g["f2_layer"] + 2) % (L - 1)
    assert np.all(st[:, 0] != st[:, 1])
    for p in g["f2_tie_p"]:
        dd = K.d2(orc.node_xy, p)
        tied = np.nonzero(dd == dd.min())[0]
        assert tied.size >= 2 and len(set(orc.node_layer[tied].tolist())) >= 2, tied
    # F3
    assert np.all(g["f3_ok"][:, 0] != g["f3_ok"][:, 1])
    # F4: B is the closest object iff its point resolves to the layer before A's
    for (l, l2), pair, lay in zip(g["f4_l"], g["f4_p"], g["f4_layer"]):
        sc = [K.f4_scenario(orc, int(l), int(l2), p) for p in pair]
        if sc[0] is None:
            continue
        obs = [K.paths_observable(orc, *s)[0] for s in sc]
        assert obs == [int(v == l) for v in lay], (l, l2, obs, lay)
    for (l, l2), p, lay in zip(g["f4_tie_l"], g["f4_tie_p"], g["f4_tie_layer"]):
        dd = K.d2(lt.refline, p)
        assert dd[l] == dd[l2] == dd.min() and lay == min(l, l2)
        sc = K.f4_scenario(orc, int(l), int(l2), p)
        if sc is not None:
            assert K.paths_observable(orc, *sc)[0] == int(lay == l)
    # F5
    assert np.all(g["f5_obs"][:, 0] != g["f5_obs"][:, 1])
    for k, c in enumerate(g["f5_eq_case"]):
        assert g["f5_eq_obs"][k] in g["f5_obs"][c].tolist()
    # F6: the constant-segment check; an object at exactly oref from the ego position is IN the segment (<=)
    assert np.all(g["f6_obs"][:, 0] != g["f6_obs"][:, 1])
    oref = np.power(2.5 + lt.veh_width / 2, 2)
    for k, c in enumerate(g["f6_eq_case"]):
        d = np.power(g["f6_ego"][c][0] - g["f6_eq_p"][k][0], 2) + np.power(g["f6_ego"][c][1] - g["f6_eq_p"][k][1], 2)
        assert d == oref and g["f6_eq_obs"][k] in g["f6_obs"][c].tolist(), k
    # F6, race line: the neighbour choice puts the object's s on one or the other side of s_start, and so the object
    # beside the segment (closest object 0) or behind the start layer (none)
    beside = g["f6r_s"] >= g["f6r_s0"]
    assert beside.any() and (~beside).any()
    for k in range(g["f6r_p"].shape[0]):
        assert g["f6r_obs"][k].startswith("(0," if beside[k] else "(-1,"), k
    # F7: both signs of the angle gap around every vertex, with different answers
    for i in np.unique(g["f7_i"]):
        m = g["f7_i"] == i
        neg, pos = g["f7_start"][m & (g["f7_gap"] < 0)], g["f7_start"][m & (g["f7_gap"] > 0)]
        if neg.size and pos.size:
            assert set(neg.tolist()).isdisjoint(pos.tolist()), i


def test_knife_edge_coverage():
    """per family and lattice: flip pairs, exact ties / equalities, cases at the seam or the track ends, cell edges,
    warp-scan fallback lanes (F4 points > 60 m off the track), exact-path angle cases (1e-14 < |gap| <= 1e-10 rad),
    the four decisions of the constant-segment check and its race-line near-ties."""
    rows = []
    for tag in SETS:
        g = K.golden_set(tag)
        orc = K.oracle_for(tag)
        L = orc.lat.num_layers
        seam4 = int(np.sum(g["f4_l"][:, 0] == L - 1))
        seam4_ties = int(np.sum(g["f4_tie_l"][:, 0] == L - 1))
        wrap3 = int(np.sum(np.abs(g["f3_psi"]) > np.pi - 0.85))
        gap = np.abs(g["f7_gap"])
        c = dict(f1=g["f1_p"].shape[0], f1_seam_end=int(np.sum(g["f1_kind"] == 2)),
                 f1_cell_edge=int(np.sum(g["f1_kind"] == 3)), f1_vertex=int(np.sum(g["f1_kind"] == 1)),
                 f2=g["f2_p"].shape[0], f2_ties=g["f2_tie_p"].shape[0], f3=g["f3_h"].shape[0], f3_wrap=wrap3,
                 f4=g["f4_p"].shape[0], f4_ties=g["f4_tie_p"].shape[0], f4_fallback=int(g["f4_far"].sum()),
                 f4_seam=seam4, f5=g["f5_p"].shape[0], f5_equal=g["f5_eq_p"].shape[0],
                 f7=int(np.sum((gap > 1e-14) & (gap <= 1.5e-10))), f4_seam_ties=seam4_ties,
                 f6_start=int(np.sum(g["f6_kind"] == 0)), f6_end=int(np.sum(g["f6_kind"] == 1)),
                 f6_oref_first=int(np.sum(g["f6_kind"] == 2)), f6_oref_mid=int(np.sum(g["f6_kind"] == 3)),
                 f6_oref_equal=g["f6_eq_p"].shape[0], f6_raceline_ties=g["f6r_p"].shape[0])
        rows.append((tag, c))
        print("knife-edge coverage %-8s %s" % (tag, c))
        assert c["f1"] >= 40 and c["f1_seam_end"] >= 4 and c["f1_cell_edge"] >= 4 and c["f1_vertex"] >= 10, c
        assert c["f2"] >= 10 and c["f2_ties"] >= 10, c
        assert c["f3"] >= 20 and c["f3_wrap"] >= 2, c
        assert c["f4"] >= 10 and c["f4_ties"] >= 10 and c["f4_fallback"] >= 3, c
        assert c["f4_seam"] >= (2 if orc.lat.closed else 0), c
        assert c["f4_seam_ties"] >= (2 if orc.lat.closed else 0), c   # the wrap tie rule of lanes_closest_point
        assert min(c["f6_start"], c["f6_end"], c["f6_oref_first"], c["f6_oref_mid"]) >= 5, c
        assert c["f6_oref_equal"] >= 5 and c["f6_raceline_ties"] >= 30, c
        assert c["f5"] >= 8 and c["f5_equal"] >= 8, c
        assert c["f7"] >= 40, c
