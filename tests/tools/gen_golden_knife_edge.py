"""Golden vectors of the planner's float64 decisions at their exact boundaries (tests/knife_edge.py): flip pairs
(adjacent doubles that decide differently), exact ties and exact equalities, on the default, "216 x 11" and open
lattices.  Writes exactly one file and nothing else under the repository:

  tests/golden/ticks_knife_edge.npz   keys '<lattice>__<array>'

The inputs are constructed on the lattices the planner builds (tests.helpers.lattice_for: the knife edges sit on THOSE
float64 values).  The decisions are taken by the UNMODIFIED reference functions, imported through
oracle/gen_golden.py's load_reference, called on those arrays:
  F1 / F1'  check_inside_bounds.py (ego and object in-track test)
  F2        closest_path_index.py over all nodes (its argpartition has no tie order, q10: exact ties keep np.argmin's
            first minimum, which the planner implements)
  F4        get_intersec_edges.py (obj_layer = min((val, idx)) over the reference line; a graph stub without edges)
  F7        get_s_coord.py on glob_rl (CVPF:166-172)
  F3        the heading test OTH:234-240 is inline code of the reference's set_initial_pose, restated in tests/knife_edge.py
            (checked here against the reference's Graph_LTPL.set_startpos on flip pairs built on the reference's own graph)
  F6        the constant-segment check MOPG:86-122: the race-line s coordinates by get_s_coord.py; the observable
            (closest object, node sequences) from the oracle, like F5
  F5        the collision observable (closest object, node sequences) needs whole first ticks on the lattice's own samples;
            it is taken from the oracle, which tests/test_oracle_golden.py pins against the reference's ticks

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_knife_edge
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

SETS = (("default", 9101), ("l216", 9102), ("open", 9103))


class _GraphStub(object):
    """what get_intersec_edges reads of a GraphBase: the reference line; no edges"""

    def __init__(self, refline):
        self.refline = refline

    def get_intersec_edges_in_range(self, **kw):
        return []


def lattice_set(tag, seed, ref):
    from graphbasedlocaltrajectoryplanner_b200 import lattice_blob as LB
    from oracle.ltpl_oracle import OracleLTPL
    from tests import helpers as H
    from tests import knife_edge as K
    lat = H.lattice_for(tag)
    LB.pack_lattice(lat)
    orc = OracleLTPL(lat)
    rng = np.random.default_rng(seed)
    inside = lambda p: bool(ref.check_inside_bounds(orc.bound1, orc.bound2, p))   # noqa: E731
    out = {}
    # F1 / F1'
    c1 = K.f1_cases(orc, rng)
    # a flip pair that ends on an exact tie of one of check_inside_bounds' arg-mins has no defined reference decision
    # (argpartition, q10): such pairs are left out
    n1 = len(c1)
    c1 = [c for c in c1 if [inside(c[0]), inside(c[1])] == [K.in_track(orc, c[0]), K.in_track(orc, c[1])]]
    print("[knife_edge %s] F1: %d flip pairs on an arg-min tie left out" % (tag, n1 - len(c1)))
    out["f1_p"] = np.array([[a, b] for a, b, _, _ in c1])
    out["f1_axis"] = np.array([ax for _, _, ax, _ in c1], dtype=np.int32)
    out["f1_kind"] = np.array([k for _, _, _, k in c1], dtype=np.int32)
    out["f1_in"] = np.array([[inside(a), inside(b)] for a, b, _, _ in c1])
    # F2
    c2 = K.f2_cases(orc, rng)
    def lay(p):
        idx, dd = ref.closest_path_index(orc.node_xy, p)
        if np.sum(dd == dd.min()) > 1:   # an exact tie (a flip pair may end on one): first minimum, q10
            return K.start_layer_of(orc, p)
        return int(orc.node_layer[int(idx[0])])
    out["f2_p"] = np.array([[a, b] for a, b, _, _ in c2])
    out["f2_axis"] = np.array([ax for _, _, ax, _ in c2], dtype=np.int32)
    out["f2_layer"] = np.array([[lay(a), lay(b)] for a, b, _, _ in c2], dtype=np.int32)
    ties = [t for c in c2 for t in c[3]]
    out["f2_tie_p"] = np.array(ties).reshape(-1, 2)
    out["f2_tie_layer"] = np.array([K.start_layer_of(orc, t) for t in ties], dtype=np.int32)   # first minimum (q10)
    # F3
    c3 = K.f3_cases(orc, rng)
    out["f3_layer"] = np.array([c[0] for c in c3], dtype=np.int32)
    out["f3_h"] = np.array([[c[2], c[3]] for c in c3])
    out["f3_psi"] = np.array([c[4] for c in c3])
    out["f3_ok"] = np.array([[K.heading_ok(orc, c[2], c[4]), K.heading_ok(orc, c[3], c[4])] for c in c3])
    # F4
    c4 = K.f4_cases(orc, rng)
    gie = lambda p: int(ref.get_intersec_edges(_GraphStub(lat.refline), p, 1.0)[1])   # noqa: E731
    out["f4_l"] = np.array([[c[0], c[1]] for c in c4], dtype=np.int32)
    out["f4_p"] = np.array([[c[2], c[3]] for c in c4])
    out["f4_far"] = np.array([c[5] for c in c4])
    out["f4_layer"] = np.array([[gie(c[2]), gie(c[3])] for c in c4], dtype=np.int32)
    t4 = [(c[0], c[1], t, c[5]) for c in c4 for t in c[4]]
    out["f4_tie_l"] = np.array([[a, b] for a, b, _, _ in t4], dtype=np.int32).reshape(-1, 2)
    out["f4_tie_p"] = np.array([t for _, _, t, _ in t4]).reshape(-1, 2)
    out["f4_tie_far"] = np.array([f for _, _, _, f in t4], dtype=bool)
    out["f4_tie_layer"] = np.array([gie(t) for _, _, t, _ in t4], dtype=np.int32)
    # F5
    c5 = K.f5_cases(orc, rng)
    out["f5_ego"] = np.array([c[0] for c in c5], dtype=np.int32)
    out["f5_p"] = np.array([[c[3], c[4]] for c in c5])
    out["f5_axis"] = np.array([c[5] for c in c5], dtype=np.int32)
    obs = lambda le, p: repr(K.paths_observable(orc, *K.ego_pose(orc, le), [K.obj(p)]))   # noqa: E731
    out["f5_obs"] = np.array([[obs(c[0], c[3]), obs(c[0], c[4])] for c in c5])
    # (kept where nothing but the equal sample decides: the observable is one of its pair's)
    e5 = [(i, e) for i, c in enumerate(c5) for e in c[6] if obs(c[0], e) in out["f5_obs"][i].tolist()]
    out["f5_eq_case"] = np.array([i for i, _ in e5], dtype=np.int32)
    out["f5_eq_p"] = np.array([e for _, e in e5]).reshape(-1, 2)
    out["f5_eq_obs"] = np.array([obs(int(out["f5_ego"][i]), e) for i, e in e5])
    # F7: only points where the object is on the track and becomes the closest object (its cobj_start is computed)
    c7 = K.f7_cases(orc, rng)
    f7 = []
    for i, pts, gaps in c7:
        for p, g in zip(pts, gaps):
            eb = K.ego_behind(orc, p)
            if abs(g) < 2e-14 or eb is None or not inside(p):
                continue
            if K.paths_observable(orc, *eb[1], [K.obj(p)])[0] != 0:
                continue
            s = int(ref.get_s_coord(K.glob_xy(orc), tuple(p), lat.glob_rl[:-1, 0], closed=True)[1][0])
            f7.append((i, p, g, s))
    out["f7_i"] = np.array([c[0] for c in f7], dtype=np.int32)
    out["f7_p"] = np.array([c[1] for c in f7]).reshape(-1, 2)
    out["f7_gap"] = np.array([c[2] for c in f7])
    out["f7_start"] = np.array([c[3] for c in f7], dtype=np.int32)
    # F6: the constant-segment check (own random stream: the arrays above stay as they were)
    rng6 = np.random.default_rng(seed + 6)
    s_ref = lambda p: float(ref.get_s_coord(lat.raceline, tuple(p), lat.s_raceline, closed=True)[0])   # noqa: E731
    c6 = K.f6_cases(orc, rng6)
    out["f6_kind"] = np.array([c[0] for c in c6], dtype=np.int32)
    out["f6_ego"] = np.array([c[1] for c in c6])
    out["f6_hd"] = np.array([c[2] for c in c6])
    out["f6_p"] = np.array([[c[3], c[4]] for c in c6])
    out["f6_axis"] = np.array([c[5] for c in c6], dtype=np.int32)
    out["f6_s"] = np.array([[s_ref(c[3]), s_ref(c[4])] for c in c6])
    obs6 = lambda c, p: repr(K.paths_observable(orc, c[1], c[2], [K.obj(p)]))   # noqa: E731
    out["f6_obs"] = np.array([[obs6(c, c[3]), obs6(c, c[4])] for c in c6])
    e6 = [(i, e) for i, c in enumerate(c6) for e in c[6]]
    out["f6_eq_case"] = np.array([i for i, _ in e6], dtype=np.int32)
    out["f6_eq_p"] = np.array([e for _, e in e6]).reshape(-1, 2)
    out["f6_eq_obs"] = np.array([obs6(c6[i], e) for i, e in e6])
    r6 = K.f6r_cases(orc, rng6)
    out["f6r_ego"] = np.array([c[0] for c in r6]).reshape(-1, 2)
    out["f6r_hd"] = np.array([c[1] for c in r6])
    out["f6r_p"] = np.array([c[2] for c in r6]).reshape(-1, 2)
    out["f6r_gap"] = np.array([c[3] for c in r6])
    out["f6r_s"] = np.array([s_ref(c[2]) for c in r6])
    out["f6r_s0"] = np.array([s_ref(c[0]) for c in r6])
    out["f6r_obs"] = np.array([repr(K.paths_observable(orc, c[0], c[1], [K.obj(c[2])])) for c in r6])
    print("[knife_edge %s] F6 %d pairs (kinds %s) + %d equalities, %d race-line near-ties" % (
        tag, len(c6), np.bincount(out["f6_kind"], minlength=4).tolist(), len(e6), len(r6)))
    print("[knife_edge %s] F1 %d pairs (kinds %s), F2 %d pairs + %d ties, F3 %d, F4 %d pairs (%d far) + %d ties, "
          "F5 %d pairs + %d equalities, F7 %d points" % (
              tag, len(c1), np.bincount(out["f1_kind"], minlength=4).tolist(), len(c2), len(ties), len(c3), len(c4),
              int(out["f4_far"].sum()), len(t4), len(c5), len(e5), len(f7)))
    return out


def check_heading_restatement(ltpl):
    """F3's decision is the inline heading test of the reference's set_initial_pose (OTH:234-240), restated in
    tests/knife_edge.heading_ok: on flip pairs built on the reference's OWN graph (its node positions and headings),
    Graph_LTPL.set_startpos must report out_of_track exactly where the restatement says the heading is off."""
    from tests import knife_edge as K
    gb = ltpl._Graph_LTPL__graph_base
    orc = K.oracle_for("default")
    n = 0
    for l in range(0, gb.num_layers - 2, 9):
        pos = np.asarray(gb.get_node_info(layer=l, node_number=int(gb.raceline_index[l]))[0], dtype=np.float64)
        goal = (l + 2) % (gb.num_layers - 1)
        psi = float(gb.get_node_info(layer=goal, node_number=int(gb.raceline_index[goal]))[1])
        f = lambda h: K.heading_ok(orc, h, psi)   # noqa: E731
        off = orc.p['max_heading_offset']
        for a, b in ((psi + off - 0.1, psi + off + 0.1), (psi - off + 0.1, psi - off - 0.1)):
            for h in K.bisect(f, a, b):
                oot = ltpl.set_startpos(pos_est=pos, heading_est=h, vel_est=10.0)
                assert bool(oot) == (not f(h)), (l, h, psi)
                n += 1
    print("[knife_edge] heading test: %d flip-pair sides agree with the reference's set_initial_pose" % n)


def main():
    GG.load_reference()
    from graph_ltpl.helper_funcs.src import closest_path_index, get_s_coord
    from graph_ltpl.online_graph.src import check_inside_bounds, get_intersec_edges

    class Ref(object):
        pass
    ref = Ref()
    ref.check_inside_bounds = check_inside_bounds.check_inside_bounds
    ref.closest_path_index = closest_path_index.closest_path_index
    ref.get_s_coord = get_s_coord.get_s_coord
    ref.get_intersec_edges = get_intersec_edges.get_intersec_edges
    check_heading_restatement(GG.make_ltpl(GG.load_reference(), "default", {})[0])
    out = {}
    for tag, seed in SETS:
        out.update({"%s__%s" % (tag, k): v for k, v in lattice_set(tag, seed, ref).items()})
    np.savez_compressed(os.path.join(GG.GOLDEN, "ticks_knife_edge.npz"), **out)


if __name__ == "__main__":
    main()
