"""The stateful tick's float64 decisions at their exact boundaries on the CPU (tests/golden/ticks_knife_edge_state.npz,
tests/knife_edge_state.py): the replays and the session oracle give the reference's decision on every fixture probe,
every flip pair changes its observable, and each family covers what it has to on every lattice."""
import numpy as np
import pytest

from tests import helpers as H
from tests import knife_edge as K
from tests import knife_edge_state as KS

SETS = ("default", "l216", "open")


def _set(tag):
    g = H.golden("ticks_knife_edge_state.npz")
    return {k.split("__", 1)[1]: g[k] for k in g.files if k.startswith(tag + "__")}


def _mem(g, h):
    n, nn = int(g["h_n"][h]), int(g["h_nn"][h])
    return dict(traj=g["h_traj"][h, :n], node_xy=g["h_node_xy"][h, :nn], nodes=g["h_nodes"][h, :nn],
                node_idx=g["h_node_idx"][h, :nn])


def _ni2(g, h):
    return g["h_node_idx2"][h, :int(g["h_nn2"][h])]


@pytest.mark.parametrize("tag", SETS)
def test_replays_reproduce_the_reference(tag):
    """next_idx / start_node_idx (G1, G2) and ref_idx (G3 - G5) on the reference's memory give the reference's start
    node, constant-segment length, cut index, cut layer, cut_index_layer, vel_plan and len(vel_course)"""
    g = _set(tag)
    for h in np.nonzero(~g["h_em"])[0]:   # every row as the predicted position (the reference's get_s_coord)
        mem = _mem(g, h)
        for r in range(int(g["h_n"][h])):
            assert KS.start_node_idx(mem["node_xy"], mem["traj"][r, 1:3]) == int(g["h_row_sni"][h, r]), (tag, h, r)
    for j in range(g["g1_T"].shape[0]):
        mem = _mem(g, int(g["g1_h"][j]))
        sni = KS.memory_start(mem, float(g["g1_T"][j]))
        assert sni == int(g["g1_sni"][j]), (tag, j)
        assert mem["nodes"][sni].tolist() == g["g1_start"][j].tolist(), (tag, j)
        assert int(mem["node_idx"][sni]) + 1 == int(g["g1_const_len"][j]), (tag, j)
    for fam in ("g3", "g4"):
        for j in range(g[fam + "_D"].shape[0]):
            h = int(g[fam + "_h"][j])
            r = KS.ref_idx(_mem(g, h)["traj"], g[fam + "_pos"][j], float(g[fam + "_D"][j]), _ni2(g, h), 0)
            assert list(r[:4]) == g[fam + "_obs"][j].tolist(), (tag, fam, j, r[:4])
            assert np.float64(r[4]).tobytes() == g[fam + "_vel_plan"][j].tobytes(), (tag, fam, j)
            assert r[5].shape[0] == r[3]


@pytest.mark.parametrize("tag", SETS)
def test_session_oracle_reproduces_the_reference(tag):
    """OracleSession's get_ref_idx and its start-node selection (oracle/ltpl_session.py), run on the reference's
    memory, give the reference's decisions"""
    from oracle.ltpl_oracle import get_s_coord
    from oracle.ltpl_session import OracleSession
    g = _set(tag)

    class _P(object):
        p = {}
    for fam in ("g3", "g4"):
        for j in range(g[fam + "_D"].shape[0]):
            h = int(g[fam + "_h"][j])
            tr = _mem(g, h)["traj"]
            bp = np.zeros((tr.shape[0], 7))
            bp[:, [0, 1, 2, 5]] = tr
            orc = _P()
            orc.p = dict(delaycomp=float(g[fam + "_D"][j]))
            ses = OracleSession(orc)
            ses.m_bp = {"straight": [bp]}
            ses.m_node_idx = {"straight": [_ni2(g, h)]}
            cut_pos, cut_layer, vel_plan, course = ses.get_ref_idx("straight", 0, g[fam + "_pos"][j])
            obs = g[fam + "_obs"][j].tolist()
            assert [cut_pos, cut_layer, cut_pos - ses.last_cut_idx, course.shape[0]] == obs, (tag, fam, j)
            assert np.float64(vel_plan).tobytes() == g[fam + "_vel_plan"][j].tobytes(), (tag, fam, j)
    # the start node: OracleSession.calc_paths takes get_s_coord(node_coords, predicted_pos)[1][1] (OTH:381-386)
    for j in range(g["g1_T"].shape[0]):
        mem = _mem(g, int(g["g1_h"][j]))
        tr = mem["traj"]
        p = tr[KS.next_idx(tr[:, 0], tr[:, 3], float(g["g1_T"][j])), 1:3]
        assert int(get_s_coord(mem["node_xy"], p, only_index=True)[1][1]) == int(g["g1_sni"][j]), (tag, j)


@pytest.mark.parametrize("tag", SETS)
def test_flip_pairs_change_the_observable(tag):
    """G1: T = cumsum[k] and its lower neighbour give different start nodes; G3: the two sides of a nearest-row or
    angle-rule flip pair give different cut indices; G4: D = cumsum[k] and its lower neighbour different vel_idx"""
    g = _set(tag)
    kind = g["g1_kind"]
    ties, below = np.nonzero(kind == KS.G1_TIE)[0], np.nonzero(kind == KS.G1_BELOW)[0]
    assert ties.size == below.size
    for a, b in zip(ties, below):
        assert g["g1_k"][a] == g["g1_k"][b] and g["g1_h"][a] == g["g1_h"][b]
        assert K.key(g["g1_T"][a]) - K.key(g["g1_T"][b]) == 1
        assert g["g1_sni"][a] != g["g1_sni"][b], (tag, a)
    for fk, obs in ((KS.G3_FLIP, lambda j: int(np.argmin(K.d2(_mem(g, int(g["g3_h"][j]))["traj"][:, 1:3],
                                                                g["g3_pos"][j])))),
                    (KS.G3_ANGLE, lambda j: int(g["g3_obs"][j, 0]))):
        idx = np.nonzero(g["g3_kind"] == fk)[0]
        assert idx.size % 2 == 0
        for a, b in zip(idx[0::2], idx[1::2]):   # the nearest row / the cut index
            assert obs(a) != obs(b), (tag, fk, a)
    t4, b4 = np.nonzero(g["g4_kind"] == KS.G4_TIE)[0], np.nonzero(g["g4_kind"] == KS.G4_BELOW)[0]
    assert t4.size == b4.size > 0
    for a, b in zip(t4, b4):
        assert K.key(g["g4_D"][a]) - K.key(g["g4_D"][b]) == 1
        nv = int(g["h_n"][g["g4_h"][a]]) - 1 - int(g["g4_obs"][a, 0])
        if int(g["g4_obs"][b, 3]) < nv - 1:   # (else the nv - 1 clamp decides both)
            assert g["g4_obs"][a, 3] != g["g4_obs"][b, 3], (tag, a)   # +1, or 1 where the tie makes all True


def test_no_last_row_cut():
    """a pos_est beyond the last row of the executed trajectory cuts at row n - 2, not at the last row: get_s_coord's
    idx2 is clipped to idx_nb there, so ang2 == 0 and ang1 >= ang2 holds; v_past keeps one row and vel_plan is the
    velocity of row n - 2.  LTPL_SC_REASON_LAST_ROW cannot arise from a trajectory of >= 3 rows."""
    n_beyond = 0
    for tag in SETS:
        g = _set(tag)
        for kind in (KS.G3_BEYOND, KS.G3_COLLINEAR):
            for j in np.nonzero(g["g3_kind"] == kind)[0]:
                h = int(g["g3_h"][j])
                n = int(g["h_n"][h])
                tr = _mem(g, h)["traj"]
                if int(np.argmin(K.d2(tr[:, 1:3], g["g3_pos"][j]))) != n - 1:
                    continue
                assert g["g3_obs"][j, 0] == n - 2 and g["g3_obs"][j, 3] == 0, (tag, j)
                assert g["g3_vel_plan"][j] == tr[n - 2, 3]
                n_beyond += 1
    assert n_beyond >= 6


MIN = {   # per lattice, from what the generator finds: G1 flip pairs (the start node moves at t_const <= 0.5 s, which
          # needs layers closer than 0.5 s of trajectory: only the "216 x 11" lattice has them), distinct rows reached
          # through t_const, G3 (flip / tie / angle / on row / before / beyond / collinear), G4 (tie pairs, all-True,
          # v == 0, probes on an executed 'emergency' trajectory)
    "default": dict(g1_pairs=0, g1_rows=10, g3=(40, 8, 30, 200, 6, 6, 4), g4_tie=18, g4_all=12, g4_inf=10, g4_em=24),
    "l216": dict(g1_pairs=2, g1_rows=20, g3=(80, 30, 40, 400, 9, 9, 6), g4_tie=30, g4_all=24, g4_inf=10, g4_em=24),
    "open": dict(g1_pairs=0, g1_rows=10, g3=(60, 20, 36, 250, 9, 9, 6), g4_tie=25, g4_all=12, g4_inf=20, g4_em=24),
}


@pytest.mark.parametrize("tag", SETS)
def test_knife_edge_state_coverage(tag):
    """counts of what the probes REACH: rows and start nodes through t_const, start nodes of every row (rows on nodes
    included), and the G3 / G4 kinds"""
    g = _set(tag)
    m = MIN[tag]
    c1 = np.bincount(g["g1_kind"], minlength=7)
    c3 = np.bincount(g["g3_kind"], minlength=7)
    c4 = np.bincount(g["g4_kind"], minlength=5)
    assert c1[KS.G1_TIE] >= m["g1_pairs"] and c1[KS.G1_ZERO] >= 1, c1
    assert all(T <= 0.5 for T in g["g1_T"]), "t_const above the reference's cap"
    reached, starts = set(), set()
    for j in range(g["g1_T"].shape[0]):
        h = int(g["g1_h"][j])
        tr = _mem(g, h)["traj"]
        reached.add((h, KS.next_idx(tr[:, 0], tr[:, 3], float(g["g1_T"][j]))))
        starts.add((h, int(g["g1_sni"][j])))
    assert len(reached) >= m["g1_rows"], sorted(reached)
    if m["g1_pairs"]:
        assert len(starts) > len({h for h, _ in starts}), "no history reaches a second start node through t_const"
    # every row of every history: the start nodes it reaches, rows on a node (the zero vector) among them
    on_node = 0
    for h in np.nonzero(~g["h_em"])[0]:
        n, mem = int(g["h_n"][h]), _mem(g, h)
        assert (g["h_row_sni"][h, :n] >= 0).all()
        assert len(set(g["h_row_sni"][h, :n].tolist())) >= 5, (tag, h)
        on_node += int(np.sum(mem["node_idx"] < n))
    assert on_node >= 10, on_node
    assert all(c3[k] >= v for k, v in enumerate(m["g3"])), c3
    assert c4[KS.G4_TIE] >= m["g4_tie"] and c4[KS.G4_ALL] >= m["g4_all"] and c4[KS.G4_INF] >= m["g4_inf"], c4
    em = np.nonzero(g["h_em"])[0]
    assert em.size == 1 and int(g["h_sel"][em[0]]) == 4
    in_em = g["g4_h"] == em[0]
    assert in_em.sum() >= m["g4_em"] and (g["g4_kind"][in_em] == KS.G4_INF).sum() >= 4
    assert (_mem(g, em[0])["traj"][:, 3] == 0.0).any(), "the executed 'emergency' trajectory reaches standstill"
    # the collinear points are bitwise collinear: both atan2 of get_s_coord's angle rule are equal
    for j in np.nonzero(g["g3_kind"] == KS.G3_COLLINEAR)[0]:
        tr = _mem(g, int(g["g3_h"][j]))["traj"]
        assert KS.collinear_angles(np.ascontiguousarray(tr[:, 1:3]), g["g3_pos"][j]) == (0.0, 0.0), (tag, j)


def test_v_zero_and_all_true_cases():
    """across the lattices: the delay compensation's cumsum reaches v == 0 (q11, inf) on the open track's end and on
    executed 'emergency' trajectories, and its all-True case is pinned; t_const's cap of 0.5 s keeps the reference's
    next_idx away from both (the device test covers them on the same replay, next_idx)"""
    c4 = sum(np.bincount(_set(t)["g4_kind"], minlength=5) for t in SETS)
    assert c4[KS.G4_INF] >= 1 and c4[KS.G4_ALL] >= 1
