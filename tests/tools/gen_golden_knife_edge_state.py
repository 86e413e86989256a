"""Golden vectors of the STATEFUL tick's float64 decisions at their exact boundaries (tests/knife_edge_state.py, families
G1-G5), on the default, "216 x 11" and open lattices.  Writes exactly one file and nothing else under the repository:

  tests/golden/ticks_knife_edge_state.npz   keys '<lattice>__<array>'

Each probe is a second tick on the memory of a HISTORY: the UNMODIFIED reference (oracle/gen_golden.py's
load_reference / make_ltpl) plans a first tick through Graph_LTPL (set_startpos, calc_paths, calc_vel_profile) for a
pose without objects, and the probe's second tick reads what it decides:
  G1 / G2   calc_paths with the executed action and a scripted clock: the reference measures calc_time = T - 0.0
            (the first tick ran at clock 0.0); with calc_time_safety = 1.0 and calc_time_buffer_len = 1, the values
            the online ini's [CALC_TIME] entries set, t_const = min(T, 0.5) = T.  Observables: the private __start_node
            after calc_paths and the constant segment's length (what OnlineTrajectoryHandler.calc_paths returns).
  G3 / G4   after one such calc_paths (t_const = T0), OnlineTrajectoryHandler.get_ref_idx -- the first call of
            Graph_LTPL.calc_vel_profile -- for each pos_est, with [DELAY] delaycomp = D (the handler's value of it) and
            __last_cut_idx restored between the calls.  Observables: cut_index_pos, cut_layer, cut_index_layer (from the
            updated __last_cut_idx), vel_plan and len(vel_course).
  G2 rows   the start node of EVERY row of the memory trajectory as the predicted position, by the reference's own
            get_s_coord on the memory's node coordinates (the call of OTH:384-386): t_const cannot reach rows behind
            0.5 s of trajectory time, and a row that lies on a node (the zero vector) is pinned here.
A history is re-planned from set_startpos for every G1 / G2 probe, since calc_paths replaces the memory.  t_const above
the reference's cap of 0.5 s is no decision of its own and is not stored.  Histories: two ordinary poses, the two
poses (of 48 candidates at 40 - 60 m/s) with the most start-node flips at or below the cap, on the open track a pose whose
trajectory stops at the track's end (v == 0), and the first pose again with its 'emergency' trajectory executed
(G4 only: get_ref_idx reads that trajectory's velocity, calc_brake_emergency.py).

The fixture stores each history's inputs and the reference's memory (executed trajectory rows s, x, y, vx, node list,
node coordinates, node indices, and the node indices of the second tick's first action), so that the replays of
tests/knife_edge_state.py run on it; this script asserts that they reproduce every observable.

Usage (from the repo root, needs the reference checkout):   python tests/tools/gen_golden_knife_edge_state.py
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

SETS = (("default", 9201, {}), ("l216", 9202, {"lat_resolution": 1.0, "lon_straight_step": 12.0}), ("open", 9203, {}))
ORDER = ("straight", "left", "right", "follow")   # the executed action: the first of these the first tick returned
T0 = 0.125          # t_const of the G3 / G4 probes' second tick
DELAY = 0.1         # [DELAY] delaycomp of the online ini (G1 - G3)
HMAX = 40
NEXP = 115
PRIV = "_OnlineTrajectoryHandler__"


TCAP = 0.5          # the reference's cap of t_const (OTH:375): larger values are not decisions of their own


def poses(tag, seed, n):
    """(pos, heading, vel) of n poses without objects (on the open track not on its last 200 m)"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    from tests import helpers as H
    tr = Track(H.track_csv_for(tag))
    sc = make_scenarios(tr, n, seed=seed, n_obj_min=0, n_obj_max=0, s_max=tr.length - 200.0 if tag == "open" else None)
    return [(sc.pos[b], float(sc.heading[b]), float(sc.vel[b])) for b in range(sc.size)]


def histories(ses, tag, seed, n_search=48):
    """[(pos, heading, vel, emergency)]: two ordinary poses; the two poses among n_search candidates (at 40 - 60 m/s)
    with the most G1 flips (start node moves) at or below TCAP, which the reference can decide; on the open track a pose on its last
    150 m (the trajectory stops there: v == 0); and the first pose once more with its 'emergency' trajectory executed"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    from tests import helpers as H
    from tests import knife_edge_state as KS
    out = [p + (False,) for p in poses(tag, seed, 2)]
    scored = []
    # fast candidates: 0.5 s of trajectory reach past the next node
    for j, c in enumerate((p, hd, 40.0 + 20.0 * (k % 3) / 2) for k, (p, hd, _) in enumerate(poses(tag, seed + 100,
                                                                                               n_search))):
        try:
            _, mem = ses.history(c + (False,))
        except AssertionError:   # a pose the reference rejects
            continue
        ties = [T for T, kind, _ in KS.g1_probes(mem) if kind == KS.G1_TIE and T <= TCAP]
        scored.append((-len(ties), j, c))
    scored.sort(key=lambda x: x[:2])
    out += [c + (False,) for nt, _, c in scored[:2] if nt < 0]
    if tag == "open":
        tr = Track(H.track_csv_for(tag))
        se = make_scenarios(tr, 1, seed=seed + 1, n_obj_min=0, n_obj_max=0, s_min=tr.length - 150.0,
                            s_max=tr.length - 60.0)
        out.append((se.pos[0], float(se.heading[0]), float(se.vel[0]), False))
    out.append(out[0][:3] + (True,))
    return out


class Session(object):
    """one reference Graph_LTPL with a scripted clock inside OnlineTrajectoryHandler"""

    def __init__(self, graph_ltpl, tag, overrides, csv):
        import graph_ltpl.online_graph.src.OnlineTrajectoryHandler as oth_mod
        self.ltpl, _ = GG.make_ltpl(graph_ltpl, "kes_" + tag, overrides, csv=csv)
        self.clock = GG.ScriptedClock()
        oth_mod.time = self.clock
        self.oth = self.ltpl._Graph_LTPL__oth
        from graph_ltpl.helper_funcs.src.get_s_coord import get_s_coord
        self.get_s_coord = get_s_coord   # the reference's own function (OTH:384-386 calls it on the memory nodes)
        self.vk = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
                       safety_d=30.0)
        self.recorded = None
        calc_paths = self.oth.calc_paths

        def recorder(*a, **kw):
            self.recorded = calc_paths(*a, **kw)
            return self.recorded
        self.oth.calc_paths = recorder

    def priv(self, name, value=None):
        if value is not None:
            setattr(self.oth, PRIV + name, value)
        return getattr(self.oth, PRIV + name)

    def history(self, h):
        """the first tick of history h at clock 0.0; returns the executed action and the memory: with h's emergency
        flag the 'emergency' trajectory (s, x, y of its base, the brake profile's vx) and the base's node lists"""
        pos, hd, vel, emerg = h
        self.clock.t = 0.0
        assert not self.ltpl.set_startpos(pos_est=np.array(pos), heading_est=hd, vel_est=vel)
        self.ltpl._Graph_LTPL__obj_zone = []
        self.ltpl._Graph_LTPL__obj_list_handler._ObjectListInterface__object_zones = []
        self.priv("calc_time_safety", 1.0)
        self.priv("calc_time_buffer_len", 1)
        self.priv("delaycomp", DELAY)
        self.ltpl.calc_paths(prev_action_id="straight", object_list=[])
        traj, _, _ = self.ltpl.calc_vel_profile(pos_est=np.array(pos), vel_est=vel, incl_emerg_traj=emerg, **self.vk)
        sel = self.priv("em_base_id") if emerg else next(a for a in ORDER if a in traj and len(traj[a]))
        bp = traj["emergency" if emerg else sel][0]
        ni = np.asarray(self.priv("last_action_set_node_idx")[sel][0])
        path = self.priv("last_action_set_path_param")[sel][0]
        nodes = [[-1 if v is None else int(v) for v in p] for p in self.priv("last_action_set_nodes")[sel][0]]
        return ("emergency" if emerg else sel), dict(traj=np.ascontiguousarray(bp[:, [0, 1, 2, 5]]),
                                                     node_xy=path[ni, 0:2].copy(), node_idx=ni,
                                                     nodes=np.array(nodes, dtype=np.int32))

    def second_paths(self, sel, T):
        """calc_paths of the second tick with t_const = T -> (start node, constant-segment length)"""
        self.clock.t = T
        self.ltpl.calc_paths(prev_action_id=sel, object_list=[])
        seg = self.recorded[3]
        return [int(v) for v in self.priv("start_node")], (0 if seg is None else int(seg.shape[0]))

    def ref_idx(self, sel, pos, D):
        """get_ref_idx of the second tick -> (cut_pos, cut_layer, cut_index_layer, vel_idx, vel_plan)"""
        keep = self.priv("last_cut_idx")
        self.priv("delaycomp", D)
        try:
            cut_pos, cut_layer, vel_plan, vel_course, _ = self.oth.get_ref_idx(action_id_sel=sel, idx_sel_traj=0,
                                                                              pos_est=np.asarray(pos))
            return int(cut_pos), int(cut_layer), int(cut_pos) - int(self.priv("last_cut_idx")), \
                int(len(vel_course)), float(vel_plan)
        finally:
            self.priv("last_cut_idx", keep)
            self.priv("delaycomp", DELAY)


def lattice_set(graph_ltpl, tag, seed, overrides):
    from tests import knife_edge_state as KS
    csv = None
    if tag == "open":
        from tests import helpers as H
        csv = H.OPEN_TRACK_CSV
    ses = Session(graph_ltpl, tag, overrides, csv)
    rng = np.random.default_rng(seed)
    hs = histories(ses, tag, seed)
    nh = len(hs)
    out = dict(h_pos=np.array([h[0] for h in hs]), h_heading=np.array([h[1] for h in hs]),
               h_vel=np.array([h[2] for h in hs]), h_em=np.array([h[3] for h in hs]),
               h_sel=np.zeros(nh, dtype=np.int32), h_n=np.zeros(nh, dtype=np.int32), h_traj=np.zeros((nh, NEXP, 4)),
               h_nn=np.zeros(nh, dtype=np.int32), h_node_xy=np.zeros((nh, HMAX, 2)),
               h_nodes=np.full((nh, HMAX, 2), -1, dtype=np.int32), h_node_idx=np.full((nh, HMAX), -1, dtype=np.int32),
               h_row_sni=np.full((nh, NEXP), -1, dtype=np.int32), h_nn2=np.zeros(nh, dtype=np.int32),
               h_node_idx2=np.full((nh, HMAX), -1, dtype=np.int32), t0=np.float64(T0), delay=np.float64(DELAY))
    g1, g3, g4 = [], [], []
    for i, h in enumerate(hs):
        sel, mem = ses.history(h)
        tr, n, nn = mem["traj"], mem["traj"].shape[0], mem["nodes"].shape[0]
        out["h_sel"][i] = 4 if h[3] else GG.ACTIONS.index(sel)
        out["h_n"][i], out["h_nn"][i] = n, nn
        out["h_traj"][i, :n] = tr
        out["h_node_xy"][i, :nn], out["h_nodes"][i, :nn], out["h_node_idx"][i, :nn] = \
            mem["node_xy"], mem["nodes"], mem["node_idx"]
        if not h[3]:
            # G2: the start node of every row as the predicted position, by the reference's get_s_coord (OTH:384-386)
            for r in range(n):
                sni = int(ses.get_s_coord(ref_line=mem["node_xy"], pos=tr[r, 1:3], only_index=True)[1][1])
                assert sni == KS.start_node_idx(mem["node_xy"], tr[r, 1:3]), (tag, i, r)
                out["h_row_sni"][i, r] = sni
            # G1 / G2 through calc_paths, one re-planned history per probe; t_const above TCAP is not a decision
            for T, kind, k in KS.g1_probes(mem) + KS.g2_probes(mem):
                if T > TCAP:
                    continue
                ses.history(h)
                start, clen = ses.second_paths(sel, T)
                sni = KS.memory_start(mem, T)
                assert start == mem["nodes"][sni].tolist(), (tag, i, T, start, sni)
                assert clen == int(mem["node_idx"][sni]) + 1, (tag, i, T, clen)
                g1.append((i, T, kind, k, start, clen, sni))
        # G3 / G4 on one second tick
        ses.history(h)
        ses.second_paths(sel, T0)
        ni2 = np.asarray(list(ses.priv("last_action_set_node_idx").values())[0][0])
        out["h_nn2"][i] = ni2.shape[0]
        out["h_node_idx2"][i, :ni2.shape[0]] = ni2
        p3 = [] if h[3] else [(p, DELAY, kind) for p, kind in KS.g3_probes(tr, rng)]
        p4 = [(p, D, kind) for p, D, kind, _ in KS.g4_probes(tr, KS.g4_rows(tr))]
        for rows, probes in ((g3, p3), (g4, p4)):
            for p, D, kind in probes:
                obs = ses.ref_idx(sel, p, D)
                rep = KS.ref_idx(tr, p, D, ni2, 0)
                assert obs[:4] == rep[:4] and obs[4] == rep[4] and rep[3] == rep[5].shape[0], (tag, i, kind, obs,
                                                                                               rep[:5])
                rows.append((i, p, D, kind) + obs)
    n1 = np.array([c[2] for c in g1])
    out.update(g1_h=np.array([c[0] for c in g1], dtype=np.int32), g1_T=np.array([c[1] for c in g1]),
               g1_kind=n1.astype(np.int32), g1_k=np.array([c[3] for c in g1], dtype=np.int32),
               g1_start=np.array([c[4] for c in g1], dtype=np.int32), g1_const_len=np.array([c[5] for c in g1],
                                                                                             dtype=np.int32),
               g1_sni=np.array([c[6] for c in g1], dtype=np.int32))
    for name, rows in (("g3", g3), ("g4", g4)):
        out.update({name + "_h": np.array([c[0] for c in rows], dtype=np.int32),
                    name + "_pos": np.array([c[1] for c in rows]).reshape(-1, 2),
                    name + "_D": np.array([c[2] for c in rows]),
                    name + "_kind": np.array([c[3] for c in rows], dtype=np.int32),
                    name + "_obs": np.array([c[4:8] for c in rows], dtype=np.int32).reshape(-1, 4),
                    name + "_vel_plan": np.array([c[8] for c in rows])})
    print("[knife_edge_state %s] %d histories (%s, emergency %s), G1/G2 %d probes (kinds %s), G3 %d (kinds %s), G4 %d (kinds %s)" % (
        tag, nh, out["h_sel"].tolist(), out["h_em"].tolist(), len(g1), np.bincount(n1, minlength=7).tolist(), len(g3),
        np.bincount(out["g3_kind"], minlength=7).tolist(), len(g4), np.bincount(out["g4_kind"], minlength=5).tolist()))
    return out


def main():
    graph_ltpl = GG.load_reference()
    out = {}
    for tag, seed, ov in SETS:
        out.update({"%s__%s" % (tag, k): v for k, v in lattice_set(graph_ltpl, tag, seed, ov).items()})
    np.savez_compressed(os.path.join(GG.GOLDEN, "ticks_knife_edge_state.npz"), **out)


if __name__ == "__main__":
    main()
