"""Drivers the feature tests share: a planner and its first tick, the export rows and per-scenario snapshots of a tick,
batch invariance and oracle samples on one batch, the closed loop against the session oracle, and the replays of the
multi-tick fixtures on the device, through the Graph_LTPL facade and on the session oracle."""
import numpy as np

from tests import helpers as H

VEL = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)
EXPORT_COLS = ("s", "x", "y", "psi", "kappa", "vx", "ax")


class Clock(object):
    """a scripted clock in place of time.time(): the caller advances t"""

    def __init__(self, t):
        self.t = t

    def __call__(self):
        return self.t


def planner(lat, windows=4, stateful=False, online=None, **vel):
    """a BatchPlanner on cuda:0 with `windows` scenario windows (None: the library's default); vel: set_vel_params
    arguments over VEL"""
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    pl = BatchPlanner(lat, online=online, device="cuda:0", stateful=stateful)
    if windows is not None:
        pl.set_subbatches(windows)
    pl.set_vel_params(**dict(VEL, **vel))
    return pl


def first_tick(pl, sc, vel_est=None, gg=False):
    """set_startpos + tick; gg: local_gg planes (H.local_gg_field) along the planned paths between the two halves"""
    pl.stage_scenarios(sc, vel_est=vel_est)
    pl.upload()
    pl.set_startpos()
    if gg:
        pl.calc_paths()
        pl.set_local_gg_planes(*H.local_gg_planes(pl))
        pl.calc_vel_profile()
    else:
        pl.tick()


def facade(tmp_path, online_ini=H.ONLINE_INI):
    """a Graph_LTPL facade on cuda:0 with its lattice built (graph_init)"""
    from graphbasedlocaltrajectoryplanner_b200.Graph_LTPL import Graph_LTPL
    pd = {'globtraj_input_path': H.TRACK_CSV, 'graph_store_path': str(tmp_path / "lattice.npz"),
          'ltpl_offline_param_path': H.OFFLINE_INI, 'ltpl_online_param_path': str(online_ini)}
    ltpl = Graph_LTPL(path_dict=pd, visual_mode=False, log_to_file=False, device="cuda:0")
    ltpl.graph_init()
    return ltpl


def export_rows(f, cut=False):
    """[NSLOT][B][rows][7] rows of the compact export, gathered through traj_row (their order there is unspecified);
    zero in empty slots and, with cut, behind traj_len"""
    rows = np.zeros(f["traj_row"].shape + f["traj"].shape[1:], dtype=np.float32)
    ok = f["traj_row"] >= 0
    rows[ok] = f["traj"][f["traj_row"][ok]]
    if cut:
        rows[np.arange(rows.shape[2])[None, None, :] >= f["traj_len"][..., None]] = 0.0
    return rows


def tick_snapshot(pl, emergency=True):
    """the results of a BatchPlanner's last tick as arrays that are byte-comparable across runs, each with the scenario
    on axis 1 (per-scenario entries get a leading axis of 1): entries behind the valid lengths are cleared.  emergency:
    with the emergency trajectory (em_len, em_rows)."""
    f = pl.fetch("action_id", "status", "n_nodes", "nodes", "path_len", "traj_len", "traj_row", "traj", "em_info",
                 "sc_flags")
    nodes = f["nodes"].copy()
    nodes[np.arange(nodes.shape[2])[None, None, :] >= f["n_nodes"][..., None]] = -1
    snap = dict(action_id=f["action_id"], status=f["status"], nodes=nodes, path_len=f["path_len"],
                traj_len=f["traj_len"], rows=export_rows(f, cut=True), flags=f["sc_flags"][None])
    if emergency:
        em = f["em_info"]
        em_rows = f["traj"][np.maximum(em[:, 0], 0)] * (em[:, 0] >= 0)[:, None, None]
        snap.update(em_len=em[None, :, 1], em_rows=em_rows[None])
    return snap


def take(snap, idx):
    """scenarios idx of a tick_snapshot"""
    return {k: v[:, idx] for k, v in snap.items()}


def assert_batch_invariance(lat, sc, perm, part, **vel):
    """sc planned with 4 scenario windows gives the bytes of 1 and 3 windows, of the permuted batch sc.subset(perm) and
    of the sub-batch sc.subset(part) (2 windows), scenario by scenario; returns the 4-window planner"""
    pl = planner(lat, 4, **vel)
    first_tick(pl, sc)
    ref = tick_snapshot(pl, emergency=False)
    for windows in (1, 3):
        pw = planner(lat, windows, **vel)
        first_tick(pw, sc)
        got = tick_snapshot(pw, emergency=False)
        for k in ref:
            assert np.array_equal(ref[k], got[k]), "'%s' differs between 4 and %d scenario windows" % (k, windows)
    pp = planner(lat, 4, **vel)
    first_tick(pp, sc.subset(perm))
    got = take(tick_snapshot(pp, emergency=False), np.argsort(perm))
    for k in ref:
        assert np.array_equal(ref[k], got[k]), "'%s' depends on the order of the batch" % k
    ps_ = planner(lat, 2, **vel)
    first_tick(ps_, sc.subset(part))
    got, want = tick_snapshot(ps_, emergency=False), take(ref, part)
    for k in want:
        assert np.array_equal(want[k], got[k]), "'%s' differs in a sub-batch" % k
    return pl


def assert_sample_matches_oracle(pl, orc, sc, pick, vk, ctx, emergency=False):
    """scenarios pick of pl's last tick on sc against OracleLTPL.tick (H.compare_records), failures collected over the
    sample.  emergency: records() lists 'emergency' with the exported rows only; it is compared apart, on the exported
    rows at the brake-profile tolerance."""
    fails = []
    for rec, b in zip(pl.records(indices=pick.tolist()), pick):
        want = orc.tick(sc.pos[b], sc.heading[b], sc.vel[b], sc.object_list(int(b)), vk)
        c = "%s scenario %d" % (ctx, b)
        try:
            em_g = em_w = None
            if emergency and not rec["out_of_track"]:
                em_g = rec["traj"].pop("emergency", None)
                rec["ids"].pop("emergency", None)
            if emergency and not want["out_of_track"]:
                em_w = want["traj"].pop("emergency", None)
                want["traj_full"].pop("emergency", None)
                want["ids"].pop("emergency", None)
            H.compare_records(rec, want, ctx=c)
            assert (em_g is None) == (em_w is None), c + " emergency presence"
            if em_w is not None:
                H.assert_close("traj[emergency]", em_g[0], em_w[0], EXPORT_COLS, c, w_rel=H.W_REL_BRAKE)
        except AssertionError as e:
            fails.append(str(e).split("\n")[0][:300])
    assert not fails, "%d/%d sampled scenarios differ from the oracle:\n%s" % (len(fails), len(pick),
                                                                              "\n".join(fails[:8]))


def _nodes(nodes):
    return [[-1 if v is None else int(v) for v in p] for p in nodes]


def closed_loop_vs_session(pl, lat, sc0, rng, vel, prefer, end_flags, batch=None, n_ticks=8):
    """a closed loop driven by the device results on the stateful planner pl: the vehicle dummy of oracle/gen_golden.py
    on the selected trajectory (the first of a rotating action preference `prefer` the tick returned), opponents moving
    straight on, t_const from the moving average of the tick times; one session oracle per sequence replays the same
    inputs tick by tick.  Every tick draws its tick times from rng first, then moves the objects.  batch: maps each
    tick's ScenarioBatch to the one planned.  A sequence leaves the loop when the device flags it out of track or with
    one of end_flags, when the oracle raises, or when no preferred trajectory is left.  Returns the counts: ticks and
    trajectories compared, sequences that fell back (state fallback) or were flagged (end_flags), ticks flagged
    SC_CAPACITY that were still compared, sequences alive at the end."""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    from oracle.gen_golden import advance_on_traj
    from oracle.ltpl_oracle import OracleLTPL
    from oracle.ltpl_session import OracleSession
    n_seq = sc0.size
    clks = [Clock(50.0) for _ in range(n_seq)]
    ses = [OracleSession(OracleLTPL(lat), clock=clks[q]) for q in range(n_seq)]
    objs = sc0.obj.copy()
    pos_est, vel_est = sc0.pos.copy(), sc0.vel.copy()
    sel = ["straight"] * n_seq
    cbuf = [[] for _ in range(n_seq)]
    alive = np.ones(n_seq, dtype=bool)
    last_traj = [None] * n_seq
    fails, n = [], dict(ticks=0, traj=0, fell_back=0, flagged=0, capacity=0)
    for k in range(n_ticks):
        dts = rng.uniform(0.04, 0.16, size=n_seq)
        tcs = np.zeros(n_seq)
        for q in range(n_seq):
            dt = float(dts[q])
            clks[q].t += dt
            m = int(sc0.n_obj[q])
            objs[q, :m, 0] -= np.sin(objs[q, :m, 2]) * objs[q, :m, 3] * dt
            objs[q, :m, 1] += np.cos(objs[q, :m, 2]) * objs[q, :m, 3] * dt
            if k > 0:
                if last_traj[q] is not None:
                    pos_est[q], vel_est[q] = advance_on_traj(last_traj[q], dt)
                if len(cbuf[q]) >= 5:
                    cbuf[q].pop(0)
                cbuf[q].append(dt)
                tcs[q] = min(float(np.sum(cbuf[q]) / len(cbuf[q])) * 2.0, 0.5)
        sc = ScenarioBatch(pos_est.copy(), sc0.heading.copy(), sc0.vel.copy(), sc0.n_obj.copy(), objs.copy(),
                           pred=sc0.pred, n_pred=sc0.n_pred)
        if batch is not None:
            sc = batch(sc)
        if k == 0:
            first_tick(pl, sc, vel_est=vel_est)
        else:
            pl.next_tick(sc, sel_action=[H.ACTIONS.index(a) for a in sel], t_const=tcs, vel_est=vel_est)
        recs = pl.records()
        for q in range(n_seq):
            if not alive[q]:
                continue
            ctx = "sequence %d tick %d (sel %s)" % (q, k, sel[q])
            rec = recs[q]
            if rec["out_of_track"] or (rec["flags"] & end_flags):
                alive[q] = False
                n["fell_back"] += int(bool(rec["flags"] & capi.SC_STATE_FALLBACK))
                n["flagged"] += int(not rec["out_of_track"])
                continue
            try:
                if k == 0:
                    assert ses[q].set_startpos(sc.pos[q], sc.heading[q], sc.vel[q]) is False
                paths = ses[q].calc_paths(sel[q], sc.object_list(q))
                traj, _ = ses[q].calc_vel_profile(sc.pos[q], float(vel_est[q]), **vel)
            except Exception:   # noqa: BLE001  (e.g. the reference's own brake-prefix failure)
                alive[q] = False
                continue
            n["capacity"] += int(bool(rec["flags"] & capi.SC_CAPACITY))
            try:
                assert sorted(rec["paths"]) == sorted(paths), "%s: paths %s vs %s" % (ctx, sorted(rec["paths"]),
                                                                                   sorted(paths))
                for act in paths:
                    if ses[q].tie.get(act) or rec["tie"].get(act):
                        continue
                    nd = _nodes(rec["nodes"][act][0])
                    want = _nodes(ses[q].m_nodes[act][0]) if act in ses[q].m_nodes else None
                    assert want is None or nd == want, "%s: nodes of %s\n got  %s\n want %s" % (ctx, act, nd, want)
                    assert rec["paths"][act][0].shape[0] == paths[act][0].shape[0], ctx + " path length " + act
                assert sorted(rec["traj"]) == sorted(traj), "%s: trajectories %s vs %s" % (ctx, sorted(rec["traj"]),
                                                                                        sorted(traj))
                for act in traj:
                    assert rec["traj"][act][0].shape == traj[act][0].shape, ctx + " rows " + act
                    H.assert_close("traj[%s]" % act, rec["traj"][act][0], traj[act][0], EXPORT_COLS, ctx)
                    n["traj"] += 1
                n["ticks"] += 1
            except AssertionError as e:
                fails.append(str(e).split("\n")[0][:400])
                alive[q] = False
                continue
            cand = [a for a in prefer[(q + k) % len(prefer)] if a in rec["traj"]]
            if not cand:
                alive[q] = False
                continue
            sel[q] = cand[0]
            last_traj[q] = rec["traj"][sel[q]][0]
    n["alive"] = int(alive.sum())
    assert not fails, "%d sequences diverged (%d ticks matched, %d fell back):\n%s" % (
        len(fails), n["ticks"], n["fell_back"], "\n".join(fails[:8]))
    print("closed loop: %d of %d ticks compared, %d trajectories, %d sequences fell back, %d alive at the end" % (
        n["ticks"], n_seq * n_ticks, n["traj"], n["fell_back"], n["alive"]))
    return n


class Rows(object):
    """the sequences `idx` of a multi-tick fixture (gg_scale is a per-batch parameter: grip-drop sequences run apart)."""

    def __init__(self, g, idx):
        self.g, self.idx, self.files = g, np.asarray(idx), g.files

    def __getitem__(self, k):
        a = self.g[k]
        return a if k == "ax_max_machines" else a[self.idx]


def t_const(dts):
    """OTH:353-375: moving average (5) of the calculation times * calc_time_safety (2.0), capped at 0.5 s."""
    buf, out = [], []
    for dt in dts:
        if len(buf) >= 5:
            buf.pop(0)
        buf.append(float(dt))
        out.append(min(float(np.sum(buf) / len(buf)) * 2.0, 0.5))
    return out


def compare_multitick_row(rec, g, q, k, ctx, emergency):
    """a tick record against sequence q, tick k of a multi-tick fixture: path and trajectory sets, node sequences and
    path lengths (unless the cost ties), exported rows at the parity tolerance, with emergency also the emergency
    trajectory; returns the number of compared trajectories"""
    compared = 0
    for a, act in enumerate(H.ACTIONS):
        n_want = int(g["path_len"][q, k, a])
        has = act in rec["paths"]
        assert has == (n_want > 0), "%s: path %s present=%s, golden %d" % (ctx, act, has, n_want)
        if has and not rec["tie"].get(act):
            nd = _nodes(rec["nodes"][act][0])
            want = g["nodes"][q, k, a, :int(g["nodes_len"][q, k, a])].tolist()
            assert nd == want, "%s: nodes of %s\n got  %s\n want %s" % (ctx, act, nd, want)
            assert rec["paths"][act][0].shape[0] == n_want, "%s: path length %s %d vs %d" % (
                ctx, act, rec["paths"][act][0].shape[0], n_want)
        t_want = int(g["traj_len"][q, k, a])
        t_has = act in rec["traj"]
        assert t_has == (t_want > 0), "%s: trajectory %s present=%s, golden %d" % (ctx, act, t_has, t_want)
        if t_has:
            assert rec["traj"][act][0].shape[0] == t_want, "%s: rows of %s %d vs %d" % (
                ctx, act, rec["traj"][act][0].shape[0], t_want)
            H.assert_close("traj[%s]" % act, rec["traj"][act][0], g["traj"][q, k, a, :t_want], EXPORT_COLS, ctx)
            compared += 1
    if emergency:
        n_em = min(int(g["em_len"][q, k]), 115)
        assert ("emergency" in rec["traj"]) == (n_em > 0), ctx + " emergency presence"
        if n_em:
            H.assert_close("traj[emergency]", rec["traj"]["emergency"][0], g["em_traj"][q, k, :n_em], EXPORT_COLS,
                           ctx, w_rel=H.W_REL_BRAKE)
    return compared


def fixture_objects(g, q, k):
    """object list of sequence q, tick k of a multi-tick fixture"""
    return [{'id': j + 1, 'type': 'physical', 'X': float(o[0]), 'Y': float(o[1]), 'theta': float(o[2]),
             'v': float(o[3]), 'length': float(o[4]), 'width': 2.5}
            for j, o in enumerate(g["obj"][q, k, :int(g["sc_n_obj"][q])])]


def replay_facade(ltpl, g, seqs, emergency):
    """sequences seqs of a multi-tick fixture through the Graph_LTPL facade with the reference's call sequence
    (main_std_example.py:99-126) and a scripted clock in place of time.time(); returns the number of compared
    trajectories"""
    clk = Clock(10.0)
    ltpl.clock = clk
    compared = 0
    for q in seqs:
        assert ltpl.set_startpos(pos_est=g["sc_pos"][q], heading_est=g["sc_heading"][q], vel_est=g["sc_vel"][q]) is False
        for k in range(int(g["n_done"][q])):
            clk.t += float(g["dt"][q, k])
            paths = ltpl.calc_paths(prev_action_id=(H.ACTIONS + ("emergency",))[int(g["sel"][q, k])],
                                    object_list=fixture_objects(g, q, k))
            traj, ids, _ = ltpl.calc_vel_profile(pos_est=g["pos_est"][q, k], vel_est=float(g["vel_est"][q, k]),
                                                 ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emergency,
                                                 **dict(VEL, gg_scale=float(g["gg_scale"][q, k])))
            ctx = "facade sequence %d tick %d" % (q, k)
            for a, act in enumerate(H.ACTIONS):
                assert (act in paths) == (int(g["path_len"][q, k, a]) > 0), ctx + " paths " + act
                t_want = int(g["traj_len"][q, k, a])
                assert (act in traj) == (t_want > 0), ctx + " trajectories " + act
                if t_want:
                    H.assert_close("traj[%s]" % act, traj[act][0], g["traj"][q, k, a, :t_want], EXPORT_COLS, ctx)
                    compared += 1
            if emergency and int(g["em_len"][q, k]):
                H.assert_close("traj[emergency]", traj["emergency"][0], g["em_traj"][q, k, :int(g["em_len"][q, k])],
                               EXPORT_COLS, ctx, w_rel=H.W_REL_BRAKE)
    return compared


def replay_session_oracle(fixture, emergency, lattice, online=None, veh=None, vel=None, ggpp=False):
    """every sequence of a multi-tick fixture on its own session oracle (oracle/ltpl_session.py) with a scripted clock,
    against the reference's path sets, node sequences, path lengths, trajectory ids and trajectories.  online, veh:
    OracleLTPL arguments; vel: calc_vel_profile arguments over VEL; ggpp: location dependent local_gg
    (H.local_gg_field) along every path."""
    from oracle.ltpl_oracle import OracleLTPL
    from oracle.ltpl_session import OracleSession
    g = H.golden(fixture)
    lat = H.lattice_for(lattice)
    vk = dict(VEL, ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emergency, **(vel or {}))
    if ggpp:
        vk.pop("local_gg")
    orc_kw = dict(veh or {}, **({} if online is None else dict(online=online)))
    n_seq, n_ticks = g["dt"].shape
    compared = 0
    for q in range(n_seq):
        if int(g["n_done"][q]) == 0:
            continue
        clock = Clock(1000.0)
        ses = OracleSession(OracleLTPL(lat, **orc_kw), clock=clock)
        assert ses.set_startpos(g["sc_pos"][q], g["sc_heading"][q], g["sc_vel"][q]) is False
        for k in range(int(g["n_done"][q])):
            ctx = "sequence %d tick %d" % (q, k)
            clock.t += float(g["dt"][q, k])
            sel = (H.ACTIONS + ("emergency",))[int(g["sel"][q, k])]   # 4: OTH:307-309
            paths = ses.calc_paths(sel, fixture_objects(g, q, k), blocked_zones=H.zone_of(g, q, k))
            for a, act in enumerate(H.ACTIONS):
                n_want = int(g["path_len"][q, k, a])
                assert (act in paths) == (n_want > 0), "%s: path %s present=%s, golden %d" % (ctx, act, act in paths,
                                                                                            n_want)
                if n_want:
                    assert paths[act][0].shape[0] == n_want, ctx + " path length " + act
                    nd = _nodes(ses.m_nodes[act][0])
                    assert nd == g["nodes"][q, k, a, :int(g["nodes_len"][q, k, a])].tolist(), ctx + " nodes " + act
            kw = dict(vk, gg_scale=float(g["gg_scale"][q, k]))   # grip-drop fixtures
            if ggpp:
                kw["local_gg"] = {a: [H.local_gg_field(p[0][:, 0:2])] for a, p in paths.items()}
            traj, ids = ses.calc_vel_profile(g["pos_est"][q, k], float(g["vel_est"][q, k]), **kw)
            for a, act in enumerate(H.ACTIONS):
                t_want = int(g["traj_len"][q, k, a])
                assert (act in traj) == (t_want > 0), "%s: trajectory %s present=%s, golden %d" % (ctx, act, act in traj,
                                                                                                 t_want)
                if t_want:
                    # the id base (+10 per calc_vel_profile call, OTH:669) is instance state of the reference
                    assert ids[act] % 10 == int(g["traj_id"][q, k, a]) % 10, ctx + " id " + act
                    H.assert_close("traj[%s]" % act, traj[act][0], g["traj"][q, k, a, :t_want], EXPORT_COLS, ctx)
                    compared += 1
            if emergency:
                n_em = int(g["em_len"][q, k])
                assert ("emergency" in traj) == (n_em > 0), ctx + " emergency"
                if n_em:
                    H.assert_close("traj[emergency]", traj["emergency"][0], g["em_traj"][q, k, :n_em], EXPORT_COLS, ctx)
    assert compared > (40 if n_seq < 12 else (80 if n_seq < 16 else 150))
