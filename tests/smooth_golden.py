"""Comparison against the first-tick velocity-smoothing fixture (tests/golden/ticks_smooth.npz, made by
tests/tools/gen_golden_smooth.py): of every trajectory it holds the columns vx, ax of the whole profile, of the emergency
trajectory its exported rows; node sequences are exact, the rest uses the tolerances of tests/helpers.py."""
from tests import helpers as H

COLS = ("vx", "ax")
IDX = (5, 6)             # the same columns in a (P, 7) trajectory
N_EXPORT = 115


def compare_smooth_record(rec, g, b, ctx, exported=False):
    """rec: a tick record (oracle tick() or BatchPlanner.records()); g: one sub-set of the fixture (helpers._Sub).
    exported: also compare the exported fp32 rows (rec['traj']) and take the emergency trajectory from there."""
    ctx = "%s scenario %d" % (ctx, b)
    assert bool(rec["out_of_track"]) == bool(g["out_of_track"][b]), ctx + " out_of_track"
    if rec["out_of_track"]:
        return 0
    n_traj = 0
    for a, act in enumerate(H.ACTIONS):
        has = act in rec["paths"] and len(rec["paths"][act]) > 0
        assert has == (int(g["path_len"][b, a]) > 0), "%s: path %s present=%s" % (ctx, act, has)
        if has:
            nodes = [[-1 if v is None else int(v) for v in p] for p in rec["nodes"][act][0]]
            assert nodes == g["nodes"][b, a, :int(g["nodes_len"][b, a])].tolist(), ctx + " nodes " + act
            assert rec["paths"][act][0].shape[0] == int(g["path_len"][b, a]), ctx + " path length " + act
        tl = int(g["traj_len"][b, a])
        assert (act in rec["traj_full"]) == (tl > 0), "%s: trajectory %s present=%s" % (ctx, act, act in rec["traj_full"])
        if not tl:
            continue
        assert int(rec["ids"][act]) % 10 == int(g["traj_id"][b, a]) % 10, ctx + " id " + act
        full = rec["traj_full"][act][0]
        assert full.shape[0] == tl, ctx + " rows of " + act
        H.assert_close("traj[%s]" % act, full[:, IDX], g["traj"][b, a, :tl], COLS, ctx)
        if exported:
            rows = rec["traj"][act][0]
            assert rows.shape[0] == min(tl, N_EXPORT), ctx + " exported rows of " + act
            H.assert_close("export[%s]" % act, rows[:, IDX], g["traj"][b, a, :rows.shape[0]], COLS, ctx)
        n_traj += 1
    n_em = int(g["em_len"][b])
    em = (rec["traj"] if exported else rec["traj_full"]).get("emergency")
    assert (em is not None) == (n_em > 0), "%s: emergency present=%s, golden rows %d" % (ctx, em is not None, n_em)
    if n_em:
        assert int(rec["ids"]["emergency"]) % 10 == int(g["em_id"][b]) % 10, ctx + " emergency id"
        ne = min(n_em, N_EXPORT)
        assert em[0].shape[0] == (ne if exported else n_em), ctx + " emergency rows"
        H.assert_close("traj[emergency]", em[0][:ne, IDX], g["em_traj"][b, :ne], COLS, ctx, w_rel=H.W_REL_BRAKE)
    return n_traj
