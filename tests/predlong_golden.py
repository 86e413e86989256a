"""Comparison against the long-prediction fixture (tests/golden/ticks_predlong.npz, made by
tests/tools/gen_golden_predlong.py).  It holds what the obstacle discs decide: the action sets, node sequences and node
indices (exact), reduced-horizon flags, the closest object, and of every trajectory its length, id and the columns vx, ax
of the whole profile (tolerances of tests/helpers.py).  Paths are compared by their length: at equal node sequences the
other first-tick fixtures pin their geometry."""
import numpy as np

from tests import helpers as H

SETS = ("default", "l216", "open")
COLS = ("vx", "ax")
IDX = (5, 6)             # the same columns in a (P, 7) trajectory
N_EXPORT = 115


class Subset(H._Sub):
    """one sub-set of the fixture; the prediction points are stored as float32 (they are float32-representable) and are
    handed out as the float64 arrays the reference was given."""

    def __getitem__(self, k):
        v = super().__getitem__(k)
        return v.astype(np.float64) if k == "sc_pred" else v


def subset(name):
    return Subset(H.golden("ticks_predlong.npz"), name)


def compare_predlong_record(rec, g, b, ctx, exported=False):
    """rec: a tick record (oracle tick() or BatchPlanner.records()); g: a Subset.  exported: also compare the exported
    fp32 rows (rec['traj'])."""
    ctx = "%s scenario %d" % (ctx, b)
    assert bool(rec["out_of_track"]) == bool(g["out_of_track"][b]), ctx + " out_of_track"
    if rec["out_of_track"]:
        return
    assert list(rec["start_node"]) == g["start_node"][b].tolist(), ctx + " start node"
    coi = -1 if rec["closest_obj_index"] is None else int(rec["closest_obj_index"])
    assert coi == int(g["closest_obj_index"][b]), ctx + " closest_obj_index %d vs %d" % (coi, int(g["closest_obj_index"][b]))
    for a, act in enumerate(H.ACTIONS):
        n_want = int(g["path_len"][b, a])
        has = act in rec["paths"] and len(rec["paths"][act]) > 0
        assert has == (n_want > 0), "%s: action %s present=%s, golden len %d" % (ctx, act, has, n_want)
        if has:
            nodes = [[-1 if v is None else int(v) for v in p] for p in rec["nodes"][act][0]]
            want = g["nodes"][b, a, :int(g["nodes_len"][b, a])].tolist()
            assert nodes == want, "%s: node sequence of %s differs\n got  %s\n want %s" % (ctx, act, nodes, want)
            ni = np.asarray(rec["node_idx"][act][0]).tolist()
            assert ni == g["node_idx"][b, a, :len(ni)].tolist(), ctx + " node_idx " + act
            assert bool(rec["red_len"][act][0]) == bool(g["red_len"][b, a]), ctx + " red_len " + act
            assert rec["paths"][act][0].shape[0] == n_want, ctx + " path length " + act
        tl = int(g["traj_len"][b, a])
        assert (act in rec["traj_full"]) == (tl > 0), "%s: trajectory %s present=%s" % (ctx, act, act in rec["traj_full"])
        if not tl:
            continue
        assert int(rec["ids"][act]) % 10 == int(g["traj_id"][b, a]) % 10, ctx + " traj id " + act
        full = rec["traj_full"][act][0]
        assert full.shape[0] == tl, ctx + " rows of " + act
        H.assert_close("traj[%s]" % act, full[:, IDX], g["traj"][b, a, :tl], COLS, ctx)
        if exported:
            rows = rec["traj"][act][0]
            assert rows.shape[0] == min(tl, N_EXPORT), ctx + " exported rows of " + act
            H.assert_close("export[%s]" % act, rows[:, IDX], g["traj"][b, a, :rows.shape[0]], COLS, ctx)
