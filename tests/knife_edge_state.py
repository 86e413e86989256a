"""Inputs within a few ulps of the STATEFUL tick's float64 decisions (k_state, k_ref; DESIGN.md section 6), pure-NumPy
replays of those decisions in the reference's operation order, and the observables through which a test sees them
(tests/golden/ticks_knife_edge_state.npz, tests/tools/gen_golden_knife_edge_state.py).

A stateful tick decides on the MEMORY of the last tick: the executed trajectory (s, x, y, vx rows) and the node list of
its path.  The device keeps the velocity rows as fp32 recurrences stored in float64, so a tie built on the reference's
memory is no tie on the device's: the device tests download the device's own memory, build the probes on it with the
constructions below and compare with the replays, which the fixture pins to the reference.

Families (kernel -> reference; G for the stateful tick, F1-F7 are the first tick's, tests/knife_edge.py):
  G1  t_const ties: next_idx = (cumsum(ds / v) <= t_const).argmin() + 1, inf where v == 0 (q11),   OTH:366-386
      all-True -> 1; T = cumsum[k] exactly, its lower neighbour (the flip pair) and +-4 ulps, where
      the flip moves the start node
  G2  every row of the memory trajectory as the predicted position -> start node (first-minimum   OTH:381-386,
      nearest node, ang1 >= ang2; a row on a node is a zero vector)                                get_s_coord.py
  G3  cut index by pos_est: nearest-row flip pairs and exact ties, angle-rule flips, points on     OTH:551-556
      rows, before the first / beyond the last row, bitwise-collinear end points
  G4  delay compensation: vel_idx = min((cumsum(ds / v) <= delaycomp).argmin() + 1, nv - 1)        OTH:558-574
  G5  cut layer max(argmin(node_idx < cut_pos) - 2, 0) and cut_index_layer: every G3 / G4 probe    OTH:580-590
"""
import numpy as np

from tests.knife_edge import W, d2, exact_ties, flip_on_axis, step

# G1 kinds
G1_TIE, G1_BELOW, G1_WINDOW, G1_ZERO, G1_ALL, G1_INF, G1_ROW = range(7)
# G3 kinds
G3_FLIP, G3_TIE, G3_ANGLE, G3_ON_ROW, G3_BEFORE, G3_BEYOND, G3_COLLINEAR = range(7)
# G4 kinds
G4_TIE, G4_BELOW, G4_WINDOW, G4_ALL, G4_INF = range(5)


# ---- replays (the reference's expressions, NumPy float64) ---------------------------------------------------------------
def t_approx(s, v):
    """np.divide(np.diff(s), v, out=inf, where=v != 0) (quirk q11)"""
    ds = np.diff(np.asarray(s, dtype=np.float64))
    v = np.asarray(v, dtype=np.float64)
    return np.divide(ds, v, out=np.full(v.shape[0], np.inf), where=v != 0)


def next_idx(s, v, t_const):
    """OTH:370-378 on the executed trajectory's s and vx columns"""
    return int((np.cumsum(t_approx(s[1:], v[1:-1])) <= t_const).argmin() + 1)


def start_node_idx(node_xy, pos):
    """OTH:381-386: get_s_coord(node_coords, predicted_pos, only_index=True)[1][1]"""
    from oracle.ltpl_oracle import get_s_coord
    return int(get_s_coord(np.asarray(node_xy, dtype=np.float64), pos, only_index=True)[1][1])


def cut_index(traj, pos):
    from oracle.ltpl_oracle import get_s_coord
    return int(get_s_coord(traj[:, 1:3], pos, traj[:, 0], only_index=True)[1][0])


def ref_idx(traj, pos, delaycomp, node_idx_first_action, last_cut):
    """OTH:551-590 on traj = rows (s, x, y, vx) of the executed trajectory -> (cut_pos, cut_layer, cut_index_layer,
    vel_idx, vel_plan, vel_course).  Raises ValueError where the reference does (np.argmin of an empty v_past)."""
    c = cut_index(traj, pos)
    v_past = traj[c:-1, 3]
    vel_idx = min(int((np.cumsum(t_approx(traj[c:, 0], v_past)) <= delaycomp).argmin()) + 1, v_past.shape[0] - 1)
    cut_pos = int(last_cut) + c
    ni = np.asarray(node_idx_first_action)
    cut_layer = max(int(np.argmin(ni < cut_pos)) - 2, 0)
    return cut_pos, cut_layer, int(ni[cut_layer]), vel_idx, float(traj[c + vel_idx, 3]), traj[c:c + vel_idx, 3].copy()


def memory_start(mem, t_const):
    """start node index in the memory node list for t_const"""
    tr = mem["traj"]
    return start_node_idx(mem["node_xy"], tr[next_idx(tr[:, 0], tr[:, 3], t_const), 1:3])


# ---- constructions on a memory: mem = dict(traj=(n, 4) rows (s, x, y, vx), node_xy=(k, 2)) ---------------------------
def cumsum_from(traj, c):
    return np.cumsum(t_approx(traj[c:, 0], traj[c:-1, 3]))


def _ulps(x, kinds):
    """x (exact), its lower neighbour and +-W ulps with their kinds"""
    tie, below, win = kinds
    return [(x, tie), (step(x, -1), below), (step(x, -W), win), (step(x, 1), win), (step(x, W), win)]


def g1_probes(mem, all_true=None):
    """[(T, kind, k)]: T = cumsum[k] where the flip pair (nextbefore(T), T) moves the start node, its +-W ulps; T = 0;
    with all_true, a T above the whole trajectory's time (all-True: next_idx = 1) when that time is finite and below
    all_true; the first inf of the cumsum (v == 0, q11) with the last finite value and ulps above it"""
    tr = mem["traj"]
    cum = np.cumsum(t_approx(tr[1:, 0], tr[1:-1, 3]))
    out = []
    for k in range(cum.shape[0]):
        T = float(cum[k])
        if not np.isfinite(T):
            last = float(cum[k - 1]) if k else 0.0
            out += [(last, G1_INF, k), (step(last, 1), G1_INF, k), (step(last, W), G1_INF, k), (1e3, G1_INF, k)]
            break
        if k and cum[k - 1] == T:
            continue
        if memory_start(mem, T) == memory_start(mem, step(T, -1)):
            continue
        out += [(t, kind, k) for t, kind in _ulps(T, (G1_TIE, G1_BELOW, G1_WINDOW))]
    out.append((0.0, G1_ZERO, -1))
    if all_true is not None and np.isfinite(cum[-1]) and cum[-1] < all_true:
        out += [(step(float(cum[-1]), 1), G1_ALL, -1), (float(all_true), G1_ALL, -1)]
    return out


def g2_probes(mem):
    """[(T, kind, row)]: one t_const per reachable row r of the memory trajectory (next_idx = r), at the middle of its
    cumsum interval (row 1: T = 0)"""
    tr = mem["traj"]
    cum = np.cumsum(t_approx(tr[1:, 0], tr[1:-1, 3]))
    out = [(0.0, G1_ROW, 1)]
    for r in range(2, cum.shape[0] + 1):
        lo, hi = cum[r - 2], cum[r - 1]
        if not (np.isfinite(hi) and hi > lo):
            break
        T = float(0.5 * (lo + hi))
        if next_idx(tr[:, 0], tr[:, 3], T) == r:
            out.append((T, G1_ROW, r))
    return out


def g3_probes(traj, rng, n_flip=12, n_angle=10):
    """[(pos, kind)] for the cut index: nearest-row flip pairs between consecutive rows (and exact distance ties there),
    angle-rule flip pairs near rows, every row itself, points before the first / beyond the last row (off the line) and
    bitwise-collinear points on the extension of the first / last segment"""
    from oracle.ltpl_oracle import angle3pt
    xy = np.ascontiguousarray(traj[:, 1:3])
    n = xy.shape[0]
    near = lambda p: int(np.argmin(d2(xy, p)))   # noqa: E731
    out = []
    for i in sorted(rng.choice(np.arange(0, n - 1), min(n_flip, n - 1), replace=False)):
        pa, pb = xy[i], xy[i + 1]
        axis = int(np.argmax(np.abs(pb - pa)))
        r = flip_on_axis(near, (pa + pb) / 2, axis, pa[axis], pb[axis])
        if r is None:
            continue
        out += [(r[0], G3_FLIP), (r[1], G3_FLIP)]
        out += [(t, G3_TIE) for t in exact_ties(xy[near(r[0])], xy[near(r[1])], r[0], axis, pts=xy)[:2]]
    # angle rule: a point beside row i moved along the track; flips where the angle comparison decides the cut
    for i in sorted(rng.choice(np.arange(1, n - 1), min(n_angle, n - 2), replace=False)):
        t = xy[i + 1] - xy[i - 1]
        t = t / np.linalg.norm(t)
        nrm = np.array([-t[1], t[0]])
        base = xy[i] + rng.choice([-1.0, 1.0]) * rng.uniform(0.2, 1.0) * nrm
        axis = int(np.argmax(np.abs(t)))
        span = 0.3 * min(np.linalg.norm(xy[i + 1] - xy[i]), np.linalg.norm(xy[i] - xy[i - 1]))
        r = flip_on_axis(lambda p: cut_index(traj, p), base, axis, base[axis] - span * abs(t[axis]),
                         base[axis] + span * abs(t[axis]))
        if r is None or near(r[0]) != i or near(r[1]) != i:
            continue
        gap = lambda p: abs(angle3pt(xy[i], p, xy[i - 1])) - abs(angle3pt(xy[i], p, xy[i + 1]))   # noqa: E731
        if min(abs(gap(r[0])), abs(gap(r[1]))) > 1e-14:   # the F7 rule: decided by more than atan2's error
            out += [(r[0], G3_ANGLE), (r[1], G3_ANGLE)]
    out += [(xy[i].copy(), G3_ON_ROW) for i in range(n)]
    for kind, a, b in ((G3_BEFORE, xy[0], xy[1]), (G3_BEYOND, xy[-1], xy[-2])):
        u = (a - b) / np.linalg.norm(a - b)
        nrm = np.array([-u[1], u[0]])
        for off, lat in ((0.5, 0.3), (3.0, -1.0), (20.0, 2.0)):
            out.append((a + off * u + lat * nrm, kind))
    out += [(p, G3_COLLINEAR) for p in collinear_ends(xy)]
    return out


def collinear_ends(xy):
    """points P on the extension of the first / last segment, away from the line, at which the two vectors the angle
    rule compares are exact multiples (P - p_a = d, P - p_b = 2 d): both atan2 values are bitwise equal, ang1 == ang2 == 0
    -- `>=` keeps the cut at n - 2 beyond the last row, `>` would take the last row"""
    out = []
    for a, b in ((xy[-1], xy[-2]), (xy[0], xy[1])):
        d = a - b
        for m in (1.0, 0.5, 0.25):
            p = a + m * d
            if np.array_equal(p - a, m * d) and np.array_equal(p - b, (m + 1.0) * d) and \
                    int(np.argmin(d2(xy, p))) in (0, xy.shape[0] - 1) and collinear_angles(xy, p) == (0.0, 0.0):
                out.append(p)
    return out


def collinear_angles(xy, p):
    """(ang1, ang2) of get_s_coord at p, as the reference computes them"""
    from oracle.ltpl_oracle import angle3pt
    n = xy.shape[0]
    nb = int(np.argmin(d2(xy, p)))
    i1, i2 = max(nb - 1, 0), min(nb + 1, n - 1)
    return abs(angle3pt(xy[nb], p, xy[i1])), abs(angle3pt(xy[nb], p, xy[i2]))


def g4_probes(traj, rows, all_true=1e3):
    """[(pos, D, kind, c)]: pos = trajectory row r (its cut index c = cut_index(traj, pos) is r or r - 1), D = the
    cumsum from c at index k exactly, its lower neighbour and +-W ulps, for k at the start, the middle and the end of the
    finite part; a D above the whole time (all-True: the nv - 1 clamp decides near the end); where the cumsum reaches
    inf (v == 0, q11), the last finite value and ulps above it"""
    out = []
    for r in rows:
        pos = traj[r, 1:3].copy()
        c = cut_index(traj, pos)
        cum = cumsum_from(traj, c)
        fin = int(np.sum(np.isfinite(cum)))
        for k in sorted({0, fin // 2, fin - 1}):
            if k < 0 or k >= fin or (k and cum[k - 1] == cum[k]):
                continue
            out += [(pos, D, kind, c) for D, kind in _ulps(float(cum[k]), (G4_TIE, G4_BELOW, G4_WINDOW))]
        if fin == cum.shape[0]:
            if fin:
                out.append((pos, step(float(cum[-1]), 1), G4_ALL, c))
            out.append((pos, all_true, G4_ALL, c))
        else:
            last = float(cum[fin - 1]) if fin else 0.0
            # (a delaycomp must be > 0: the library refuses 0, where the cumsum is inf from its first term)
            out += [(pos, D, G4_INF, c) for D in (last, step(last, 1), step(last, W), all_true) if D > 0.0]
    return out


def g4_rows(traj):
    """trajectory rows of G4: the first, the middle and near the end (the all-True case and the nv - 1 clamp)"""
    n = traj.shape[0]
    return sorted({1, n // 2, n - 3, n - 1})
