"""Inputs within a few ulps of the planner's float64 decision boundaries (first tick), and the observables through which a
test sees each decision (tests/golden/ticks_knife_edge.npz, tests/tools/gen_golden_knife_edge.py).

One primitive: along a line in input space (one coordinate of a position or the heading, everything else fixed) a
decision flips; bisection over the ordered integer view of the float64 coordinate ends at the FLIP PAIR x-, x+ =
nextafter(x-), whose two sides decide differently.  Around it the tests take +-4 ulps; where a short ulp search finds
them, points of EXACT equality (two squared distances equal, a distance equal to its bound) separate `<` from `<=` and
exercise the first-minimum tie rules.  No transcendental function sits between an input and its decision: objects have
v = 0 (X - sin(theta) * v * 0.2 is X bit for bit) or explicit 'prediction' points.

Families (kernel -> reference):
  F1  / F1'  in-track test of the ego (k_startpos) / of an object (k_plan's chunk_objects)     check_inside_bounds.py
  F2  nearest node of the ego over all nodes -> start layer                                     GB:341-345
  F3  heading test hd > max_heading_offset                                                      OTH:234-240
  F4  nearest reference-line layer of a disc (the last one sets the object's layer, q14)        GIE:41-42
  F5  collision test x^2 + y^2 <= ref of a lattice sample                                       GB:640-643
  F6  object beside / in the constant segment: s_start <= s_obj <= s_end, d2 <= oref (q15), and    MOPG:86-122
      the race-line near-ties of get_s_coord that decide s_start <= s_obj
  F7  neighbour choice of get_s_coord on near-ties (angle_cmp -> angle_cmp_exact), glob_rl       get_s_coord.py:60-77
"""
import math

import numpy as np

SIGN = 1 << 63
W = 4   # ulps on either side of a flip pair


# ---- ordered integer view of float64 ------------------------------------------------------------------------------------
def key(x):
    i = int(np.float64(x).view(np.int64))
    return i if i >= 0 else -(i & (SIGN - 1))


def unkey(k):
    return float(np.uint64(k).view(np.float64)) if k >= 0 else float(np.uint64((-k) | SIGN).view(np.float64))


def step(x, n):
    """x moved by n ulps"""
    return unkey(key(x) + n)


def window(x, n=W):
    return [step(x, k) for k in range(-n, n + 1)]


def bisect(f, a, b):
    """a, b with f(a) != f(b) -> (x-, x+), adjacent doubles between a and b, f(x-) == f(a), f(x+) == f(b)"""
    fa = f(a)
    assert f(b) != fa
    ka, kb = key(a), key(b)
    while abs(kb - ka) > 1:
        km = (ka + kb) // 2
        if f(unkey(km)) == fa:
            ka = km
        else:
            kb = km
    return unkey(ka), unkey(kb)


def at(base, axis, v):
    p = np.array(base, dtype=np.float64)
    p[axis] = v
    return p


def flip_on_axis(f, base, axis, lo, hi):
    """flip pair of f along coordinate `axis` of base between lo and hi: (p-, p+) or None when f(lo) == f(hi)"""
    g = lambda v: f(at(base, axis, v))   # noqa: E731
    if g(lo) == g(hi):
        return None
    a, b = bisect(g, lo, hi)
    return at(base, axis, a), at(base, axis, b)


def d2(pts, p):
    """np.power(x - px, 2) + np.power(y - py, 2), the reference's expression (float64, no fma)"""
    return np.power(pts[:, 0] - p[0], 2) + np.power(pts[:, 1] - p[1], 2)


def exact_ties(pa, pb, base, axis, rng=64, other=512, pts=None):
    """points near base (axis +-rng ulps, the other coordinate +-other ulps) at which the squared distances to pa and pb
    are EQUAL in float64 -- and, with pts given, the minimum over pts"""
    o = 1 - axis
    xs = np.array([step(base[axis], k) for k in range(-rng, rng + 1)])
    ys = np.array([step(base[o], k) for k in range(-other, other + 1)])
    P = np.empty((xs.size, ys.size, 2))
    P[..., axis] = xs[:, None]
    P[..., o] = ys[None, :]
    da = np.power(P[..., 0] - pa[0], 2) + np.power(P[..., 1] - pa[1], 2)
    db = np.power(P[..., 0] - pb[0], 2) + np.power(P[..., 1] - pb[1], 2)
    out = []
    for i, j in zip(*np.nonzero(da == db)):
        p = P[i, j].copy()
        if pts is None or d2(pts, p).min() == da[i, j]:
            out.append(p)
    return out


# ---- geometry of a lattice ----------------------------------------------------------------------------------------------
def center(orc):
    return (orc.bound1 + orc.bound2) / 2


def ego_pose(orc, layer):
    """ego on the race-line node of `layer`, with the heading of its goal node (OTH:226: no heading mismatch)"""
    lt = orc.lat
    g = lt.node_off[layer] + lt.raceline_index[layer]
    goal = (layer + 2) % (lt.num_layers - 1)
    psi = lt.node_psi[lt.node_off[goal] + lt.raceline_index[goal]]
    return orc.node_xy[g].copy(), float(psi)


def ego_behind(orc, p, gap=25.0):
    """layer of an ego vehicle whose start node (two layers on, q5) lies >= gap metres of race line before the position
    p, and the pose there; None when the track does not reach that far back (open track)"""
    lt = orc.lat
    lp = int(np.argmin(d2(lt.refline, p)))
    s = lt.s_raceline
    for k in range(1, lt.num_layers):
        le = lp - k
        if le < 0:
            if not lt.closed:
                return None
            le += lt.num_layers
        ls = (le + 2) % (lt.num_layers - 1)
        ds = s[lp] - s[ls] if s[lp] >= s[ls] else s[lp] + s[-1] - s[ls]
        if ds >= gap and ds < 150.0:
            return le, ego_pose(orc, le)
    return None


def obj(p, length=5.0, pred=None):
    o = {'id': 1, 'type': 'physical', 'X': float(p[0]), 'Y': float(p[1]), 'theta': 0.0, 'v': 0.0, 'length': length,
         'width': 2.5}
    if pred is not None:
        o['prediction'] = np.asarray(pred, dtype=np.float64).reshape(-1, 2)
    return o


FAR = (1.0e4, 1.0e4)   # an object beyond every bound and every grid cell (whole-polyline scan)


def pad_objects(n):
    return [obj(FAR) for _ in range(n)]


# ---- the decisions, as the oracle restates them -----------------------------------------------------------------------
def in_track(orc, p):
    from oracle.ltpl_oracle import check_inside_bounds
    return bool(check_inside_bounds(orc.bound1, orc.bound2, p))


def start_layer_of(orc, p):
    return int(orc.node_layer[int(np.argmin(d2(orc.node_xy, p)))])


def heading_ok(orc, heading, psi_e):
    hd = abs(heading - psi_e)
    if hd > np.pi:
        hd = abs(2 * np.pi - hd)
    return not hd > orc.p['max_heading_offset']


def ref_layer(orc, p):
    return int(np.argmin(d2(orc.lat.refline, p)))


def glob_xy(orc):
    return np.ascontiguousarray(orc.lat.glob_rl[:-1, 1:3])


def glob_start(orc, p):
    """get_s_coord(glob_rl[:, 1:3], pos, glob_rl[:, 0], closed=True)[1][0] (CVPF:166-172)"""
    from oracle.ltpl_oracle import get_s_coord
    return int(get_s_coord(glob_xy(orc), tuple(p), orc.lat.glob_rl[:-1, 0], closed=True)[1][0])


def angle_gap(orc, p, i):
    """|angle3pt(pn, p, p1)| - |angle3pt(pn, p, p2)| at glob_rl vertex i"""
    from oracle.ltpl_oracle import angle3pt
    G = glob_xy(orc)
    n = G.shape[0]
    return abs(angle3pt(G[i], p, G[i - 1])) - abs(angle3pt(G[i], p, G[(i + 1) % n]))


def paths_observable(orc, pos, heading, objs):
    """what the object decisions of a first tick show: closest object and {action: node sequence}"""
    st = orc.set_startpos(np.asarray(pos, dtype=np.float64), float(heading), 10.0)
    if not (st['in_track'] and st['cor_heading']):
        return None
    res = orc.calc_paths(st, orc.process_object_list(objs))
    return observable(res['closest_obj_index'], res['nodes'])


def observable(coi, nodes):
    return (-1 if coi is None else int(coi),
            tuple(sorted((a, tuple(tuple(-1 if v is None else int(v) for v in p) for p in n[0]))
                         for a, n in nodes.items())))


# ---- scenarios through which a test sees an object decision -------------------------------------------------------
def golden_set(tag):
    from tests import helpers as H
    g = H.golden("ticks_knife_edge.npz")
    return {k.split("__", 1)[1]: g[k] for k in g.files if k.startswith(tag + "__")}


def oracle_for(tag):
    from graphbasedlocaltrajectoryplanner_b200 import lattice_blob as LB
    from oracle.ltpl_oracle import OracleLTPL
    from tests import helpers as H
    lat = H.lattice_for(tag)
    LB.pack_lattice(lat)   # the nearest-vertex grids (cell edges of F1)
    return OracleLTPL(lat)


def f1_scenario(orc, p, chunk2=False):
    """F1': one v = 0 object at p, ahead of an ordinary ego (None: the track does not reach back far enough); with
    chunk2 behind 33 objects beyond every bound, so that k_plan's second object chunk decides it.  The object is the
    closest object (index 0) iff it is on the track."""
    eb = ego_behind(orc, p)
    if eb is None:
        return None
    return eb[1][0], eb[1][1], (pad_objects(33) if chunk2 else []) + [obj(p)]


def f4_scenario(orc, l, l2, p):
    """F4: object A (v = 0, no prediction) at reference-line vertex l2, object B with its last (only) prediction
    point at p: the closest object is B (1) iff p's layer resolves to l, the layer before l2, else A (0)."""
    eb = ego_behind(orc, orc.lat.refline[l])
    if eb is None:
        return None
    r = orc.lat.refline[l2]
    return eb[1][0], eb[1][1], [obj(r), obj(r, pred=[p])]


def f7_scenario(orc, p):
    eb = ego_behind(orc, p)
    return eb[1][0], eb[1][1], [obj(p)]


# ---- constructions -----------------------------------------------------------------------------------------------------
def f1_cases(orc, rng, n_vertex=10, n_mid=14):
    """flip pairs of the in-track test across bound1 and bound2: at centre-line vertices, mid-segment, at the closed
    track's seam (L-1 <-> 0) or the open track's ends, and with the fixed coordinate on a 4 m grid-cell edge.
    Returns [(p-, p+, axis, kind)], kind: 0 mid-segment, 1 vertex, 2 seam / track end, 3 cell edge."""
    from graphbasedlocaltrajectoryplanner_b200 import lattice_blob as LB
    lt = orc.lat
    L = lt.num_layers
    c = center(orc)
    x0, y0 = lt._nearest_grids["x0"], lt._nearest_grids["y0"]
    verts = [(int(i), 0.0, 1) for i in rng.choice(np.arange(2, L - 2), n_vertex, replace=False)]
    mids = [(int(i), float(f), 0) for i, f in zip(rng.choice(np.arange(2, L - 3), n_mid, replace=False),
                                                   rng.uniform(0.05, 0.95, n_mid))]
    ends = [(0, 0.0, 2), (L - 1, 0.0, 2), (L - 1 if lt.closed else 0, 0.5, 2), (0, 0.3, 2)] if lt.closed else \
        [(0, 0.0, 2), (L - 1, 0.0, 2), (0, 0.5, 2), (L - 2, 0.5, 2)]
    cells = [(int(i), float(f), 3) for i, f in zip(rng.choice(np.arange(2, L - 3), 6, replace=False),
                                                   rng.uniform(0.1, 0.9, 6))]
    out = []
    for i, f, kind in verts + mids + ends + cells:
        j = (i + 1) % L
        for bnd in (orc.bound1, orc.bound2):
            base = bnd[i] + f * (bnd[j] - bnd[i])
            cc = c[i] + f * (c[j] - c[i])
            u = (base - cc) / np.linalg.norm(base - cc)
            axis = int(np.argmax(np.abs(u)))
            if kind == 3:   # the other coordinate on a grid-cell edge x0 + 4k / y0 + 4k
                o = 1 - axis
                g0 = (x0, y0)[o]
                base[o] = g0 + LB.GRID_CELL * np.round((base[o] - g0) / LB.GRID_CELL)
            lo, hi = base[axis] - 0.6 * u[axis], base[axis] + 0.6 * u[axis]
            r = flip_on_axis(lambda p: in_track(orc, p), base, axis, lo, hi)
            if r is not None:
                out.append((r[0], r[1], axis, kind))
    return out


def f2_cases(orc, rng, n=16):
    """flip pairs of the start layer (nearest node over all nodes) between the race-line nodes of adjacent layers, and
    exact ties of the two nearest nodes (first minimum: the lower global index).  [(p-, p+, axis, ties)]"""
    lt = orc.lat
    L = lt.num_layers
    # (not at the seam: layers L-1 and 0 lead to the same start layer, (l + 2) % (L - 1), quirk q5)
    layers = list(rng.choice(np.arange(1, L - 3), n, replace=False))
    out = []
    for l in layers:
        l2 = (l + 1) % L
        ga = lt.node_off[l] + lt.raceline_index[l]
        gb = lt.node_off[l2] + lt.raceline_index[l2]
        pa, pb = orc.node_xy[ga], orc.node_xy[gb]
        base = (pa + pb) / 2
        axis = int(np.argmax(np.abs(pb - pa)))
        r = flip_on_axis(lambda p: start_layer_of(orc, p), base, axis, pa[axis], pb[axis])
        if r is None:
            continue
        if not (in_track(orc, r[0]) and in_track(orc, r[1])):
            continue
        na, nb = (int(np.argmin(d2(orc.node_xy, q))) for q in r)
        ties = exact_ties(orc.node_xy[na], orc.node_xy[nb], r[0], axis, pts=orc.node_xy)[:2]
        out.append((r[0], r[1], axis, ties))
    return out


def f3_cases(orc, rng, n=10):
    """flip pairs of the heading test at psi_e +- max_heading_offset, incl. goal nodes with |psi_e| near pi where the
    heading sits on the other side of +-pi (the 2 pi - hd branch).  [(layer, pos, h-, h+, psi_e)]"""
    lt = orc.lat
    L = lt.num_layers
    off = orc.p['max_heading_offset']
    pose = [ego_pose(orc, int(l)) + (int(l),) for l in range(L - 2)]
    wrap = [q for q in pose if abs(q[1]) > np.pi - off - 0.05]
    pick = [pose[int(i)] for i in rng.choice(len(pose), n, replace=False)] + wrap[:6]
    out = []
    for pos, psi, l in pick:
        cands = [(psi + off - 0.1, psi + off + 0.1), (psi - off + 0.1, psi - off - 0.1)]
        if abs(psi) > np.pi - off - 0.05:
            sgn = 1.0 if psi > 0 else -1.0
            cands.append((psi + sgn * (off - 0.1) - sgn * 2 * np.pi, psi + sgn * (off + 0.1) - sgn * 2 * np.pi))
        for a, b in cands:
            f = lambda h: heading_ok(orc, h, psi)   # noqa: E731
            if f(a) == f(b):
                continue
            h0, h1 = bisect(f, a, b)
            out.append((l, pos, h0, h1, psi))
    return out


def f4_cases(orc, rng, n=10):
    """flip pairs and exact ties of the nearest reference-line layer between vertices l and l + 1: on the track, > 60 m
    off the track (no grid bound: warp-scan fallback), and at the closed track's seam (L-1 <-> 0).
    [(l_lo, l_hi, p-, p+, ties, far)]"""
    lt = orc.lat
    L = lt.num_layers
    R = lt.refline
    layers = [int(l) for l in rng.choice(np.arange(3, L - 3), n, replace=False)]
    if lt.closed:
        layers += [L - 1, L - 1]
    out = []
    for k, l in enumerate(layers):
        l2 = (l + 1) % L
        pa, pb = R[l], R[l2]
        t = (pb - pa) / np.linalg.norm(pb - pa)
        nrm = np.array([-t[1], t[0]])
        for off, far in ((0.0, False), (70.0 if k % 2 else -70.0, True)):
            base = (pa + pb) / 2 + off * nrm
            axis = int(np.argmax(np.abs(pb - pa)))
            r = flip_on_axis(lambda p: ref_layer(orc, p), base, axis, base[axis] - 0.6 * (pb - pa)[axis],
                             base[axis] + 0.6 * (pb - pa)[axis])
            if r is None or {ref_layer(orc, r[0]), ref_layer(orc, r[1])} != {l, l2}:
                continue
            ties = exact_ties(pa, pb, r[0], axis, pts=R)[:2]
            out.append((l, l2, r[0], r[1], ties, far))
    return out


def f5_cases(orc, rng, n=8, samples=16):
    """flip pairs of the collision test: one v = 0 object moved across the track at a layer ~40-150 m ahead of the ego;
    bisection on the first tick's observable (closest object, node sequences), kept where only the blocked-edge set
    differs between the two sides (same in-track decision, same layer), plus points where the deciding sample's
    x^2 + y^2 EQUALS ref.  [(ego_layer, pos, heading, p-, p+, axis, equal_points)]"""
    lt = orc.lat
    L = lt.num_layers
    out = []
    for l in rng.choice(np.arange(4, L - 6), n, replace=False):
        l = int(l)
        eb = ego_behind(orc, lt.refline[l], gap=40.0)
        if eb is None:
            continue
        le, (pos, hd) = eb
        nrm = lt.normvec[l]
        axis = int(np.argmax(np.abs(nrm)))
        base = lt.refline[l].copy()
        s_lo, s_hi = -(lt.w_left[l] - 1.0), lt.w_right[l] - 1.0
        vs = base[axis] + np.linspace(s_lo, s_hi, samples) * nrm[axis]
        obs = lambda v: paths_observable(orc, pos, hd, [obj(at(base, axis, v))])   # noqa: E731
        ob = [obs(v) for v in vs]
        st = orc.set_startpos(pos, hd, 10.0)
        for k in range(samples - 1):
            if ob[k] == ob[k + 1] or ob[k] is None or ob[k + 1] is None:
                continue
            a, b = bisect(obs, float(vs[k]), float(vs[k + 1]))
            pa, pb = at(base, axis, a), at(base, axis, b)
            va, vb = (orc.process_object_list([obj(p)]) for p in (pa, pb))
            if len(va) != 1 or len(vb) != 1:
                continue
            ta, tb = (orc.gen_local_node_template(st['start_node'], v) for v in (va, vb))
            if ta[1:3] != tb[1:3] or ta[3] == tb[3]:
                continue
            out.append((le, pos, hd, pa, pb, axis, collision_equalities(orc, pa, pb, ta[3] ^ tb[3], axis)))
    return out


def collision_equalities(orc, pa, pb, edges, axis, rng=256, other=256):
    """object positions near pa at which a sample of one of `edges` lies EXACTLY at x^2 + y^2 == ref (5 m object)"""
    lt = orc.lat
    ref = np.power(2.5 + lt.veh_width / 2, 2) + np.power(lt.sampled_resolution, 2) / 4
    S = np.concatenate([orc.samp_xy[lt.samp_off[e]:lt.samp_off[e + 1]] for e in sorted(edges)])
    s = S[int(np.argmin(np.abs(d2(S, pa) - ref)))]
    o = 1 - axis
    xs = np.array([step(pa[axis], k) for k in range(-rng, rng + 1)])
    ys = np.array([step(pa[o], k) for k in range(-other, other + 1)])
    P = np.empty((xs.size, ys.size, 2))
    P[..., axis] = xs[:, None]
    P[..., o] = ys[None, :]
    x, y = s[0] - P[..., 0], s[1] - P[..., 1]
    hit = np.nonzero(x * x + y * y == ref)
    return [P[i, j].copy() for i, j in zip(*hit)][:2]


def rl_s(orc, p):
    """race-line s coordinate (MOPG:90-97)"""
    from oracle.ltpl_oracle import get_s_coord
    lt = orc.lat
    return float(get_s_coord(lt.raceline, tuple(p), lt.s_raceline, closed=True)[0])


def rl_s_via(orc, p, a_idx, b_idx):
    """get_s_coord.py:66-85 with the neighbour segment (a_idx, b_idx) forced"""
    lt = orc.lat
    a, b = lt.raceline[a_idx], lt.raceline[b_idx]
    t = ((p[0] - a[0]) * (b[0] - a[0]) + (p[1] - a[1]) * (b[1] - a[1])) / \
        (np.power(b[0] - a[0], 2) + np.power(b[1] - a[1], 2))
    sp = [a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1])]
    return float(lt.s_raceline[a_idx] + np.sqrt(np.power(a[0] - sp[0], 2) + np.power(a[1] - sp[1], 2)))


def heading_at(orc, p):
    """the goal node's heading for an ego at p (no heading mismatch)"""
    lt = orc.lat
    goal = (start_layer_of(orc, p) + 2) % (lt.num_layers - 1)
    return float(lt.node_psi[lt.node_off[goal] + lt.raceline_index[goal]])


def const_seg(orc, pos, heading):
    st = orc.set_startpos(np.asarray(pos, dtype=np.float64), float(heading), 10.0)
    return st['path_param']


def replay_observable(orc, pos, heading, objs, seg):
    """paths_observable with the constant segment replaced by `seg` (x, y, psi, kappa, el rows): the device's own
    segment, whose points come out of float64 sin / cos and may differ from the oracle's by an ulp"""
    st = orc.set_startpos(np.asarray(pos, dtype=np.float64), float(heading), 10.0)
    if not (st['in_track'] and st['cor_heading']):
        return None
    st['path_param'] = np.asarray(seg, dtype=np.float64)
    st['node_idx'] = [0, st['path_param'].shape[0] - 1]
    res = orc.calc_paths(st, orc.process_object_list(objs))
    return observable(res['closest_obj_index'], res['nodes'])


def f6_cases(orc, rng, n=10):
    """the constant-segment check of a v = 0 object (MOPG:86-122, q15): flip pairs of s_start <= s_obj (kind 0),
    s_obj <= s_end (kind 1), d2 <= oref against the segment's first point = the ego position (kind 2) and against a
    point inside the segment (kind 3), and object positions at EXACTLY oref from the ego position.  Kinds 1 and 3
    depend on segment points that come out of sin / cos: the device tests replay them on the device's segment.
    [(kind, ego, heading, p-, p+, axis, equal_points)]"""
    lt = orc.lat
    L = lt.num_layers
    oref = np.power(2.5 + lt.veh_width / 2, 2)
    out = []
    for l in rng.choice(np.arange(2, L - 6), n, replace=False):
        ego, hd = ego_pose(orc, int(l))
        seg = const_seg(orc, ego, hd)
        if seg is None or seg.shape[0] < 4:
            continue
        t = np.array([np.cos(hd + np.pi / 2), np.sin(hd + np.pi / 2)])   # driving direction
        nrm = np.array([-t[1], t[0]])
        s0, s1 = rl_s(orc, seg[0, 0:2]), rl_s(orc, seg[-1, 0:2])
        pobs = lambda p: paths_observable(orc, ego, hd, [obj(p)])   # noqa: E731
        for side in (1.0, -1.0):
            # kind 0 / 1: 5 m beside the segment's first / last point (outside oref), moved along the track
            for kind, anchor, s_ref in ((0, seg[0, 0:2], s0), (1, seg[-1, 0:2], s1)):
                base = anchor + side * 5.0 * nrm
                axis = int(np.argmax(np.abs(t)))
                f = (lambda p: s_ref <= rl_s(orc, p)) if kind == 0 else (lambda p: rl_s(orc, p) <= s_ref)
                r = flip_on_axis(f, base, axis, base[axis] - 1.5 * abs(t[axis]), base[axis] + 1.5 * abs(t[axis]))
                if r is not None and all(in_track(orc, p) for p in r) and pobs(r[0]) != pobs(r[1]):
                    out.append((kind, ego, hd, r[0], r[1], axis, []))
            # kind 2: sqrt(oref) from the ego position, a quarter step ahead (nearer to the first point than to the
            # second, and beside the segment); kind 3: sqrt(oref) beside a point in the middle of the segment
            step_len = float(np.linalg.norm(seg[1, 0:2] - seg[0, 0:2]))
            R = float(np.sqrt(oref))
            ca = step_len / (4.0 * R)
            for kind, anchor, u in ((2, seg[0, 0:2], ca * t + side * np.sqrt(1 - ca * ca) * nrm),
                                    (3, seg[seg.shape[0] // 2, 0:2], side * nrm)):
                base = anchor + R * u
                axis = int(np.argmax(np.abs(u)))
                f = lambda p: bool(np.any(d2(seg, p) <= oref))   # noqa: E731
                r = flip_on_axis(f, base, axis, base[axis] - 0.3 * u[axis], base[axis] + 0.3 * u[axis])
                if r is None or not all(in_track(orc, p) for p in r) or pobs(r[0]) == pobs(r[1]):
                    continue
                eq = []
                if kind == 2:
                    for e in exact_distance(seg[0, 0:2], oref, r[0], axis):
                        if pobs(e) in (pobs(r[0]), pobs(r[1])):
                            eq.append(e)
                out.append((kind, ego, hd, r[0], r[1], axis, eq[:2]))
    return out


def exact_distance(c, ref, p, axis, rng=256, other=256):
    """positions near p at which np.power(c - q, 2) summed over x, y EQUALS ref"""
    o = 1 - axis
    xs = np.array([step(p[axis], k) for k in range(-rng, rng + 1)])
    ys = np.array([step(p[o], k) for k in range(-other, other + 1)])
    P = np.empty((xs.size, ys.size, 2))
    P[..., axis] = xs[:, None]
    P[..., o] = ys[None, :]
    dd = np.power(c[0] - P[..., 0], 2) + np.power(c[1] - P[..., 1], 2)
    return [P[i, j].copy() for i, j in zip(*np.nonzero(dd == ref))]


def f6r_cases(orc, rng, n=12, gaps=(1e-13, 1e-11, 1e-10)):
    """race-line near-ties of get_s_coord (angle gap 1e-13 .. 1e-10 rad at race-line vertex i: angle_cmp_exact): the
    two neighbour segments give the object two s coordinates s_a < s_b; the ego is placed on the race line so that its
    own s, s_start, lies between them.  The object is then beside the constant segment iff the neighbour choice is the
    one with s_b.  [(ego, heading, p, gap)]"""
    from oracle.ltpl_oracle import angle3pt
    lt = orc.lat
    Rl = lt.raceline
    nr = Rl.shape[0]
    out = []
    for i in rng.choice(np.arange(3, nr - 3), n, replace=False):
        i = int(i)
        tv = Rl[i + 1] - Rl[i - 1]
        tv /= np.linalg.norm(tv)
        nrm = np.array([-tv[1], tv[0]])
        base = Rl[i] + rng.choice([-1.0, 1.0]) * rng.uniform(0.5, 2.0) * nrm
        axis = int(np.argmax(np.abs(tv)))
        gapf = lambda p: abs(angle3pt(Rl[i], p, Rl[i - 1])) - abs(angle3pt(Rl[i], p, Rl[i + 1]))   # noqa: E731
        seg = 0.3 * min(np.linalg.norm(Rl[i + 1] - Rl[i]), np.linalg.norm(Rl[i] - Rl[i - 1]))
        r = flip_on_axis(lambda p: gapf(p) >= 0.0, base, axis, base[axis] - seg * abs(tv[axis]),
                         base[axis] + seg * abs(tv[axis]))
        if r is None:
            continue
        h = 1e-6
        sl = (gapf(at(r[0], axis, r[0][axis] + h)) - gapf(at(r[0], axis, r[0][axis] - h))) / (2 * h)
        if sl == 0.0 or not math.isfinite(sl):
            continue
        for g in gaps:
            for sg in (-1.0, 1.0):
                p = at(r[0], axis, r[0][axis] + sg * g / sl)
                gp = gapf(p)
                if abs(gp) < 2e-14 or int(np.argmin(d2(Rl, p))) != i or not in_track(orc, p):
                    continue
                sa, sb = sorted((rl_s_via(orc, p, i - 1, i), rl_s_via(orc, p, i, i + 1)))
                if not sb - sa > 1e-9:
                    continue
                # ego on the race line near vertex i with s_start in the middle of (s_a, s_b)
                q0, q1 = Rl[i] - 1.0 * tv, Rl[i] + 1.0 * tv
                qa = int(np.argmax(np.abs(tv)))
                mid = 0.5 * (sa + sb)
                rq = flip_on_axis(lambda q: rl_s(orc, q) < mid, q0, qa, q0[qa], q1[qa])
                if rq is None:
                    continue
                ego = rq[0]
                if not (sa < rl_s(orc, ego) < sb) or not in_track(orc, ego):
                    continue
                out.append((ego, heading_at(orc, ego), p, gp))
    return out


def f7_cases(orc, rng, n=12, gaps=(1e-13, 1e-12, 1e-11, 1e-10)):
    """points near glob_rl vertex i at which the two neighbour angles of get_s_coord differ by 1e-13 .. 1e-10 rad (both
    signs): below angle_cmp's cosine margin, far above atan2's error.  [(i, points, gaps)]"""
    G = glob_xy(orc)
    ng = G.shape[0]
    out = []
    for i in rng.choice(np.arange(2, ng - 2), n, replace=False):
        i = int(i)
        t = G[i + 1] - G[i - 1]
        t /= np.linalg.norm(t)
        nrm = np.array([-t[1], t[0]])
        base = G[i] + rng.choice([-1.0, 1.0]) * rng.uniform(0.3, 2.0) * nrm
        axis = int(np.argmax(np.abs(t)))
        seg = 0.3 * min(np.linalg.norm(G[i + 1] - G[i]), np.linalg.norm(G[i] - G[i - 1]))
        r = flip_on_axis(lambda p: angle_gap(orc, p, i) >= 0.0, base, axis, base[axis] - seg * abs(t[axis]),
                         base[axis] + seg * abs(t[axis]))
        if r is None:
            continue
        # slope of the gap along the axis, from points 1e-6 m away
        h = 1e-6
        sl = (angle_gap(orc, at(r[0], axis, r[0][axis] + h), i) - angle_gap(orc, at(r[0], axis, r[0][axis] - h), i)) / (2 * h)
        if sl == 0.0 or not math.isfinite(sl):
            continue
        pts, gp = [], []
        for g in gaps:
            for s in (-1.0, 1.0):
                p = at(r[0], axis, r[0][axis] + s * g / sl)
                if int(np.argmin(d2(G, p))) != i:
                    continue
                pts.append(p)
                gp.append(angle_gap(orc, p, i))
        if pts:
            out.append((i, np.array(pts), np.array(gp)))
    return out
