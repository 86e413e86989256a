"""Golden vectors of the reference's position helpers get_s_coord (helper_funcs/src/get_s_coord.py), closest_path_index
(helper_funcs/src/closest_path_index.py) and check_inside_bounds (online_graph/src/check_inside_bounds.py), made by
running the UNMODIFIED reference on the shims of oracle/gen_golden.py and recording the arguments and results of every
call.  Writes exactly one file under the repository:

  tests/golden/path_coord.npz

Two kinds of call (`kind`):
  0   the reference's own calls (outermost only, not the helpers' calls of each other) inside closed loops
      (oracle/gen_golden.multitick_fixture) on the default and "216 x 11" lattices: OTH:214 (set_startpos bound check),
      384, 401, 556, 774-782 (follow object distance), MOPG:86-98 (the closed race line with its s values), CVPF:172 and
      OLI:107 (object filter);
  1   direct calls on synthetic lines, kept so that every label of LABELS occurs.

Lines are stored once each (`line_xy`, rows line_off[i] .. line_off[i + 1]), s arrays likewise (`sarr`, `sarr_off`).
Per call: fn (0 get_s_coord, 1 closest_path_index, 2 check_inside_bounds), line_a (ref_line / path / bound1), line_b
(bound2, -1), sarr (-1: None), pos, only_index, closed; results s (NaN for only_index and where the reference raises,
raised = 1), closest (the index pair), idx, inside; and two margins:
  ang_margin    |ang1 - ang2| of the neighbour choice (for check_inside_bounds: on the centre line)
  bound_margin  min(|d_b1_2 - d_track_2|, |d_b2_2 - d_track_2|) (check_inside_bounds only, else inf)
The device's float64 atan2 is not libm's: every recorded call has ang_margin > 1e-12 rad or is an exact tie of zeros
(ang1 == ang2 == 0).  This generator asserts it for the closed loops and drops direct candidates that miss it.  Calls
whose nearest point is tied (argpartition's order is undefined) are not kept either.

Usage (from the repo root, needs the reference checkout):   python -m tests.tools.gen_golden_path_coord
"""
import ast
import math
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

from oracle import gen_golden as GG  # noqa: E402

LABELS = ("closed_wrap_0", "closed_wrap_end", "open_start", "open_end", "on_vertex", "before_start", "beyond_end",
          "dup_points", "sarr_none_ins", "sarr_none_noins", "sarr_given_ins", "sarr_given_noins", "index_error",
          "only_index", "inside", "outside", "far_off", "angle_tie")
MARGIN_A = 1e-12
FN_S, FN_CLOSEST, FN_INSIDE = 0, 1, 2
RECORDS = []
_LINES, _SARR = {}, {}
_CUR = {"kind": 0, "depth": 0}


def _intern(table, a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    key = (a.shape, a.tobytes())
    if key not in table:
        table[key] = (len(table), a)
    return table[key][0]


def _ties(line, pos):
    d2 = np.power(line[:, 0] - pos[0], 2) + np.power(line[:, 1] - pos[1], 2)
    return int(np.sum(d2 == np.nanmin(d2))) > 1


def angles(ref, line, pos, closed):
    """the reference's ang1, ang2 (get_s_coord.py:34-49) with its own angle3pt and closest_path_index"""
    gs = ref.helper_funcs.src.get_s_coord
    nb = ref.helper_funcs.src.closest_path_index.closest_path_index(path=line, pos=pos, n_closest=1)[0][0]
    n = line.shape[0]
    if closed:
        i1, i2 = nb - 1, (0 if nb + 1 > n - 1 else nb + 1)
    else:
        i1, i2 = max(nb - 1, 0), min(nb + 1, n - 1)
    return abs(gs.angle3pt(line[nb, :], pos, line[i1, :])), abs(gs.angle3pt(line[nb, :], pos, line[i2, :])), nb, n


def ang_ok(a1, a2):
    return abs(a1 - a2) > MARGIN_A or (a1 == 0.0 and a2 == 0.0)


def bound_margin(b1, b2, pos, pair):
    l1 = np.column_stack((np.linspace(b1[pair[0], 0], b1[pair[1], 0]), np.linspace(b1[pair[0], 1], b1[pair[1], 1])))
    l2 = np.column_stack((np.linspace(b2[pair[0], 0], b2[pair[1], 0]), np.linspace(b2[pair[0], 1], b2[pair[1], 1])))
    c = (b1 + b2) / 2
    cl = np.column_stack((np.linspace(c[pair[0], 0], c[pair[1], 0]), np.linspace(c[pair[0], 1], c[pair[1], 1])))
    d = np.power(cl[:, 0] - pos[0], 2) + np.power(cl[:, 1] - pos[1], 2)
    i = int(np.argmin(d))
    dt = np.power(l1[i, 0] - l2[i, 0], 2) + np.power(l1[i, 1] - l2[i, 1], 2)
    d1 = np.power(l1[i, 0] - pos[0], 2) + np.power(l1[i, 1] - pos[1], 2)
    d2 = np.power(l2[i, 0] - pos[0], 2) + np.power(l2[i, 1] - pos[1], 2)
    return float(min(abs(d1 - dt), abs(d2 - dt))), int(np.sum(d == d.min())) > 1


def install(ref):
    """wrap the three module functions the reference calls through module attributes"""
    gs_mod = ref.helper_funcs.src.get_s_coord
    cp_mod = ref.helper_funcs.src.closest_path_index
    ib_mod = ref.online_graph.src.check_inside_bounds
    orig_gs, orig_cp, orig_ib = gs_mod.get_s_coord, cp_mod.closest_path_index, ib_mod.check_inside_bounds

    def outer(fn):
        def wrapped(*a, **k):
            _CUR["depth"] += 1
            try:
                return fn(_CUR["depth"] == 1, *a, **k)
            finally:
                _CUR["depth"] -= 1
        return wrapped

    @outer
    def get_s_coord(top, ref_line, pos, s_array=None, only_index=False, closed=False):
        line = np.array(ref_line, dtype=np.float64)
        p = np.asarray(pos, dtype=np.float64).reshape(-1)[:2]
        raised = False
        try:
            s, ci = orig_gs(ref_line=ref_line, pos=pos, s_array=s_array, only_index=only_index, closed=closed)
        except IndexError:
            if _CUR["kind"] == 0:
                raise
            raised = True
            s, ci = None, orig_gs(ref_line=ref_line, pos=pos, only_index=True, closed=closed)[1]
        if top:
            assert line.ndim == 2 and line.shape[1] == 2, line.shape
            a1, a2, nb, n = angles(ref, line, tuple(p), closed)
            RECORDS.append(dict(fn=FN_S, a=_intern(_LINES, line), b=-1,
                                sarr=-1 if s_array is None else _intern(_SARR, np.asarray(s_array).reshape(-1)),
                                pos=p, only_index=bool(only_index), closed=bool(closed),
                                s=np.nan if s is None else float(s), ci=[int(ci[0]), int(ci[1])], idx=-1, inside=-1,
                                ang_margin=abs(a1 - a2), ang_ok=ang_ok(a1, a2), bound_margin=np.inf,
                                tie=_ties(line, p), raised=raised, nb=int(nb), n=n, kind=_CUR["kind"],
                                labels=set(_CUR.get("labels", ()))))
        if raised:
            raise IndexError("recorded")
        return s, ci

    @outer
    def closest_path_index(top, path, pos, n_closest=1):
        res = orig_cp(path=path, pos=pos, n_closest=n_closest)
        if top:
            assert n_closest == 1
            line = np.array(path, dtype=np.float64)[:, :2]
            p = np.asarray(pos, dtype=np.float64).reshape(-1)[:2]
            RECORDS.append(dict(fn=FN_CLOSEST, a=_intern(_LINES, line), b=-1, sarr=-1, pos=p, only_index=False,
                                closed=False, s=np.nan, ci=[-1, -1], idx=int(res[0][0]), inside=-1, ang_margin=np.inf,
                                ang_ok=True, bound_margin=np.inf, tie=_ties(line, p), raised=False, nb=int(res[0][0]),
                                n=line.shape[0], kind=_CUR["kind"], labels=set(_CUR.get("labels", ()))))
        return res

    @outer
    def check_inside_bounds(top, bound1, bound2, pos):
        res = orig_ib(bound1=bound1, bound2=bound2, pos=pos)
        if top:
            b1, b2 = np.array(bound1, dtype=np.float64), np.array(bound2, dtype=np.float64)
            p = np.asarray(pos, dtype=np.float64).reshape(-1)[:2]
            c = (b1 + b2) / 2
            a1, a2, nb, n = angles(ref, c, tuple(p), True)
            pair = orig_gs(ref_line=c, pos=tuple(p), only_index=True, closed=True)[1]
            bm, tie2 = bound_margin(b1, b2, p, pair)
            RECORDS.append(dict(fn=FN_INSIDE, a=_intern(_LINES, b1), b=_intern(_LINES, b2), sarr=-1, pos=p,
                                only_index=False, closed=True, s=np.nan, ci=[int(pair[0]), int(pair[1])], idx=-1,
                                inside=int(bool(res)), ang_margin=abs(a1 - a2), ang_ok=ang_ok(a1, a2),
                                bound_margin=bm, tie=_ties(c, p) or tie2, raised=False, nb=int(nb), n=n,
                                kind=_CUR["kind"], labels=set(_CUR.get("labels", ()))))
        return res

    gs_mod.get_s_coord, cp_mod.closest_path_index, ib_mod.check_inside_bounds = \
        get_s_coord, closest_path_index, check_inside_bounds


def label(r):
    """the labels a recorded call shows"""
    b = set(r["labels"])
    if r["fn"] == FN_INSIDE:
        b.add("inside" if r["inside"] == 1 else "outside")
        return b
    if r["fn"] != FN_S:
        return b
    n, nb = r["n"], r["nb"]
    if r["closed"]:
        if nb == 0:
            b.add("closed_wrap_0")
        if nb == n - 1:
            b.add("closed_wrap_end")
    else:
        if nb == 0:
            b.add("open_start")
        if nb == n - 1:
            b.add("open_end")
    if r["only_index"]:
        b.add("only_index")
    if r["raised"]:
        b.add("index_error")
    if r["ang_margin"] == 0.0:
        b.add("angle_tie")   # ang1 == ang2: `>` (segment for s) and `>=` (index pair) disagree
    return b


def loop_calls(ref, ltpl, track, tag, n_seq, n_ticks, seed):
    vk = dict(vel_max=70.0, gg_scale=0.95, local_gg=(5.0, 5.0), ax_max_machines=GG.ax_max_machines_table(),
              safety_d=25.0, incl_emerg_traj=False)
    n0 = len(RECORDS)
    _CUR["kind"] = 0
    GG.multitick_fixture(ref, ltpl, track, n_seq, n_ticks, vk, seed=seed, n_obj=(1, 3))
    fns = np.bincount([r["fn"] for r in RECORDS[n0:]], minlength=3)
    print("[%s closed loops] %d calls (get_s_coord %d, closest_path_index %d, check_inside_bounds %d)"
          % (tag, len(RECORDS) - n0, fns[0], fns[1], fns[2]))


def direct_calls(ref, raceline, b1, b2, seed=4242):
    """kind 1: synthetic calls; each candidate is kept when its labels are still rare (or always, `force`)"""
    gs = ref.helper_funcs.src.get_s_coord.get_s_coord
    cp = ref.helper_funcs.src.closest_path_index.closest_path_index
    ib = ref.online_graph.src.check_inside_bounds.check_inside_bounds
    rng = np.random.default_rng(seed)
    _CUR["kind"] = 1
    kept = {b: 0 for b in LABELS}

    def one(fn, labels=(), force=False):
        n0 = len(RECORDS)
        _CUR["labels"] = set(labels)
        try:
            fn()
        except IndexError:
            pass
        _CUR["labels"] = set()
        if len(RECORDS) == n0:
            return False
        r = RECORDS[-1]
        bits = label(r)
        if r["ang_ok"] and not r["tie"] and (force or any(kept[b] < 12 for b in bits) or len(RECORDS) % 7 == 0):
            for b in bits:
                kept[b] += 1
            return True
        del RECORDS[n0:]
        return False

    def path(m, step=(0.5, 3.0)):
        el = rng.uniform(*step, size=m - 1)
        s = np.concatenate(([0.0], np.cumsum(el)))
        psi = rng.uniform(-3.1, 3.1) + np.cumsum(rng.normal(0.0, 0.08, size=m))
        xy = np.column_stack((np.cumsum(np.concatenate(([0.0], el * np.cos(psi[:-1])))),
                              np.cumsum(np.concatenate(([0.0], el * np.sin(psi[:-1]))))))
        return xy + rng.uniform(-500, 500, size=2), s

    for c in range(1500):
        m = int(rng.choice([2, 3, 5, 17, 60, 115]))
        xy, s = path(m, (0.01, 0.04) if c % 9 == 0 else (0.5, 3.0))
        k = int(rng.integers(0, m))
        u = c % 6
        if u == 0:
            p = xy[k] + rng.normal(0.0, 1.5, size=2)
        elif u == 1:   # beyond either end, along the line
            e = int(rng.integers(0, 2))
            d = xy[0] - xy[1] if e == 0 else xy[-1] - xy[-2]
            p = (xy[0] if e == 0 else xy[-1]) + d * rng.uniform(0.2, 3.0) + rng.normal(0, 0.05, size=2)
            lab = ("before_start",) if e == 0 else ("beyond_end",)
        elif u == 2:   # exactly on a vertex
            p = xy[k].copy()
        elif u == 3:   # duplicate consecutive points
            if m > 2:
                j = int(rng.integers(0, m - 1))
                xy[j + 1] = xy[j]
            p = xy[k] + rng.normal(0.0, 0.5, size=2)
        elif u == 4:   # far off
            p = xy[k] + rng.normal(0.0, 300.0, size=2)
        else:
            p = xy[k] + rng.normal(0.0, 0.3, size=2)
        labs = {1: lab if u == 1 else (), 2: ("on_vertex",), 3: ("dup_points",), 4: ("far_off",)}.get(u, ())
        closed = bool(c % 4 == 3)
        sel = c % 5
        if sel == 0:
            sa, sl = None, ("sarr_none_ins" if math.hypot(*(xy[1] - xy[0])) > 0.05 else "sarr_none_noins",)
        elif sel == 1:
            sa, sl = s + (0.0 if c % 2 else 0.3), ("sarr_given_noins" if c % 2 else "sarr_given_ins",)
        elif sel == 2:
            sa, sl = s + 0.02, ("sarr_given_noins",)
        else:
            sa, sl = None, ("sarr_none_ins" if math.hypot(*(xy[1] - xy[0])) > 0.05 else "sarr_none_noins",)
        only = c % 11 == 5
        if only:
            sl = ()
        one(lambda: gs(ref_line=xy, pos=tuple(p), s_array=sa, only_index=only, closed=closed), labs + sl)
        if c % 3 == 0:
            one(lambda: cp(path=xy, pos=tuple(p), n_closest=1), labs)
    # exact angle ties (ang1 == ang2 == 0): positions collinear before the start or beyond the end of axis-aligned open
    # lines with dyadic coordinates, so that every difference is exact.  Beyond the end the segment is (nb, nb) (s NaN,
    # t = 0 / 0) while the pair is (nb - 1, nb); before the start the segment is (0, 1) while the pair is (0, 0).
    for c, m in enumerate((2, 3, 5, 17)):
        for vertical in (False, True):
            h = (0.5, 1.25, 2.0, 0.75)[c]
            t = 64.0 * (c - 1) + h * np.arange(m)
            other = np.full(m, -32.25 + 8.0 * c)
            xy = np.column_stack((other, t)) if vertical else np.column_stack((t, other))
            step = xy[1] - xy[0]
            for e, dist in ((0, 1.0), (0, 3.5), (1, 1.0), (1, 6.0)):
                p = xy[0] - dist * step if e == 0 else xy[-1] + dist * step
                for sa in (None, t - t[0], t - t[0] + 0.5):
                    one(lambda: gs(ref_line=xy, pos=tuple(p), s_array=sa), ("before_start",) if e == 0 else
                        ("beyond_end",), force=True)
                one(lambda: gs(ref_line=xy, pos=tuple(p), only_index=True), (), force=True)
    # the shared lines: the closed race line and the track bounds
    n = raceline.shape[0]
    for c in range(400):
        k = int(rng.integers(0, n)) if c % 4 else int(rng.choice([0, 1, n - 2, n - 1]))
        p = raceline[k] + rng.normal(0.0, (0.5, 4.0, 15.0, 60.0)[c % 4], size=2)
        if c % 10 == 0:
            p = raceline[k].copy()
        one(lambda: gs(ref_line=raceline, pos=tuple(p), closed=True), ("on_vertex",) if c % 10 == 0 else ())
        one(lambda: ib(bound1=b1, bound2=b2, pos=list(p)), ("far_off",) if c % 4 == 3 else ())
    # inside / outside by a small margin: points on the segment from the centre to a bound, just before and behind it
    cl = (b1 + b2) / 2
    for c in range(300):
        k = int(rng.integers(0, b1.shape[0]))
        bb = b1 if c % 2 else b2
        f = 1.0 + (1.0 if c % 4 < 2 else -1.0) * 10.0 ** rng.uniform(-7, -3)
        one(lambda: ib(bound1=b1, bound2=b2, pos=list(cl[k] + f * (bb[k] - cl[k]))), force=c < 60)
    print("[direct] labels kept %s" % kept)


def pack():
    lines = [a for _, a in sorted(_LINES.values(), key=lambda t: t[0])]
    sarr = [a for _, a in sorted(_SARR.values(), key=lambda t: t[0])]
    used_l = sorted(set(r["a"] for r in RECORDS) | set(r["b"] for r in RECORDS if r["b"] >= 0))
    used_s = sorted(set(r["sarr"] for r in RECORDS if r["sarr"] >= 0))
    lmap, smap = {o: i for i, o in enumerate(used_l)}, {o: i for i, o in enumerate(used_s)}
    lines, sarr = [lines[i] for i in used_l], [sarr[i] for i in used_s]
    out = dict(line_xy=np.concatenate(lines), line_off=np.cumsum([0] + [a.shape[0] for a in lines]).astype(np.int64),
               sarr=np.concatenate(sarr) if sarr else np.zeros(0),
               sarr_off=np.cumsum([0] + [a.size for a in sarr]).astype(np.int64), label_names=np.array(LABELS))
    out["fn"] = np.array([r["fn"] for r in RECORDS], dtype=np.int32)
    out["line_a"] = np.array([lmap[r["a"]] for r in RECORDS], dtype=np.int32)
    out["line_b"] = np.array([lmap[r["b"]] if r["b"] >= 0 else -1 for r in RECORDS], dtype=np.int32)
    out["sarr_id"] = np.array([smap[r["sarr"]] if r["sarr"] >= 0 else -1 for r in RECORDS], dtype=np.int32)
    out["pos"] = np.array([r["pos"] for r in RECORDS], dtype=np.float64)
    for k in ("only_index", "closed", "raised"):
        out[k] = np.array([r[k] for r in RECORDS], dtype=bool)
    for k in ("s", "ang_margin", "bound_margin"):
        out[k] = np.array([r[k] for r in RECORDS], dtype=np.float64)
    out["closest"] = np.array([r["ci"] for r in RECORDS], dtype=np.int32)
    for k in ("idx", "inside", "kind"):
        out[k] = np.array([r[k] for r in RECORDS], dtype=np.int32)
    out["labels"] = np.array([sum(1 << LABELS.index(b) for b in label(r) if b in LABELS) for r in RECORDS],
                             dtype=np.int64)
    return out


def main():
    ref = GG.load_reference()
    import graph_ltpl.helper_funcs.src.get_s_coord  # noqa: F401
    import graph_ltpl.helper_funcs.src.closest_path_index  # noqa: F401
    import graph_ltpl.online_graph.src.check_inside_bounds  # noqa: F401
    install(ref)
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    track = Track(GG.REF + "/inputs/traj_ltpl_cl/traj_ltpl_cl_monteblanco.csv")
    ltpl, _ = GG.make_ltpl(ref, "default", {})
    loop_calls(ref, ltpl, track, "default", 6, 6, 951)
    l216 = dict(ast.literal_eval(str(np.load(os.path.join(GG.GOLDEN, "ticks_l216.npz"))["overrides"])))
    l216_ltpl, _ = GG.make_ltpl(ref, "l216", l216)
    loop_calls(ref, l216_ltpl, track, "l216", 4, 6, 952)
    for r in RECORDS:
        assert r["ang_ok"] and not r["tie"] and not r["raised"], r
    gb = ltpl._Graph_LTPL__graph_base
    b1 = gb.refline + gb.normvec_normalized * np.expand_dims(gb.track_width_right, 1)   # OTH:207-210
    b2 = gb.refline - gb.normvec_normalized * np.expand_dims(gb.track_width_left, 1)
    direct_calls(ref, np.array(gb.raceline, dtype=np.float64), b1, b2)
    out = pack()
    missing = [b for i, b in enumerate(LABELS) if not np.any(out["labels"] & (1 << i))]
    assert not missing, missing
    np.savez_compressed(os.path.join(GG.GOLDEN, "path_coord.npz"), **out)
    fin = out["ang_margin"][np.isfinite(out["ang_margin"]) & (out["ang_margin"] > 0)]
    print("path_coord.npz: %d calls (%d from closed loops, %d direct; get_s_coord %d, closest_path_index %d, "
          "check_inside_bounds %d), %d lines (%d points), smallest angle margin %.3g rad, smallest bound margin %.3g"
          % (out["fn"].size, int((out["kind"] == 0).sum()), int((out["kind"] == 1).sum()),
             int((out["fn"] == 0).sum()), int((out["fn"] == 1).sum()), int((out["fn"] == 2).sum()),
             out["line_off"].size - 1, out["line_xy"].shape[0], float(fin.min()),
             float(out["bound_margin"][out["fn"] == 2].min())))


if __name__ == "__main__":
    main()
