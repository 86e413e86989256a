"""Positions on polylines on the device (pathcoord.get_s_coord, closest_path_index, check_inside_bounds;
ltpl_path_coord_batch): every call of tests/golden/path_coord.npz replayed in ragged batches, per query and on shared
lines; strided selection rows; bytes behind n_pts never read; invalid rows; no host synchronisation; a CUDA graph
replay; NumPy in and out; and the follow mode's object distance from a tick's selected trajectories."""
import numpy as np
import pytest
import torch

from tests import drivers as D
from tests import helpers as H
from tests import path_coord_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _t(a, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def _run(fn, lines, pos, **kw):
    from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P
    if fn == R.FN_S:
        s, ci = P.get_s_coord(lines[0], pos, **kw)
        return s.cpu().numpy(), ci.cpu().numpy(), None, None
    if fn == R.FN_CLOSEST:
        return None, None, P.closest_path_index(lines[0], pos, **kw).cpu().numpy(), None
    return None, None, None, P.check_inside_bounds(lines[0], lines[1], pos, **kw).cpu().numpy()


def _check(g, calls, res, ctx):
    s, ci, idx, inside = res
    for j, c in enumerate(calls):
        fn = int(g["fn"][c])
        if fn == R.FN_S:
            assert R.same_s(float(s[j]), float(g["s"][c])), (ctx, c, s[j], g["s"][c])
            assert tuple(ci[j]) == tuple(g["closest"][c]), (ctx, c)
        elif fn == R.FN_CLOSEST:
            assert idx[j] == g["idx"][c], (ctx, c)
        else:
            assert inside[j] == g["inside"][c], (ctx, c)


def _groups(g, key):
    out = {}
    for c in range(g["fn"].size):
        out.setdefault(key(c), []).append(c)
    return out


@pytest.mark.parametrize("pad", ["nan", "decoy"])
def test_recorded_calls_in_ragged_batches(pad):
    """each call on its own row of a batch of mixed lengths; behind every row's end NaN (an over-read in the neighbour
    or chord stages would show) or the query's own position (a decoy nearer than any point: an over-read in the
    nearest-point scan would take it)"""
    g = H.golden("path_coord.npz")
    rng = np.random.default_rng(3)
    groups = _groups(g, lambda c: (int(g["fn"][c]), bool(g["closed"][c]), bool(g["only_index"][c]),
                                   int(g["sarr_id"][c]) >= 0))
    for (fn, closed, only, has_s), calls in groups.items():
        calls = list(rng.permutation(calls))
        n = np.array([R.line(g, int(g["line_a"][c])).shape[0] for c in calls], dtype=np.int32)
        m = int(n.max()) + 3
        lines = [np.full((len(calls), m, 2), np.nan) for _ in range(2 if fn == R.FN_INSIDE else 1)]
        sa = np.full((len(calls), m), np.nan) if has_s else None
        for j, c in enumerate(calls):
            if pad == "decoy":
                for a in lines:
                    a[j, n[j]:] = g["pos"][c]
            lines[0][j, :n[j]] = R.line(g, int(g["line_a"][c]))
            if fn == R.FN_INSIDE:
                lines[1][j, :n[j]] = R.line(g, int(g["line_b"][c]))
            if has_s:
                sa[j, :n[j]] = R.s_array(g, c)
        kw = dict(n_pts=_t(n, torch.int32))
        if fn == R.FN_S:
            kw.update(closed=closed, only_index=only, s_array=_t(sa) if has_s else None)
        res = _run(fn, [_t(a) for a in lines], _t(g["pos"][calls]), **kw)
        _check(g, calls, res, (fn, closed, only, has_s))


def test_recorded_calls_on_shared_lines():
    """the calls that share one line (race line, track bounds, a path with several queries) as one [M][2] line"""
    g = H.golden("path_coord.npz")
    groups = _groups(g, lambda c: (int(g["fn"][c]), int(g["line_a"][c]), int(g["line_b"][c]), int(g["sarr_id"][c]),
                                   bool(g["closed"][c]), bool(g["only_index"][c])))
    n_shared = 0
    for (fn, a, b, sid, closed, only), calls in groups.items():
        if len(calls) < 2:
            continue
        n_shared += len(calls)
        lines = [_t(R.line(g, a))] + ([_t(R.line(g, b))] if fn == R.FN_INSIDE else [])
        kw = {}
        if fn == R.FN_S:
            kw = dict(closed=closed, only_index=only, s_array=_t(R.s_array(g, calls[0])) if sid >= 0 else None)
        _check(g, calls, _run(fn, lines, _t(g["pos"][calls]), **kw), ("shared", fn, a))
    assert n_shared > 100


def test_strided_selection_rows_give_the_bytes_of_contiguous_ones():
    """x / y columns of a [B][115][7] selection, read in place, against the same values made contiguous; a column
    view of pos too"""
    from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P
    rng = np.random.default_rng(5)
    b = 257
    rows = np.zeros((b, 115, 7))
    s = np.cumsum(rng.uniform(0.5, 2.5, size=(b, 115)), axis=1) - 1.0
    rows[:, :, 0] = s
    rows[:, :, 1] = s * np.cos(0.01 * s) + rng.normal(0, 0.01, size=(b, 115))
    rows[:, :, 2] = 30.0 * np.sin(0.02 * s)
    sel = _t(rows)
    view = sel[:, :, 1:3]
    assert not view.is_contiguous()
    posb = _t(np.column_stack((rows[:, 40, 1] + rng.normal(0, 2, b), rows[:, 40, 2] + rng.normal(0, 2, b),
                               np.zeros(b))))
    pos = posb[:, 0:2]
    n = _t(rng.integers(2, 116, size=b), torch.int32)
    for kw in (dict(), dict(s_array=sel[:, :, 0]), dict(closed=True), dict(only_index=True)):
        a = P.get_s_coord(view, pos, n_pts=n, **kw)
        c = P.get_s_coord(view.contiguous(), pos.contiguous(), n_pts=n,
                          **{k: (v.contiguous() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
        assert a[0].cpu().numpy().tobytes() == c[0].cpu().numpy().tobytes() and torch.equal(a[1], c[1]), kw
    assert torch.equal(P.closest_path_index(view, pos, n_pts=n), P.closest_path_index(view.contiguous(), pos, n_pts=n))
    # the s column (element stride 7) is read in place: with out= the call allocates nothing
    out = (torch.empty(b, dtype=torch.float64, device=DEV), torch.empty((b, 2), dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    P.get_s_coord(view, pos, s_array=sel[:, :, 0], n_pts=n, out=out)
    assert torch.cuda.max_memory_allocated() == m0
    b2 = view + 3.0
    assert torch.equal(P.check_inside_bounds(view, b2, pos, n_pts=n),
                       P.check_inside_bounds(view.contiguous(), b2.contiguous(), pos, n_pts=n))


def test_invalid_rows():
    """device lengths out of range, a position that is not finite, and a row without a point at a finite distance: s NaN,
    closest (-2, -2), idx -1, inside -1; the valid rows of the same batch as computed alone"""
    from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P
    m = 20
    t = np.linspace(0.0, 40.0, m)
    line = np.stack([np.column_stack((t, 0.1 * t * t))] * 7)
    line2 = line + np.array([0.0, 5.0])
    pos = np.tile([10.0, 12.0], (7, 1))
    n = np.array([0, 1, m + 1, m, m, m, 7], dtype=np.int32)
    pos[3] = [np.nan, 1.0]
    pos[4] = [1.0, np.inf]
    line[5] = np.nan
    line2[5] = np.nan
    bad = np.array([1, 1, 1, 1, 1, 1, 0], dtype=bool)
    args = (_t(line), _t(pos))
    for kw in (dict(), dict(closed=True), dict(only_index=True), dict(s_array=_t(np.tile(t, (7, 1))))):
        s, ci = P.get_s_coord(*args, n_pts=_t(n, torch.int32), **kw)
        s, ci = s.cpu().numpy(), ci.cpu().numpy()
        assert np.all(np.isnan(s[bad])) and np.all(ci[bad] == -2), kw
        kw1 = {k: (v[6:] if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
        s1, ci1 = P.get_s_coord(_t(line[6:]), _t(pos[6:]), n_pts=_t(n[6:], torch.int32), **kw1)
        assert R.same_s(float(s[6]), float(s1.cpu()[0])) and np.array_equal(ci[6], ci1.cpu().numpy()[0]), kw
        assert np.all(ci[6] >= 0)
    idx = P.closest_path_index(*args, n_pts=_t(n, torch.int32)).cpu().numpy()
    assert np.all(idx[bad] == -1) and idx[6] >= 0
    ins = P.check_inside_bounds(_t(line), _t(line2), _t(pos), n_pts=_t(n, torch.int32)).cpu().numpy()
    assert ins.dtype == np.int8 and np.all(ins[bad] == -1) and ins[6] in (0, 1)


def test_empty_batches():
    """N = 0: empty results of the right types, device and NumPy, per query and on a shared line"""
    from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P
    pos = torch.empty((0, 2), dtype=torch.float64, device=DEV)
    for line in (torch.empty((0, 5, 2), dtype=torch.float64, device=DEV), _t(np.arange(10.0).reshape(5, 2))):
        s, ci = P.get_s_coord(line, pos, s_array=None)
        assert s.shape == (0,) and ci.shape == (0, 2) and ci.dtype == torch.int32
        assert P.closest_path_index(line, pos).shape == (0,)
        ins = P.check_inside_bounds(line, line, pos)
        assert ins.shape == (0,) and ins.dtype == torch.int8
    hs, hci = P.get_s_coord(np.zeros((0, 5, 2)), np.zeros((0, 2)))
    assert isinstance(hs, np.ndarray) and hs.shape == (0,) and hci.shape == (0, 2)


def test_no_host_sync_graph_replay_and_numpy():
    """device in / out under sync debug mode "error"; a CUDA graph captured with out= replays to the eager bytes; NumPy
    in gives NumPy out with the same values"""
    from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P
    g = H.golden("path_coord.npz")
    calls = np.flatnonzero((g["fn"] == R.FN_S) & g["closed"] & (g["sarr_id"] < 0))
    a = int(g["line_a"][calls[0]])
    calls = calls[g["line_a"][calls] == a]
    line, pos = _t(R.line(g, a)), _t(g["pos"][calls])
    n = len(calls)
    ref = [x.clone() for x in P.get_s_coord(line, pos, closed=True)]
    out = (torch.empty(n, dtype=torch.float64, device=DEV), torch.empty((n, 2), dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        P.get_s_coord(line, pos, closed=True, out=out)
        P.closest_path_index(line, pos)
        P.check_inside_bounds(line, line + 1.0, pos)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(ref[0], out[0]) and torch.equal(ref[1], out[1])
    for x in out:
        x.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            P.get_s_coord(line, pos, closed=True, out=out)
    torch.cuda.current_stream().wait_stream(s)
    for x in out:
        x.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(ref[0], out[0]) and torch.equal(ref[1], out[1])
    hs, hci = P.get_s_coord(R.line(g, a), g["pos"][calls], closed=True)
    assert isinstance(hs, np.ndarray) and hs.tobytes() == ref[0].cpu().numpy().tobytes()
    assert np.array_equal(hci, ref[1].cpu().numpy())
    m = R.line(g, a).shape[0]
    hidx = P.closest_path_index(R.line(g, a), g["pos"][calls], n_pts=np.full(n, 2))
    assert isinstance(hidx, np.ndarray) and hidx.dtype == np.int32 and np.all(hidx < 2) and m >= 2


def test_follow_object_distance_from_selected_trajectories():
    """obj_dist = get_s_coord(path, obj_pos, s)[0] - get_s_coord(path, pos, s)[0] (OTH:774-782) on the selected rows of a
    tick, on the device, is the oracle's on the downloaded rows; calc_vel_profile_follow gives the same bytes with
    either"""
    from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner
    from oracle import ltpl_oracle as O
    from tests import vel_follow_ref as VR
    lat = H.lattice_for("default")
    sc = make_scenarios(Track(H.TRACK_CSV), 64, seed=21, n_obj_min=1, n_obj_max=2)
    pl = D.planner(lat, ax_max_machines=H.golden("ticks_default.npz")["ax_max_machines"])
    D.first_tick(pl, sc)
    sel = pl.select(["follow", "straight", "left", "right"])
    rows = sel["sel_info"][:, 2].to(torch.int32)
    keep = torch.nonzero(rows >= 2).flatten()   # (outside the timed path: the test picks scenarios with a trajectory)
    traj = sel["sel_traj"].double()[keep]
    n_pts = rows[keep]
    obj = np.array([[sc.object_list(b)[0]["X"], sc.object_list(b)[0]["Y"]] for b in keep.cpu().numpy()])
    obj_pos, ego = _t(obj), traj[:, 0, 1:3] + 0.3
    line, s_arr = traj[:, :, 1:3], traj[:, :, 0]
    d = P.get_s_coord(line, obj_pos, s_array=s_arr, n_pts=n_pts)[0] - P.get_s_coord(line, ego, s_array=s_arr,
                                                                                      n_pts=n_pts)[0]
    h, hn, he = traj.cpu().numpy(), n_pts.cpu().numpy(), ego.cpu().numpy()
    want = np.array([O.get_s_coord(h[i, :hn[i], 1:3], tuple(obj[i]), h[i, :hn[i], 0])[0]
                     - O.get_s_coord(h[i, :hn[i], 1:3], tuple(he[i]), h[i, :hn[i], 0])[0] for i in range(len(hn))])
    got = d.cpu().numpy()
    assert all(R.same_s(float(a), float(b)) for a, b in zip(got, want))
    vp = VelocityPlanner(device=DEV, len_veh=4.7, follow_control_type="PD",
                         follow_control_params={"c_p": 1.25, "k_d": 0.025, "k_p": 0.2}, glob_rl=VR.race_line())
    vp.update_dyn_parameters(vel_max=60.0, gg_scale=1.0, ax_max_machines=H.golden("ticks_default.npz")["ax_max_machines"])
    kappa = traj[:, :, 4].contiguous()
    el = torch.zeros_like(kappa)
    el[:, :-1] = traj[:, 1:, 0] - traj[:, :-1, 0]
    k = kappa.shape[0]
    v = traj[:, 0, 5].contiguous()
    args = (kappa, el, (5.0, 5.0), v, v, 0.5 * v, torch.full((k,), 20.0, dtype=torch.float64, device=DEV))
    a = vp.calc_vel_profile_follow(*args, torch.nan_to_num(d, nan=50.0), obj_pos, n_pts=n_pts)
    b = vp.calc_vel_profile_follow(*args, _t(np.nan_to_num(want, nan=50.0)), obj_pos, n_pts=n_pts)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
