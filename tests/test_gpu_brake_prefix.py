"""VelocityPlanner.check_brake_prefix on the device: every call of the reference recorded in
tests/golden/brake_prefix.npz (batched ragged calls per kind, and each chain in order with its memory carried), the
float64 boundary of the branch, per-point friction against the oracle with an old gg scale other than the current one,
strided rows, device lengths out of range, calls without a host synchronisation and from a CUDA graph, and the README's
re-timing chain."""
import numpy as np
import pytest
import torch

from tests import brake_prefix_ref as R
from tests import helpers as H

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
RTOL = ATOL = 1e-9   # the float64 brake chain against tph (test_brake_profile_matches_tph)


def _axm():
    return H.golden("ticks_default.npz")["ax_max_machines"]


def _planner(exp=1.0, drag=0.85, mass=1000.0, vel_max=30.0, gg_scale=0.9):
    from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner
    vp = VelocityPlanner(veh_param_dyn_model_exp=exp, veh_param_dragcoeff=drag, veh_param_mass=mass, device=DEV)
    vp.update_dyn_parameters(vel_max=vel_max, gg_scale=gg_scale, ax_max_machines=_axm())
    return vp


def _d(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _check_rows(got, want, ctx):
    """got: (vx_prefix, n_prefix, pref_idx, vel_start, old) as NumPy; want: one (vx_prefix, pref_idx, vel_start, old, c)
    per row.  Exact: n_prefix, pref_idx, the memory and the course part; 1e-9 relative + 1e-9 m/s: the brake part and
    vel_start; zeros behind n_prefix."""
    vx, n_prefix, pref_idx, vel_start, old = got
    for r, (wvx, widx, wvs, wold, c) in enumerate(want):
        n = wvx.size
        assert int(pref_idx[r]) == widx and int(n_prefix[r]) == n, "%s row %d: pref_idx %d n_prefix %d, want %d %d" % (
            ctx, r, pref_idx[r], n_prefix[r], widx, n)
        assert old[r] == wold, "%s row %d: memory %r, want %r" % (ctx, r, old[r], wold)
        assert vx[r, :c].tobytes() == wvx[:c].tobytes(), "%s row %d: course part" % (ctx, r)
        assert np.all(np.abs(vx[r, c:n] - wvx[c:]) <= ATOL + RTOL * np.abs(wvx[c:])), "%s row %d: brake part" % (ctx, r)
        assert abs(vel_start[r] - wvs) <= ATOL + RTOL * abs(wvs), "%s row %d: vel_start %r, want %r" % (
            ctx, r, vel_start[r], wvs)
        assert not np.any(vx[r, n:]), "%s row %d: not zero behind n_prefix" % (ctx, r)


def _run(vp, rows, g, gg):
    """one batched ragged call over recorded calls `rows` with their recorded memory; returns NumPy results + memory"""
    n = len(rows)
    p = int(g["n_pts"][rows].max())
    cap = int(g["n_course"][rows].max())
    old = _d(g["old_before"][rows])
    res = vp.check_brake_prefix(_d(g["vel_plan"][rows]), _d(g["vel_course"][rows, :cap]), _d(g["kappa"][rows, :p]),
                                _d(g["el"][rows, :p - 1]), gg if isinstance(gg, tuple) else _d(g["loc_gg"][rows, :p]),
                                old, n_course=_d(g["n_course"][rows], torch.int32),
                                n_pts=_d(g["n_pts"][rows], torch.int32))
    torch.cuda.synchronize()
    assert res[0].shape == (n, cap + p - 1)
    return [t.cpu().numpy() for t in res] + [old.cpu().numpy()]


def _want(g, c):
    return (g["vx_prefix"][c, :int(g["n_prefix"][c])], int(g["pref_idx"][c]), float(g["vel_start"][c]),
            float(g["old_after"][c]), int(g["n_course"][c]))


def _params_key(g, c):
    return tuple(float(g[k][c]) for k in ("vel_max", "gg_scale", "dyn_model_exp", "drag", "mass"))


def _planners():
    cache = {}

    def get(key):
        if key not in cache:
            vel_max, gg_scale, exp, drag, mass = key
            cache[key] = _planner(exp, drag, mass, vel_max, gg_scale)
        return cache[key]
    return get


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_fixture_calls_batched(kind):
    """the recorded calls of one kind as batched ragged calls, one per parameter set, each row from its recorded
    memory; rows of constant friction go through the constant-friction instance"""
    g = H.golden("brake_prefix.npz")
    planners = _planners()
    groups = {}
    for c in np.flatnonzero(g["kind"] == kind):
        const = not bool(g["has_gg"][c])
        key = _params_key(g, c) + ((True,) + tuple(g["loc_gg"][c, 0]) if const else (False, 0.0, 0.0))
        groups.setdefault(key, []).append(c)
    assert groups
    for key, rows in groups.items():
        gg = (float(key[6]), float(key[7])) if key[5] else None
        got = _run(planners(key[:5]), rows, g, gg)
        _check_rows(got, [_want(g, c) for c in rows], "kind %d %s" % (kind, key))


def test_fixture_chains_in_order():
    """every chain (one reference instance's calls in order) replayed call by call with the memory tensor carried from
    call to call, starting from the instance's first memory"""
    g = H.golden("brake_prefix.npz")
    planners = _planners()
    for ch in np.unique(g["chain"]):
        idx = np.flatnonzero(g["chain"] == ch)
        idx = idx[np.argsort(g["step"][idx])]
        old = _d(g["old_before"][idx[:1]])
        outs = []
        for c in idx:
            p, cap = int(g["n_pts"][c]), int(g["n_course"][c])
            res = planners(_params_key(g, c)).check_brake_prefix(
                _d(g["vel_plan"][c:c + 1]), _d(g["vel_course"][c:c + 1, :cap]), _d(g["kappa"][c:c + 1, :p]),
                _d(g["el"][c:c + 1, :p - 1]), _d(g["loc_gg"][c:c + 1, :p]), old)
            outs.append([t.clone() for t in res] + [old.clone()])
        torch.cuda.synchronize()
        for c, o in zip(idx, outs):
            _check_rows([t.cpu().numpy() for t in o], [_want(g, c)], "chain %d step %d" % (ch, g["step"][c]))


def test_boundary_calls_take_the_reference_branch():
    """vel_plan = nextafter(vel_max + 0.1, -inf) and vel_max + 0.1 need no brake, nextafter(.., +inf) brakes"""
    g = H.golden("brake_prefix.npz")
    rows = np.flatnonzero(R.has(g, "boundary"))
    planners = _planners()
    sides = 0
    for c in rows:
        got = _run(planners(_params_key(g, c)), [c], g, None)
        _check_rows(got, [_want(g, c)], "boundary call %d" % c)
        sides += int(g["pref_idx"][c] > 0)
    assert 0 < sides < rows.size


def _random(n, p, cap, seed, frac_brake=0.5, vel_max=30.0):
    rng = np.random.default_rng(seed)
    el = rng.uniform(0.8, 3.0, size=(n, p - 1))
    s = np.concatenate((np.zeros((n, 1)), np.cumsum(el, axis=1)), axis=1)
    kappa = rng.uniform(0.0, 0.02, size=(n, 1)) * np.sin(s / rng.uniform(20.0, 150.0, size=(n, 1)))
    gg = np.stack((4.0 + 1.5 * np.sin(s / 37.0), 4.5 + np.cos(s / 53.0)), axis=-1)
    brake = rng.random(n) < frac_brake
    vel_plan = np.where(brake, vel_max + 0.1 + rng.uniform(0.5, 40.0, size=n), rng.uniform(0.0, vel_max + 0.1, size=n))
    return dict(kappa=kappa, el=el, gg=gg, vel_plan=vel_plan, vel_course=rng.uniform(10.0, 60.0, size=(n, cap)),
                n_pts=rng.integers(2, p + 1, size=n).astype(np.int32),
                n_course=rng.integers(0, cap + 1, size=n).astype(np.int32),
                old=rng.uniform(0.5, 1.0, size=n))


def _oracle_rows(d, vel_max, gg_scale, exp, gg=None):
    out = []
    for i in range(d["kappa"].shape[0]):
        m, c = int(d["n_pts"][i]), int(d["n_course"][i])
        vx, idx, vs, old = R.prefix_ref(d["vel_plan"][i], d["vel_course"][i, :c], d["kappa"][i, :m],
                                        d["el"][i, :m - 1], d["gg"][i, :m] if gg is None else gg, d["old"][i],
                                        vel_max, gg_scale, exp, 0.85, 1000.0)
        out.append((vx, idx, vs, old, c))
    return out


@pytest.mark.parametrize("exp", [1.0, 1.5])
def test_per_point_friction_against_the_oracle(exp):
    """random ragged paths and courses, per-point and constant friction, the memory other than gg_scale; about half of
    the paths brake"""
    d = _random(300, 160, 5, 7 + int(exp * 2))
    vp = _planner(exp=exp, vel_max=30.0, gg_scale=0.9)
    for gg in (None, (4.5, 5.5)):
        old = d["old"].copy()
        got = vp.check_brake_prefix(d["vel_plan"], d["vel_course"], d["kappa"], d["el"],
                                    d["gg"] if gg is None else gg, old, n_course=d["n_course"], n_pts=d["n_pts"])
        _check_rows(list(got) + [old], _oracle_rows(d, 30.0, 0.9, exp, gg), "exp %g gg %s" % (exp, gg))
        assert 100 < int((got[2] > 0).sum()) < 200


def test_strided_rows_give_the_bytes_of_contiguous_ones():
    d = _random(100, 70, 4, 21)
    vp = _planner()
    t = {k: _d(d[k]) for k in ("kappa", "el", "gg", "vel_plan", "vel_course")}
    nl = {k: _d(d[k], torch.int32) for k in ("n_pts", "n_course")}
    old0 = _d(d["old"])
    ref = [x.clone() for x in vp.check_brake_prefix(t["vel_plan"], t["vel_course"], t["kappa"], t["el"], t["gg"],
                                                     old0, **nl)]

    def wide(x, extra):
        w = torch.full((x.shape[0], x.shape[1] + extra) + tuple(x.shape[2:]), 7.0, dtype=x.dtype, device=DEV)
        w[:, :x.shape[1]] = x
        return w[:, :x.shape[1]]
    old1 = _d(d["old"])
    out = (wide(torch.empty((100, 4 + 69), dtype=torch.float64, device=DEV), 9),
           torch.empty(100, dtype=torch.int32, device=DEV), torch.empty(100, dtype=torch.int32, device=DEV),
           torch.empty(100, dtype=torch.float64, device=DEV))
    got = vp.check_brake_prefix(t["vel_plan"], wide(t["vel_course"], 3), wide(t["kappa"], 5), wide(t["el"], 2),
                                wide(t["gg"], 1), old1, out=out, **nl)
    torch.cuda.synchronize()
    assert got[0].stride(0) == 82
    for a, b in zip(ref, got):
        assert a.cpu().numpy().tobytes() == b.contiguous().cpu().numpy().tobytes()
    assert torch.equal(old0, old1)


def test_out_of_range_device_lengths_give_nan_rows_and_keep_the_memory():
    d = _random(64, 40, 3, 33, frac_brake=0.0)   # no path brakes: every valid row writes its memory
    vp = _planner(gg_scale=0.75)
    n_pts, n_course = d["n_pts"].copy(), d["n_course"].copy()
    n_pts[[3, 9]] = (1, 41)
    n_course[[20, 50]] = (-1, 4)
    bad = np.zeros(64, dtype=bool)
    bad[[3, 9, 20, 50]] = True
    old = _d(d["old"])
    vx, n_prefix, pref_idx, vel_start = (x.cpu().numpy() for x in vp.check_brake_prefix(
        _d(d["vel_plan"]), _d(d["vel_course"]), _d(d["kappa"]), _d(d["el"]), _d(d["gg"]), old,
        n_course=_d(n_course, torch.int32), n_pts=_d(n_pts, torch.int32)))
    old = old.cpu().numpy()
    assert np.all(np.isnan(vx[bad])) and np.all(np.isnan(vel_start[bad]))
    assert np.all(n_prefix[bad] == -1) and np.all(pref_idx[bad] == -1)
    assert np.array_equal(old[bad], d["old"][bad]) and np.all(old[~bad] == 0.75)
    assert not np.any(np.isnan(vx[~bad])) and np.all(n_prefix[~bad] == n_course[~bad])


def test_no_host_sync_and_cuda_graph_replay_carrying_the_memory():
    """a device call under sync debug mode "error"; one call captured in a CUDA graph and replayed three times with the
    memory carried gives the bytes of three eager calls"""
    d = _random(300, 120, 4, 45)
    d["old"][::3] = 0.9   # some rows already hold the current scale
    vp = _planner(gg_scale=0.8)
    t = {k: _d(d[k]) for k in ("kappa", "el", "gg", "vel_plan", "vel_course")}
    nl = {k: _d(d[k], torch.int32) for k in ("n_pts", "n_course")}
    args = (t["vel_plan"], t["vel_course"], t["kappa"], t["el"], t["gg"])

    def outs():
        return (torch.empty((300, 4 + 119), dtype=torch.float64, device=DEV),
                torch.empty(300, dtype=torch.int32, device=DEV), torch.empty(300, dtype=torch.int32, device=DEV),
                torch.empty(300, dtype=torch.float64, device=DEV))
    eager_old = _d(d["old"])
    eager = []
    for _ in range(3):
        eager.append([x.clone() for x in vp.check_brake_prefix(*args, eager_old, **nl)] + [eager_old.clone()])
    torch.cuda.synchronize()
    out = outs()
    old = _d(d["old"])
    torch.cuda.set_sync_debug_mode("error")
    try:
        vp.check_brake_prefix(*args, old, out=out, **nl)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    for a, b in zip(eager[0], list(out) + [old]):
        assert torch.equal(a, b)
    old.copy_(_d(d["old"]))
    for x in out:
        x.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            vp.check_brake_prefix(*args, old, out=out, **nl)
    torch.cuda.current_stream().wait_stream(s)
    old.copy_(_d(d["old"]))   # capture does not run the kernel; start from the same memory as the eager calls
    for k in range(3):
        for x in out:
            x.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(eager[k], list(out) + [old]):
            assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), k
    assert not torch.equal(eager[0][4], _d(d["old"]))   # the first call changed the memory


def test_readme_chain_matches_the_oracle_per_path():
    """README: prefix, shift each row by pref_idx with torch.gather (no synchronisation), plan the remainder from
    vel_start; against check_brake_prefix and calc_vel_profile of the oracle per path.  The prefix at 1e-9 relative +
    1e-9 m/s, the re-timed profile at the fp32 velocity planner's tolerances (helpers.assert_close)."""
    from oracle.ltpl_oracle import OracleLTPL
    import types
    n, p = 200, 150
    d = _random(n, p, 0, 57, frac_brake=0.6, vel_max=35.0)
    d["n_pts"] = np.maximum(d["n_pts"], 100).astype(np.int32)
    d["vel_plan"] = np.minimum(d["vel_plan"], 50.0)
    vp = _planner(vel_max=35.0, gg_scale=0.85)
    kappa, el, gg = _d(d["kappa"]), _d(np.concatenate((d["el"], np.zeros((n, 1))), axis=1)), _d(d["gg"])
    n_pts = _d(d["n_pts"], torch.int32)
    old = _d(d["old"])
    vx_prefix, n_prefix, pref_idx, vel_start = vp.check_brake_prefix(_d(d["vel_plan"]), torch.zeros((n, 0),
                                                                      dtype=torch.float64, device=DEV),
                                                                      kappa, el, gg, old, n_pts=n_pts)
    # shift every row by its pref_idx: point j of the remainder is point pref_idx + j of the path
    cols = (torch.arange(p, device=DEV).unsqueeze(0) + pref_idx.long().unsqueeze(1)).clamp_(max=p - 1)
    k2, e2 = torch.gather(kappa, 1, cols), torch.gather(el, 1, cols)
    g2 = torch.gather(gg, 1, cols.unsqueeze(-1).expand(n, p, 2))
    vx, ax = vp.calc_vel_profile(k2, e2, g2, vel_start, torch.zeros(n, dtype=torch.float64, device=DEV),
                                 n_pts=n_pts - pref_idx)
    torch.cuda.synchronize()
    vx, vx_prefix, pref_idx, vel_start = (t.cpu().numpy() for t in (vx, vx_prefix, pref_idx, vel_start))
    assert 60 < int((pref_idx > 0).sum()) < 180
    rows = _oracle_rows(dict(d, vel_course=np.zeros((n, 0)), n_course=np.zeros(n, dtype=np.int32)), 35.0, 0.85, 1.0)
    ns = types.SimpleNamespace(dyn_model_exp=1.0, drag_coeff=0.85, m_veh=1000.0)
    vk = dict(vel_max=35.0, gg_scale=0.85, ax_max_machines=_axm())
    for i, (wvx, widx, wvs, _, _) in enumerate(rows):
        assert int(pref_idx[i]) == widx
        assert np.allclose(vx_prefix[i, :widx], wvx, rtol=RTOL, atol=ATOL) and abs(vel_start[i] - wvs) <= ATOL + RTOL * wvs
        m = int(d["n_pts"][i])
        if widx == m - 1:   # the brake used the whole path: one point is left, a length the planner refuses (NaN)
            assert np.all(np.isnan(vx[i]))
            continue
        ref = OracleLTPL.vp_calc_vel_profile(ns, d["kappa"][i, widx:m], d["el"][i, widx:m - 1], d["gg"][i, widx:m],
                                             wvs, 0.0, vk)
        H.assert_close("readme chain", vx[i, :m - widx, None], np.asarray(ref)[:, None], ["vx"], ctx="row %d" % i)


@pytest.mark.parametrize("p", [33, 65])
@pytest.mark.parametrize("per_point", [False, True])
def test_cut_at_the_last_point_without_a_course(p, per_point):
    """C = 0 and full-length paths whose brake reaches vel_max only at their last point, or not at all: the cut falls on
    point P - 1, one behind the last prefix position (P - 1 = 32, 64 is a whole number of tiles).  The first half of
    the rows start at a speed bisected on the oracle so that the last point is the first at or below vel_max, the
    second half too fast to get there.  Every row against the oracle; rows whose brake profile comes within 1e-6 m/s of
    vel_max are left out, so the cut is the same on both sides"""
    from oracle import tph_port
    n, vel_max = 128, 30.0
    d = _random(n, p, 0, p + 7 + per_point, frac_brake=1.0, vel_max=vel_max)
    d["n_pts"] = np.full(n, p, dtype=np.int32)
    gg = None if per_point else (4.5, 5.5)

    def profile(i, v):
        loc = d["gg"][i] if per_point else np.tile(gg, (p, 1))
        return tph_port.calc_vel_profile_brake(loc_gg=loc * d["old"][i], kappa=d["kappa"][i], el_lengths=d["el"][i],
                                               v_start=v, dyn_model_exp=1.0, drag_coeff=0.85, m_veh=1000.0)

    def first(i, v):   # the first point at or below vel_max, p if none
        below = np.flatnonzero(profile(i, v) <= vel_max)
        return int(below[0]) if below.size else p

    def least(i, k):   # the least start speed whose first point at or below vel_max is >= k
        lo, hi = vel_max + 0.1, 200.0
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            lo, hi = (lo, mid) if first(i, mid) >= k else (mid, hi)
        return hi
    for i in range(n):
        d["vel_plan"][i] = 0.5 * (least(i, p - 1) + least(i, p)) if i < n // 2 else least(i, p) + 5.0
    keep, last = [], {"reached": 0, "unreached": 0}
    for i in range(n):
        vx = profile(i, d["vel_plan"][i])
        if np.min(np.abs(vx - vel_max)) < 1e-6:
            continue
        keep.append(i)
        if first(i, d["vel_plan"][i]) >= p - 1:
            last["reached" if vx[-1] <= vel_max else "unreached"] += 1
    assert last["reached"] >= 40 and last["unreached"] >= 40, last
    d = {k: v[keep] for k, v in d.items()}
    vp = _planner(vel_max=vel_max, gg_scale=0.9)
    old = _d(d["old"])
    got = vp.check_brake_prefix(_d(d["vel_plan"]), torch.zeros((len(keep), 0), dtype=torch.float64, device=DEV),
                                _d(d["kappa"]), _d(d["el"]), _d(d["gg"]) if per_point else gg, old)
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in got] + [old.cpu().numpy()]
    assert got[0].shape == (len(keep), p - 1) and np.sum(got[2] == p - 1) >= 80
    _check_rows(got, _oracle_rows(d, vel_max, 0.9, 1.0, gg), "P %d per_point %s" % (p, per_point))
