"""Location dependent friction computed on the device between the two halves of a tick: set_local_gg_planes from
device tensors gives the bytes of the same planes uploaded from NumPy (first and stateful ticks, non-contiguous views,
planes narrower than p_max) and still reproduces the reference's ggpp closed loop; split ticks replayed from CUDA graphs
(capture_split_tick / capture_next_split_tick, SplitTickGraph) give the bytes of the same split calls run eagerly, on
three lattices and in the ggpp closed loop from both parities, interleaved with eager full and split ticks.  Neither
does host work, and refusals change nothing."""
import numpy as np
import pytest
import torch

from tests import drivers as D
from tests import gg_map_ref as M
from tests import helpers as H
from tests.test_gpu_device_inputs import MAP, _assert_inputs_equal, _assert_same, _fixture_inputs, _scenarios
from tests.test_gpu_tick_graph import _axm, _dev, _ids, _refused, _results, _state

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
NSLOT = 3
GGPP = "ticks_multitick_ggpp_default.npz"


def _field(path, batch, n=None):
    """H.local_gg_field evaluated by torch on the device along the path planes [5][NSLOT * B][p_max] (device_results()
    ["path"]), points [0, n): the planes (ax, ay) [NSLOT][B][n] as the two columns of one [..][2] tensor, so both are
    non-contiguous views"""
    x, y = (path[0], path[1]) if n is None else (path[0, :, :n], path[1, :, :n])
    gg = torch.stack((4.2 + 1.1 * torch.sin(0.011 * x + 0.5), 4.6 + 0.9 * torch.cos(0.013 * y - 0.3)), dim=-1)
    gg = gg.view(NSLOT, batch, -1, 2)
    return gg[..., 0], gg[..., 1]


def _like(pl, batch):
    """example planes of the full width for a capture"""
    ones = torch.ones((NSLOT, batch, pl.cap["p_max"]), dtype=torch.float64, device=DEV)
    return ones, ones.clone()


def _first_split(pl, dsc, pos, vel, planes=True):
    """the eager first tick in halves: stage + set_startpos + calc_paths, the estimates and the torch field along the
    new paths, calc_vel_profile"""
    pl.stage_scenarios(dsc)
    pl.set_startpos()
    pl.calc_paths()
    pl.set_estimates(pos, vel)
    if planes:
        pl.set_local_gg_planes(*_field(pl.device_results()["path"], dsc.size))
    pl.calc_vel_profile()


def _next_split(pl, dsc, sel, t_c, pos, vel):
    pl.next_calc_paths(dsc, sel, t_c)
    pl.set_local_gg_planes(*_field(pl.device_results()["path"], dsc.size))
    pl.next_calc_vel_profile(pos_est=pos, vel_est=vel)


def _replay(graph, pos, vel, planes=True):
    pl = graph.planner
    graph.replay_paths()
    gg = _field(pl.device_results()["path"], pl.dims.batch) if planes else None
    graph.vel_inputs.copy_(pos, vel, gg)
    graph.replay_vel_profile()


# ---- device planes == host planes ----------------------------------------------------------------------------------
def test_device_planes_equal_host_planes():
    """the ggpp closed loop on two stateful planners, first tick included: one takes NumPy planes, the other the same
    values as device tensors (views with stride 2; on odd ticks narrower than p_max).  The values are evaluated once,
    by torch on the device, and copied to the host for the first planner.  Packed inputs, the planes, results and
    memory are byte-equal after every tick."""
    g = H.golden(GGPP)
    n_seq, n_ticks = g["dt"].shape
    lat = H.lattice_for("default")
    vel_kw = dict(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True)
    ph, pd = (D.planner(lat, 1 + n_seq % 4, stateful=True, **vel_kw) for _ in range(2))
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)])
    n_traj = 0
    for k in range(n_ticks):
        sc, sel, t_c, v_est, _, gg_scale = _fixture_inputs(g, "ggpp", k, tc)
        for pl in (ph, pd):
            pl.set_vel_params(**dict(D.VEL, gg_scale=gg_scale, **vel_kw))
        dsc = sc.to_device(DEV)
        if k == 0:
            for pl, batch in ((ph, sc), (pd, dsc)):
                pl.stage_scenarios(batch, vel_est=v_est if pl is ph else _dev(v_est))
                pl.upload()
                pl.set_startpos()
                pl.calc_paths()
        else:
            ph.next_calc_paths(sc, sel, t_c)
            pd.next_calc_paths(dsc, _dev(sel, np.int32), _dev(t_c))
        _assert_inputs_equal(ph, pd, "tick %d" % k)
        assert torch.equal(pd.device_results()["path"], ph.device_results()["path"]), "tick %d: path" % k
        n = pd.dims.p_max - 37 if k % 2 else None
        ax, ay = _field(pd.device_results()["path"], sc.size, n)
        assert not ax.is_contiguous() and ax.shape[2] == (n or pd.dims.p_max)
        ph.set_local_gg_planes(ax.cpu().numpy(), ay.cpu().numpy())
        pd.set_local_gg_planes(ax, ay)
        assert torch.equal(pd.t["gg"], ph.t["gg"]), "tick %d: the planes differ" % k
        if k == 0:
            for pl in (ph, pd):
                pl.calc_vel_profile()
        else:
            ph.next_calc_vel_profile(pos_est=g["pos_est"][:, k], vel_est=v_est)
            pd.next_calc_vel_profile(pos_est=_dev(g["pos_est"][:, k]), vel_est=_dev(v_est))
        _assert_same(_state(pd), _state(ph), "tick %d" % k)
        n_traj += int((ph.fetch("traj_len")["traj_len"] > 0).sum())
    assert n_traj > n_seq * n_ticks


@pytest.mark.parametrize("group", [0, 1])
def test_device_planes_match_the_reference(group):
    """the ggpp fixture (grip drop on the odd sequences: gg_scale is per batch, so each half runs apart) from device
    batches, with the planes of H.local_gg_field evaluated on the host along device_results()["path"] and given as
    device tensors: every tick matches the reference within the parity tolerances"""
    from graphbasedlocaltrajectoryplanner_b200 import capi
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    g = D.Rows(H.golden(GGPP), np.arange(group, H.golden(GGPP)["dt"].shape[0], 2))
    n_seq, n_ticks = g["dt"].shape
    pl = D.planner(H.lattice_for("default"), 1 + n_seq % 4, stateful=True, ax_max_machines=g["ax_max_machines"],
                   incl_emerg_traj=True)
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)])
    fails, compared = [], 0
    alive = np.ones(n_seq, dtype=bool)
    for k in range(n_ticks):
        sc = ScenarioBatch(g["pos_est"][:, k].copy(), g["sc_heading"].copy(), g["sc_vel"].copy(), g["sc_n_obj"].copy(),
                           g["obj"][:, k].copy())
        pl.set_vel_params(**dict(D.VEL, ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True,
                                 gg_scale=float(g["gg_scale"][0, k])))
        dsc = sc.to_device(DEV)
        if k == 0:
            pl.stage_scenarios(dsc, vel_est=_dev(g["vel_est"][:, k]))
            pl.set_startpos()
            pl.calc_paths()
        else:
            pl.next_calc_paths(dsc, _dev(g["sel"][:, k], np.int32), _dev(tc[:, k - 1]))
        path = pl.device_results()["path"].cpu().numpy()
        gg = H.local_gg_field(np.column_stack((path[0].ravel(), path[1].ravel())))
        shape = (NSLOT, n_seq, path.shape[2])
        pl.set_local_gg_planes(_dev(gg[:, 0].reshape(shape)), _dev(gg[:, 1].reshape(shape)))
        if k == 0:
            pl.calc_vel_profile()
        else:
            pl.next_calc_vel_profile(vel_est=_dev(g["vel_est"][:, k]))
        recs = pl.records()
        for q in range(n_seq):
            if not alive[q] or k >= int(g["n_done"][q]):
                continue
            ctx = "sequence %d tick %d" % (q, k)
            try:
                assert not (recs[q]["flags"] & capi.SC_STATE_FALLBACK), ctx + " fell back"
                assert not recs[q]["out_of_track"] and "error" not in recs[q], ctx + " flags %d" % recs[q]["flags"]
                compared += D.compare_multitick_row(recs[q], g, q, k, ctx, True)
            except AssertionError as e:
                fails.append(str(e).split("\n")[0][:400])
                alive[q] = False
    assert not fails, "%d sequences diverged:\n%s" % (len(fails), "\n".join(fails[:8]))
    assert compared > 30


# ---- split replays == eager split calls ----------------------------------------------------------------------------
@pytest.mark.parametrize("tag,n,windows", [("default", 384, 4), ("l216", 257, 3), ("open", 200, 1)])
def test_first_split_replays_equal_eager_split_calls(tag, n, windows):
    """capture_split_tick once, then 4 seeded device batches: paths_inputs.copy_ + replay_paths, the torch field along
    device_results()["path"] and the estimates into vel_inputs, replay_vel_profile == the eager split calls of the same
    tensors on a twin planner, every result incl. the ids (10, 20, 30, 40)"""
    lat = H.lattice_for(tag)
    vel_kw = dict(ax_max_machines=_axm(tag), incl_emerg_traj=True)
    pg, pe = D.planner(lat, windows, **vel_kw), D.planner(lat, windows, **vel_kw)
    sc0 = _scenarios(tag, n, 9600).to_device(DEV)
    graph = pg.capture_split_tick(sc0, vel_est=sc0.vel, pos_est=sc0.pos, local_gg=_like(pg, n))
    assert graph.n_graphs == 2 and graph.vel_inputs.ax.shape == (NSLOT, n, pg.cap["p_max"])
    for i in range(1, 5):
        dsc = _scenarios(tag, n, 9600 + i).to_device(DEV)
        pos, vel = dsc.pos + 0.05 * i, dsc.vel * 0.97
        graph.paths_inputs.copy_(dsc)
        _replay(graph, pos, vel)
        _first_split(pe, dsc, pos, vel)
        got, want = _results(pg), _results(pe)
        _assert_same(got, want, "%s replay %d" % (tag, i))
        assert (want["traj_len"] > 0).sum() > n
        assert list(_ids(pg)) == [i]


@pytest.mark.parametrize("shift", [0, 1])
def test_closed_loop_split_replays_equal_eager_split_calls(shift):
    """the ggpp closed loop from device tensors: the twin runs eager split calls (a full next_tick where the other
    does), the other interleaves eager split calls, an eager full next_tick and split replays, the graph captured at
    either parity (after `shift` eager stateful ticks) and anew after the full tick, whose buffers leave the captured
    states (three states then: the planes were unused in the tick before).  Results, memory and ids byte-equal after
    every tick."""
    g = H.golden(GGPP)
    n_seq, n_ticks = g["dt"].shape
    lat = H.lattice_for("default")
    vel_kw = dict(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True)
    pe, pg = (D.planner(lat, 1 + n_seq % 4, stateful=True, **vel_kw) for _ in range(2))
    tc = np.array([D.t_const(g["dt"][q, 1:]) for q in range(n_seq)])
    pattern = (["split"] * shift + ["replay", "replay", "split", "replay", "full", "replay", "replay"])[:n_ticks - 1]
    graph, scale, n_graphs = None, None, []
    for k, how in enumerate(["first"] + pattern):
        sc, sel, t_c, v_est, _, gg_scale = _fixture_inputs(g, "ggpp", k, tc)
        if gg_scale != scale:
            for pl in (pe, pg):
                pl.set_vel_params(**dict(D.VEL, gg_scale=gg_scale, **vel_kw))
            scale, graph = gg_scale, None
        dsc = sc.to_device(DEV)
        args, pos, vel = (_dev(sel, np.int32), _dev(t_c)), _dev(g["pos_est"][:, k]), _dev(v_est)
        if how == "first":
            for pl in (pe, pg):
                _first_split(pl, dsc, pos, vel)
        elif how == "full":
            for pl in (pe, pg):
                pl.next_tick(dsc, *args, vel_est=vel)
            graph = None
        else:
            _next_split(pe, dsc, *args, pos, vel)
            if how == "split":
                _next_split(pg, dsc, *args, pos, vel)
            else:
                if graph is None:
                    graph = pg.capture_next_split_tick(dsc, *args, vel_est=vel, pos_est=pos, local_gg=_like(pg, n_seq))
                    n_graphs.append(graph.n_graphs)
                graph.paths_inputs.copy_(dsc, *args)
                _replay(graph, pos, vel)
        _assert_same(_state(pg), _state(pe), "tick %d (%s)" % (k, how))
        assert list(_ids(pg)) == [k + 1], (k, how)
    assert pg._tick_count == pe._tick_count == len(pattern) + 1
    assert n_graphs == [4, 6], n_graphs


# ---- no host work --------------------------------------------------------------------------------------------------
def test_device_planes_and_split_replays_do_no_host_work():
    """an eager stateful tick with device planes and split replays under torch.cuda.set_sync_debug_mode('error'); a
    replay makes no library call (launch count unchanged); both equal their eager twin"""
    sc = _scenarios("default", 256, 9700)
    lat = H.lattice_for("default")
    pe, pg = (D.planner(lat, 4, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True) for _ in range(2))
    dsc = sc.to_device(DEV)
    for pl in (pe, pg):
        _first_split(pl, dsc, dsc.pos, dsc.vel)
    sel = pe.device_results()["action_id"].max(dim=0).values.clamp(min=0)
    graph = pg.capture_next_split_tick(dsc, sel, 0.15, vel_est=dsc.vel, pos_est=dsc.pos, local_gg=_like(pg, sc.size))
    for k in range(3):
        sel = pe.device_results()["action_id"].max(dim=0).values.clamp(min=0)
        vel = dsc.vel * (0.9 + 0.02 * k)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            _next_split(pe, dsc, sel, 0.15, dsc.pos, vel)
            n0 = pg.launch_count()
            graph.paths_inputs.copy_(dsc, sel)
            _replay(graph, dsc.pos, vel)
            n1 = pg.launch_count()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert n1 == n0
        _assert_same(_state(pg), _state(pe), "replay %d" % k)


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_bad_planes_are_refused_before_writing():
    """wrong device, dtype, rank, batch, slot count, width > p_max, unequal shapes, a host array next to a tensor:
    ValueError, no buffer and no launch changed, and a friction map set before stays"""
    sc = _scenarios("default", 96, 9800)
    pl = D.planner(H.lattice_for("default"), 2, stateful=True, ax_max_machines=_axm())
    _first_split(pl, sc.to_device(DEV), sc.to_device(DEV).pos, sc.to_device(DEV).vel)
    pl.set_gg_map(*M.surface_map(MAP[2], x0=MAP[0], y0=MAP[1], width=500.0, height=350.0), *MAP)
    B, P = sc.size, pl.dims.p_max
    ok = torch.ones((NSLOT, B, P), dtype=torch.float64, device=DEV)
    bad = [(ok.cpu(), ok.cpu()), (ok.float(), ok.float()), (ok[0], ok[0]), (ok[:, :-1], ok[:, :-1]),
           (ok[:2], ok[:2]), (torch.ones((NSLOT, B, P + 1), dtype=torch.float64, device=DEV),) * 2,
           (ok, ok[:, :, :-1]), (ok, np.ones((NSLOT, B, P)))]
    generation = pl._generation
    for ax, ay in bad:
        _refused(pl, lambda: pl.set_local_gg_planes(ax, ay), "local_gg planes")
    assert pl._gg_map is not None and pl.buf.gg_map is not None and pl._generation == generation


def test_split_replays_in_the_wrong_order_are_refused():
    sc = _scenarios("default", 96, 9810)
    dsc = sc.to_device(DEV)
    lat = H.lattice_for("default")
    pl = D.planner(lat, 2, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True)
    _first_split(pl, dsc, dsc.pos, dsc.vel)
    sel = pl.device_results()["action_id"].max(dim=0).values.clamp(min=0)
    graph = pl.capture_next_split_tick(dsc, sel, 0.1, vel_est=dsc.vel, local_gg=_like(pl, sc.size))
    other = pl.capture_next_split_tick(dsc, sel, 0.1)
    _refused(pl, graph.replay_vel_profile, "last call")
    graph.replay_paths()
    ticks = pl._tick_count
    _refused(pl, graph.replay_paths, "velocity half")
    _refused(pl, other.replay_paths, "velocity half")
    _refused(pl, other.replay_vel_profile, "last call")
    graph.vel_inputs.copy_(None, dsc.vel, _field(pl.device_results()["path"], sc.size))
    graph.replay_vel_profile()
    assert pl._tick_count == ticks + 1
    _refused(pl, graph.replay_vel_profile, "last call")
    graph.replay_paths()
    pl.set_estimates(vel_est=dsc.vel)   # any other call in between: the velocity half is refused
    _refused(pl, graph.replay_vel_profile, "last call")
    with pytest.raises(ValueError, match="is required"):
        graph.vel_inputs.copy_(None, None, None)
    with pytest.raises(ValueError, match="was not captured"):
        other.vel_inputs.copy_(dsc.pos)


def test_refused_split_captures_change_nothing():
    sc = _scenarios("default", 96, 9820)
    dsc = sc.to_device(DEV)
    lat = H.lattice_for("default")
    fresh = D.planner(lat, 2, stateful=True, ax_max_machines=_axm())
    fresh.allocate(sc.size, 3)
    sel = torch.zeros(sc.size, dtype=torch.int32, device=DEV)
    _refused(fresh, lambda: fresh.capture_next_split_tick(dsc, sel, 0.1), "no previous tick")
    pl = D.planner(lat, 2, stateful=True, ax_max_machines=_axm())
    _first_split(pl, dsc, dsc.pos, dsc.vel)
    planes = _like(pl, sc.size)
    _refused(pl, lambda: pl.capture_split_tick(sc), "DeviceScenarioBatch")
    _refused(pl, lambda: pl.capture_next_split_tick(sc, sel, 0.1, local_gg=planes), "DeviceScenarioBatch")
    _refused(pl, lambda: pl.capture_next_split_tick(dsc, sel, 0.1, local_gg=(planes[0].float(), planes[1])),
             "float64")
    _refused(pl, lambda: pl.capture_next_split_tick(dsc, sel, 0.1, local_gg=planes[0]), "pair")
    _refused(pl, lambda: pl.capture_next_split_tick(dsc, sel, 0.1, pos_est=dsc.pos.t()), "pos_est")
    pl.set_local_gg_planes(*H.local_gg_planes(pl))   # uploaded from the host
    _refused(pl, lambda: pl.capture_split_tick(dsc, local_gg=planes), "local_gg planes")
    _refused(pl, lambda: pl.capture_next_split_tick(dsc, sel, 0.1), "local_gg planes")
    pl.set_gg_map(*M.surface_map(MAP[2], x0=MAP[0], y0=MAP[1], width=500.0, height=350.0), *MAP)
    _refused(pl, lambda: pl.capture_next_split_tick(dsc, sel, 0.1, local_gg=planes), "friction map")
    assert pl._traj_base is None and pl.buf.traj_base is None   # nothing was prepared either


def test_stale_split_graphs_refuse_to_replay():
    """set_vel_params makes every split graph stale; set_local_gg_planes makes a graph without planes stale, while
    one that sets its own planes replays on and equals the eager twin"""
    sc = _scenarios("default", 96, 9830)
    dsc = sc.to_device(DEV)
    lat = H.lattice_for("default")
    pe, pl = (D.planner(lat, 2, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True) for _ in range(2))
    for p in (pe, pl):
        _first_split(p, dsc, dsc.pos, dsc.vel)
    sel = pe.device_results()["action_id"].max(dim=0).values.clamp(min=0)
    own = pl.capture_next_split_tick(dsc, sel, 0.1, pos_est=dsc.pos, vel_est=dsc.vel, local_gg=_like(pl, sc.size))
    bare = pl.capture_next_split_tick(dsc, sel, 0.1)
    pl.set_local_gg_planes(None)
    pe.set_local_gg_planes(None)
    _refused(pl, bare.replay_paths, "changed since the capture")
    _next_split(pe, dsc, sel, 0.1, dsc.pos, dsc.vel)
    own.paths_inputs.copy_(dsc, sel)
    _replay(own, dsc.pos, dsc.vel)
    _assert_same(_state(pl), _state(pe), "own planes after set_local_gg_planes(None)")
    own.replay_paths()
    pl.set_vel_params(**dict(D.VEL, ax_max_machines=_axm(), incl_emerg_traj=True))
    ticks = pl._tick_count
    _refused(pl, own.replay_vel_profile, "changed since the capture")
    _refused(pl, own.replay_paths, "velocity half")
    assert pl._tick_count == ticks
    own.close()
    pl.set_estimates(vel_est=dsc.vel)   # any other call ends the wait for the velocity half
    with pytest.raises(ValueError, match="closed"):
        own.replay_paths()
    bare.close()
