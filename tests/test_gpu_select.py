"""The trajectory each scenario takes, on the device (BatchPlanner.select, k_select): the rule of tests/select_ref.py on
the results as the tick left them, over first and stateful ticks with restarts, emergency off and on, and preference
lists of every integer width, strided and broadcast; closed loops fed by sel_action="selected" against host-computed
actions; graph replays that end with the selection against eager ticks; plan_batch / plan_stream with prefer against
the full download; and the refusals."""
from dataclasses import replace

import numpy as np
import pytest
import torch

from tests import drivers as D
from tests import helpers as H
from tests.select_ref import select_ref
from tests.test_gpu_device_inputs import _scenarios
from tests.test_gpu_tick_graph import _axm, _state

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
N = 1000
# the rotating preference orders of the closed loops (tests/drivers.closed_loop_vs_session, oracle/gen_golden.py)
ORDERS = (("right", "left", "straight", "follow"), ("follow", "straight", "left", "right"),
          ("left", "straight", "follow", "right"))
IDS = dict(straight=0, follow=1, left=2, right=3, emergency=4)
T_CONST = 0.15


def _order_ids(n, k, emergency_first=False):
    """[n][L] int64: scenario b prefers ORDERS[(b + k) % 3] (with 'emergency' in front)"""
    rows = [[IDS[a] for a in ORDERS[(b + k) % 3]] for b in range(n)]
    ids = np.array(rows, dtype=np.int64)
    if emergency_first:
        ids = np.concatenate((np.full((n, 1), 4), ids), axis=1)
    return ids


def _step(sel, pos, vel):
    """the vehicle dummy on the device: to row 1 of the selected trajectory (position and velocity), where one was
    selected"""
    ok = sel["sel_info"][:, :1] >= 0
    pos = torch.where(ok, sel["sel_traj"][:, 1, 1:3].double(), pos)
    vel = torch.where(ok[:, 0], sel["sel_traj"][:, 1, 5].double(), vel)
    return pos, vel


def _selection(sel_info, sel_traj):
    """a selection comparable across planners: the compact row a trajectory gets is unspecified, and a row holds what an
    earlier tick wrote there behind its length, so the row index is left out and the rows are cleared behind it"""
    info, rows = sel_info.cpu().numpy(), sel_traj.cpu().numpy().copy()
    rows[np.arange(rows.shape[1])[None, :] >= info[:, 2:3]] = 0.0
    return info[:, [0, 2, 3]], rows


def _check(pl, sel, prefer, emerg, ctx):
    """select()'s outputs against select_ref on the fetched results; sel_traj byte-equal to the selected export row,
    zero without a selection"""
    f = pl.fetch("action_id", "traj_row", "traj_len", "traj_id", "em_info")
    traj = pl.device_results()["traj"].cpu().numpy()
    want_act, want_info = select_ref(f["action_id"], f["traj_row"], f["traj_len"], f["traj_id"], f["em_info"], emerg,
                                     prefer)
    info = sel["sel_info"].cpu().numpy()
    assert np.array_equal(sel["sel_action"].cpu().numpy(), want_act), ctx
    assert np.array_equal(info, want_info), ctx
    rows = sel["sel_traj"].cpu().numpy()
    ok = info[:, 1] >= 0
    assert np.array_equal(rows[ok].view(np.uint32), traj[info[ok, 1]].view(np.uint32)), ctx + ": sel_traj"
    assert not rows[~ok].any(), ctx + ": sel_traj behind no selection"
    return want_act


def _prefer_variants(n, k, rng):
    """(prefer as passed, its ids [n or 1][L] for select_ref, name): int8 per scenario with ids outside the five, an
    int32 column slice, a broadcast int64 row, names and a host array"""
    out = []
    i8 = torch.as_tensor(rng.integers(-2, 7, size=(n, 6)), dtype=torch.int8, device=DEV)
    out.append((i8, i8.cpu().numpy(), "int8"))
    wide = torch.as_tensor(np.repeat(_order_ids(n, k, emergency_first=k % 2 == 1), 2, axis=1), dtype=torch.int32,
                           device=DEV)
    sl = wide[:, ::2]
    out.append((sl, sl.cpu().numpy(), "int32 strided"))
    row = torch.as_tensor([[3, 4, 1, 0, 2]], dtype=torch.int64, device=DEV).expand(n, 5)
    out.append((row, row[:1].cpu().numpy(), "int64 broadcast"))
    names = ["emergency", "left", "follow", "straight", "right"][k % 2:]
    out.append((names, np.array([[IDS[a] for a in names]]), "names"))
    host = _order_ids(n, k + 1)
    out.append((host, host, "host array"))
    out.append(([], np.zeros((1, 0), dtype=np.int64), "empty"))
    return out


@pytest.mark.parametrize("emerg", [False, True])
def test_select_equals_rule_over_ticks(emerg):
    """l216, 1000 scenarios: a first tick and 8 stateful ticks (restarts at ticks 3 and 6), every preference variant
    selected after each tick against the rule; the loop drives on the selection of the names variant through
    sel_action="selected"; on a planner with the trajectory id counter (a graph captured first) for emergency on"""
    lat = H.lattice_for("l216")
    rng = np.random.default_rng(77 + emerg)
    sc = _scenarios("l216", N, 5100)
    pl = D.planner(lat, 4, stateful=True, ax_max_machines=_axm("l216"), incl_emerg_traj=emerg)
    dsc = sc.to_device(DEV)
    if emerg:   # ids from the device counter (k_traj_base) from here on
        pl.capture_tick(dsc).close()
    D.first_tick(pl, dsc)
    pos, vel = dsc.pos.clone(), dsc.vel.clone()
    acts = set()
    for k in range(9):
        if k:
            restart = torch.zeros(N, dtype=torch.bool, device=DEV)
            if k in (3, 6):
                restart[k::11] = True
            pl.next_tick(replace(dsc, pos=pos), "selected", T_CONST, vel_est=vel, restart=restart)
        for prefer, ids, name in _prefer_variants(N, k, rng):
            sel = pl.select(prefer)
            acts |= set(_check(pl, sel, ids, emerg, "tick %d %s" % (k, name)).tolist())
        sel = pl.select(["left", "follow", "straight", "right"])
        pos, vel = _step(sel, pos, vel)
    assert {0, 1, 2, 3} <= acts and (4 in acts) == emerg


def test_stale_emergency_is_not_selected():
    """a stateless planner keeps em_info of an earlier call with the emergency trajectory; after a call without it,
    'emergency' is not returned"""
    lat = H.lattice_for("l216")
    sc = _scenarios("l216", N, 5200)
    pl = D.planner(lat, 4, ax_max_machines=_axm("l216"), incl_emerg_traj=True)
    D.first_tick(pl, sc)
    sel = pl.select(["emergency"])
    assert (sel["sel_action"] == 4).any()
    pl.set_vel_params(**dict(D.VEL, ax_max_machines=_axm("l216"), incl_emerg_traj=False))
    D.first_tick(pl, sc)
    assert (pl.fetch("em_info")["em_info"][:, 0] >= 0).any()   # stale
    sel = pl.select(["emergency", "right"])
    act = _check(pl, sel, np.array([[4, 3]]), False, "stale em_info")
    assert not (act == 4).any() and (act == 3).any()


def test_closed_loop_selected_equals_host_actions():
    """three stateful planners on the same inputs for 8 ticks: a device batch with sel_action="selected", a host batch
    with sel_action="selected" and a host batch with the actions the rule gives on the host; every result and memory
    record byte-equal after every tick"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import ScenarioBatch
    lat = H.lattice_for("l216")
    sc = _scenarios("l216", N, 5300)
    vel = dict(ax_max_machines=_axm("l216"), incl_emerg_traj=True)
    pd, ph, pr = (D.planner(lat, 4, stateful=True, **vel) for _ in range(3))
    for pl in (pd, ph, pr):
        D.first_tick(pl, sc)
    pos, v = torch.as_tensor(sc.pos, device=DEV), torch.as_tensor(sc.vel, device=DEV)
    for k in range(8):
        ids = _order_ids(N, k, emergency_first=k in (2, 5))
        sel_d = pd.select(torch.as_tensor(ids, device=DEV))
        ph.select(ids)
        f = pr.fetch("action_id", "traj_row", "traj_len", "traj_id", "em_info")
        host_sel, _ = select_ref(f["action_id"], f["traj_row"], f["traj_len"], f["traj_id"], f["em_info"], True, ids)
        pos, v = _step(sel_d, pos, v)
        hsc = ScenarioBatch(pos.cpu().numpy(), sc.heading, sc.vel, sc.n_obj, sc.obj)
        dsc = hsc.to_device(DEV)
        pd.next_tick(dsc, "selected", T_CONST, vel_est=v)
        ph.next_tick(hsc, "selected", T_CONST, vel_est=v.cpu().numpy())
        pr.next_tick(hsc, host_sel, T_CONST, vel_est=v.cpu().numpy())
        want = _state(pr)
        for name, pl in (("device selected", pd), ("host selected", ph)):
            got = _state(pl)
            for key in want:
                assert np.array_equal(got[key], want[key]), "tick %d %s: %s" % (k, name, key)


def test_graph_replays_with_selection_equal_eager_ticks():
    """capture_tick(prefer=P) and capture_next_tick(sc, "selected", prefer=P): 8 replays (both parities) equal eager
    ticks + select(P), selection included; then replays and an eager device tick with its selection under
    torch.cuda.set_sync_debug_mode('error')"""
    lat = H.lattice_for("l216")
    sc = _scenarios("l216", N, 5400)
    vel = dict(ax_max_machines=_axm("l216"), incl_emerg_traj=True)
    pg, pe = D.planner(lat, 4, stateful=True, **vel), D.planner(lat, 4, stateful=True, **vel)
    prefer = torch.as_tensor(_order_ids(N, 0, emergency_first=True), device=DEV)
    dsc = sc.to_device(DEV)
    pos, v = dsc.pos.clone(), dsc.vel.clone()
    t_const = torch.full((N,), T_CONST, dtype=torch.float64, device=DEV)
    g0 = pg.capture_tick(dsc, prefer=prefer)
    g0.replay()
    gn = pg.capture_next_tick(dsc, "selected", t_const, vel_est=v, prefer=prefer)
    assert gn.n_graphs == 2
    pe.capture_tick(dsc).close()   # the same id counter
    D.first_tick(pe, dsc)
    sel_e = pe.select(prefer)

    def same(k):
        a, b = _state(pg), _state(pe)
        for key in a:
            assert np.array_equal(a[key], b[key]), "tick %d: %s" % (k, key)
        for got, want in zip(_selection(pg._sel[0]["info"], pg._sel[0]["traj"]),
                             _selection(pe._sel[0]["info"], pe._sel[0]["traj"])):
            assert np.array_equal(got, want), "tick %d: selection" % k

    same(0)
    for k in range(1, 9):
        pos, v = _step(sel_e, pos, v)
        nsc = replace(dsc, pos=pos)
        gn.inputs.copy_(nsc, t_const=t_const, vel_est=v)
        gn.replay()
        pe.next_tick(nsc, "selected", t_const, vel_est=v)
        sel_e = pe.select(prefer)
        same(k)
    sel_g = dict(sel_info=pg._sel[0]["info"], sel_traj=pg._sel[0]["traj"])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            pos, v = _step(sel_g, pos, v)
            gn.inputs.sc.pos.copy_(pos)
            gn.inputs.vel_est.copy_(v)
            gn.replay()
        pos, v = _step(sel_g, pos, v)
        pg.next_tick(replace(dsc, pos=pos), "selected", t_const, vel_est=v)
        out = pg.select(prefer)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _check(pg, out, prefer.cpu().numpy(), True, "after the device loop")
    for g in (g0, gn):
        g.close()


def _host_pick(full, ids):
    """the rule on a full download: per scenario (action, rows) and the selected rows of the compact export"""
    act, info = select_ref(full["action_id"].numpy(), full["traj_row"].numpy(), full["traj_len"].numpy(),
                           full["traj_id"].numpy(), full["em_info"].numpy(), full["incl_emerg_traj"], ids)
    rows = full["traj"].numpy()[np.maximum(info[:, 1], 0)].copy()
    return act, info, rows


def _assert_selected(out, full, ids, ctx):
    act, info, rows = _host_pick(full, ids)
    B, NE = act.shape[0], rows.shape[1]
    assert out["sel_traj"].numpy().nbytes == B * NE * 28 and out["sel_info"].numpy().nbytes == B * 16, ctx
    assert np.array_equal(out["sel_action"].numpy(), act), ctx
    got = out["sel_info"].numpy()
    assert np.array_equal(got[:, 2], info[:, 2]), ctx + ": rows"
    assert np.array_equal(got[:, 3] % 10, info[:, 3] % 10) and np.array_equal(got[:, 3] < 0, info[:, 3] < 0), ctx
    st = out["sel_traj"].numpy()
    for b in range(B):   # compact rows are in an unspecified order: compare the selected rows themselves
        n = info[b, 2]
        assert np.array_equal(st[b, :n], rows[b, :n]), "%s scenario %d" % (ctx, b)
        assert info[b, 1] >= 0 or not st[b].any()


@pytest.mark.parametrize("emerg", [False, True])
def test_plan_batch_and_stream_with_prefer(tmp_path, emerg):
    """plan_batch / plan_stream with prefer give the selected rows of the full download, B * n_export * 28 bytes of
    rows; without prefer, launches and results are those of the plain calls; a bad prefer is refused before anything
    is staged or launched"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    ltpl = D.facade(tmp_path)
    pl = ltpl.planner
    pl.set_vel_params(**dict(D.VEL, incl_emerg_traj=emerg))
    track = Track(H.TRACK_CSV)
    batches = [make_scenarios(track, 600, seed=5500 + i, n_obj_min=0, n_obj_max=3) for i in range(4)]
    names = ["emergency", "right", "left", "follow", "straight"] if emerg else ["right", "straight", "follow", "left"]
    ids = np.array([[IDS[a] for a in names]])
    for i, sc in enumerate(batches):
        n0 = pl.launch_count()
        full = {k: (v.copy() if isinstance(v, np.ndarray) else (v.clone() if hasattr(v, "clone") else v))
                for k, v in ltpl.plan_batch(sc).items()}
        n_plain = pl.launch_count() - n0
        out = ltpl.plan_batch(sc, prefer=names)
        assert pl.launch_count() - n0 == 2 * n_plain + 1   # k_select is the only extra launch
        _assert_selected(out, full, ids, "plan_batch %d" % i)
    fulls = [{k: (v.clone() if hasattr(v, "clone") else v) for k, v in o.items()} for o in ltpl.plan_stream(batches)]
    for i, out in enumerate(ltpl.plan_stream(batches, prefer=names)):
        _assert_selected(out, fulls[i], ids, "plan_stream %d" % i)
    assert pl.h_out_sets[0]["traj"].shape[0] == 4 * 600   # the compact-row buffers are as they were
    n0 = pl.launch_count()
    for bad in (["straight", "overtake"], np.zeros((599, 2), dtype=np.int32), torch.zeros((600, 2), device=DEV)):
        with pytest.raises(ValueError):
            ltpl.plan_batch(batches[0], prefer=bad)
        with pytest.raises(ValueError):
            next(iter(ltpl.plan_stream(batches[:1], prefer=bad)))
    assert pl.launch_count() == n0


def test_select_refusals():
    """select before a velocity call, with a bad sel_action tensor or with buffers.traj elsewhere (a PeerGather);
    sel_action="selected" without a select after the last tick; a capture with "selected" but without prefer: each a
    ValueError with nothing launched"""
    lat = H.lattice_for("l216")
    sc = _scenarios("l216", 256, 5600)
    pl = D.planner(lat, 2, stateful=True, ax_max_machines=_axm("l216"))
    dsc = sc.to_device(DEV)
    pl.stage_scenarios(dsc)
    n0 = pl.launch_count()
    with pytest.raises(ValueError, match="no velocity call"):
        pl.select(["left"])
    assert pl.launch_count() == n0
    D.first_tick(pl, dsc)
    n0 = pl.launch_count()
    with pytest.raises(ValueError, match="no select"):
        pl.next_tick(dsc, "selected", T_CONST)
    with pytest.raises(ValueError, match="needs prefer"):
        pl.capture_next_tick(dsc, "selected", T_CONST)
    for bad in (torch.zeros(256, dtype=torch.int64, device=DEV), torch.zeros(255, dtype=torch.int32, device=DEV),
                np.zeros(256, dtype=np.int32)):
        with pytest.raises(ValueError, match="sel_action"):
            pl.select(["left"], sel_action=bad)
    with pytest.raises(ValueError, match="selected"):
        pl.next_tick(dsc, "chosen", T_CONST)
    saved, other = pl.buf.traj, torch.zeros(16, dtype=torch.float32, device=DEV)
    pl.buf.traj = other.data_ptr()
    try:
        with pytest.raises(ValueError, match="PeerGather"):
            pl.select(["left"])
    finally:
        pl.buf.traj = saved
    assert pl.launch_count() == n0
    # a caller tensor receives the actions (any stride); sel_info keeps them for "selected"
    dst = torch.full((256, 2), 9, dtype=torch.int32, device=DEV)
    out = pl.select(["left", "right", "straight", "follow"], sel_action=dst[:, 1])
    assert out["sel_action"].data_ptr() == dst[:, 1].data_ptr()
    assert torch.equal(dst[:, 1], out["sel_info"][:, 0]) and (dst[:, 0] == 9).all()
    pl.next_tick(dsc, "selected", T_CONST)
    assert torch.equal(pl.t["sel_action"], out["sel_info"][:, 0])
