"""Edges of ticks replayed from CUDA graphs: a stateful capture whose example batch grows the input buffers keeps the last
tick's positions for pos_last; k_traj_base leaves the ids a repeated velocity call did not write; refused settings calls
leave captured graphs valid; a TickGraph collected during the caller's own capture does not disturb it."""
import gc

import numpy as np
import pytest
import torch

from tests import drivers as D
from tests import helpers as H
from tests.test_gpu_device_inputs import _assert_same, _outputs, _scenarios, _with_pred

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MEMORY = ("st_info", "vel_plan", "course", "zone_s0")


def _axm():
    return H.golden("ticks_default.npz")["ax_max_machines"]


def _state(pl):
    """every result of the last tick with the emergency rows cleared behind their length (a compact export row keeps
    what an earlier tick wrote behind it), and the memory records"""
    out = _outputs(pl)
    em_rows = out["em_rows"].copy()
    em_rows[0][np.arange(em_rows.shape[2])[None, :] >= out["em_len"][0][:, None]] = 0.0
    out["em_rows"] = em_rows
    torch.cuda.synchronize()
    out.update({k: pl._state[k].cpu().numpy() for k in MEMORY})
    out["trim"] = pl.t["trim"].cpu().numpy()
    return out


def _sel(pl):
    return pl.device_results()["action_id"].max(dim=0).values.clamp(min=0)


def test_capture_that_grows_the_inputs_keeps_the_last_positions():
    """a first tick with 3 object slots, then capture_next_tick of a batch with 5 slots and 4 prediction points (the
    input copies are re-created before the capture): replay, eager next_tick, replay on the capturing planner equal the
    eager twin, which grows inside its first next_tick, byte for byte in results and memory"""
    lat = H.lattice_for("default")
    pe, pg = (D.planner(lat, 3, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True) for _ in range(2))
    sc3 = _scenarios("default", 128, 9860, omax=3)
    sc5 = _with_pred(_scenarios("default", 128, 9860, omax=5), 4, 9861)
    assert np.array_equal(sc3.pos, sc5.pos) and sc5.obj.shape[1] == 5
    for pl in (pe, pg):
        D.first_tick(pl, sc3.to_device(DEV))
    dsc = sc5.to_device(DEV)
    graph = pg.capture_next_tick(dsc, _sel(pe), 0.15)
    assert pg.dims.k_obj == 5 and pg._k_pred_cap == 4
    for k, how in enumerate(("replay", "eager", "replay")):
        sel = _sel(pe)
        pe.next_tick(dsc, sel, 0.15)
        if how == "eager":
            pg.next_tick(dsc, sel, 0.15)
        else:
            graph.inputs.copy_(dsc, sel)
            graph.replay()
        got, want = _state(pg), _state(pe)
        _assert_same(got, want, "tick %d (%s)" % (k + 1, how))
        assert (want["traj_len"] > 0).sum() > 128


def test_repeated_velocity_call_keeps_the_ids_it_did_not_write():
    """ids of paths a velocity call leaves without a trajectory keep their value with the device counter as they do
    with params.traj_base_id: stale ids planted between two calc_vel_profile calls after one calc_paths survive, and
    traj_id / em_info equal the eager planner's after the second call"""
    sc = _scenarios("default", 160, 9870)
    dsc = sc.to_device(DEV)
    lat = H.lattice_for("default")
    pe, pg = (D.planner(lat, 2, ax_max_machines=_axm(), incl_emerg_traj=True) for _ in range(2))
    pg.capture_tick(dsc).close()   # from now on pg numbers its trajectories with the device counter
    assert pg.buf.traj_base is not None
    for pl in (pe, pg):
        pl.stage_scenarios(dsc)
        pl.set_startpos()
        pl.calc_paths()
        pl.calc_vel_profile()
    stale = None
    for pl in (pe, pg):
        tid = pl.t["traj_id"]
        if stale is None:
            stale = (tid < 0).nonzero()[::2]
        assert stale.shape[0] > 0
        tid[stale[:, 0], stale[:, 1]] = 57   # ids an earlier call would have left (base 50, action 'right' + 4)
        pl.calc_vel_profile()
    f_e, f_g = pe.fetch("traj_id", "em_info"), pg.fetch("traj_id", "em_info")
    assert np.array_equal(f_g["traj_id"], f_e["traj_id"])
    # em_info: rows and id (the export row of the emergency trajectory is unspecified)
    assert np.array_equal(f_g["em_info"][:, 1:], f_e["em_info"][:, 1:])
    assert np.array_equal(f_g["em_info"][:, 0] >= 0, f_e["em_info"][:, 0] >= 0)
    assert (f_g["traj_id"][stale[:, 0].cpu().numpy(), stale[:, 1].cpu().numpy()] == 57).all()
    assert set(np.unique(f_g["traj_id"][f_g["traj_id"] >= 0] // 10)) == {2, 5}


def test_refused_settings_calls_keep_graphs_valid():
    """set_vel_params and set_local_gg_planes that raise change nothing, so a graph captured before still replays and
    equals the eager twin"""
    sc = _scenarios("default", 96, 9880)
    dsc = sc.to_device(DEV)
    lat = H.lattice_for("default")
    pe, pg = (D.planner(lat, 2, stateful=True, ax_max_machines=_axm(), incl_emerg_traj=True) for _ in range(2))
    for pl in (pe, pg):
        D.first_tick(pl, dsc)
    graph = pg.capture_next_tick(dsc, _sel(pe), 0.1)
    with pytest.raises(RuntimeError):
        pg.set_vel_params(**dict(D.VEL, vel_max=1e4, ax_max_machines=_axm()))
    with pytest.raises(ValueError):
        pg.set_local_gg_planes(np.ones((2, 2, 2)), np.ones((2, 2, 2)))
    sel = _sel(pe)
    pe.next_tick(dsc, sel, 0.1)
    graph.inputs.copy_(dsc, sel)
    graph.replay()
    _assert_same(_state(pg), _state(pe), "replay after refused calls")


def test_graph_collected_during_the_callers_capture():
    """a TickGraph that the garbage collector collects while the caller captures a graph of its own neither
    synchronises nor destroys its graphs then, so that capture completes and replays; the graphs are released by the
    next capture"""
    sc = _scenarios("default", 64, 9890)
    pl = D.planner(H.lattice_for("default"), 2, stateful=True, ax_max_machines=_axm())
    D.first_tick(pl, sc.to_device(DEV))
    graph = pl.capture_next_tick(sc.to_device(DEV), _sel(pl), 0.1)
    graph.replay()
    torch.cuda.synchronize()
    x = torch.zeros(16, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    mine = torch.cuda.CUDAGraph()
    with torch.cuda.graph(mine, stream=side):
        x.add_(1.0)
        del graph
        gc.collect()
        x.add_(1.0)
    torch.cuda.current_stream().wait_stream(side)
    mine.replay()
    torch.cuda.synchronize()
    assert torch.equal(x, torch.full((16,), 2.0, device=DEV))
    from graphbasedlocaltrajectoryplanner_b200 import tick_graph
    assert len(tick_graph._DEFERRED) == 2            # released at the next chance outside a capture
    again = pl.capture_next_tick(sc.to_device(DEV), _sel(pl), 0.1)
    assert not tick_graph._DEFERRED
    again.replay()
    again.close()
