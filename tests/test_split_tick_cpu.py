"""Friction planes from device tensors and split-tick graphs, without a GPU: the checks of plane tensors
(planner.check_gg_planes) and the copy rule of a SplitTickGraph's velocity inputs (tick_graph.VelInputs), on CPU
tensors standing in for device ones."""
import numpy as np
import pytest
import torch

from graphbasedlocaltrajectoryplanner_b200.planner import NSLOT, check_gg_planes
from graphbasedlocaltrajectoryplanner_b200.tick_graph import VelInputs

CPU = torch.device("cpu")
B, P = 5, 12


def _planes(n=P, dtype=torch.float64):
    return torch.ones((NSLOT, B, n), dtype=dtype), torch.ones((NSLOT, B, n), dtype=dtype)


def test_plane_tensors_pass_in_any_width_and_strides():
    check_gg_planes(*_planes(), B, P, CPU)
    check_gg_planes(*_planes(3), B, P, CPU)
    wide = torch.ones((NSLOT, B, P, 2), dtype=torch.float64)
    check_gg_planes(wide[..., 0], wide[..., 1], B, P, CPU)   # stride 2: the columns of one (P, 2) array per path
    check_gg_planes(*(a[:, :, :0] for a in _planes()), B, P, CPU)


@pytest.mark.parametrize("case", ["dtype", "device", "rank", "batch", "slots", "wide", "unequal", "numpy"])
def test_bad_plane_tensors_raise(case):
    ax, ay = _planes()
    if case == "dtype":
        ax, ay = _planes(dtype=torch.float32)
    elif case == "device":
        ax = ax.to("meta")
    elif case == "rank":
        ax, ay = ax[0], ay[0]
    elif case == "batch":
        ax, ay = ax[:, 1:], ay[:, 1:]
    elif case == "slots":
        ax, ay = ax[1:], ay[1:]
    elif case == "wide":
        ax, ay = _planes(P + 1)
    elif case == "unequal":
        ay = ay[:, :, 1:]
    else:
        ay = np.ones((NSLOT, B, P))
    with pytest.raises(ValueError, match="local_gg planes"):
        check_gg_planes(ax, ay, B, P, CPU)


def test_vel_inputs_take_what_was_captured_and_nothing_else():
    pos, vel = torch.zeros((B, 2), dtype=torch.float64), torch.zeros(B, dtype=torch.float64)
    vi = VelInputs(pos.clone(), vel.clone(), *_planes())
    ax, ay = (a * 2.5 for a in _planes())
    vi.copy_(pos + 1.0, vel + 2.0, (ax, ay))
    assert torch.equal(vi.pos_est, pos + 1.0) and torch.equal(vi.vel_est, vel + 2.0)
    assert torch.equal(vi.ax, ax) and torch.equal(vi.ay, ay)
    before = [a.clone() for a in (vi.pos_est, vi.vel_est, vi.ax, vi.ay)]
    for args, match in [((pos, vel), "is required"), ((pos, None, (ax, ay)), "is required"),
                        ((pos, vel, (ax, ay[:, :, 1:])), "must be a tensor"), ((pos, vel.float(), (ax, ay)), "tensor"),
                        ((pos, vel, ax), "pair")]:
        with pytest.raises(ValueError, match=match):
            vi.copy_(*args)
    for a, b in zip(before, (vi.pos_est, vi.vel_est, vi.ax, vi.ay)):
        assert torch.equal(a, b)   # a refused copy wrote nothing
    bare = VelInputs(vel_est=vel.clone())
    with pytest.raises(ValueError, match="was not captured"):
        bare.copy_(pos, vel)
    with pytest.raises(ValueError, match="was not captured"):
        bare.copy_(None, vel, (ax, ay))
    bare.copy_(vel_est=vel + 3.0)
    assert torch.equal(bare.vel_est, vel + 3.0)
