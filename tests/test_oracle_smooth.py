"""Velocity smoothing ([SMOOTHING] filt_window_width > 1, tph.conv_filt on every kept profile, OTH:926-941 / 986-1004):
the oracle against golden vectors of the unmodified reference run with a modified online ini (tests/golden/
ticks_smooth.npz, ticks_multitick_smooth_default.npz, made by tests/tools/gen_golden_smooth.py), and the window checks of
the host, which need no GPU."""
import numpy as np
import pytest

from tests import drivers as D
from tests import helpers as H

SMOOTH_SETS = ("w3_default", "w7_default", "w5_open")


@pytest.mark.parametrize("name", SMOOTH_SETS)
def test_oracle_matches_reference_smoothed_first_ticks(name):
    """first ticks at windows 3, 7 (default lattice) and 5 (open track: reduced horizons ending in the zero tail), with the
    emergency trajectory, which is built on the smoothed trajectory but reads only its first row and path columns."""
    from oracle.ltpl_oracle import OracleLTPL
    g = H.golden("ticks_smooth.npz")
    sub = H._Sub(g, name)
    w = int(sub["filt_window"])
    orc = OracleLTPL(H.lattice_for(str(sub["lattice"])), online=dict(filt_window_width=w))
    vk = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), ax_max_machines=g["ax_max_machines"], safety_d=30.0,
              incl_emerg_traj=True)
    n = sub["sc_pos"].shape[0]
    smoothed = 0
    for b in range(n):
        rec = orc.tick(sub["sc_pos"][b], sub["sc_heading"][b], sub["sc_vel"][b], H.object_list(sub, b), vk)
        H.compare_first_tick(rec, sub, b, ctx=name, emergency=True)
        smoothed += sum(int(t[0].shape[0] >= w) for t in rec.get("traj_full", {}).values())
    assert smoothed >= n


def test_oracle_session_matches_reference_smoothed_sequences():
    """closed loop at window 5 with the emergency trajectory; the grip drops on the odd sequences, so the brake profile on
    the backup plan and its vel_course seam are smoothed too, and the next tick's memory holds smoothed values."""
    D.replay_session_oracle("ticks_multitick_smooth_default.npz", True, "default", online=dict(filt_window_width=5))


def test_conv_filt_semantics():
    """tph.conv_filt on an open signal: the first and last h = (w - 1) / 2 rows keep their values, the rows between are the
    window mean; a signal shorter than the window is returned unchanged; an even window raises."""
    from oracle.tph_port import conv_filt
    x = np.array([0.0, 3.0, 6.0, 3.0, 9.0, 12.0, 0.0])
    f = conv_filt(signal=x, filt_window=3, closed=False)
    assert f[0] == x[0] and f[-1] == x[-1]
    assert np.allclose(f[1:-1], [(x[i - 1] + x[i] + x[i + 1]) / 3.0 for i in range(1, 6)])
    assert np.array_equal(conv_filt(signal=x[:4], filt_window=5, closed=False), x[:4])
    assert np.array_equal(conv_filt(signal=x, filt_window=1, closed=False), x)
    with pytest.raises(RuntimeError, match="must be odd"):
        conv_filt(signal=x, filt_window=4, closed=False)


def _online_ini(tmp_path, w):
    txt = open(H.ONLINE_INI).read()
    assert txt.count("filt_window_width=1\n") == 1
    p = tmp_path / ("online_w%d.ini" % w)
    p.write_text(txt.replace("filt_window_width=1\n", "filt_window_width=%d\n" % w))
    return str(p)


def test_window_is_checked_without_a_gpu(tmp_path):
    """an even window is refused with tph.conv_filt's RuntimeError, a window < 1 with a ValueError -- by
    read_online_config and by BatchPlanner, before any device is touched."""
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner, read_online_config
    assert read_online_config(_online_ini(tmp_path, 5))["filt_window_width"] == 5
    assert read_online_config(H.ONLINE_INI)["filt_window_width"] == 1
    with pytest.raises(RuntimeError, match="Window width of moving average filter must be odd!"):
        read_online_config(_online_ini(tmp_path, 4))
    with pytest.raises(ValueError):
        read_online_config(_online_ini(tmp_path, 0))
    with pytest.raises(RuntimeError, match="Window width of moving average filter must be odd!"):
        BatchPlanner(None, online=dict(filt_window_width=4))
    for bad in (0, -3):
        with pytest.raises(ValueError):
            BatchPlanner(None, online=dict(filt_window_width=bad))
