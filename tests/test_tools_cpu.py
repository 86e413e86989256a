"""The measurement tools' shared module (tools/workload.py) and tools/bench_variant.py without a GPU.  The workload
transforms and the closed-loop step compute, bit for bit, what the per-script copies they replaced computed: the SHA-256
digests below were taken from those copies on the same seeded inputs."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import helpers as H
from tools import workload

NSLOT = 3
DT = 0.1


def _digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def _bench_batch():
    """bench.make_batch("l216", 2000)"""
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios
    return make_scenarios(Track(H.TRACK_CSV), 2000, seed=20260924, n_obj_min=1, n_obj_max=3)


def _result_block(seed=11, batch=64, n_export=24):
    """a downloaded stateful result in miniature: fp32 trajectory rows (arc length with repeated points, junk behind each
    row's length), ragged traj_len down to 1, empty slots, and scenarios without any kept trajectory"""
    rng = np.random.default_rng(seed)
    n_rows = NSLOT * batch
    ds = rng.uniform(0.0, 3.0, (n_rows, n_export))
    ds[rng.random(ds.shape) < 0.05] = 0.0
    traj = np.empty((n_rows, n_export, 7), dtype=np.float32)
    traj[:, :, 0] = rng.uniform(0.0, 3000.0, (n_rows, 1)) + np.cumsum(ds, axis=1)
    traj[:, :, 1:5] = rng.normal(size=(n_rows, n_export, 4)) * (100.0, 100.0, 3.0, 0.05)
    traj[:, :, 5] = rng.uniform(0.0, 80.0, (n_rows, n_export))
    traj[:, :, 6] = rng.uniform(-15.0, 10.0, (n_rows, n_export))
    traj_row = rng.permutation(n_rows).reshape(NSLOT, batch).astype(np.int32)
    traj_row[rng.random(traj_row.shape) < 0.4] = -1
    traj_row[:, :5] = -1
    traj_len = rng.integers(1, n_export + 1, traj_row.shape).astype(np.int32)
    traj_len[traj_row < 0] = 0
    for r, n in zip(traj_row[traj_row >= 0], traj_len[traj_row >= 0]):
        traj[r, n:] = rng.uniform(-50.0, 50.0, (n_export - n, 7))
    action_id = np.where(traj_row >= 0, rng.integers(0, 4, traj_row.shape), -1).astype(np.int32)
    return dict(traj_row=traj_row, traj_len=traj_len, action_id=action_id, traj=traj)


def _float64_rows(seed=12, count=200):
    """trajectories of one scenario each as the session oracle returns them (float64, 2 .. 40 rows)"""
    rng = np.random.default_rng(seed)
    out = []
    for n in rng.integers(2, 41, count):
        ds = np.where(rng.random(n) < 0.05, 0.0, rng.uniform(0.0, 3.0, n))
        tr = np.empty((n, 7))
        tr[:, 0] = rng.uniform(0.0, 3000.0) + np.cumsum(ds)
        tr[:, 1:5] = rng.normal(size=(n, 4)) * (100.0, 100.0, 3.0, 0.05)
        tr[:, 5] = rng.uniform(0.0, 80.0, n)
        tr[:, 6] = rng.uniform(-15.0, 10.0, n)
        out.append(tr)
    return out


def test_workload_transforms_keep_their_draws():
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    track = Track(H.TRACK_CSV)
    sc = workload.with_objects(_bench_batch(), 64, track)
    assert _digest(sc.obj, sc.n_obj) == "0886fa06b081ec8d16105c653c9b2ddc77232ae4a80093076aecc6e7e15c964d"
    sc = workload.with_predictions(_bench_batch(), 50)
    assert _digest(sc.pred, sc.n_pred) == "97d48692a9cd9c0bae3b5bde6f5c6e45259ad2187959087c42b200f6c26fd8f0"
    sc = workload.with_predictions(workload.with_objects(_bench_batch(), 64, track), 50)   # bench_variant.py's order
    assert _digest(sc.obj, sc.n_obj, sc.pred, sc.n_pred) == \
        "6805a80957d1de77aa13050e1007cd1ab1d86d7795f7ee3534d506548fad542d"


def test_closed_loop_step_matches_the_vehicle_dummy():
    res = _result_block()
    pos, vel, sel, ok, heading = workload.closed_loop_step(res, DT)
    assert 0 < ok.sum() < ok.size and sel.dtype == np.int32
    assert _digest(pos, vel, sel, ok, heading) == "8c3651d0e0a35fdc2f574181cfb0350b87c111b862f180069b0255676eb76830"


def test_step_along_one_scenario():
    """the one-scenario use (float64 rows of the session oracle, tests/tools/cpu_stateful_diag.py)"""
    steps = [workload.step_along(tr[None], [tr.shape[0]], DT) for tr in _float64_rows()]
    pos = np.array([p[0] for p, _, _ in steps])
    vel = np.array([v[0] for _, v, _ in steps])
    assert _digest(pos, vel) == "00192c5992f0b5b677703aa4c1aebfb24e7c21b95c2aca10c251d8899a43925b"


def test_online_ini_with_window():
    from graphbasedlocaltrajectoryplanner_b200.planner import read_online_config
    with open(H.ONLINE_INI) as f:
        shipped = f.read().splitlines()
    with workload.online_ini_with_window(H.ONLINE_INI, 5) as ini:
        with open(ini) as f:
            got = f.read().splitlines()
        assert read_online_config(ini) == dict(read_online_config(H.ONLINE_INI), filt_window_width=5)
    assert not os.path.exists(os.path.dirname(ini))
    assert len(got) == len(shipped)
    assert [(a, b) for a, b in zip(shipped, got) if a != b] == [("filt_window_width=1", "filt_window_width=5")]


@pytest.mark.parametrize("args", [
    ["--objects", "64", "--gpus", "2"], ["--objects", "64", "--gpus=1"], ["--pred-points", "50", "--impl", "reference"],
    ["--objects", "0"], ["--pred-points", "-1"], ["--filt-window", "4"], ["--filt-window", "0"], ["--filt-window", "-3"]])
def test_bench_variant_refuses(args):
    r = subprocess.run([sys.executable, os.path.join(H.REPO, "tools", "bench_variant.py")] + args + ["--steps", "1"],
                       cwd=H.REPO, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120)
    assert r.returncode != 0, r.stderr[-400:]
    assert not [ln for ln in r.stdout.splitlines() if ln.strip().startswith("{")]
