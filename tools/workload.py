"""What the measurement and diagnostic scripts share: the benchmark workload's variants (long object lists, prediction
arrays, a smoothing window in the online ini), the closed-loop vehicle dummy, one L2-flushed event timing and the card
the numbers were taken on.  bench.py is not imported here: importing it points file descriptor 1 at stderr."""
import contextlib
import os
import subprocess
import tempfile

import numpy as np
import torch

OBJECTS_SEED = 4242
PRED_DT = 0.1


def with_objects(sc, n, track):
    """the batch with its objects filled up to n per scenario (OLI:96-141; a fixed seed: the same objects on every
    call).  The added objects stand 20-500 m ahead of the ego vehicle, every second one 3-15 m beyond the track bounds
    (an off-track entry the object filter drops on the device), the others on the track."""
    k0 = sc.obj.shape[1]
    if n <= k0:
        return sc
    rng = np.random.default_rng(OBJECTS_SEED)
    B = sc.size
    # arc length of every ego pose: its nearest race-line point
    s_e = np.empty(B)
    for i in range(0, B, 512):
        d2 = np.sum((sc.pos[i:i + 512, None, :] - track.raceline[None, :, :]) ** 2, axis=2)
        s_e[i:i + 512] = track.s[np.argmin(d2, axis=1)]
    obj = np.zeros((B, n, 5))
    obj[:, :k0] = sc.obj
    for j in range(n):
        ref, nv, wl, wr, psi, vrl = track.frame(s_e + rng.uniform(20.0, 500.0, size=B))
        if j % 2:
            d = np.where(rng.random(B) < 0.5, -(wl + rng.uniform(3.0, 15.0, size=B)), wr + rng.uniform(3.0, 15.0, size=B))
        else:
            d = -(wl - 1.4) + rng.uniform(0.0, 1.0, size=B) * ((wr - 1.4) + (wl - 1.4))
        new = np.arange(B) if j >= k0 else np.nonzero(sc.n_obj <= j)[0]   # slots behind the scenario's own objects
        obj[new, j, 0:2] = (ref + nv * d[:, None])[new]
        obj[new, j, 2] = psi[new]
        obj[new, j, 3] = (rng.uniform(0.0, 0.5, size=B) * vrl)[new]
        obj[new, j, 4] = 5.0
    sc.obj = obj
    sc.n_obj = np.full(B, n, dtype=np.int32)
    return sc


def with_predictions(sc, n):
    """the batch with an n-point constant-velocity prediction at 0.1 s spacing on every object (n more obstacle discs
    per object, OLI:117-119, GLNT:169-189; n = 0: unchanged, the built-in 0.2 s point)."""
    if n == 0:
        return sc
    k = sc.obj.shape[1]
    t = PRED_DT * np.arange(1, n + 1)
    x, y, th, v = (sc.obj[:, :, i][..., None] for i in range(4))
    sc.pred = np.stack((x - np.sin(th) * v * t, y + np.cos(th) * v * t), axis=-1)
    sc.n_pred = np.where(np.arange(k)[None, :] < sc.n_obj[:, None], n, -1).astype(np.int32)
    return sc


@contextlib.contextmanager
def online_ini_with_window(online_ini, width):
    """path of a copy of the online ini with [SMOOTHING] filt_window_width = width and every other line unchanged; the
    copy is removed on exit."""
    with open(online_ini) as f:
        txt = f.read()
    assert txt.count("filt_window_width=1\n") == 1
    with tempfile.TemporaryDirectory(prefix="ltpl_online_ini_", ignore_cleanup_errors=True) as tmp:
        ini = os.path.join(tmp, "ltpl_config_online.ini")
        with open(ini, "w") as f:
            f.write(txt.replace("filt_window_width=1\n", "filt_window_width=%d\n" % width))
        yield ini


def step_along(tr, n, dt):
    """position (B, 2), velocity and heading of every scenario after dt along its trajectory rows tr (B, L, 7, float64,
    the first n of them valid): the arc length moves by vx dt + ax dt^2 / 2 (never backwards) and the row values are
    interpolated linearly between the rows around it."""
    b = np.arange(tr.shape[0])
    n = np.maximum(n, 2)
    s_t = tr[:, 0, 0] + np.maximum(tr[:, 0, 5] * dt + 0.5 * tr[:, 0, 6] * dt ** 2, 0.0)
    valid = np.arange(tr.shape[1])[None, :] < n[:, None]
    i0 = np.clip((np.where(valid, tr[:, :, 0], np.inf) <= s_t[:, None]).sum(axis=1) - 1, 0, n - 2)
    s0, s1 = tr[b, i0, 0], tr[b, i0 + 1, 0]
    w = np.clip((s_t - s0) / np.maximum(s1 - s0, 1e-9), 0.0, 1.0)
    lerp = lambda c: tr[b, i0, c] * (1 - w) + tr[b, i0 + 1, c] * w   # noqa: E731
    return np.column_stack((lerp(1), lerp(2))), lerp(5), tr[b, i0, 3]


def closed_loop_step(res, dt):
    """the vehicle dummy of the closed loop: every scenario drives dt along its first kept trajectory.  res holds the
    host arrays traj_row, traj_len, action_id and traj of a result.  Returns position, velocity, the executed action
    (int32, 0 where nothing was kept), the mask of scenarios that kept a trajectory and the heading of the row the step
    started from."""
    rows = res["traj_row"]
    slot = np.argmax(rows >= 0, axis=0)
    b = np.arange(rows.shape[1])
    ok = rows[slot, b] >= 0
    tr = res["traj"][np.where(ok, rows[slot, b], 0)].astype(np.float64)
    pos, vel, heading = step_along(tr, res["traj_len"][slot, b], dt)
    return pos, vel, np.where(ok, res["action_id"][slot, b], 0).astype(np.int32), ok, heading


_FLUSH = []


def timed_ms(fn):
    """device time of fn() in ms: CUDA events on the current stream around it, with L2 flushed (a 256 MB buffer written,
    L2 = 50 MB) and the device idle before it starts."""
    if not _FLUSH:
        _FLUSH.append(torch.empty(256 << 20, dtype=torch.uint8, device="cuda"))
    _FLUSH[0].fill_(1)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def card():
    """name and power limit of the current GPU as nvidia-smi reports them (its name alone without nvidia-smi)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()
