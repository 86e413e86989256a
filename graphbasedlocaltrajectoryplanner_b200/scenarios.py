"""
Synthetic scenario batches (ego start pose x dynamic-obstacle set) for the batched planning tick.

The reference has no scenario generator -- its only fixtures are the static dummy object of
/root/reference/graph_ltpl/testing_tools/src/objectlist_dummy.py:175-176 and the start pose of
/root/reference/main_min_example.py:63-67.  The batches here follow SURVEY.md section 8(d) (configs 2 / 4 / 5):
ego placed on the race line at a uniformly drawn arc length, 1..n dynamic objects 30..280 m ahead with a uniformly
drawn lateral offset inside the track, object dicts in exactly the format ``Graph_LTPL.calc_paths`` consumes
(/root/reference/graph_ltpl/data_objects/ObjectListInterface.py:75-141).
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from .lattice import import_globtraj_csv

DEFAULT_SEED = 20260924
OBJ_FIELDS = ("X", "Y", "theta", "v", "length")


@dataclass
class ScenarioBatch:
    """SoA scenario batch.  obj[:, k, :] = (X, Y, theta, v, length); entries k >= n_obj[b] are ignored."""
    pos: np.ndarray        # (B, 2) float64
    heading: np.ndarray    # (B,)   float64
    vel: np.ndarray        # (B,)   float64
    n_obj: np.ndarray      # (B,)   int32
    obj: np.ndarray        # (B, K, 5) float64
    # blocked zones (calc_paths(blocked_zones=...), LTPL:311-312, 'nodes' type): distinct zones as (layer ids, node ids)
    # pairs and, per scenario, the index of its zone or -1.  None: no zones in this batch.
    zones: list = None
    zone_sel: np.ndarray = None   # (B,) int32
    zone_key: np.ndarray = None   # (B,) int64 crc of the zone id (0: none): a stateful planner processes a zone anew when
    #                               its id changes between ticks (ObjectListInterface.update_zone, OLI:155-237)
    # explicit prediction arrays of the objects (dict key 'prediction', OLI:117-119): n_pred[b, k] points (-1: none
    # given -> the built-in constant-velocity point at 0.2 s, OLI:121-127).  None: no object carries a prediction.
    pred: np.ndarray = None       # (B, K, KP, 2) float64
    n_pred: np.ndarray = None     # (B, K) int32

    @property
    def size(self) -> int:
        return int(self.pos.shape[0])

    def object_list(self, b: int) -> list:
        """object dicts of scenario b in the reference's format (OLI:96-141)."""
        out = []
        for k in range(int(self.n_obj[b])):
            x, y, th, v, ln = (float(a) for a in self.obj[b, k])
            out.append({'id': k + 1, 'type': 'physical', 'X': x, 'Y': y, 'theta': th, 'v': v, 'length': ln,
                        'width': 2.5})
            if self.n_pred is not None and self.n_pred[b, k] >= 0:
                out[-1]['prediction'] = self.pred[b, k, :int(self.n_pred[b, k])].copy()
        return out

    def subset(self, idx) -> "ScenarioBatch":
        idx = np.asarray(idx)
        return ScenarioBatch(self.pos[idx].copy(), self.heading[idx].copy(), self.vel[idx].copy(),
                             self.n_obj[idx].copy(), self.obj[idx].copy(), self.zones,
                             None if self.zone_sel is None else self.zone_sel[idx].copy(),
                             None if self.zone_key is None else self.zone_key[idx].copy(),
                             None if self.pred is None else self.pred[idx].copy(),
                             None if self.n_pred is None else self.n_pred[idx].copy())

    def set_zones(self, blocked_zones) -> None:
        """blocked_zones: one entry per scenario, each None or a dict {zone id: [layer ids, node ids, left bound, right
        bound]} exactly as Graph_LTPL.calc_paths takes it (LTPL:311-312).  A scenario may carry ONE zone: with several
        keys the reference's update_zone (OLI:155-237, called once per key at LTPL:326-329) flags all but the last as
        removed and GLNT:69-83 then fails on them."""
        import zlib
        zones, index, sel = [], {}, np.full(self.size, -1, dtype=np.int32)
        zkey = np.zeros(self.size, dtype=np.int64)
        for i, bz in enumerate(blocked_zones):
            if not bz:
                continue
            zkey[i] = 1 + zlib.crc32(str(next(iter(bz))).encode())
            if len(bz) != 1:
                raise NotImplementedError("more than one blocked zone per scenario is not a defined input of the reference")
            zid, z = next(iter(bz.items()))
            lay, nod = np.asarray(z[0], dtype=np.int64), np.asarray(z[1], dtype=np.int64)
            if lay.shape != nod.shape or lay.ndim != 1:
                raise ValueError("zone '%s': layer ids and node ids must be two lists of equal length" % zid)
            key = (lay.tobytes(), nod.tobytes())
            if key not in index:
                index[key] = len(zones)
                zones.append((lay, nod))
            sel[i] = index[key]
        self.zones, self.zone_sel = (zones, sel) if zones else (None, None)
        self.zone_key = zkey if zones else None

    def shard(self, rank: int, world: int) -> "ScenarioBatch":
        """scenario i goes to rank i % world (SURVEY 8(e))."""
        return self.subset(np.arange(rank, self.size, world))

    def to_device(self, device) -> "DeviceScenarioBatch":
        """the same batch as torch tensors on `device` (DeviceScenarioBatch); DeviceScenarioBatch.cpu() gives it back
        exactly"""
        def dev(a, dt):
            return None if a is None else torch.as_tensor(np.ascontiguousarray(a, dtype=dt)).to(device)
        return DeviceScenarioBatch(dev(self.pos, np.float64), dev(self.heading, np.float64), dev(self.vel, np.float64),
                                   dev(self.n_obj, np.int32), dev(self.obj, np.float64), self.zones,
                                   dev(self.zone_sel, np.int32), dev(self.zone_key, np.int64),
                                   dev(self.pred, np.float64), dev(self.n_pred, np.int32))

    @staticmethod
    def from_object_lists(pos, heading, vel, object_lists, k_max=None, blocked_zones=None) -> "ScenarioBatch":
        b = len(object_lists)
        n_obj = np.array([len(o) if o is not None else 0 for o in object_lists], dtype=np.int32)
        k = int(max(1, n_obj.max() if b else 1)) if k_max is None else int(k_max)
        obj = np.zeros((b, k, 5))
        kp = max([np.atleast_2d(o['prediction']).shape[0] for ol in object_lists for o in (ol or [])
                  if 'prediction' in o and np.size(o['prediction'])] + [0])
        has_pred = any('prediction' in o for ol in object_lists for o in (ol or []))
        pred = np.zeros((b, k, max(kp, 1), 2)) if has_pred else None
        n_pred = np.full((b, k), -1, dtype=np.int32) if has_pred else None
        for i, ol in enumerate(object_lists):
            for j, o in enumerate(ol or []):
                obj[i, j] = [o['X'], o['Y'], o['theta'], o['v'], o['length']]
                if 'prediction' in o:
                    pr = np.asarray(o['prediction'], dtype=np.float64).reshape(-1, 2)
                    n_pred[i, j] = pr.shape[0]
                    pred[i, j, :pr.shape[0]] = pr
        sc = ScenarioBatch(np.asarray(pos, dtype=np.float64).reshape(b, 2),
                           np.asarray(heading, dtype=np.float64).reshape(b),
                           np.asarray(vel, dtype=np.float64).reshape(b), n_obj, obj, pred=pred, n_pred=n_pred)
        if blocked_zones is not None:
            sc.set_zones(blocked_zones)
        return sc


@dataclass
class DeviceScenarioBatch:
    """A ScenarioBatch whose arrays already live on the device: torch tensors on the planner's device with the fields,
    shapes and dtypes of ScenarioBatch.  Every tick entry point of BatchPlanner except plan_stream stages it with one
    kernel (k_stage) instead of a host copy and an upload, and without a host synchronisation.  The tensors may be
    non-contiguous: they are read through their strides, and ``obj`` may carry more than five columns, of which the
    first five are used.  ``zones`` stays host data, as in ScenarioBatch; its bitmasks are uploaded when it changes."""
    pos: torch.Tensor          # (B, 2)  float64
    heading: torch.Tensor      # (B,)    float64
    vel: torch.Tensor          # (B,)    float64
    n_obj: torch.Tensor        # (B,)    int32
    obj: torch.Tensor          # (B, K, >= 5) float64
    zones: list = None
    zone_sel: torch.Tensor = None   # (B,) int32
    zone_key: torch.Tensor = None   # (B,) int64
    pred: torch.Tensor = None       # (B, K, KP, 2) float64
    n_pred: torch.Tensor = None     # (B, K) int32

    _SPEC = (("pos", 2, torch.float64), ("heading", 1, torch.float64), ("vel", 1, torch.float64),
             ("n_obj", 1, torch.int32), ("obj", 3, torch.float64), ("zone_sel", 1, torch.int32),
             ("zone_key", 1, torch.int64), ("pred", 4, torch.float64), ("n_pred", 2, torch.int32))

    @property
    def size(self) -> int:
        return int(self.pos.shape[0])

    def subset(self, idx) -> "DeviceScenarioBatch":
        """scenarios idx (a device index tensor, or anything torch indexing takes), as new tensors"""
        def take(a):
            return None if a is None else a[idx]
        return DeviceScenarioBatch(take(self.pos), take(self.heading), take(self.vel), take(self.n_obj),
                                   take(self.obj), self.zones, take(self.zone_sel), take(self.zone_key),
                                   take(self.pred), take(self.n_pred))

    def cpu(self) -> ScenarioBatch:
        """the host ScenarioBatch of the same values (obj: its first five columns)"""
        def host(a):
            return None if a is None else a.cpu().numpy().copy()
        return ScenarioBatch(host(self.pos), host(self.heading), host(self.vel), host(self.n_obj),
                             host(self.obj[:, :, :5]), self.zones, host(self.zone_sel), host(self.zone_key),
                             host(self.pred), host(self.n_pred))

    def check(self, device) -> None:
        """device, dtype, dimensionality and batch size of every tensor (ValueError); reads shapes only, no values"""
        dev = torch.device(device)
        for name, ndim, dt in self._SPEC:
            a = getattr(self, name)
            if a is None:
                if name in ("pos", "heading", "vel", "n_obj", "obj"):
                    raise ValueError("DeviceScenarioBatch.%s is required" % name)
                continue
            if not isinstance(a, torch.Tensor):
                raise ValueError("DeviceScenarioBatch.%s must be a torch tensor, got %s" % (name, type(a).__name__))
            if a.device.type != dev.type or (dev.index is not None and a.device.index != dev.index):
                raise ValueError("DeviceScenarioBatch.%s is on %s, the planner on %s" % (name, a.device, dev))
            if a.dtype != dt:
                raise ValueError("DeviceScenarioBatch.%s must be %s, got %s" % (name, dt, a.dtype))
            if a.dim() != ndim:
                raise ValueError("DeviceScenarioBatch.%s must have %d dimensions, got shape %s" % (name, ndim,
                                                                                                   tuple(a.shape)))
        B, K = self.size, int(self.obj.shape[1])
        if B < 1:
            raise ValueError("DeviceScenarioBatch: the batch is empty")
        want = dict(pos=(B, 2), obj=(B, K), n_pred=(B, K))
        if self.pred is not None:
            want["pred"] = (B, K, int(self.pred.shape[2]), 2)
        for name, ndim, _ in self._SPEC:
            a = getattr(self, name)
            if a is None:
                continue
            shape = tuple(a.shape)
            w = want.get(name, (B,))
            if shape[:len(w)] != w:
                raise ValueError("DeviceScenarioBatch.%s has shape %s, expected %s" % (name, shape, w + ("...",) *
                                                                                       (ndim - len(w))))
        if int(self.obj.shape[2]) < 5:
            raise ValueError("DeviceScenarioBatch.obj needs at least 5 columns (X, Y, theta, v, length), got %d"
                             % int(self.obj.shape[2]))
        if (self.pred is None) != (self.n_pred is None):
            raise ValueError("DeviceScenarioBatch: pred and n_pred come together")


class Track(object):
    """Full-resolution track / race line arrays of a 12-column global trajectory CSV."""

    def __init__(self, globtraj_input_path: str):
        t = import_globtraj_csv(globtraj_input_path)
        self.refline = t["refline"]
        self.normvec = t["normvec"]
        self.w_right = t["width_right"]
        self.w_left = t["width_left"]
        self.alpha = t["alpha"]
        self.s = t["s_rl"][:-1]
        self.length = float(t["s_rl"][-1])
        self.psi = t["psi_rl"]
        self.vel = t["vel_rl"]
        self.raceline = self.refline + self.normvec * self.alpha[:, None]

    def _seg(self, s):
        s = np.mod(s, self.length)
        i = np.clip(np.searchsorted(self.s, s, side="right") - 1, 0, self.s.size - 1)
        j = (i + 1) % self.s.size
        s_next = np.where(j == 0, self.length, self.s[j])
        f = (s - self.s[i]) / (s_next - self.s[i])
        return i, j, f

    def raceline_pose(self, s):
        """(x, y), heading, race line velocity at arc length s (linear interpolation between race line points)."""
        i, j, f = self._seg(s)
        xy = self.raceline[i] * (1.0 - f)[:, None] + self.raceline[j] * f[:, None]
        dpsi = np.mod(self.psi[j] - self.psi[i] + np.pi, 2 * np.pi) - np.pi
        psi = np.mod(self.psi[i] + f * dpsi + np.pi, 2 * np.pi) - np.pi
        vel = self.vel[i] * (1.0 - f) + self.vel[j] * f
        return xy, psi, vel

    def frame(self, s):
        """reference-line point, normal vector and track widths at (the race line point preceding) arc length s."""
        i, _, _ = self._seg(s)
        return self.refline[i], self.normvec[i], self.w_left[i], self.w_right[i], self.psi[i], self.vel[i]


def make_scenarios(track: Track, batch: int, seed: int = DEFAULT_SEED, n_obj_min: int = 1, n_obj_max: int = 3,
                   k_max: int = None, obj_margin: float = 1.4, ahead=(30.0, 280.0), s_max: float = None,
                   s_min: float = 0.0) -> ScenarioBatch:
    """SURVEY 8(d) config 2 (n_obj 1..3) / config 4 (n_obj_min = n_obj_max = 5).  s_max: upper bound of the ego arc
    length (open tracks: stay in front of the last race line point), s_min: lower bound."""
    rng = np.random.default_rng(seed)
    s_e = rng.uniform(s_min, track.length if s_max is None else s_max, size=batch)
    pos, heading, v_rl = track.raceline_pose(s_e)
    vel = rng.uniform(5.0, np.maximum(0.9 * v_rl, 5.0))
    n_obj = rng.integers(n_obj_min, n_obj_max + 1, size=batch).astype(np.int32)
    k = int(n_obj_max if k_max is None else k_max)
    obj = np.zeros((batch, k, 5))
    ds = rng.uniform(ahead[0], ahead[1], size=(batch, k))
    u = rng.uniform(0.0, 1.0, size=(batch, k))
    uv = rng.uniform(0.0, 1.0, size=(batch, k))
    for j in range(k):
        ref, nv, wl, wr, psi, vrl = track.frame(s_e + ds[:, j])
        lo = -(wl - obj_margin)
        hi = (wr - obj_margin)
        d = lo + u[:, j] * (hi - lo)
        obj[:, j, 0:2] = ref + nv * d[:, None]
        obj[:, j, 2] = psi
        obj[:, j, 3] = uv[:, j] * 0.5 * vrl
        obj[:, j, 4] = 5.0
    mask = np.arange(k)[None, :] >= n_obj[:, None]
    obj[mask] = 0.0
    return ScenarioBatch(pos=pos, heading=heading, vel=vel, n_obj=n_obj, obj=obj)


def make_velocity_microbench(n_paths: int, n_points: int, seed: int = DEFAULT_SEED) -> dict:
    """SURVEY 8(d) config 5: smooth random curvature profiles for the stand-alone forward/backward solver."""
    rng = np.random.default_rng(seed)
    el = 2.5 + rng.uniform(-0.1, 0.1, size=(n_paths, n_points)).astype(np.float64)
    s = np.cumsum(el, axis=1) - el
    amp = rng.uniform(0.0, 0.04 / 3.0, size=(n_paths, 3, 1))
    wl = rng.uniform(60.0, 600.0, size=(n_paths, 3, 1))
    ph = rng.uniform(0.0, 2 * np.pi, size=(n_paths, 3, 1))
    kappa = np.sum(amp * np.sin(2 * np.pi * s[:, None, :] / wl + ph), axis=1)
    return dict(kappa=kappa, el=el, v_start=rng.uniform(0.0, 40.0, size=n_paths),
                v_end=rng.uniform(0.0, 40.0, size=n_paths), v_max=60.0, gg=(5.0, 5.0), drag_coeff=0.85, m_veh=1000.0,
                dyn_model_exp=1.0)
